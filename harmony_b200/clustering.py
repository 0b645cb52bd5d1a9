"""k-means of an embedding and the NMI / ARI scores of a clustering (DESIGN.md §15): scib's bio-conservation score
``nmi_ari_cluster_labels_kmeans``, k-means into as many clusters as there are cell types, compared with the cell types
by sklearn's ``normalized_mutual_info_score`` (arithmetic mean) and ``adjusted_rand_score``.

``kmeans`` clusters an embedding; ``kmeans_on`` (``harmony.kmeans``) runs ``hb_kmeans`` on an existing object;
``nmi_ari`` folds two labelings; ``nmi_ari_cluster_labels_kmeans`` does both.  Argument errors are raised before the
CUDA library is loaded.
"""
import math

import numpy as np

from ._arrays import (call, device_of, download, embedding, factorise, handle, label_columns, ptr, resolve_device,
                      rows_on)
from .utils import is_cuda_tensor

MAX_CLUSTERS = 1024   # the seeding makes about K passes over the rows


def _integer(v, what, low):
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
        raise ValueError(f"{what} must be an integer, not {v!r}")
    if v < low:
        raise ValueError(f"{what} = {v}, at least {low} is needed")
    return int(v)


def check_kmeans(N, n_clusters, seed, n_init, max_iter, tol):
    """The arguments of a k-means call of N rows -> (n_clusters, seed, n_init, max_iter, tol), checked."""
    if N < 1:
        raise ValueError("X has no rows")
    n_clusters = _integer(n_clusters, "n_clusters", 1)
    if n_clusters > min(N, MAX_CLUSTERS):
        raise ValueError(f"n_clusters = {n_clusters} is not supported (1 <= n_clusters <= min(N, {MAX_CLUSTERS}) = "
                         f"{min(N, MAX_CLUSTERS)})")
    seed = _integer(seed, "seed", 0)
    if seed >= 2 ** 64:
        raise ValueError(f"seed = {seed} does not fit 64 bits")
    n_init = _integer(n_init, "n_init", 1)
    max_iter = _integer(max_iter, "max_iter", 0)
    for name, v in (("n_init", n_init), ("max_iter", max_iter)):
        if v >= 2 ** 31:
            raise ValueError(f"{name} = {v} does not fit 32 bits")
    if isinstance(tol, bool) or not isinstance(tol, (int, float, np.integer, np.floating)) or not (
            math.isfinite(tol) and tol >= 0):
        raise ValueError(f"tol must be a finite number >= 0, not {tol!r}")
    return n_clusters, seed, n_init, max_iter, float(tol)


def kmeans_on(obj, X, n_clusters, seed=0, n_init=1, max_iter=300, tol=1e-4, return_seeds=False):
    """``hb_kmeans`` on an existing ``harmony`` object (any state: the call needs no setup and changes none) ->
    ``(labels, centres, inertia, n_iter)``: labels [N] int32 (-1 for a row with a non-finite value) and centres [K, d]
    float64 of the init with the lowest inertia, and each init's inertia [n_init] float64 and iterations [n_init]
    int32; with ``return_seeds`` also the seed rows [n_init, K] int32.  numpy arrays for host rows, CUDA tensors
    otherwise.  ``RuntimeError`` (status 3) when fewer than K rows are finite."""
    X = embedding(X, "X")
    N, d = X.shape
    K, seed, n_init, max_iter, tol = check_kmeans(N, n_clusters, seed, n_init, max_iter, tol)
    import torch
    device = device_of(obj)
    host, x, x_args = rows_on(obj, X, "X")
    labels = torch.empty(N, dtype=torch.int32, device=device)
    centres = torch.empty((K, d), dtype=torch.float64, device=device)
    inertia = torch.empty(n_init, dtype=torch.float64, device=device)
    n_iter = torch.empty(n_init, dtype=torch.int32, device=device)
    seeds = torch.empty((n_init, K), dtype=torch.int32, device=device) if return_seeds else None
    call(obj, "hb_kmeans", *x_args, N, int(d), K, seed, n_init, max_iter, tol, ptr(labels), ptr(centres), ptr(inertia),
         ptr(n_iter), ptr(seeds))
    out = download(host, labels, centres, inertia, n_iter, seeds)
    return tuple(out) if return_seeds else tuple(out[:4])


def kmeans(X, n_clusters, seed=0, n_init=1, max_iter=300, tol=1e-4, return_seeds=False, device=None):
    """k-means of the rows of ``X`` [N, d] (d <= 128) into ``n_clusters`` clusters (1 <= K <= min(N, 1024)): greedy
    k-means++ seeds, then sklearn's ``algorithm="lloyd"`` iteration (stop when the labels repeat or the squared centre
    shift is at most ``tol`` times the mean column variance), ``n_init`` times; the init of the lowest inertia is
    returned.  Returns ``(labels, centres, inertia, n_iter)`` as ``kmeans_on`` does.  A row with a NaN or an infinity
    takes no part and gets label -1.  A CUDA ``X`` (float32 / float64) stays on its device and the outputs are CUDA
    tensors; fp32 rows are assigned on 3xTF32 scores (DESIGN §9's band), means and inertia are fp64."""
    X = embedding(X, "X")
    check_kmeans(X.shape[0], n_clusters, seed, n_init, max_iter, tol)
    return kmeans_on(handle(resolve_device(device, X, "X")), X, n_clusters, seed, n_init, max_iter, tol, return_seeds)


def _codes(v):
    """A label vector -> int64 codes 0..n-1 (on the device for a CUDA tensor, numpy otherwise)."""
    if is_cuda_tensor(v):
        import torch
        return torch.unique(v, return_inverse=True)[1].reshape(-1).to(torch.int64)
    return np.unique(np.asarray(v), return_inverse=True)[1].reshape(-1).astype(np.int64)


def _assigned(p):
    """The rows of a prediction that are not -1 (the rows k-means assigned): a bool vector where p lives."""
    if is_cuda_tensor(p):
        return p != -1
    p = np.asarray(p)
    return p != -1 if p.dtype.kind in "iuf" else np.ones(len(p), bool)


def contingency(labels_true, labels_pred):
    """The contingency table [classes, clusters] (int64, host) of two labelings of the same rows, the rows whose
    ``labels_pred`` is -1 left out.  When either is a CUDA tensor the table is counted on its device; host labels of
    any values (strings, categories) are factorised to integer codes on the host and only the codes are uploaded."""
    keep = _assigned(labels_pred)
    if is_cuda_tensor(labels_true) or is_cuda_tensor(labels_pred):
        import torch
        dev = (labels_pred if is_cuda_tensor(labels_pred) else labels_true).device
        on = lambda v: v if is_cuda_tensor(v) else torch.as_tensor(_codes(v), device=dev)  # noqa: E731
        keep = keep if is_cuda_tensor(keep) else torch.as_tensor(keep, device=dev)
        t, p = _codes(on(labels_true)[keep]), _codes(on(labels_pred)[keep])
        if not len(t):
            return np.zeros((0, 0), np.int64)
        nc = int(p.max()) + 1
        table = torch.bincount(t * nc + p, minlength=(int(t.max()) + 1) * nc)
        return table.reshape(-1, nc).cpu().numpy().astype(np.int64)
    t, p = _codes(np.asarray(labels_true)[keep]), _codes(np.asarray(labels_pred)[keep])
    if not len(t):
        return np.zeros((0, 0), np.int64)
    nc = int(p.max()) + 1
    return np.bincount(t * nc + p, minlength=(int(t.max()) + 1) * nc).reshape(-1, nc).astype(np.int64)


def _entropy(counts):
    """sklearn's entropy of a labeling from its class sizes."""
    pi = counts[counts > 0].astype(np.float64)
    if pi.size <= 1:
        return 0.0
    s = pi.sum()
    return float(-np.sum((pi / s) * (np.log(pi) - math.log(s))))


def nmi_ari_fold(C):
    """(NMI, ARI) of a contingency table, as sklearn's ``normalized_mutual_info_score`` (arithmetic mean) and
    ``adjusted_rand_score`` compute them, including their special cases."""
    C = np.asarray(C, dtype=np.int64)
    n = int(C.sum())
    a, b = C.sum(axis=1), C.sum(axis=0)
    # ---- NMI
    if (len(a) == len(b) == 1) or n == 0:
        nmi = 1.0
    else:
        nzx, nzy = np.nonzero(C)
        nz = C[nzx, nzy].astype(np.float64)
        if len(a) == 1 or len(b) == 1:
            mi = 0.0
        else:
            cnm = nz / n
            outer = a[nzx].astype(np.int64) * b[nzy].astype(np.int64)
            log_outer = -np.log(outer.astype(np.float64)) + math.log(a.sum()) + math.log(b.sum())
            terms = cnm * (np.log(nz) - math.log(n)) + cnm * log_outer
            terms = np.where(np.abs(terms) < np.finfo(np.float64).eps, 0.0, terms)
            mi = max(float(terms.sum()), 0.0)
        if mi == 0.0:
            nmi = 0.0
        else:
            nmi = float(mi / ((_entropy(a) + _entropy(b)) / 2.0))
    # ---- ARI from the pair confusion matrix, in exact integers
    Co = C.astype(object)  # Python integers: N^2 overflows int64 beyond 3e9 rows
    sq = int((Co ** 2).sum())
    tp = sq - n
    fp = int((Co * b.astype(object)[None, :]).sum()) - sq
    fn = int((Co * a.astype(object)[:, None]).sum()) - sq
    tn = n * n - fp - fn - sq
    if fn == 0 and fp == 0:
        ari = 1.0
    else:
        ari = 2.0 * (tp * tn - fn * fp) / ((tp + fn) * (fn + tn) + (tp + fp) * (fp + tn))
    return nmi, float(ari)


def nmi_ari(labels_true, labels_pred):
    """(NMI, ARI) of two labelings of the same rows: sklearn's ``normalized_mutual_info_score(labels_true,
    labels_pred)`` (arithmetic mean) and ``adjusted_rand_score``, with their special cases.  Labels of any values;
    rows whose ``labels_pred`` is -1 (k-means' non-finite rows) are left out.  CUDA tensors are counted on their
    device; only the contingency table comes to the host."""
    nt, np_ = len(labels_true), len(labels_pred)
    if nt != np_:
        raise ValueError(f"labels_true has {nt} rows and labels_pred {np_}: they must label the same rows")
    for name, v in (("labels_true", labels_true), ("labels_pred", labels_pred)):
        if getattr(v, "ndim", 1) != 1:
            raise ValueError(f"{name} must be a vector")
    return nmi_ari_fold(contingency(labels_true, labels_pred))


def nmi_ari_cluster_labels_kmeans(X, meta_data, label_key, seed=0, n_init=1, device=None):
    """scib-metrics' ``nmi_ari_cluster_labels_kmeans``: k-means of ``X`` [N, d] into as many clusters as
    ``meta_data[label_key]`` has distinct labels among the finite rows, then ``{"nmi": ..., "ari": ...}`` of the labels
    against the clusters (``nmi_ari``).  ``meta_data`` as ``compute_lisi`` takes it.  A CUDA ``X`` stays on its device
    until the fold."""
    on_device = is_cuda_tensor(X)
    X = embedding(X, "X")
    labels = label_columns(meta_data, [label_key], X)[0]
    seed = _integer(seed, "seed", 0)
    n_init = _integer(n_init, "n_init", 1)
    device = resolve_device(device, X, "X")
    if on_device:
        import torch
        fin = torch.isfinite(X).all(dim=1)
        if not is_cuda_tensor(labels):  # host labels of any values: their integer codes go to the device
            labels = factorise(labels, X.device)[1]
        K = int(torch.unique(labels[fin]).numel())
    else:
        fin = np.isfinite(X).all(axis=1)
        K = len(np.unique(np.asarray(labels)[fin]))
    if K < 1:
        raise ValueError("X has no finite row")
    check_kmeans(X.shape[0], K, seed, n_init, 300, 1e-4)
    pred = kmeans(X, K, seed=seed, n_init=n_init, device=device)[0]
    nmi, ari = nmi_ari(labels, pred)
    return {"nmi": nmi, "ari": ari}
