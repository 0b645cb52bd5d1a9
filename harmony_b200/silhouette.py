"""Silhouette widths of an embedding (DESIGN.md §11): per cell, how much closer it lies to the cells of its own label
than to those of the nearest other label, over all pairs of cells (within a group, when groups are given).  The
scores scib reports as ``silhouette`` (cell-type ASW) and ``silhouette_batch`` (batch ASW within each cell type) are
folds of these per-cell values.

``silhouette_samples`` mirrors ``sklearn.metrics.silhouette_samples`` (with optional groups); ``silhouette_on``
(``harmony.silhouette``) runs ``hb_silhouette`` on an existing object.  Argument errors are raised before the CUDA
library is loaded.
"""
import ctypes

import numpy as np

from ._arrays import current_stream, device_rows, factorise, resolve_device, to_device
from .lisi import _check_rows, _missing
from .utils import is_cuda_tensor


def _check_codes(codes, n, what):
    """int32-representable codes [N] (numpy or an int32 CUDA tensor) -> the same, and their count (largest + 1)."""
    if is_cuda_tensor(codes):
        import torch
        if codes.dtype != torch.int32:
            raise TypeError(f"CUDA {what} must be int32, not {codes.dtype}")
        if codes.ndim != 1 or codes.shape[0] != n:
            raise ValueError(f"{what} must be [{n}], not {tuple(codes.shape)}")
        return codes, int(codes.max()) + 1 if n else 0
    codes = np.asarray(codes)
    if codes.dtype.kind not in "iu":
        raise TypeError(f"{what} must be integers, not {codes.dtype}")
    if codes.ndim != 1 or codes.shape[0] != n:
        raise ValueError(f"{what} must be [{n}], not {codes.shape}")
    if codes.size and (codes.min() < 0 or codes.max() >= 2 ** 31 - 1):
        raise ValueError(f"{what} must be codes in 0..2^31 - 2")
    return codes, int(codes.max()) + 1 if n else 0


def silhouette_on(obj, X, labels, groups=None):
    """``hb_silhouette`` on an existing ``harmony`` object (any state: the call needs no setup and changes none).
    ``labels`` / ``groups``: dense codes 0..n-1 (numpy or int32 CUDA tensors on the object's device)."""
    X = _check_rows(X)
    N, d = X.shape
    if N < 2:
        raise ValueError(f"X has {N} rows, at least 2 are needed")
    labels, n_labels = _check_codes(labels, N, "labels")
    n_groups = 0
    if groups is not None:
        groups, n_groups = _check_codes(groups, N, "groups")
    import torch
    host = not is_cuda_tensor(X)
    device = torch.device("cuda", obj._scalar("device"))
    if host:
        X = to_device(obj, X)
    x, *x_args = device_rows(obj, X, "X")
    codes = []
    for c in (labels, groups):
        if c is not None and not is_cuda_tensor(c):
            c = torch.as_tensor(np.ascontiguousarray(c, dtype=np.int32)).to(device)
        if c is not None:
            if c.device != device:
                raise ValueError(f"codes are on {c.device}, the harmony object on {device}")
            c = c.contiguous()
        codes.append(c)
    out = torch.empty(N, dtype=torch.float64, device=device)
    ptr = lambda t: ctypes.c_void_p(None if t is None else t.data_ptr())  # noqa: E731
    obj._check(obj._L.hb_silhouette(obj._h, *x_args, N, int(d), ptr(codes[0]), int(n_labels), ptr(codes[1]),
                                    int(n_groups), ptr(out), current_stream(device)))
    return out.cpu().numpy() if host else out


def _column(cols, name, n):
    if name not in cols:
        raise ValueError(f"meta_data has no column {name!r}")
    if cols[name].ndim != 1 or len(cols[name]) != n:
        raise ValueError(f"column {name!r} must hold one label per row of X ({n})")
    if not is_cuda_tensor(cols[name]) and _missing(cols[name]):
        raise ValueError(f"column {name!r} holds missing labels")
    return cols[name]


def _vector(v, n, what):
    if not is_cuda_tensor(v):
        v = np.asarray(v)
    if v.ndim != 1 or len(v) != n:
        raise ValueError(f"{what} must hold one label per row of X ({n})")
    if not is_cuda_tensor(v) and _missing(v):
        raise ValueError(f"{what} holds missing labels")
    return v


def _n_levels(codes):
    return int(codes.max()) + 1 if len(codes) else 0


def silhouette_samples(X, labels, groups=None, device=None):
    """The silhouette width of every row of ``X`` [N, d] -> [N] float64: with ``a`` the mean Euclidean distance to
    the other rows of its label and ``b`` the smallest mean distance to the rows of another label, ``(b - a) /
    max(a, b)``; 0 for a row alone in its label.  With ``groups`` only rows of one group interact (a row of a group
    with one label gets NaN).  Without groups this is ``sklearn.metrics.silhouette_samples(X, labels)``, which it
    refuses the same way: fewer than 2 labels, or as many labels as rows.

    ``labels`` / ``groups``: any values, one per row (CUDA integer tensors on ``X``'s device when ``X`` is a CUDA
    tensor).  Host ``X`` in -> numpy out; a CUDA ``X`` (float32 / float64) -> a CUDA tensor, ordered on the device's
    current torch stream.  A row with a non-finite value gets NaN and takes no part.  d <= 128."""
    on_device = is_cuda_tensor(X)
    X = _check_rows(X)
    N = X.shape[0]
    if N < 2:
        raise ValueError(f"X has {N} rows, at least 2 are needed")
    cols = {"labels": _vector(labels, N, "labels")}
    if groups is not None:
        cols["groups"] = _vector(groups, N, "groups")
    from .ui import _label_device
    _label_device(cols, list(cols), X, on_device)
    device = resolve_device(device, X, "X")
    dev = X.device if on_device else None
    codes = factorise(cols["labels"], dev)[1]
    gcodes = factorise(cols["groups"], dev)[1] if groups is not None else None
    n = _n_levels(codes)
    if groups is None and not 1 < n < N:
        raise ValueError(f"Number of labels is {n}. Valid values are 2 to n_samples - 1 (inclusive)")
    from .harmony import harmony  # needs the CUDA extension; fails loudly when it is missing
    return silhouette_on(harmony(device=device), X, codes, gcodes)


def _columns(X, meta_data, names):
    on_device = is_cuda_tensor(X)
    X = _check_rows(X)
    if not isinstance(meta_data, dict) and not hasattr(meta_data, "columns"):
        raise ValueError("meta_data must be a DataFrame or a dict of columns")
    from .ui import _as_columns, _label_device
    cols, _ = _as_columns(meta_data, ())
    used = [_column(cols, v, X.shape[0]) for v in names]
    _label_device(cols, names, X, on_device)
    return X, used


def silhouette_label(X, meta_data, label_key, scale=True):
    """Cell-type ASW, scib's ``silhouette``: the mean silhouette width of ``meta_data[label_key]`` over ``X``,
    scaled to ``(s + 1) / 2`` (1 best) unless ``scale`` is False.  Labels are taken as ``compute_lisi`` takes them."""
    X, (labels,) = _columns(X, meta_data, [label_key])
    s = silhouette_samples(X, labels)
    asw = float(s.mean())
    return (asw + 1) / 2 if scale else asw


def batch_fold(s, batch, label, scale=True):
    """scib's fold of per-cell batch silhouettes ``s`` (scored within each cell type) -> (batch ASW, {cell type: its
    mean of 1 - |s|}, or of |s| unless ``scale``).  A cell type with one batch, or as many batches as cells, is skipped;
    the ASW is NaN when every one is.  Host arrays."""
    types, tcodes = factorise(np.asarray(label))
    bcodes = factorise(np.asarray(batch))[1]
    s = np.asarray(s, dtype=np.float64)
    means = {}
    for t in range(len(types)):
        rows = tcodes == t
        nb = len(np.unique(bcodes[rows]))
        if nb == 1 or nb == rows.sum():
            continue
        v = np.abs(s[rows])
        means[types[t].item() if hasattr(types[t], "item") else types[t]] = float((1 - v if scale else v).mean())
    asw = float(np.mean(list(means.values()))) if means else float("nan")
    return asw, means


def silhouette_batch(X, meta_data, batch_key, label_key, scale=True, return_all=False):
    """Batch ASW, scib's ``silhouette_batch``: within each cell type (``label_key``), the silhouette width of the
    batches (``batch_key``) of its cells, taken as ``1 - |s|`` (``|s|`` unless ``scale``), averaged per cell type and
    then over the cell types.  A cell type with one batch, or with as many batches as cells, is skipped; NaN when all
    are.  One device call scores every cell type.  With ``return_all`` also ``{cell type: its mean}``."""
    X, (batch, label) = _columns(X, meta_data, [batch_key, label_key])
    s = silhouette_samples(X, batch, groups=label)
    host = lambda v: v.cpu().numpy() if is_cuda_tensor(v) else np.asarray(v)  # noqa: E731
    asw, means = batch_fold(host(s), host(batch), host(label), scale)
    return (asw, means) if return_all else asw
