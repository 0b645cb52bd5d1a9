"""kBET, the k-nearest-neighbour batch effect test (DESIGN.md §13): per cell, a chi-square test of whether the batches
among the cell and its nearest neighbours of the same cell type are mixed as the batches of that cell type are.  The
score scib reports as ``kBET`` is one minus the mean rejection rate over the cell types.

``kbet`` takes labels by column name, as scib's ``kBET`` does; ``kbet_on`` (``harmony.kbet``) runs ``hb_kbet`` on an
existing object.  Argument errors are raised before the CUDA library is loaded.
"""
import numpy as np

from ._arrays import (call, check_two_rows, dense_codes, dense_on, device_of, download, embedding, factorise_for,
                      handle, label_columns, ptr, resolve_device, rows_on, to_host)

MAX_K0 = 129       # the cell and the sweep's longest list of 128 neighbours
RULE_MAX_K0 = 70   # scib's rule: min(70, max(10, floor(mean batch size / 4)))


def check_k0(k0):
    """k0: None or 0 for scib's rule, else an integer 2..MAX_K0 -> 0 or that integer."""
    if k0 is None:
        return 0
    if isinstance(k0, bool) or not isinstance(k0, (int, np.integer)):
        raise ValueError(f"k0 must be None or an integer, not {k0!r}")
    if k0 != 0 and not 2 <= k0 <= MAX_K0:
        raise ValueError(f"k0 = {k0} is not supported (None or 0 for scib's rule, or 2 <= k0 <= {MAX_K0})")
    return int(k0)


def kbet_on(obj, X, batches, labels=None, k0=0, return_neighbors=False):
    """``hb_kbet`` on an existing ``harmony`` object (any state: the call needs no setup and changes none) -> ``(stat,
    pval, k0)``: each row's chi-square statistic and p-value (NaN for a row that is not tested) and each label's
    neighbourhood size (0 for a label that is not tested).  ``batches`` / ``labels``: dense codes 0..n-1, [N] (numpy or
    int32 CUDA tensors on the object's device); no labels: one label.  ``k0``: 0 for scib's rule, else 2..129.  With
    ``return_neighbors`` also ``idx`` [N, max k0 - 1]: each tested row's neighbours by ascending distance, -1 after them
    and for the other rows."""
    X = embedding(X, "X")
    N, d = X.shape
    check_two_rows(X)
    k0 = check_k0(k0)
    batches, n_batches = dense_codes(batches, N, "batches")
    n_labels = 0
    if labels is not None:
        labels, n_labels = dense_codes(labels, N, "labels")
    import torch
    device = device_of(obj)
    host, x, x_args = rows_on(obj, X, "X")
    batches, labels = dense_on(obj, batches), dense_on(obj, labels)
    stat = torch.empty(N, dtype=torch.float64, device=device)
    pval = torch.empty(N, dtype=torch.float64, device=device)
    k0_out = torch.empty(max(n_labels, 1), dtype=torch.int32, device=device)
    width = (k0 or RULE_MAX_K0) - 1
    idx = torch.empty((N, width), dtype=torch.int32, device=device) if return_neighbors else None
    call(obj, "hb_kbet", *x_args, N, int(d), ptr(batches), int(n_batches), ptr(labels), int(n_labels), int(k0), ptr(stat),
         ptr(pval), ptr(k0_out), ptr(idx), int(width))
    if return_neighbors:
        idx = idx[:, :max(int(k0_out.max()) - 1, 0)]
    out = download(host, stat, pval, k0_out, idx)
    return tuple(out) if return_neighbors else tuple(out[:3])


def kbet_fold(pval, codes, k0, alpha=0.05):
    """The rejection rate of each label: the share of its tested rows (p-value not NaN) with p < alpha, NaN for a label
    with k0 = 0 (not tested).  Host arrays."""
    pval, codes = np.asarray(pval, np.float64), np.asarray(codes)
    rates = np.full(len(k0), np.nan)
    for l in np.nonzero(np.asarray(k0) > 0)[0]:
        p = pval[(codes == l) & ~np.isnan(pval)]
        if len(p):
            rates[l] = float((p < alpha).mean())
    return rates


def kbet(X, meta_data, batch_key, label_key=None, k0=None, alpha=0.05, scaled=True, return_all=False, device=None):
    """kBET, scib's ``kBET``: within each cell type of ``meta_data[label_key]`` (all cells when None), every cell's
    batches (``batch_key``) among itself and its ``k0 - 1`` nearest other cells of its type in ``X`` [N, d] are tested
    against the cell type's batch frequencies with a chi-square test at level ``alpha``; the rejection rate is the share
    of rejected cells.  Returns 1 - the mean rejection rate over the tested cell types (1: batches well mixed), or the
    mean rate itself unless ``scaled``; NaN when no cell type is tested.  A cell type with fewer than 10 cells or one
    batch is not tested.  ``k0``: None for scib's rule (min(70, max(10, floor(mean batch size / 4))) per cell type), else
    a fixed 2..129, and a cell type with fewer cells is not tested.  With ``return_all`` also ``{cell type: rejection
    rate, NaN if not tested}`` (key None without ``label_key``) and the per-cell ``(stat, pval)``.

    The neighbours are exact and Euclidean; a cell with a non-finite value takes no part and gets NaN.  ``meta_data``
    as ``compute_lisi`` takes it.  A CUDA ``X`` (float32 / float64) stays on its device until the final fold, and
    ``(stat, pval)`` are then CUDA tensors; d <= 128."""
    X = embedding(X, "X")
    N = X.shape[0]
    check_two_rows(X)
    k0 = check_k0(k0)
    if isinstance(alpha, bool) or not isinstance(alpha, (int, float, np.integer, np.floating)) or not 0 < alpha < 1:
        raise ValueError(f"alpha must be a number in (0, 1), not {alpha!r}")
    names = [batch_key] + ([label_key] if label_key is not None else [])
    cols = label_columns(meta_data, names, X)
    obj = handle(resolve_device(device, X, "X"))
    bcodes = factorise_for(cols[0], X)[1]
    levels, lcodes = factorise_for(cols[1], X) if label_key is not None else (None, None)
    stat, pval, k0_out = kbet_on(obj, X, bcodes, lcodes, k0)
    codes = to_host(lcodes) if lcodes is not None else np.zeros(N, np.int32)
    rates = kbet_fold(to_host(pval), codes, to_host(k0_out), alpha)
    tested = rates[~np.isnan(rates)]
    score = float("nan") if not len(tested) else float(1 - tested.mean() if scaled else tested.mean())
    if not return_all:
        return score
    keys = [None] if levels is None else [v.item() if hasattr(v, "item") else v for v in to_host(levels)]
    return score, dict(zip(keys, rates.tolist())), (stat, pval)
