"""Principal component regression (DESIGN.md §14): the share of an embedding's variance that its batches explain,
scib's ``pcr`` / ``pcr_comparison``.  The embedding's principal components are regressed one by one on the one-hot
batches, and each component's R^2 is weighted by its variance.

``pcr`` takes the batches by column name, as ``compute_lisi`` does, and treats any column as categorical;
``pcr_comparison`` folds the scores of one embedding before and after an integration; ``pcr_on`` (``harmony.pcr``)
runs ``hb_pcr`` on an existing object.  Argument errors are raised before the CUDA library is loaded.
"""
import warnings

import numpy as np

from ._arrays import (call, check_two_rows, dense_codes, dense_on, device_of, download, embedding, factorise_for,
                      handle, label_columns, ptr, resolve_device, rows_on)


def check_n_comps(n_comps):
    """n_comps: an integer >= 1 -> that integer."""
    if isinstance(n_comps, bool) or not isinstance(n_comps, (int, np.integer)):
        raise ValueError(f"n_comps must be an integer, not {n_comps!r}")
    if n_comps < 1:
        raise ValueError(f"n_comps = {n_comps}, at least one component is needed")
    return int(n_comps)


def pcr_on(obj, X, batches, n_comps=50):
    """``hb_pcr`` on an existing ``harmony`` object (any state: the call needs no setup and changes none) -> ``(var, r2,
    components, score)``: with m = min(n_comps, N, d), the variance of each of the m leading principal components
    (eigenvalue / (n - 1) over the n finite rows), the R^2 of regressing each on the one-hot batches, the components
    [m, d] and the variance-weighted R^2 as a float.  ``batches``: dense codes 0..n-1, [N] (numpy or an int32 CUDA
    tensor on the object's device).  The arrays come back as numpy arrays for host rows, CUDA tensors otherwise."""
    X = embedding(X, "X")
    N, d = X.shape
    check_two_rows(X)
    n_comps = check_n_comps(n_comps)
    batches, n_batches = dense_codes(batches, N, "batches")
    import torch
    device = device_of(obj)
    host, x, x_args = rows_on(obj, X, "X")
    batches = dense_on(obj, batches)
    m = min(n_comps, N, d)
    var = torch.empty(m, dtype=torch.float64, device=device)
    r2 = torch.empty(m, dtype=torch.float64, device=device)
    comps = torch.empty((m, d), dtype=torch.float64, device=device)
    score = torch.empty(1, dtype=torch.float64, device=device)
    call(obj, "hb_pcr", *x_args, N, int(d), ptr(batches), int(n_batches), int(n_comps), ptr(var), ptr(r2), ptr(comps),
         ptr(score))
    var, r2, comps = download(host, var, r2, comps)
    return var, r2, comps, float(score.item())


def pcr(X, meta_data, batch_key, n_comps=50, return_all=False, device=None):
    """scib's ``pcr``: the principal components of ``X`` [N, d] (at most ``n_comps``), each regressed on the batches
    of ``meta_data[batch_key]`` (any values, always categorical); returns sum_j R^2_j var_j / sum_j var_j, in [0, 1]
    (0: the batches explain none of the variance).  NaN when fewer than two rows are finite or X has no variance.
    With ``return_all`` also ``(var, r2, components)`` of the m = min(n_comps, N, d) components.

    A row with a non-finite value takes no part.  ``meta_data`` as ``compute_lisi`` takes it.  A CUDA ``X`` (float32
    / float64) stays on its device, and the arrays are then CUDA tensors; d <= 128."""
    X = embedding(X, "X")
    check_two_rows(X)
    n_comps = check_n_comps(n_comps)
    col = label_columns(meta_data, [batch_key], X)[0]
    obj = handle(resolve_device(device, X, "X"))
    codes = factorise_for(col, X)[1]
    var, r2, comps, score = pcr_on(obj, X, codes, n_comps)
    return (score, var, r2, comps) if return_all else score


def pcr_fold(before, after, scale=True):
    """scib's fold of two PCR scores: (before - after) / before, 0 (with a warning) where it is negative; unscaled,
    after - before."""
    before, after = np.float64(before), np.float64(after)
    if not scale:
        return float(after - before)
    with np.errstate(divide="ignore", invalid="ignore"):
        score = (before - after) / before
    if score < 0:
        warnings.warn("the batches explain more variance after integration than before; the PCR comparison is set "
                      "to 0", stacklevel=3)
        score = 0.0
    return float(score)


def pcr_comparison(X_before, X_after, meta_data, batch_key, n_comps=50, scale=True, device=None):
    """scib's ``pcr_comparison``: the PCR scores of one set of cells before (``X_before``) and after (``X_after``) an
    integration, both [N, d] with the batches of ``meta_data[batch_key]``, folded as (before - after) / before (1: the
    batch variance is gone, 0: it did not shrink; set to 0 with a warning when it grew) or, unless ``scale``, as
    after - before.  Harmony: ``pcr_comparison(obj.getZorig().T, obj.getZcorr().T, meta, "dataset")``."""
    X_before, X_after = embedding(X_before, "X_before"), embedding(X_after, "X_after")
    check_two_rows(X_before, "X_before")
    check_two_rows(X_after, "X_after")
    if X_before.shape[0] != X_after.shape[0]:
        raise ValueError(f"X_before has {X_before.shape[0]} rows and X_after {X_after.shape[0]}: they must hold the "
                         f"same cells")
    check_n_comps(n_comps)
    label_columns(meta_data, [batch_key], X_before)
    before = pcr(X_before, meta_data, batch_key, n_comps, device=device)
    after = pcr(X_after, meta_data, batch_key, n_comps, device=device)
    return pcr_fold(before, after, scale)
