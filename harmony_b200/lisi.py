"""LISI, the Local Inverse Simpson's Index of an embedding (DESIGN.md §10): per cell, the effective number of batches
(iLISI) or of cell types (cLISI) among its nearest neighbours, the score Harmony's authors introduced with it.

``compute_lisi`` mirrors the LISI package's function of that name; ``lisi_on`` (``harmony.lisi``) runs ``hb_lisi`` on
an existing object.  Argument errors are raised before the CUDA library is loaded.
"""
import math

import numpy as np

from ._arrays import (call, code_sets, codes_on, device_of, download, embedding, factorise_for, handle, label_columns,
                      ptr, resolve_device, row_layout, rows_on)
from .utils import is_cuda_tensor

MAX_K = 128   # the neighbour lists of hb_lisi's search: perplexity < 43 1/3


def neighbours_for(perplexity, n):
    """k = floor(3 p) - 1, the neighbours LISI weighs at perplexity p (the package searches 3 p rows including the cell
    itself and drops the first); ValueError for a perplexity hb_lisi refuses or one that n rows cannot serve."""
    if isinstance(perplexity, bool) or not isinstance(perplexity, (int, float, np.integer, np.floating)):
        raise ValueError(f"perplexity must be a number, not {perplexity!r}")
    p = float(perplexity)
    if not math.isfinite(p) or p < 1:
        raise ValueError(f"perplexity must be finite and at least 1, not {perplexity!r}")
    k = math.floor(3 * p) - 1
    if k > MAX_K:
        raise ValueError(f"perplexity {perplexity!r} needs k = floor(3 p) - 1 = {k} neighbours; at most {MAX_K} "
                         f"(perplexity < 43 1/3)")
    if k > n - 1:
        raise ValueError(f"perplexity {perplexity!r} needs k = {k} neighbours, {n} rows have {max(n - 1, 0)}")
    return k


def lisi_on(obj, X, codes, perplexity=30, return_neighbors=False):
    """``hb_lisi`` on an existing ``harmony`` object (any state: the call needs no setup and changes none)."""
    X = embedding(X, "X")
    N, d = X.shape
    k = neighbours_for(perplexity, N)
    codes = code_sets(codes, N)
    import torch
    device = device_of(obj)
    host, x, x_args = rows_on(obj, X, "X")
    codes, ld = row_layout(codes_on(obj, codes), N)
    out = torch.empty((N, codes.shape[0]), dtype=torch.float64, device=device)
    idx = dist = None
    if return_neighbors:
        idx = torch.empty((N, k), dtype=torch.int32, device=device)
        dist = torch.empty((N, k), dtype=torch.float32, device=device)
    call(obj, "hb_lisi", *x_args, N, int(d), ptr(codes), ld, int(codes.shape[0]), float(perplexity), ptr(out), ptr(idx),
         ptr(dist))
    out, idx, dist = download(host, out, idx, dist)
    return (out, idx, dist) if return_neighbors else out


def compute_lisi(X, meta_data, label_colnames, perplexity=30, device=None, return_neighbors=False):
    """The LISI package's ``compute_lisi``: for every row of ``X`` [N, d] and every column named in ``label_colnames``,
    the inverse Simpson's index of that column's labels among the row's ``floor(3 perplexity) - 1`` nearest other rows,
    weighted by a Gaussian kernel calibrated to ``perplexity`` -> [N, len(label_colnames)] float64: how many labels are
    mixed around the row (1: one label; at most the number of labels).  iLISI on batch labels should be high after an
    integration, cLISI on cell types near 1.

    ``meta_data``: a DataFrame or a dict of columns, one label per row, as ``RunHarmony`` takes it; any values, missing
    ones refused.  Host ``X`` in -> numpy out; a CUDA ``X`` (float32 / float64) -> a CUDA tensor, ordered on the
    device's current torch stream, and its labels may be integer CUDA tensors on the same device.  A row with a
    non-finite value has no neighbours and gets NaN; a row whose weights all fall on one neighbour gets -1, the
    package's marker.  With ``return_neighbors`` also the neighbours searched, ``(lisi, idx, dist)`` as ``knn``
    returns them.  1 <= perplexity < 43 1/3, d <= 128."""
    on_device = is_cuda_tensor(X)
    X = embedding(X, "X")
    neighbours_for(perplexity, X.shape[0])
    names = [label_colnames] if isinstance(label_colnames, str) else list(label_colnames)
    if not names:
        raise ValueError("label_colnames names no column")
    cols = label_columns(meta_data, names, X)
    obj = handle(resolve_device(device, X, "X"))
    codes = [factorise_for(c, X)[1] for c in cols]
    if on_device:
        import torch
        codes = torch.stack(codes)
    else:
        codes = np.stack(codes)
    return lisi_on(obj, X, codes, perplexity, return_neighbors)
