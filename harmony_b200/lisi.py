"""LISI, the Local Inverse Simpson's Index of an embedding (DESIGN.md §10): per cell, the effective number of batches
(iLISI) or of cell types (cLISI) among its nearest neighbours, the score Harmony's authors introduced with it.

``compute_lisi`` mirrors the LISI package's function of that name; ``lisi_on`` (``harmony.lisi``) runs ``hb_lisi`` on
an existing object.  Argument errors are raised before the CUDA library is loaded.
"""
import ctypes
import math

import numpy as np

from ._arrays import current_stream, device_rows, factorise, resolve_device, to_device
from .neighbors import MAX_D
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


def _check_rows(X):
    if not is_cuda_tensor(X):
        X = np.asarray(X)
    if X.ndim != 2:
        raise ValueError("X must be an [N, d] matrix")
    if not 1 <= X.shape[1] <= MAX_D:
        raise ValueError(f"d = {X.shape[1]} is not supported (1 <= d <= {MAX_D})")
    return X


def _check_codes(codes, n):
    """int32 codes [N] or [n_sets, N] (numpy or a CUDA tensor) -> the same as [n_sets, N]."""
    if is_cuda_tensor(codes):
        import torch
        if codes.dtype != torch.int32:
            raise TypeError(f"CUDA codes must be int32, not {codes.dtype}")
    else:
        codes = np.asarray(codes)
        if codes.dtype.kind not in "iu":
            raise TypeError(f"codes must be integers, not {codes.dtype}")
        if codes.size and (codes.min() < -2 ** 31 or codes.max() >= 2 ** 31):
            raise ValueError("codes must fit int32")
    if codes.ndim == 1:
        codes = codes[None]
    if codes.ndim != 2 or codes.shape[0] < 1 or codes.shape[1] != n:
        raise ValueError(f"codes must be [{n}] or [n_sets, {n}] with n_sets >= 1, not {tuple(codes.shape)}")
    return codes


def lisi_on(obj, X, codes, perplexity=30, return_neighbors=False):
    """``hb_lisi`` on an existing ``harmony`` object (any state: the call needs no setup and changes none)."""
    X = _check_rows(X)
    N, d = X.shape
    k = neighbours_for(perplexity, N)
    codes = _check_codes(codes, N)
    import torch
    host = not is_cuda_tensor(X)
    device = torch.device("cuda", obj._scalar("device"))
    if host:
        X = to_device(obj, X)
    x, *x_args = device_rows(obj, X, "X")
    if not is_cuda_tensor(codes):
        codes = torch.as_tensor(np.ascontiguousarray(codes, dtype=np.int32)).to(device)
    if codes.device != device:
        raise ValueError(f"codes are on {codes.device}, the harmony object on {device}")
    if not (codes.stride(1) == 1 and (codes.shape[0] == 1 or codes.stride(0) >= N)):
        codes = codes.contiguous()
    ld = codes.stride(0) if codes.shape[0] > 1 else N
    out = torch.empty((N, codes.shape[0]), dtype=torch.float64, device=device)
    idx = dist = None
    if return_neighbors:
        idx = torch.empty((N, k), dtype=torch.int32, device=device)
        dist = torch.empty((N, k), dtype=torch.float32, device=device)
    ptr = lambda t: ctypes.c_void_p(None if t is None else t.data_ptr())  # noqa: E731
    obj._check(obj._L.hb_lisi(obj._h, *x_args, N, int(d), ptr(codes), int(ld), int(codes.shape[0]), float(perplexity),
                              ptr(out), ptr(idx), ptr(dist), current_stream(device)))
    if host:
        out = out.cpu().numpy()
        if return_neighbors:
            idx, dist = idx.cpu().numpy(), dist.cpu().numpy()
    return (out, idx, dist) if return_neighbors else out


def _missing(a):
    if a.dtype.kind == "f":
        return bool(np.isnan(a).any())
    if a.dtype.kind == "O":
        return any(v is None or (isinstance(v, float) and v != v) or type(v).__name__ in ("NAType", "NaTType") for v in a)
    return False


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
    from .ui import _as_columns, _label_device
    on_device = is_cuda_tensor(X)
    X = _check_rows(X)
    N = X.shape[0]
    neighbours_for(perplexity, N)
    names = [label_colnames] if isinstance(label_colnames, str) else list(label_colnames)
    if not names:
        raise ValueError("label_colnames names no column")
    if not isinstance(meta_data, dict) and not hasattr(meta_data, "columns"):
        raise ValueError("meta_data must be a DataFrame or a dict of columns")
    cols, _ = _as_columns(meta_data, ())
    for v in names:
        if v not in cols:
            raise ValueError(f"meta_data has no column {v!r}")
        if cols[v].ndim != 1 or len(cols[v]) != N:
            raise ValueError(f"column {v!r} must hold one label per row of X ({N})")
        if not is_cuda_tensor(cols[v]) and _missing(cols[v]):
            raise ValueError(f"column {v!r} holds missing labels")
    _label_device(cols, names, X, on_device)
    device = resolve_device(device, X, "X")
    from .harmony import harmony  # needs the CUDA extension; fails loudly when it is missing
    obj = harmony(device=device)
    codes = [factorise(cols[v], X.device if on_device else None)[1] for v in names]
    if on_device:
        import torch
        codes = torch.stack(codes)
    else:
        codes = np.stack(codes)
    return lisi_on(obj, X, codes, perplexity, return_neighbors)
