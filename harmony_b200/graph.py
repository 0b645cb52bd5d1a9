"""Connected components of a neighbour graph, and scib's graph connectivity score (DESIGN.md §12): for each cell type,
whether its cells form one connected piece of the k-nearest-neighbour graph or whether the batches keep them apart.

``graph_components`` runs ``hb_graph_components`` on neighbour lists (``knn``'s ``idx``); ``graph_connectivity`` builds
the graph with ``hb_knn`` and folds the largest component of each label; ``components_on`` (``harmony.graph_components``)
runs on an existing object.  Argument errors are raised before the CUDA library is loaded.
"""
import numpy as np

from ._arrays import (call, codes_on, dense_codes, dense_on, device_of, download, embedding, factorise_for, handle,
                      label_columns, label_vector, ptr, resolve_device, row_layout, rows_on, to_host)
from .utils import is_cuda_tensor

MAX_NEIGHBORS = 65   # hb_knn's k <= 64 other cells, plus the cell itself


def _check_idx(idx):
    """Neighbour lists [N, k]: a CUDA tensor must be int32 (its range is checked on the device); a host array must be
    integers in -1..N-1 -> the same, host arrays as int32."""
    if is_cuda_tensor(idx):
        import torch
        if idx.dtype != torch.int32:
            raise TypeError(f"CUDA idx must be int32, not {idx.dtype}")
    else:
        idx = np.asarray(idx)
        if idx.dtype.kind not in "iu":
            raise TypeError(f"idx must be integers, not {idx.dtype}")
    if idx.ndim != 2 or idx.shape[0] < 1 or idx.shape[1] < 1:
        raise ValueError(f"idx must be an [N, k] matrix with N, k >= 1, not {tuple(idx.shape)}")
    N = idx.shape[0]
    if N >= 2 ** 31:
        raise ValueError(f"N = {N} rows are not supported (N < 2^31)")
    if not is_cuda_tensor(idx):
        if idx.min() < -1 or idx.max() >= N:
            raise ValueError(f"idx entries must be -1 or rows in 0..{N - 1}")
        idx = idx.astype(np.int32, copy=False)
    return idx


def components_on(obj, idx, labels=None):
    """``hb_graph_components`` on an existing ``harmony`` object (any state: the call needs no setup and changes none)
    -> ``(comp, largest)``.  ``idx``: [N, k] int32 neighbour lists, -1 for none (numpy or a CUDA tensor on the object's
    device); ``labels``: dense codes 0..n-1, [N] (numpy or an int32 CUDA tensor), or None for one label."""
    idx = _check_idx(idx)
    N, k = idx.shape
    n_labels = 0
    if labels is not None:
        labels, n_labels = dense_codes(labels, N, "labels")
    import torch
    device = device_of(obj)
    host = not is_cuda_tensor(idx)
    idx, ld = row_layout(codes_on(obj, idx), k)
    labels = dense_on(obj, labels)
    comp = torch.empty(N, dtype=torch.int32, device=device)
    largest = torch.empty(max(n_labels, 1), dtype=torch.int32, device=device)
    call(obj, "hb_graph_components", ptr(idx), ld, int(N), int(k), ptr(labels), int(n_labels), ptr(comp), ptr(largest))
    return tuple(download(host, comp, largest))


def graph_components(idx, labels=None, device=None):
    """The connected components of the neighbour graph ``idx`` [N, k] -> ``(comp, largest)``.  Entry j of row i is the
    undirected edge {i, j}; -1 is no neighbour (``knn``'s fill), and self or repeated entries add nothing.  ``comp``
    [N] int32 is the smallest row of each row's component.  With ``labels`` (any values, one per row) only edges between
    rows of one label count, and ``largest`` [n_levels] int32 holds the size of the largest component of each label in
    the order of the sorted levels; without, ``largest`` is [1], the largest component.  Host ``idx`` in -> numpy out; a
    CUDA ``idx`` (int32) -> CUDA tensors, ordered on the device's current torch stream."""
    idx = _check_idx(idx)
    on_device = is_cuda_tensor(idx)
    codes = None
    if labels is not None:
        if not is_cuda_tensor(labels):
            labels = np.asarray(labels)
        if labels.ndim != 1 or len(labels) != idx.shape[0]:
            raise ValueError(f"labels must hold one label per row of idx ({idx.shape[0]})")
        labels = label_vector(labels, idx.shape[0], "labels")
        if is_cuda_tensor(labels) and not on_device:
            raise ValueError("labels are a CUDA tensor but idx is not: device labels go with a device idx")
        if is_cuda_tensor(labels) and labels.device != idx.device:
            raise ValueError(f"labels are on {labels.device}, idx on {idx.device}")
        codes = factorise_for(labels, idx)[1]
    return components_on(handle(resolve_device(device, idx, "idx")), idx, codes)


def connectivity_fold(largest, counts):
    """scib's fold: the mean over the labels with rows of (largest component) / (rows of the label)."""
    largest, counts = np.asarray(largest, np.float64), np.asarray(counts, np.float64)
    present = counts > 0
    return float(np.mean(largest[present] / counts[present]))


def graph_connectivity(X, meta_data, label_key, n_neighbors=15, device=None, return_all=False):
    """Graph connectivity, scib's ``graph_connectivity``: for each label of ``meta_data[label_key]`` (a cell type), the
    share of its cells in the largest connected component of its cells' subgraph of the ``n_neighbors`` nearest
    neighbour graph of ``X`` [N, d], averaged over the labels -> a float in (0, 1], 1 when no cell type is split.  With
    ``return_all`` also ``{label: share}``.

    ``n_neighbors`` counts the cell itself, as scanpy's does: the graph is ``knn`` of ``X`` against itself with
    ``n_neighbors - 1`` others, exact and Euclidean, 2 <= n_neighbors <= 65.  A row with a non-finite value has no
    neighbours and is nobody's neighbour: a component of its own.  ``meta_data`` as ``compute_lisi`` takes it.  A CUDA
    ``X`` (float32 / float64) stays on its device until the final fold; d <= 128."""
    X = embedding(X, "X")
    N = X.shape[0]
    if isinstance(n_neighbors, bool) or int(n_neighbors) != n_neighbors:
        raise ValueError(f"n_neighbors must be an integer, not {n_neighbors!r}")
    if not 2 <= n_neighbors <= min(MAX_NEIGHBORS, N):
        raise ValueError(f"n_neighbors = {n_neighbors} is not supported here (2 <= n_neighbors <= "
                         f"{min(MAX_NEIGHBORS, N)}: at most {MAX_NEIGHBORS}, and the N = {N} rows)")
    (labels,) = label_columns(meta_data, [label_key], X)
    obj = handle(resolve_device(device, X, "X"))
    from .neighbors import knn_on
    levels, codes = factorise_for(labels, X)
    _, x, _ = rows_on(obj, X, "X")
    idx, _ = knn_on(obj, x, None, int(n_neighbors) - 1)
    codes = codes_on(obj, codes)
    _, largest = components_on(obj, idx, codes)
    import torch
    counts = torch.bincount(codes.long(), minlength=len(levels)).cpu().numpy()
    largest = largest.cpu().numpy()
    score = connectivity_fold(largest, counts)
    if not return_all:
        return score
    levels = to_host(levels)
    return score, {(v.item() if hasattr(v, "item") else v): float(largest[i] / counts[i]) for i, v in enumerate(levels)}
