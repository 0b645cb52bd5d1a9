"""UMAP connectivities of a neighbour graph and deterministic Leiden clustering (DESIGN.md §16): scanpy's
``neighbors`` -> ``leiden`` on the GPU, and scib's ``nmi_ari_cluster_labels_leiden``, which keeps the best NMI over a
sweep of resolutions.

``umap_connectivities`` builds the symmetric CSR of an embedding's exact neighbour graph (``hb_knn`` then
``hb_umap_graph``); ``leiden`` clusters an embedding or a graph (``hb_leiden``); ``umap_on`` / ``leiden_on``
(``harmony.umap_connectivities`` / ``harmony.leiden``) run on an existing object.  Argument errors are raised before the
CUDA library is loaded.
"""
import ctypes
import math

import numpy as np

from ._arrays import DTYPE, call, device_of, embedding, handle, label_columns, ptr, resolve_device, rows_on
from .clustering import nmi_ari
from .utils import is_cuda_tensor

MAX_NEIGHBORS = 65   # hb_knn's k <= 64 other cells, plus the cell itself
SCIB_RESOLUTIONS = tuple(round(0.1 * i, 1) for i in range(1, 21))


def _n_neighbors(n_neighbors, N):
    if isinstance(n_neighbors, bool) or not isinstance(n_neighbors, (int, np.integer)):
        raise ValueError(f"n_neighbors must be an integer, not {n_neighbors!r}")
    if not 2 <= n_neighbors <= min(MAX_NEIGHBORS, max(N, 2)):
        raise ValueError(f"n_neighbors = {n_neighbors} is not supported here (2 <= n_neighbors <= "
                         f"{min(MAX_NEIGHBORS, max(N, 2))}: at most {MAX_NEIGHBORS}, and the N = {N} rows)")
    return int(n_neighbors)


def _resolution(r):
    if isinstance(r, bool) or not isinstance(r, (int, float, np.integer, np.floating)) or not (
            math.isfinite(r) and r > 0):
        raise ValueError(f"resolution must be a finite number > 0, not {r!r}")
    return float(r)


def _n_iterations(n):
    if isinstance(n, bool) or not isinstance(n, (int, np.integer)) or n < -1 or n >= 2 ** 31:
        raise ValueError(f"n_iterations must be -1 (until no label changes) or an integer >= 0, not {n!r}")
    return int(n)


def _check_graph(G):
    """A graph: a scipy sparse matrix (host) or a CUDA triple (indptr int64, indices int32, data fp32 / fp64) ->
    ('host', csr) or ('cuda', (indptr, indices, data)).  Symmetry, order and diagonal are checked on the device."""
    if isinstance(G, tuple):
        if len(G) != 3 or not all(is_cuda_tensor(t) for t in G):
            raise ValueError("a device graph is the CUDA triple (indptr, indices, data)")
        import torch
        indptr, indices, data = G
        if indptr.dtype != torch.int64 or indices.dtype != torch.int32 or data.dtype not in (torch.float32,
                                                                                            torch.float64):
            raise TypeError("a device graph needs int64 indptr, int32 indices and float32 / float64 data")
        if indptr.ndim != 1 or indices.ndim != 1 or data.ndim != 1 or indptr.numel() < 2 or \
                indices.numel() != data.numel():
            raise ValueError("indptr must be [N + 1] with N >= 1, and indices and data of one length")
        if len({indptr.device, indices.device, data.device}) != 1:
            raise ValueError("indptr, indices and data must be on one device")
        return "cuda", (indptr.contiguous(), indices.contiguous(), data.contiguous())
    import scipy.sparse as sp
    if not sp.issparse(G):
        raise ValueError("a graph must be a scipy sparse matrix or the CUDA triple (indptr, indices, data)")
    if G.shape[0] != G.shape[1] or G.shape[0] < 1:
        raise ValueError(f"a graph must be square with at least one row, not {G.shape}")
    G = sp.csr_matrix(G, copy=True)
    if G.dtype not in (np.float32, np.float64):
        G = G.astype(np.float64)
    G.sum_duplicates()   # a canonical copy: sorted rows, no repeated or explicitly stored zero entry
    G.eliminate_zeros()
    G.sort_indices()
    return "host", G


def umap_graph_on(obj, idx, dist, n_neighbors):
    """``hb_umap_graph`` of CUDA neighbour lists ``idx`` / ``dist`` [N, k] -> the CUDA triple (indptr, indices, data)."""
    import torch
    device = device_of(obj)
    N, k = idx.shape
    idx, dist = idx.contiguous(), dist.contiguous()
    indptr = torch.empty(N + 1, dtype=torch.int64, device=device)
    indices = torch.empty(max(2 * N * k, 1), dtype=torch.int32, device=device)
    data = torch.empty(max(2 * N * k, 1), dtype=torch.float32, device=device)
    nnz = ctypes.c_int64(0)
    call(obj, "hb_umap_graph", ptr(idx), int(k), ptr(dist), int(k), int(N), int(k), int(n_neighbors), ptr(indptr),
         ptr(indices), ptr(data), ctypes.byref(nnz))
    return indptr, indices[:nnz.value], data[:nnz.value]


def _graph_of(obj, X, n_neighbors):
    """An embedding -> (whether it came from the host, the device CSR triple, the finite rows)."""
    from .neighbors import knn_on
    host, x, _ = rows_on(obj, X, "X")
    import torch
    if x.shape[0] < 2:
        indptr = torch.zeros(x.shape[0] + 1, dtype=torch.int64, device=x.device)
        empty = torch.empty(0, dtype=torch.int32, device=x.device)
        return host, (indptr, empty, empty.float()), torch.isfinite(x).all(dim=1)
    idx, dist = knn_on(obj, x, None, n_neighbors - 1)
    return host, umap_graph_on(obj, idx, dist, n_neighbors), torch.isfinite(x).all(dim=1)


def umap_on(obj, X, n_neighbors=15):
    """``umap_connectivities`` on an existing ``harmony`` object (any state: the call needs no setup and changes none)."""
    X = embedding(X, "X")
    n_neighbors = _n_neighbors(n_neighbors, X.shape[0])
    host, (indptr, indices, data), _ = _graph_of(obj, X, n_neighbors)
    if not host:
        return indptr, indices, data
    import scipy.sparse as sp
    N = X.shape[0]
    return sp.csr_matrix((data.cpu().numpy(), indices.cpu().numpy(), indptr.cpu().numpy()), shape=(N, N))


def umap_connectivities(X, n_neighbors=15, device=None):
    """scanpy's ``obsp["connectivities"]`` of ``X`` [N, d] (d <= 128): the exact Euclidean ``n_neighbors`` graph (the
    cell itself counted, 2 <= n_neighbors <= 65) through umap-learn's ``fuzzy_simplicial_set`` in fp64, weights fp32.
    Host ``X`` -> a ``scipy.sparse.csr_matrix``; a CUDA ``X`` -> the CUDA triple (indptr int64, indices int32, data
    float32), rows ascending.  A row with a non-finite value has no edges."""
    X = embedding(X, "X")
    _n_neighbors(n_neighbors, X.shape[0])
    return umap_on(handle(resolve_device(device, X, "X")), X, n_neighbors)


def leiden_graph_on(obj, graph, resolution=1.0, n_iterations=-1, return_info=False):
    """``hb_leiden`` of a device CSR triple -> int32 labels on the device (with ``return_info`` also
    ``{"n_communities", "quality", "iterations", "levels", "sweeps", "rounds"}``)."""
    import torch
    indptr, indices, data = graph
    N = indptr.numel() - 1
    labels = torch.empty(N, dtype=torch.int32, device=device_of(obj))
    n_comm, q, iters = ctypes.c_int(0), ctypes.c_double(0.0), ctypes.c_int(0)
    stats = (ctypes.c_int64 * 3)()
    call(obj, "hb_leiden", ptr(indptr), ptr(indices if indices.numel() else None), ptr(data if data.numel() else None),
         DTYPE[str(data.dtype)[6:]], int(N), int(indices.numel()), float(resolution), int(n_iterations), ptr(labels),
         ctypes.byref(n_comm), ctypes.byref(q), ctypes.byref(iters), stats)
    info = {"n_communities": n_comm.value, "quality": q.value, "iterations": iters.value, "levels": stats[0],
            "sweeps": stats[1], "rounds": stats[2]}
    return (labels, info) if return_info else labels


def _compact(labels, keep):
    """Labels with the rows outside ``keep`` set to -1 and the rest renumbered 0.. in their order (they were numbered by
    size, so the order stays)."""
    import torch
    out = torch.full_like(labels, -1)
    if bool(keep.any()):
        out[keep] = torch.unique(labels[keep], sorted=True, return_inverse=True)[1].to(torch.int32)
    return out


def leiden_on(obj, X_or_graph, resolution=1.0, n_neighbors=15, n_iterations=-1, return_info=False):
    """``leiden`` on an existing ``harmony`` object (any state: the call needs no setup and changes none)."""
    resolution = _resolution(resolution)
    n_iterations = _n_iterations(n_iterations)
    import scipy.sparse as sp
    if isinstance(X_or_graph, tuple) or sp.issparse(X_or_graph):
        where, G = _check_graph(X_or_graph)
        import torch
        if where == "host":
            dev = device_of(obj)
            G = (torch.as_tensor(G.indptr.astype(np.int64)).to(dev), torch.as_tensor(G.indices.astype(np.int32)).to(dev),
                 torch.as_tensor(G.data).to(dev))
        out = leiden_graph_on(obj, G, resolution, n_iterations, True)
        labels = out[0].cpu().numpy() if where == "host" else out[0]
        return (labels, out[1]) if return_info else labels
    X = embedding(X_or_graph, "X")
    n_neighbors = _n_neighbors(n_neighbors, X.shape[0])
    host, G, finite = _graph_of(obj, X, n_neighbors)
    labels, info = leiden_graph_on(obj, G, resolution, n_iterations, True)
    if not bool(finite.all()):
        labels = _compact(labels, finite)
        info["n_communities"] = int(labels.max()) + 1 if bool(finite.any()) else 0
    labels = labels.cpu().numpy() if host else labels
    return (labels, info) if return_info else labels


def _check_input(X_or_graph):
    import scipy.sparse as sp
    if isinstance(X_or_graph, tuple) or sp.issparse(X_or_graph):
        where, G = _check_graph(X_or_graph)
        return G[0].device.index if where == "cuda" else None, True
    X = embedding(X_or_graph, "X")
    return (X.device.index if is_cuda_tensor(X) else None), False


def leiden(X_or_graph, resolution=1.0, n_neighbors=15, n_iterations=-1, return_info=False, device=None):
    """Deterministic Leiden communities (modularity with resolution γ, scanpy's default partition type) -> int32
    labels numbered by decreasing community size, ties by the smallest member row.  Takes an embedding [N, d] (the
    ``umap_connectivities`` graph is built on the device; a row with a non-finite value gets -1) or a symmetric graph
    without diagonal: a scipy sparse matrix, or the CUDA triple (indptr int64, indices int32, data fp32 / fp64); a
    vertex without edges is a community of its own.  ``n_iterations`` -1 repeats until no label changes.  Host input ->
    numpy labels; CUDA input -> a CUDA tensor.  With ``return_info`` also the number of communities, Q, iterations,
    levels, sweeps and refinement rounds."""
    _resolution(resolution)
    _n_iterations(n_iterations)
    dev, is_graph = _check_input(X_or_graph)
    if not is_graph:
        X_or_graph = embedding(X_or_graph, "X")
        _n_neighbors(n_neighbors, X_or_graph.shape[0])
    if device is not None and dev is not None and int(device) != dev:
        raise ValueError(f"device={device} differs from the input's device (cuda:{dev})")
    return leiden_on(handle(dev if dev is not None else device), X_or_graph, resolution, n_neighbors, n_iterations,
                     return_info)


def best_resolution(scores):
    """scib's choice over ``[(resolution, nmi, ari)]``: the highest NMI, the lower resolution on a tie ->
    ``{"nmi", "ari", "resolution"}``."""
    best = None
    for r, nmi, ari in sorted(scores, key=lambda t: t[0]):
        if best is None or nmi > best[1]:
            best = (r, nmi, ari)
    return {"nmi": best[1], "ari": best[2], "resolution": best[0]}


def nmi_ari_cluster_labels_leiden(X, meta_data, label_key, resolutions=None, n_neighbors=15, device=None):
    """scib's ``nmi_ari_cluster_labels_leiden``: the neighbour graph of ``X`` is built once, Leiden runs at each
    resolution (scib's grid 0.1, 0.2, ..., 2.0 by default), and the clustering with the highest NMI against
    ``meta_data[label_key]`` (the lower resolution on a tie) gives ``{"nmi", "ari", "resolution"}`` (``nmi_ari``)."""
    X = embedding(X, "X")
    labels = label_columns(meta_data, [label_key], X)[0]
    n_neighbors = _n_neighbors(n_neighbors, X.shape[0])
    resolutions = SCIB_RESOLUTIONS if resolutions is None else tuple(_resolution(r) for r in resolutions)
    if not resolutions:
        raise ValueError("resolutions is empty")
    obj = handle(resolve_device(device, X, "X"))
    host, G, finite = _graph_of(obj, X, n_neighbors)
    scores = []
    for r in resolutions:
        pred = leiden_graph_on(obj, G, r, -1)
        if not bool(finite.all()):
            pred = _compact(pred, finite)
        pred = pred.cpu().numpy() if host else pred
        scores.append((r, *nmi_ari(labels, pred)))
    return best_resolution(scores)
