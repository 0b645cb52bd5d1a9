"""Exact k nearest neighbours in an embedding, and label transfer with them (DESIGN.md §9).

``knn`` is the brute-force search of ``hb_knn`` (tensor-core scores, distances recomputed directly in fp32);
``TransferLabels`` is Symphony's ``knnPredict`` on top of it: every query cell takes the majority label of its k nearest
reference cells.  Argument errors are raised before the CUDA library is loaded.
"""
import numpy as np

from ._arrays import call, device_of, download, embedding, factorise, handle, ptr, resolve_device, rows_on
from .utils import is_cuda_tensor

METRIC = {"euclidean": 0, "cosine": 1}   # enum hb_metric
MAX_K = 64


def _check_args(query, ref, k, metric):
    """The refusals that need no device -> (query, ref or None) with host inputs as arrays."""
    if metric not in METRIC:
        raise ValueError(f"metric must be one of {sorted(METRIC)}, not {metric!r}")
    if isinstance(k, bool) or int(k) != k:
        raise ValueError(f"k must be an integer, not {k!r}")
    on_device = is_cuda_tensor(query)
    if ref is not None and is_cuda_tensor(ref) != on_device:
        raise ValueError("query and ref must both be CUDA tensors or both be host arrays")
    if not on_device:
        query = np.asarray(query)
        ref = None if ref is None else np.asarray(ref)
    if query.ndim != 2 or (ref is not None and ref.ndim != 2):
        raise ValueError("query and ref must be [rows, d] matrices")
    nq, d = query.shape
    nx = nq if ref is None else ref.shape[0]
    if ref is not None and ref.shape[1] != d:
        raise ValueError(f"query has {d} dimensions, ref {ref.shape[1]}")
    embedding(query, "query")
    if nq < 1 or nx < 1:
        raise ValueError("query and ref need at least one row")
    limit = min(MAX_K, nx - (1 if ref is None else 0))
    if not 1 <= k <= limit:
        raise ValueError(f"k = {k} is not supported here (1 <= k <= {limit}: at most {MAX_K}, and the "
                         f"{'other rows' if ref is None else 'rows of ref'})")
    return query, ref


def knn_on(obj, query, ref=None, k=15, metric="euclidean"):
    """``knn`` on an existing ``harmony`` object (any state: the search needs no setup and changes none)."""
    query, ref = _check_args(query, ref, k, metric)
    import torch
    device = device_of(obj)
    host, q, q_args = rows_on(obj, query, "query")
    _, x, x_args = (host, q, q_args) if ref is None else rows_on(obj, ref, "ref")
    idx = torch.empty((q.shape[0], int(k)), dtype=torch.int32, device=device)
    dist = torch.empty((q.shape[0], int(k)), dtype=torch.float32, device=device)
    call(obj, "hb_knn", *q_args, q.shape[0], *x_args, x.shape[0], int(q.shape[1]), int(k), METRIC[metric],
         int(ref is None), ptr(idx), ptr(dist))
    return tuple(download(host, idx, dist))


def knn(query, ref=None, k=15, metric="euclidean", device=None):
    """The exact ``k`` nearest rows of ``ref`` for every row of ``query`` -> ``(idx, dist)``, both [Nq, k], each row by
    ascending distance: ``idx`` int32 rows of ``ref``, ``dist`` float32 (Euclidean distance, or 1 - cosine).

    ``ref=None`` searches ``query`` against itself and leaves every row out of its own neighbours (the neighbour graph
    of an embedding).  Host arrays in -> numpy out; CUDA tensors (float32 / float64, both on one device) in -> CUDA
    tensors out, ordered on the device's current torch stream, nothing visiting the host.  1 <= k <= 64, d <= 128.
    Rows with non-finite values have no neighbours and are nobody's neighbour (``idx = -1``, ``dist = inf`` fill a row
    with fewer than k candidates)."""
    query, ref = _check_args(query, ref, k, metric)
    return knn_on(handle(resolve_device(device, query, "query")), query, ref, k, metric)


def vote(idx, dist, codes, n_labels):
    """The label code each row of ``idx`` elects, and its vote share: the code most frequent among ``codes[idx]``;
    among tied codes the one whose nearest member is closest, then the smaller code.  Entries ``idx < 0`` do not vote;
    a row without votes gets code -1 and share 0.  numpy arrays or torch tensors (the work stays where they are)."""
    if is_cuda_tensor(idx):
        import torch
        valid = idx >= 0
        lab = codes[idx.clamp(min=0).long()].long()
        rows = torch.arange(idx.shape[0], device=idx.device)[:, None].expand_as(idx)
        counts = torch.zeros((idx.shape[0], n_labels), dtype=torch.float64, device=idx.device)
        counts.index_put_((rows[valid], lab[valid]), torch.ones((), dtype=torch.float64, device=idx.device), accumulate=True)
        near = torch.full((idx.shape[0], n_labels), float("inf"), dtype=torch.float64, device=idx.device)
        near = near.reshape(-1).scatter_reduce(0, (rows * n_labels + lab)[valid], dist.double()[valid], "amin").reshape(near.shape)
        top = counts.max(dim=1, keepdim=True).values
        near = torch.where(counts == top, near, torch.full_like(near, float("inf")))
        best = (near == near.min(dim=1, keepdim=True).values) & (counts == top)
        code = best.to(torch.int8).argmax(dim=1)          # the first maximum: the smaller code
        total = valid.sum(dim=1)
        share = torch.where(total > 0, top[:, 0] / total.clamp(min=1), torch.zeros_like(top[:, 0]))
        return torch.where(total > 0, code, torch.full_like(code, -1)), share
    idx, dist, codes = np.asarray(idx), np.asarray(dist, dtype=np.float64), np.asarray(codes)
    valid = idx >= 0
    lab = codes[np.clip(idx, 0, None)]
    rows = np.broadcast_to(np.arange(idx.shape[0])[:, None], idx.shape)
    counts = np.zeros((idx.shape[0], n_labels))
    np.add.at(counts, (rows[valid], lab[valid]), 1.0)
    near = np.full((idx.shape[0], n_labels), np.inf)
    np.minimum.at(near, (rows[valid], lab[valid]), dist[valid])
    top = counts.max(axis=1, keepdims=True)
    near = np.where(counts == top, near, np.inf)
    best = (near == near.min(axis=1, keepdims=True)) & (counts == top)
    code = best.argmax(axis=1)
    total = valid.sum(axis=1)
    share = np.where(total > 0, top[:, 0] / np.maximum(total, 1), 0.0)
    return np.where(total > 0, code, -1), share


def TransferLabels(query, ref, ref_labels, k=5, metric="euclidean", return_prob=False, device=None):
    """Symphony's ``knnPredict``: every row of ``query`` gets the majority label of its ``k`` nearest rows of ``ref``
    (both in one embedding, e.g. ``MapQuery``'s output and the reference's ``Z_corr``), and with ``return_prob`` the
    winning label's share of the votes.

    ``ref_labels``: one label per row of ``ref`` — strings, integers, or anything with ``categories`` and ``codes``
    (a pandas Categorical); the result has the same dtype / categories.  With CUDA ``query`` and ``ref`` the vote runs
    on the device and integer CUDA ``ref_labels`` give CUDA labels back.  ``class::knn``, which ``knnPredict`` calls,
    breaks vote ties at random; here the tied label whose nearest member is closest wins, then the smaller code
    (the label earlier in sorted order or in ``categories``)."""
    query, ref = _check_args(query, ref, k, metric)
    if ref is None:
        raise ValueError("TransferLabels needs a reference embedding")
    labels_on_device = is_cuda_tensor(ref_labels)
    if labels_on_device:
        if not is_cuda_tensor(query):
            raise ValueError("ref_labels is a CUDA tensor but the embeddings are not")
        import torch
        if ref_labels.dtype not in (torch.int32, torch.int64) or ref_labels.ndim != 1:
            raise ValueError("CUDA ref_labels must be a 1-d int32 / int64 tensor")
        n_given = ref_labels.shape[0]
    elif hasattr(ref_labels, "categories") and hasattr(ref_labels, "codes"):
        categories, codes = np.asarray(ref_labels.categories), np.asarray(ref_labels.codes, dtype=np.int64)
        if (codes < 0).any():
            raise ValueError("ref_labels holds missing values")
        n_given = len(codes)
    else:
        given = np.asarray(ref_labels)
        if given.ndim != 1:
            raise ValueError("ref_labels must hold one label per row of ref")
        categories, codes = factorise(given)
        n_given = len(given)
    if n_given != ref.shape[0]:
        raise ValueError(f"ref has {ref.shape[0]} rows, ref_labels {n_given} labels")
    idx, dist = knn(query, ref, k, metric, device)
    if labels_on_device:
        categories, codes = factorise(ref_labels)
    elif is_cuda_tensor(idx):
        import torch
        codes = torch.as_tensor(codes, device=idx.device)
    code, share = vote(idx, dist, codes, len(categories))
    if labels_on_device:
        pred = torch.where(code >= 0, categories[code.clamp(min=0)], torch.full_like(code, -1).to(categories.dtype))
    else:
        if is_cuda_tensor(code):
            code, share = code.cpu().numpy(), share.cpu().numpy()
        if (code < 0).any():
            raise ValueError("a query row has no neighbour to vote (non-finite values in the embeddings)")
        pred = categories[code]
        if hasattr(ref_labels, "categories") and hasattr(ref_labels, "from_codes"):
            pred = type(ref_labels).from_codes(code, categories=ref_labels.categories)
    return (pred, share) if return_prob else pred
