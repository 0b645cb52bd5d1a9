"""Silhouette widths of an embedding (DESIGN.md §11): per cell, how much closer it lies to the cells of its own label
than to those of the nearest other label, over all pairs of cells (within a group, when groups are given).  The
scores scib reports as ``silhouette`` (cell-type ASW) and ``silhouette_batch`` (batch ASW within each cell type) are
folds of these per-cell values.

``silhouette_samples`` mirrors ``sklearn.metrics.silhouette_samples`` (with optional groups); ``silhouette_on``
(``harmony.silhouette``) runs ``hb_silhouette`` on an existing object.  Argument errors are raised before the CUDA
library is loaded.
"""
import numpy as np

from ._arrays import (call, check_two_rows, dense_codes, dense_on, device_of, download, embedding, factorise,
                      factorise_for, handle, label_columns, label_device, label_vector, ptr, resolve_device, rows_on,
                      to_host)
from .utils import is_cuda_tensor


def silhouette_on(obj, X, labels, groups=None):
    """``hb_silhouette`` on an existing ``harmony`` object (any state: the call needs no setup and changes none).
    ``labels`` / ``groups``: dense codes 0..n-1 (numpy or int32 CUDA tensors on the object's device)."""
    X = embedding(X, "X")
    N, d = X.shape
    check_two_rows(X)
    labels, n_labels = dense_codes(labels, N, "labels")
    n_groups = 0
    if groups is not None:
        groups, n_groups = dense_codes(groups, N, "groups")
    import torch
    host, x, x_args = rows_on(obj, X, "X")
    labels, groups = dense_on(obj, labels), dense_on(obj, groups)
    out = torch.empty(N, dtype=torch.float64, device=device_of(obj))
    call(obj, "hb_silhouette", *x_args, N, int(d), ptr(labels), int(n_labels), ptr(groups), int(n_groups), ptr(out))
    return download(host, out)[0]


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
    X = embedding(X, "X")
    N = X.shape[0]
    check_two_rows(X)
    cols = {"labels": label_vector(labels, N, "labels")}
    if groups is not None:
        cols["groups"] = label_vector(groups, N, "groups")
    label_device(cols, list(cols), X, on_device)
    device = resolve_device(device, X, "X")
    codes = factorise_for(cols["labels"], X)[1]
    gcodes = factorise_for(cols["groups"], X)[1] if groups is not None else None
    n = _n_levels(codes)
    if groups is None and not 1 < n < N:
        raise ValueError(f"Number of labels is {n}. Valid values are 2 to n_samples - 1 (inclusive)")
    return silhouette_on(handle(device), X, codes, gcodes)


def silhouette_label(X, meta_data, label_key, scale=True):
    """Cell-type ASW, scib's ``silhouette``: the mean silhouette width of ``meta_data[label_key]`` over ``X``,
    scaled to ``(s + 1) / 2`` (1 best) unless ``scale`` is False.  Labels are taken as ``compute_lisi`` takes them."""
    X = embedding(X, "X")
    (labels,) = label_columns(meta_data, [label_key], X)
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
    X = embedding(X, "X")
    batch, label = label_columns(meta_data, [batch_key, label_key], X)
    s = silhouette_samples(X, batch, groups=label)
    asw, means = batch_fold(to_host(s), to_host(batch), to_host(label), scale)
    return (asw, means) if return_all else asw
