"""hb_graph_components restated (DESIGN §12): scipy's connected components of the kept edges, each component named by
its smallest row, and scib's fold of the largest components into graph connectivity."""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components


def kept_edges(idx, labels=None):
    """The (i, j) entries of idx [N, k] that are edges: not -1, not i itself and, with labels, within one label."""
    idx = np.asarray(idx)
    N, k = idx.shape
    i = np.repeat(np.arange(N, dtype=np.int32), k)   # int32: the 4M x 14 case keeps to a few hundred MB
    j = idx.reshape(-1).astype(np.int32)
    keep = (j >= 0) & (j != i)
    if labels is not None:
        labels = np.asarray(labels)
        keep &= labels[i] == labels[np.clip(j, 0, None)]
    return i[keep], j[keep]


def components(idx, labels=None, n_labels=None):
    """-> (comp [N] int32: the smallest row of each row's component, largest [n_labels] int32: the largest component
    among the rows of each label, 0 for a code no row has; [1] without labels)."""
    N = np.asarray(idx).shape[0]
    i, j = kept_edges(idx, labels)
    A = coo_matrix((np.ones(len(i), np.int8), (i, j)), shape=(N, N)).tocsr()
    n, lab = connected_components(A, directed=False)
    first = np.full(n, N, np.int64)
    np.minimum.at(first, lab, np.arange(N))
    comp = first[lab].astype(np.int32)
    size = np.bincount(lab, minlength=n)
    if labels is None:
        return comp, np.array([size.max()], np.int32)
    labels = np.asarray(labels)
    largest = np.zeros(n_labels if n_labels is not None else int(labels.max()) + 1, np.int64)
    np.maximum.at(largest, labels[first], size)
    return comp, largest.astype(np.int32)


def connectivity_fold(largest, counts):
    """scib's graph connectivity from each label's largest component and its rows: the mean over the labels with rows."""
    largest, counts = np.asarray(largest, np.float64), np.asarray(counts)
    present = counts > 0
    return float((largest[present] / counts[present]).mean())


def knn_idx(X, n_neighbors):
    """Exact Euclidean neighbour lists [N, n_neighbors - 1] in fp64 (cKDTree), the row itself left out; rows with a
    non-finite value have none (-1) and are nobody's neighbour."""
    from scipy.spatial import cKDTree
    X = np.asarray(X, np.float64)
    N, k = X.shape[0], n_neighbors - 1
    fin = np.nonzero(np.isfinite(X).all(axis=1))[0]
    out = np.full((N, k), -1, np.int64)
    m = min(k + 1, len(fin))
    _, nb = cKDTree(X[fin]).query(X[fin], k=m)
    nb = np.asarray(nb).reshape(len(fin), m)
    for r in range(len(fin)):
        row = [fin[v] for v in nb[r] if fin[v] != fin[r]][:k]
        out[fin[r], :len(row)] = row
    return out.astype(np.int32)
