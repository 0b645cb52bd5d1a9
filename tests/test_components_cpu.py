"""hb_graph_components without a GPU: the scipy restatement against a literal one-edge-at-a-time union-find, the fold
against a literal transcription of scib's graph_connectivity loop, and the Python refusals before the library loads."""
import numpy as np
import pytest
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import connected_components

import components_restatement as cr
from harmony_b200 import graph_components, graph_connectivity
from harmony_b200.graph import connectivity_fold


def union_find(idx, labels=None):
    """One edge at a time, the textbook way: comp = smallest row of each set, largest per label."""
    N, k = idx.shape
    parent = list(range(N))

    def find(v):
        while parent[v] != v:
            v = parent[v]
        return v

    for i in range(N):
        for m in range(k):
            j = int(idx[i, m])
            if j < 0 or j == i or (labels is not None and labels[i] != labels[j]):
                continue
            a, b = find(i), find(j)
            if a != b:
                parent[max(a, b)] = min(a, b)
    comp = np.array([find(v) for v in range(N)], np.int32)
    n_labels = 1 if labels is None else int(max(labels)) + 1
    largest = np.zeros(n_labels, np.int32)
    for r in set(comp.tolist()):
        size = int((comp == r).sum())
        lab = 0 if labels is None else labels[r]
        largest[lab] = max(largest[lab], size)
    return comp, largest


def random_graph(rng, N, k):
    """Sparse random lists with -1 entries, self entries and repeated entries."""
    idx = rng.integers(0, N, (N, k))
    idx[rng.random((N, k)) < 0.5] = -1
    self_rows = rng.random(N) < 0.1
    idx[self_rows, 0] = np.nonzero(self_rows)[0]
    if k > 1:
        idx[:, -1] = np.where(rng.random(N) < 0.2, idx[:, 0], idx[:, -1])
    return idx.astype(np.int32)


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("labelled", [False, True])
def test_restatement_is_union_find(seed, labelled):
    rng = np.random.default_rng(seed)
    N, k = int(rng.integers(1, 300)), int(rng.integers(1, 6))
    idx = random_graph(rng, N, k)
    labels = rng.integers(0, 4, N) if labelled else None
    comp, largest = cr.components(idx, labels, 4 if labelled else None)
    want_comp, want_largest = union_find(idx, labels)
    np.testing.assert_array_equal(comp, want_comp)
    np.testing.assert_array_equal(largest[:len(want_largest)], want_largest)
    assert (largest[len(want_largest):] == 0).all()    # codes no row has
    assert (comp <= np.arange(N)).all()


def test_restatement_edge_cases():
    comp, largest = cr.components(np.full((5, 3), -1, np.int32))         # no edges: singletons
    assert (comp == np.arange(5)).all() and largest.tolist() == [1]
    comp, largest = cr.components(np.arange(5, dtype=np.int32)[:, None])  # self entries only
    assert (comp == np.arange(5)).all() and largest.tolist() == [1]
    path = np.array([[1], [2], [3], [4], [-1]], np.int32)
    comp, largest = cr.components(path, np.arange(5) % 2, 2)             # every edge cut by the labels
    assert (comp == np.arange(5)).all() and largest.tolist() == [1, 1]
    comp, largest = cr.components(path[::-1].copy() * 0 + 4)             # a star on the last row, listed one way
    assert (comp == 0).all() and largest.tolist() == [5]


def scib_graph_connectivity(idx, labels):
    """scib.metrics.graph_connectivity as published, with the AnnData parts spelled out: the symmetric connectivities
    of the neighbour lists, each category's subgraph, its strongly connected components, value_counts().max() / sum."""
    N, k = idx.shape
    rows = np.repeat(np.arange(N), k)
    cols = idx.reshape(-1)
    ok = cols >= 0
    conn = csr_matrix((np.ones(int(ok.sum())), (rows[ok], cols[ok])), shape=(N, N))
    conn = ((conn + conn.T) > 0).astype(np.float64)
    conn.setdiag(0)
    clust_res = []
    for label in sorted(set(labels.tolist())):                 # adata.obs[label_key].cat.categories
        sub = np.nonzero(labels == label)[0]
        _, comp_labels = connected_components(conn[sub][:, sub], connection="strong")
        tab = np.bincount(comp_labels)                         # pd.value_counts(labels)
        tab = tab[tab > 0]
        clust_res.append(tab.max() / sum(tab))
    return np.mean(clust_res)


@pytest.mark.parametrize("seed", range(4))
def test_fold_is_scib(seed):
    rng = np.random.default_rng(100 + seed)
    N, k = 400, 4
    idx = random_graph(rng, N, k)
    labels = rng.integers(0, 5, N)
    labels[labels == 3] = 4                                    # a code no row has
    _, largest = cr.components(idx, labels, 5)
    counts = np.bincount(labels, minlength=5)
    want = scib_graph_connectivity(idx, labels)
    assert cr.connectivity_fold(largest, counts) == pytest.approx(want, abs=1e-12)
    assert connectivity_fold(largest, counts) == pytest.approx(want, abs=1e-12)


def test_knn_restatement_leaves_out_non_finite_rows():
    rng = np.random.default_rng(7)
    X = rng.standard_normal((200, 3))
    X[[4, 50]] = np.nan
    idx = cr.knn_idx(X, 6)
    assert idx.shape == (200, 5) and (idx[[4, 50]] == -1).all() and not np.isin(idx, [4, 50]).any()
    assert (idx != np.arange(200)[:, None]).all()
    comp, _ = cr.components(idx)
    assert comp[4] == 4 and comp[50] == 50 and (comp == comp[4]).sum() == 1


def test_refusals_need_no_device(monkeypatch):
    from harmony_b200 import _lib
    monkeypatch.setattr(_lib, "lib", lambda: pytest.fail("the library was loaded"))
    rng = np.random.default_rng(8)
    X = rng.standard_normal((50, 4))
    t = rng.integers(0, 3, 50)
    idx = rng.integers(-1, 50, (50, 4)).astype(np.int32)
    meta = {"type": t}
    nn = "n_neighbors = {} is not supported here (2 <= n_neighbors <= {}: at most 65, and the N = {} rows)"
    calls = [(graph_components, dict(idx=idx[:, 0]), ValueError, "idx must be an [N, k] matrix with N, k >= 1, not (50,)"),
             (graph_components, dict(idx=idx[:, :0]), ValueError,
              "idx must be an [N, k] matrix with N, k >= 1, not (50, 0)"),
             (graph_components, dict(idx=np.zeros((0, 3), np.int32)), ValueError,
              "idx must be an [N, k] matrix with N, k >= 1, not (0, 3)"),
             (graph_components, dict(idx=idx.astype(np.float32)), TypeError, "idx must be integers, not float32"),
             (graph_components, dict(idx=np.where(idx == 0, -2, idx)), ValueError,
              "idx entries must be -1 or rows in 0..49"),
             (graph_components, dict(idx=np.where(idx == 0, 50, idx)), ValueError,
              "idx entries must be -1 or rows in 0..49"),
             (graph_components, dict(idx=idx, labels=t[:49]), ValueError, "labels must hold one label per row of idx (50)"),
             (graph_components, dict(idx=idx, labels=np.where(t == 1, np.nan, t)), ValueError,
              "labels holds missing labels"),
             (graph_connectivity, dict(X=X[:, 0], meta_data=meta, label_key="type"), ValueError,
              "X must be an [N, d] matrix"),
             (graph_connectivity, dict(X=np.zeros((50, 129)), meta_data=meta, label_key="type"), ValueError,
              "d = 129 is not supported (1 <= d <= 128)"),
             (graph_connectivity, dict(X=X, meta_data=meta, label_key="type", n_neighbors=1), ValueError,
              nn.format(1, 50, 50)),
             (graph_connectivity, dict(X=X, meta_data=meta, label_key="type", n_neighbors=51), ValueError,
              nn.format(51, 50, 50)),
             (graph_connectivity, dict(X=np.zeros((100, 4)), meta_data={"type": np.zeros(100)}, label_key="type",
                                       n_neighbors=66), ValueError, nn.format(66, 65, 100)),
             (graph_connectivity, dict(X=X, meta_data=meta, label_key="type", n_neighbors=2.5), ValueError,
              "n_neighbors must be an integer, not 2.5"),
             (graph_connectivity, dict(X=X, meta_data=meta, label_key="type", n_neighbors=True), ValueError,
              "n_neighbors must be an integer, not True"),
             (graph_connectivity, dict(X=X, meta_data=meta, label_key="nope"), ValueError,
              "meta_data has no column 'nope'"),
             (graph_connectivity, dict(X=X, meta_data=t, label_key="type"), ValueError,
              "meta_data must be a DataFrame or a dict of columns"),
             (graph_connectivity, dict(X=X, meta_data={"type": t[:49]}, label_key="type"), ValueError,
              "column 'type' must hold one label per row of X (50)")]
    for f, kw, exc, msg in calls:
        with pytest.raises(exc) as e:
            f(**kw)
        assert e.type is exc and str(e.value) == msg, (f.__name__, kw, str(e.value))
