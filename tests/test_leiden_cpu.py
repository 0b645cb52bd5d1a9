"""CPU checks of DESIGN §16: the restatement's connectivities against a loop transcription of umap's, its Leiden
against networkx, the resolution choice of nmi_ari_cluster_labels_leiden, and the Python refusals (no library)."""
import math

import networkx as nx
import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components

import leiden_restatement as lr
from harmony_b200 import community as L


def _knn(X, k):
    d = np.sqrt(((X[:, None] - X[None]) ** 2).sum(-1))
    np.fill_diagonal(d, np.inf)
    idx = np.argsort(d, axis=1, kind="stable")[:, :k]
    return idx.astype(np.int32), np.take_along_axis(d, idx, 1).astype(np.float32)


def _umap_loops(idx, dist, n_neighbors):
    """umap's smooth_knn_dist / compute_membership_strengths / fuzzy union, one loop at a time, self column prepended."""
    N, k = idx.shape
    D = np.concatenate([np.zeros((N, 1)), dist.astype(np.float64)], 1)
    I = np.concatenate([np.arange(N)[:, None], idx], 1)
    target = math.log2(n_neighbors)
    mean_distances = D.mean()
    rows, cols, vals = [], [], []
    for i in range(N):
        ith = D[i]
        nz = ith[ith > 0.0]
        rho = nz[0] if nz.shape[0] >= 1 else 0.0
        lo, hi, mid = 0.0, np.inf, 1.0
        for _ in range(64):
            psum = 0.0
            for j in range(1, D.shape[1]):
                d = D[i, j] - rho
                psum += np.exp(-(d / mid)) if d > 0 else 1.0
            if abs(psum - target) < 1e-5:
                break
            if psum > target:
                hi = mid
                mid = (lo + hi) / 2.0
            else:
                lo = mid
                mid = mid * 2 if hi == np.inf else (lo + hi) / 2.0
        s = mid
        if rho > 0.0:
            s = max(s, 1e-3 * ith.mean())
        else:
            s = max(s, 1e-3 * mean_distances)
        for j in range(D.shape[1]):
            if I[i, j] == i:
                v = 0.0
            elif D[i, j] - rho <= 0.0 or s == 0.0:
                v = 1.0
            else:
                v = np.exp(-((D[i, j] - rho) / s))
            rows.append(i)
            cols.append(I[i, j])
            vals.append(v)
    W = sp.coo_matrix((vals, (rows, cols)), shape=(N, N)).tocsr()
    W.eliminate_zeros()
    P = W + W.T - W.multiply(W.T)
    P = sp.csr_matrix(P)
    P.eliminate_zeros()
    P.sort_indices()
    return P


def test_connectivities_match_umap_loops():
    rng = np.random.default_rng(0)
    X = rng.normal(size=(120, 5))
    idx, dist = _knn(X, 9)
    P, Q = lr.umap_graph(idx, dist, 10), _umap_loops(idx, dist, 10)
    assert (P.indptr == Q.indptr).all() and (P.indices == Q.indices).all()
    np.testing.assert_allclose(P.data, Q.data, rtol=1e-12, atol=0)


def planted(n_blocks, size, p_in, p_out, seed, weighted=False):
    rng = np.random.default_rng(seed)
    N = n_blocks * size
    b = np.arange(N) // size
    P = np.where(b[:, None] == b[None], p_in, p_out)
    U = np.triu(rng.random((N, N)) < P, 1)
    W = U * (rng.integers(1, 5, (N, N)) if not weighted else rng.random((N, N)) + 0.1)
    A = sp.csr_matrix(W + W.T)
    A.sort_indices()
    return A


def _graphs():
    yield "karate", sp.csr_matrix(nx.to_scipy_sparse_array(nx.karate_club_graph(), weight="weight", dtype=float))
    yield "planted", planted(6, 40, 0.3, 0.01, 1)
    yield "planted_w", planted(8, 30, 0.25, 0.02, 2, weighted=True)
    rng = np.random.default_rng(3)
    X = np.concatenate([rng.normal(c, 1.0, (60, 8)) for c in range(0, 40, 8)])
    idx, dist = _knn(X, 14)
    yield "knn", lr.umap_graph(idx, dist, 15)


def _nx(A):
    return nx.from_scipy_sparse_array(sp.csr_matrix(A), edge_attribute="weight")


@pytest.mark.parametrize("name,A", list(_graphs()), ids=[g[0] for g in _graphs()])
def test_restatement_properties(name, A):
    labels, nc, Q, iters, near, _ = lr.leiden(A, 1.0)
    G = _nx(A)
    parts = [set(np.flatnonzero(labels == c)) for c in range(nc)]
    assert abs(Q - nx.community.modularity(G, parts, weight="weight", resolution=1.0)) <= 1e-12
    for c in range(nc):
        m = np.flatnonzero(labels == c)
        assert connected_components(A[m][:, m], directed=False)[0] == 1
    assert lr.improving_move(A, labels, 1.0) <= 1e-12 * abs(Q)
    best = max(nx.community.modularity(G, nx.community.louvain_communities(G, weight="weight", seed=s), weight="weight")
               for s in range(3))
    # measured: karate 0.969, the planted and kNN graphs 1.000-1.001 of networkx's best Louvain (DESIGN §16)
    assert Q >= (0.96 if name == "karate" else 0.99) * best, (Q, best)


def test_resolution_choice():
    got = L.best_resolution([(0.3, 0.8, 0.7), (0.1, 0.9, 0.5), (0.2, 0.9, 0.6)])
    assert got == {"nmi": 0.9, "ari": 0.5, "resolution": 0.1}
    assert L.SCIB_RESOLUTIONS[0] == 0.1 and L.SCIB_RESOLUTIONS[-1] == 2.0 and len(L.SCIB_RESOLUTIONS) == 20


def test_cell_lines_pinned():
    import os
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "cell_lines.npz"), allow_pickle=True)
    X = np.asarray(z["scaled_pcs"], np.float64)
    ct = np.asarray(z["cell_type"])
    idx, dist = _knn(X, 14)
    A = lr.umap_graph(idx, dist, 15)
    labels = lr.leiden(A, 1.0)[0]
    from harmony_b200.clustering import nmi_ari
    nmi, ari = nmi_ari(ct, labels)
    assert labels.max() + 1 == 11
    assert abs(nmi - 0.45222666200200246) <= 1e-12 and abs(ari - 0.19859704227135855) <= 1e-12


@pytest.mark.parametrize("kw,msg", [
    (dict(resolution=0.0), "resolution"), (dict(resolution=float("nan")), "resolution"),
    (dict(n_iterations=-2), "n_iterations"), (dict(n_neighbors=1), "n_neighbors"), (dict(n_neighbors=66), "n_neighbors"),
])
def test_refusals_before_the_library(kw, msg, monkeypatch):
    import harmony_b200._lib as lib
    monkeypatch.setattr(lib, "lib", lambda: (_ for _ in ()).throw(AssertionError("library loaded")))
    with pytest.raises(ValueError, match=msg):
        L.leiden(np.zeros((100, 3)), **kw)


def test_graph_refusals_before_the_library():
    with pytest.raises(ValueError, match="square"):
        L.leiden(sp.csr_matrix(np.ones((2, 3))))
    with pytest.raises(ValueError, match="CUDA triple"):
        L.leiden((1, 2))
    with pytest.raises(ValueError, match="d = "):
        L.umap_connectivities(np.zeros((5, 0)))
