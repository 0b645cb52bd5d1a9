"""GPU checks of hb_umap_graph and hb_leiden (DESIGN §16) against the fp64 restatement: exact replays, weighted and
large graphs against networkx and the restatement, the refusals, the handle's state, stream order, the cap's warning
and the NMI / ARI scores end to end."""
import ctypes

import networkx as nx
import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components

import leiden_restatement as lr
from harmony_b200._arrays import ptr
from helpers import gpu_harmony, load_cell_lines, make_Y0, run_oracle
from score_helpers import handle_state_untouched, refusals_launch_nothing, unwritten

pytestmark = pytest.mark.gpu


def _ring_of_cliques(n_cliques, size):
    N = n_cliques * size
    A = np.zeros((N, N))
    for c in range(n_cliques):
        b = c * size
        A[b:b + size, b:b + size] = 1
        A[b, (b + size) % N] = A[(b + size) % N, b] = 1
    np.fill_diagonal(A, 0)
    return sp.csr_matrix(A)


def _planted(n_blocks, size, p_in, p_out, seed, weighted=False):
    rng = np.random.default_rng(seed)
    N = n_blocks * size
    b = np.arange(N) // size
    U = np.triu(rng.random((N, N)) < np.where(b[:, None] == b[None], p_in, p_out), 1)
    W = U * (rng.random((N, N)) + 0.1 if weighted else rng.integers(1, 5, (N, N)))
    return sp.csr_matrix(W + W.T)


def _star(N, hub):
    rows = np.array([hub] * (N - 1))
    cols = np.array([j for j in range(N) if j != hub])
    A = sp.csr_matrix((np.ones(N - 1), (rows, cols)), shape=(N, N))
    return sp.csr_matrix(A + A.T)


def _integer_graphs():
    yield "planted", _planted(5, 40, 0.3, 0.02, 1)
    yield "cliques", _ring_of_cliques(12, 6)
    yield "star0", _star(300, 0)
    yield "starN", _star(300, 299)
    yield "pieces", sp.block_diag([_planted(3, 20, 0.4, 0.05, 2), _ring_of_cliques(4, 5), sp.csr_matrix((7, 7))]).tocsr()
    yield "empty", sp.csr_matrix((10, 10))
    yield "one", sp.csr_matrix((1, 1))


@pytest.mark.parametrize("name,A", list(_integer_graphs()), ids=[g[0] for g in _integer_graphs()])
@pytest.mark.parametrize("gamma", [1.0, 0.3, 2.5])
def test_exact_replay_on_integer_graphs(name, A, gamma):
    from harmony_b200 import leiden
    labels, info = leiden(A, resolution=gamma, return_info=True)
    want, nc, Q, iters, _, stats = lr.leiden(A, gamma)
    np.testing.assert_array_equal(labels, want)
    assert info["n_communities"] == nc and info["iterations"] == iters
    assert info["quality"] == Q  # integer weights: every sum exact, and Q in the same form on both sides
    assert (info["levels"], info["sweeps"], info["rounds"]) == (stats["levels"], stats["sweeps"], stats["rounds"])


def _networkx_checks(A, labels, gamma, Q):
    """Connected communities, no improving single move, Q to networkx's to 1e-9 and the quality bar of §16."""
    G = nx.from_scipy_sparse_array(sp.csr_matrix(A), edge_attribute="weight")
    parts = [set(np.flatnonzero(labels == c)) for c in range(labels.max() + 1)]
    assert lr.connected_communities(A, labels)
    assert lr.improving_move(A, labels, gamma) <= 1e-12 * abs(Q)
    assert abs(nx.community.modularity(G, parts, weight="weight", resolution=gamma) - Q) <= 1e-9
    best = max(nx.community.modularity(G, nx.community.louvain_communities(G, weight="weight", seed=s),
                                       weight="weight", resolution=gamma) for s in range(3))
    assert Q >= 0.99 * best, (Q, best)


@pytest.mark.parametrize("seed", [5, 6, 7])
def test_weighted_graphs(seed):
    from harmony_b200 import leiden
    A = _planted(8, 50, 0.2, 0.02, seed, weighted=True)
    labels, info = leiden(A, return_info=True)
    want, nc, Q, _, near, _ = lr.leiden(A, 1.0)
    if not near:
        np.testing.assert_array_equal(labels, want)
    _networkx_checks(A, labels, 1.0, info["quality"])


def _blobs(n, d=20, types=8, seed=0):
    rng = np.random.default_rng(seed)
    centres = rng.normal(0, 6, (types, d))
    t = rng.integers(0, types, n)
    return (centres[t] + rng.normal(size=(n, d))).astype(np.float32), t


def test_connectivities_match_the_restatement():
    import torch
    from harmony_b200 import knn
    from harmony_b200.community import umap_graph_on
    from harmony_b200._arrays import handle
    X, _ = _blobs(3000)
    X[5] = np.nan
    Xd = torch.as_tensor(X, device="cuda")
    idx, dist = knn(Xd, None, 14)
    ip, ind, data = umap_graph_on(handle(None), idx, dist, 15)
    P = lr.umap_graph(idx.cpu().numpy(), dist.cpu().numpy(), 15)
    np.testing.assert_array_equal(ip.cpu().numpy(), P.indptr)
    np.testing.assert_array_equal(ind.cpu().numpy(), P.indices)
    np.testing.assert_allclose(data.cpu().numpy(), P.data.astype(np.float32), rtol=1e-6, atol=0)
    again = umap_graph_on(handle(None), idx, dist, 15)
    assert all(torch.equal(a, b) for a, b in zip((ip, ind, data), again))


@pytest.mark.parametrize("N", [1, 2, 3, 1000, 100_003])
def test_embedding_path_sizes(N):
    import torch
    from harmony_b200 import leiden
    X, _ = _blobs(N, seed=N)
    X[N // 2] = np.inf  # a non-finite row: label -1, the others numbered from 0
    k = min(15, max(N, 2))
    lab = leiden(torch.as_tensor(X, device="cuda"), n_neighbors=k)
    again = leiden(torch.as_tensor(X, device="cuda"), n_neighbors=k)
    assert torch.equal(lab, again)
    host = leiden(X, n_neighbors=k)
    np.testing.assert_array_equal(host, lab.cpu().numpy())
    assert host[N // 2] == -1 and (np.delete(host, N // 2) >= 0).all()


def test_large_graph_properties():
    """2^20 + 5 rows: connected communities, no improving single move, and Q of the GPU's labels (restated on the
    host) equal to the Q it reports, to 1e-9."""
    import torch
    from harmony_b200 import knn
    from harmony_b200.community import leiden_graph_on, umap_graph_on
    from harmony_b200._arrays import handle
    X, _ = _blobs(2 ** 20 + 5, seed=7)
    obj = handle(None)
    Xd = torch.as_tensor(X, device="cuda")
    idx, dist = knn(Xd, None, 14)
    G = umap_graph_on(obj, idx, dist, 15)
    labels, info = leiden_graph_on(obj, G, 1.0, -1, True)
    A = sp.csr_matrix((G[2].double().cpu().numpy(), G[1].cpu().numpy(), G[0].cpu().numpy()))
    lab = labels.cpu().numpy()
    assert abs(lr.modularity(A, lab, 1.0) - info["quality"]) <= 1e-9
    assert lr.connected_communities(A, lab)
    assert info["n_communities"] >= 8


def test_gamma_extremes():
    from harmony_b200 import leiden
    A = sp.block_diag([_planted(3, 20, 0.4, 0.05, 2), _ring_of_cliques(4, 5)]).tocsr()
    lab = leiden(A, resolution=1e-6)
    assert lab.max() + 1 == connected_components(A, directed=False)[0]
    lab = leiden(A, resolution=1e6)
    assert lab.max() + 1 == A.shape[0]


def _device_graph(M, dtype=np.float64):
    import torch
    return (torch.as_tensor(np.asarray(M.indptr, np.int64), device="cuda"),
            torch.as_tensor(np.asarray(M.indices, np.int32), device="cuda"),
            torch.as_tensor(np.asarray(M.data, dtype), device="cuda"))


def _leiden_call(L, g, a):
    return L.hb_leiden(g._h, a["indptr"], a["indices"], a["data"], a["dtype"], a["N"], a["nnz"], a["gamma"], a["n_iter"],
                       a["labels"], a["n_comm"], a["Q"], a["iters"], None, None)


def _umap_call(L, g, a):
    return L.hb_umap_graph(g._h, a["idx"], a["idx_ld"], a["dist"], a["dist_ld"], a["N"], a["k"], a["n_neighbors"],
                           a["indptr"], a["indices"], a["data"], a["nnz"], None)


def test_refusals_launch_nothing():
    import torch
    from harmony_b200 import _lib
    L = _lib.lib()
    A = _planted(3, 20, 0.4, 0.05, 2)
    ip, ind, dat = _device_graph(A)
    labels = torch.zeros(A.shape[0], dtype=torch.int32, device="cuda")
    host = np.zeros(A.shape[0] + 1, np.int64)
    ref = lambda t: ctypes.byref(t)  # noqa: E731
    g = gpu_harmony()
    good = dict(indptr=ptr(ip), indices=ptr(ind), data=ptr(dat), dtype=1, N=A.shape[0], nnz=A.nnz, gamma=1.0, n_iter=-1,
                labels=ptr(labels), n_comm=ref(ctypes.c_int()), Q=ref(ctypes.c_double()), iters=ref(ctypes.c_int()))
    bad = [dict(N=0), dict(N=2 ** 31), dict(nnz=-1), dict(nnz=2 ** 31), dict(gamma=0.0), dict(gamma=-1.0),
           dict(gamma=float("nan")), dict(gamma=float("inf")), dict(n_iter=-2), dict(dtype=2),
           dict(indptr=ptr(None)), dict(indices=ptr(None)), dict(data=ptr(None)), dict(labels=ptr(None)),
           dict(indptr=ctypes.c_void_p(host.ctypes.data)), dict(labels=ctypes.c_void_p(host.ctypes.data)),
           dict(n_comm=None), dict(Q=None), dict(iters=None)]
    refusals_launch_nothing(g, lambda a: _leiden_call(L, g, a), good, bad)
    N, k = 50, 6
    idx = torch.zeros((N, k), dtype=torch.int32, device="cuda")
    dist = torch.ones((N, k), dtype=torch.float32, device="cuda")
    out_ip = torch.zeros(N + 1, dtype=torch.int64, device="cuda")
    out_ind = torch.zeros(2 * N * k, dtype=torch.int32, device="cuda")
    out_dat = torch.zeros(2 * N * k, dtype=torch.float32, device="cuda")
    good = dict(idx=ptr(idx), idx_ld=k, dist=ptr(dist), dist_ld=k, N=N, k=k, n_neighbors=k + 1, indptr=ptr(out_ip),
                indices=ptr(out_ind), data=ptr(out_dat), nnz=ref(ctypes.c_int64()))
    hostf = np.zeros(N * k, np.float32)
    bad = [dict(N=0), dict(k=0), dict(k=129), dict(idx_ld=k + 1), dict(dist_ld=k - 1), dict(n_neighbors=1),
           dict(idx=ptr(None)), dict(dist=ptr(None)), dict(dist=ctypes.c_void_p(hostf.ctypes.data)),
           dict(indptr=ptr(None)), dict(indices=ptr(None)), dict(data=ptr(None)), dict(nnz=None)]
    refusals_launch_nothing(g, lambda a: _umap_call(L, g, a), good, bad)


def test_bad_graphs_write_nothing():
    """Order, diagonal, range, weight, missing-mirror and mirror-weight faults: status 2 naming the row and the fault,
    the labels unwritten.  An unsorted row is named as such, not as another row's missing mirror."""
    import torch
    from harmony_b200 import _lib
    L = _lib.lib()
    g = gpu_harmony()
    A = _planted(3, 20, 0.4, 0.05, 2).astype(np.float64).tocsr()
    A.sort_indices()
    cases = []
    B = A.copy()
    r = 5
    a, b = B.indptr[r], B.indptr[r + 1]
    B.indices[a:b] = B.indices[a:b][::-1].copy()  # row 5 descends: its mirrors' searches must not be blamed
    B.data[a:b] = B.data[a:b][::-1].copy()
    cases.append((B, "row 5, .* does not ascend"))
    B = A.tolil()
    B[7, 7] = 1.0
    cases.append((B.tocsr(), "row 7, .* on the diagonal"))
    B = A.copy()
    B.data[B.indptr[3]] = 9.5  # (3, j) without (j, 3) of that weight: the pair's first row is named
    cases.append((B, f"row {min(3, A.indices[A.indptr[3]])}, .* differs from its mirror"))
    B = A.copy()
    B.data[B.indptr[4]] = -1.0
    cases.append((B, "row 4, .* not finite and > 0"))
    B = A.tolil()
    B[0, 59] = 1.0 if A[0, 59] == 0 else 0.0
    B = B.tocsr()
    B.eliminate_zeros()
    cases.append((B, "row (0|59), .*no mirror"))
    for M, msg in cases:
        ip, ind, dat = _device_graph(M)
        labels = torch.full((M.shape[0],), -7, dtype=torch.int32, device="cuda")
        a = dict(indptr=ptr(ip), indices=ptr(ind), data=ptr(dat), dtype=1, N=M.shape[0], nnz=M.nnz, gamma=1.0,
                 n_iter=-1, labels=ptr(labels), n_comm=ctypes.byref(ctypes.c_int()), Q=ctypes.byref(ctypes.c_double()),
                 iters=ctypes.byref(ctypes.c_int()))
        assert _leiden_call(L, g, a) == 2, msg
        import re
        assert re.search(msg, L.hb_last_error(g._h).decode()), (msg, L.hb_last_error(g._h))
        unwritten(-7, labels)


def test_bad_neighbour_lists_write_nothing():
    import torch
    from harmony_b200 import _lib
    L = _lib.lib()
    g = gpu_harmony()
    N, k = 40, 5
    base = (np.arange(N)[:, None] + np.arange(1, k + 1)[None]) % N
    for row, col, value, msg in ((3, 2, N, "idx\\[3\\]\\[2\\] = 40 is not -1"), (4, 1, -2, "idx\\[4\\]\\[1\\] = -2"),
                                 (6, 3, None, "idx\\[6\\]\\[3\\] = .* repeats")):
        I = base.copy()
        I[row, col] = value if value is not None else I[row, 0]
        idx = torch.as_tensor(I.astype(np.int32), device="cuda")
        dist = torch.ones((N, k), dtype=torch.float32, device="cuda")
        out = [torch.full((N + 1,), -7, dtype=torch.int64, device="cuda"),
               torch.full((2 * N * k,), -7, dtype=torch.int32, device="cuda"),
               torch.full((2 * N * k,), -7.0, dtype=torch.float32, device="cuda")]
        a = dict(idx=ptr(idx), idx_ld=k, dist=ptr(dist), dist_ld=k, N=N, k=k, n_neighbors=k + 1, indptr=ptr(out[0]),
                 indices=ptr(out[1]), data=ptr(out[2]), nnz=ctypes.byref(ctypes.c_int64()))
        assert _umap_call(L, g, a) == 2
        import re
        assert re.search(msg, L.hb_last_error(g._h).decode()), (msg, L.hb_last_error(g._h))
        unwritten(-7, *out)


def test_handle_state_untouched():
    def call(h, phase, data):
        G = h.umap_connectivities(data.probe)
        assert G[0].numel() == data.probe.shape[0] + 1
        assert (h.leiden(data.probe) >= 0).all()
        assert (h.leiden(G) >= 0).all()
    handle_state_untouched(call)


def test_cap_warning():
    """The synchronous up/down sweeps of this graph at gamma = 2.5 do not settle within a level's 128 sweeps: the call
    warns, and still replays the restatement exactly."""
    from harmony_b200 import leiden
    A = dict(_integer_graphs())["pieces"]
    with pytest.warns(UserWarning, match="cap"):
        labels = leiden(A, resolution=2.5)
    np.testing.assert_array_equal(labels, lr.leiden(A, 2.5)[0])


def test_canonical_host_graph():
    """A host graph stored with unsorted rows and explicit zeros is the same graph: the same labels."""
    from harmony_b200 import leiden
    A = _planted(5, 40, 0.3, 0.02, 1).astype(np.float64).tocsr()
    B = A.copy()
    for r in range(B.shape[0]):
        a, b = B.indptr[r], B.indptr[r + 1]
        B.indices[a:b], B.data[a:b] = B.indices[a:b][::-1].copy(), B.data[a:b][::-1].copy()
    B.has_sorted_indices = False
    C = A.copy()
    C.data[C.indptr[2]] = 0.0  # an explicitly stored zero, on both sides of the pair
    C = C.tolil()
    j = A.indices[A.indptr[2]]
    C[j, 2] = 0.0
    C = sp.csr_matrix(C)
    D = A.copy()
    D[2, j] = 0.0
    D[j, 2] = 0.0
    D.eliminate_zeros()
    np.testing.assert_array_equal(leiden(B), leiden(A))
    np.testing.assert_array_equal(leiden(C), leiden(D))
    assert leiden([[0.0, 1.0], [1.0, 0.0], [5.0, 5.0]], n_neighbors=2).shape == (3,)


def test_state_untouched_and_side_stream():
    import torch
    from harmony_b200 import leiden
    X, _ = _blobs(5000, seed=3)
    Xd = torch.as_tensor(X, device="cuda")
    want = leiden(Xd)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        Y = torch.zeros_like(Xd)
        torch.cuda._sleep(50_000_000)
        Y.copy_(Xd)
        got = leiden(Y)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def test_nmi_ari_leiden_end_to_end():
    from harmony_b200 import nmi_ari_cluster_labels_leiden
    X, t = _blobs(20000, seed=11)
    out = nmi_ari_cluster_labels_leiden(X, {"cell_type": t}, "cell_type")
    assert out["nmi"] > 0.95 and out["ari"] > 0.9, out
    assert 0.1 <= out["resolution"] <= 2.0


RES = (0.2, 0.5, 1.0)


def _restated_scores(Z, labels):
    """nmi_ari_cluster_labels_leiden restated on the host: fp64 exact neighbours, the restatement's connectivities and
    Leiden at RES, the NMI / ARI fold and scib's choice."""
    from harmony_b200 import nmi_ari
    from harmony_b200.community import best_resolution
    Z = np.asarray(Z, np.float64)
    D = ((Z[:, None] - Z[None]) ** 2).sum(-1)
    np.fill_diagonal(D, np.inf)
    idx = np.argsort(D, axis=1, kind="stable")[:, :14]
    A = lr.umap_graph(idx, np.sqrt(np.take_along_axis(D, idx, 1)), 15)
    return best_resolution([(r, *nmi_ari(labels, lr.leiden(A, r)[0])) for r in RES])


def test_cell_lines_raw_and_integrated():
    """cell_lines by cell_type, raw and integrated over the datasets: the GPU's scores against the restatement's on
    the same rows, and RunHarmony on the GPU against the CPU oracle's fp64 integration (make_Y0 centroids, 10 rounds)
    clustered by the restatement."""
    import torch
    from harmony_b200 import RunHarmony, nmi_ari_cluster_labels_leiden, prepare_inputs
    Z, meta = load_cell_lines(False)
    raw = nmi_ari_cluster_labels_leiden(Z, meta, "cell_type", resolutions=RES)
    raw_host = _restated_scores(Z, meta["cell_type"])
    a = prepare_inputs(Z, meta, "dataset")
    o, _, _ = run_oracle(a, make_Y0(Z, a["K"]), 10, double=True)
    integ_host = _restated_scores(o.get("Z_corr"), meta["cell_type"])
    Zc = RunHarmony(torch.as_tensor(Z, device="cuda:0"), meta, "dataset", verbose=False, seed=1)
    integ = nmi_ari_cluster_labels_leiden(Zc, meta, "cell_type", resolutions=RES)
    print(f"[leiden cell_lines] raw {raw} restated {raw_host}; integrated {integ} oracle {integ_host}")
    for k in ("nmi", "ari"):
        assert abs(raw[k] - raw_host[k]) <= 0.02
        assert abs(integ[k] - integ_host[k]) <= 0.05
    assert integ["nmi"] >= raw["nmi"]
