"""hb_kmeans on the GPU against the fp64 restatement (kmeans_score_restatement.py): the seeding replayed round by round,
one Lloyd step within §9's band, whole runs on well-separated data, n_init, degenerate inputs, repeatability, the
handle's state, the refusals, stream order, the launch count and the NMI / ARI scores end to end (DESIGN §15)."""
import ctypes

import numpy as np
import pytest

import kmeans_score_restatement as kr
import knn_restatement as knr
from harmony_b200 import RunHarmony, kmeans, nmi_ari, nmi_ari_cluster_labels_kmeans
from harmony_b200._arrays import ptr, to_host
from helpers import gpu_harmony, load_cell_lines
from score_helpers import Frame, after_late_write, handle_state_untouched, refusals_launch_nothing, strided, unwritten

pytestmark = pytest.mark.gpu


def _data(N, d, types, rng, spread=8.0, offset=0.0):
    M = rng.standard_normal((types, d)) * spread
    t = rng.integers(0, types, N)
    return M[t] + rng.standard_normal((N, d)) + offset, t


SEEDING = [
    # name, N, d, K, dtype, options
    ("N1_d1_K1", 1, 1, 1, np.float64, {}),
    ("N2_d7_K2", 2, 7, 2, np.float32, {}),
    ("N17_d8_K17", 17, 8, 17, np.float32, {}),
    ("N1000_d50_K7_f64", 1000, 50, 7, np.float64, {}),
    ("N1000_d64_K63_strided", 1000, 64, 63, np.float32, dict(strided=True)),
    ("N1000_d127_K64_nonfinite", 1000, 127, 64, np.float32, dict(nan=True)),
    ("N1000_d128_K65_offset", 1000, 128, 65, np.float64, dict(offset=1e4)),
    ("N1000_d8_K200_host", 1000, 8, 200, np.float32, dict(host=True)),
    ("N100k_d50_K1024", 100000, 50, 1024, np.float32, {}),
]


def _input(X, dtype, o):
    import torch
    X = X.astype(dtype)
    if o.get("host"):
        return X
    return strided(X) if o.get("strided") else torch.as_tensor(X, device="cuda:0")


def _case(name, N, d, K, o):
    rng = np.random.default_rng(sum(map(ord, name)))
    X, _ = _data(N, d, max(K // 2, 1), rng, offset=o.get("offset", 0.0))
    if o.get("nan"):
        X[[3, 700]] = np.nan
        X[11, 5] = np.inf
    return X


@pytest.mark.parametrize("row", SEEDING, ids=[r[0] for r in SEEDING])
def test_seeding_replays(row):
    name, N, d, K, dtype, o = row
    X = _case(name, N, d, K, o)
    labels, centres, inertia, n_iter, seeds = kmeans(_input(X, dtype, o), K, seed=5, max_iter=0, return_seeds=True)
    seeds = to_host(seeds)[0]
    fin, P, _ = kr.prepare(X.astype(dtype))
    if N <= 20000:
        exact = kr.replay_seeds(P, fin, K, 5, 0, seeds)
        if exact == K:
            np.testing.assert_array_equal(seeds, kr.seeding(P, fin, K, 5))
    assert len(set(seeds.tolist())) == K or N == K
    assert fin[seeds].all()
    assert int(to_host(n_iter)[0]) == 0
    C = to_host(centres)
    np.testing.assert_array_equal(C, X.astype(dtype).astype(np.float64)[seeds])


LLOYD = [
    ("N1000_d7_K7", 1000, 7, 7, np.float32, {}),
    ("N1000_d50_K63_f64", 1000, 50, 63, np.float64, {}),
    ("N100k_d50_K20", 100000, 50, 20, np.float32, {}),
    ("N100k_d128_K200_strided", 100000, 128, 200, np.float32, dict(strided=True)),
    ("N100k_d64_K64_nonfinite_offset", 100000, 64, 64, np.float32, dict(nan=True, offset=1e4)),
    ("N2^20+5_d50_K20", 2 ** 20 + 5, 50, 20, np.float32, {}),
]


@pytest.mark.parametrize("row", LLOYD, ids=[r[0] for r in LLOYD])
def test_one_step_within_band(row):
    """max_iter = 1: the centres are the fp64 means of the seeds' assignment (max_iter = 0, the same seeds; an empty
    cluster keeps its seed row) to 1e-12 relative, and every returned label, the assignment to those centres, is the
    fp64 argmin within §9's band."""
    name, N, d, K, dtype, o = row
    X = _case(name, N, d, K, o)
    lab0, C0, _, _, seeds = map(to_host, kmeans(_input(X, dtype, o), K, seed=1, max_iter=0, return_seeds=True))
    labels, C, _, n_iter = map(to_host, kmeans(_input(X, dtype, o), K, seed=1, max_iter=1, tol=0.0))
    assert int(n_iter[0]) == 1
    Xd = X.astype(dtype).astype(np.float64)
    fin = np.isfinite(Xd).all(axis=1)
    assert (labels[~fin] == -1).all() and (labels[fin] >= 0).all() and (lab0[~fin] == -1).all()
    want = Xd[seeds[0]].copy()
    for k in range(K):
        mk = lab0 == k
        if mk.any():
            want[k] = Xd[mk].mean(axis=0)
    assert np.abs(C - want).max() <= 1e-12 * (np.abs(Xd[fin]).max() + 1.0)
    m = Xd[fin].mean(axis=0)
    xn = float(np.linalg.norm(C - m, axis=1).max())
    Xf, lf = Xd[fin], labels[fin]
    for s in range(0, len(Xf), 20000):
        _, D = kr.assign(Xf[s:s + 20000] - m, C - m)
        got = D[np.arange(len(D)), lf[s:s + 20000]]
        b = knr.band(np.linalg.norm(Xf[s:s + 20000] - m, axis=1), xn, d)
        assert (got <= D.min(axis=1) + b).all()


def test_whole_runs_match_restatement():
    """Well-separated clusters (every row's margin beyond the band): labels and n_iter equal the restatement run from
    the GPU's seeds, centres and inertia to 1e-9."""
    import torch
    rng = np.random.default_rng(4)
    for N, d, K, dtype in [(20000, 16, 8, np.float64), (50000, 50, 20, np.float32), (2000, 128, 7, np.float32)]:
        X, _ = _data(N, d, K, rng, spread=20.0)
        Xd = X.astype(dtype).astype(np.float64)
        for tol in (1e-4, 0.0):
            labels, C, inertia, n_iter, seeds = kmeans(torch.as_tensor(X.astype(dtype), device="cuda:0"), K, seed=3,
                                                       tol=tol, return_seeds=True)
            seeds = seeds.cpu().numpy()[0]
            wl, wc, wi, wn = kr.lloyd(Xd, Xd[seeds], 300, tol)
            _, D = kr.assign(Xd, wc)
            Ds = np.sort(D, axis=1)
            assert (Ds[:, 1] - Ds[:, 0] > 1e-3 * Ds[:, 1]).all()
            np.testing.assert_array_equal(labels.cpu().numpy(), wl)
            assert int(n_iter[0]) == wn
            assert abs(float(inertia[0]) - wi) <= 1e-9 * wi
            assert np.abs(C.cpu().numpy() - wc).max() <= 1e-9 * (np.abs(wc).max() + 1)


def test_n_init_returns_the_lowest_inertia():
    rng = np.random.default_rng(9)
    X, _ = _data(5000, 10, 12, rng, spread=3.0)
    labels, C, inertia, n_iter = kmeans(X, 12, seed=2, n_init=3)
    assert len(inertia) == 3 and len(n_iter) == 3
    best = int(np.argmin(inertia))
    one = kmeans(X, 12, seed=2, n_init=1)
    assert one[2][0] == inertia[0]
    assert abs(((X - C[labels]) ** 2).sum() - inertia[best]) <= 1e-9 * inertia[best]  # host fp64 rows stay fp64


def test_duplicates_and_empty_clusters_are_deterministic():
    rng = np.random.default_rng(2)
    X = np.repeat(rng.standard_normal((3, 4)), 40, axis=0)   # 3 distinct rows, K = 5
    a = kmeans(X, 5, seed=1, return_seeds=True)
    b = kmeans(X, 5, seed=1, return_seeds=True)
    for u, v in zip(a, b):
        np.testing.assert_array_equal(u, v)
    labels, C = a[0], a[1]
    assert len(np.unique(labels)) == 3
    for k in set(range(5)) - set(labels.tolist()):  # an empty cluster keeps its seed row
        np.testing.assert_array_equal(C[k], X[a[4][0][k]])
    assert float(a[2][0]) <= 1e-20  # every row sits on its centre, the fp64 mean of identical rows


def _sevens(K):
    """The outputs of a 10-row, 3-column call into K clusters, filled with 7: labels, centres, inertia, n_iter."""
    import torch
    return [torch.full(s, 7, dtype=t, device="cuda:0")
            for s, t in (((10,), torch.int32), ((K, 3), torch.float64), ((1,), torch.float64), ((1,), torch.int32))]


def test_too_few_finite_rows_is_status_3_outputs_untouched():
    import torch
    from harmony_b200 import _lib
    X = torch.full((10, 3), float("nan"), device="cuda:0", dtype=torch.float64)
    X[:4] = 1.0
    g = gpu_harmony()
    labels, C, ine, nit = _sevens(5)
    st = _lib.lib().hb_kmeans(g._h, ptr(X), 1, 3, 10, 3, 5, 0, 1, 300, 1e-4, ptr(labels), ptr(C), ptr(ine), ptr(nit),
                              ptr(None), None)
    torch.cuda.synchronize()
    assert st == 3 and b"finite" in _lib.lib().hb_last_error(g._h)
    unwritten(7, labels, C, ine, nit)


def test_row_beyond_fp32_range_is_status_2_outputs_untouched():
    """fp64 rows are assigned in fp32 after centring: a finite row with |x - m|^2 > 2^124 is refused, not dropped."""
    import torch
    from harmony_b200 import _lib
    X = torch.zeros((10, 3), device="cuda:0", dtype=torch.float64)
    X[:, 0] = torch.arange(10, device="cuda:0")
    X[4, 1] = 1e20
    g = gpu_harmony()
    labels, C, ine, nit = _sevens(2)
    st = _lib.lib().hb_kmeans(g._h, ptr(X), 1, 3, 10, 3, 2, 0, 1, 300, 1e-4, ptr(labels), ptr(C), ptr(ine), ptr(nit),
                              ptr(None), None)
    torch.cuda.synchronize()
    assert st == 2 and b"2^124" in _lib.lib().hb_last_error(g._h)
    unwritten(7, labels, C, ine, nit)
    X[4, 1] = 1e18  # |x - m|^2 ~ 1e36 < 2^124: runs, and every row takes part
    out = kmeans(X, 2, seed=0)
    assert (out[0] >= 0).all()


def test_two_calls_bit_identical():
    import torch
    rng = np.random.default_rng(11)
    X = torch.as_tensor(_data(200000, 50, 30, rng, spread=2.0)[0].astype(np.float32), device="cuda:0")
    a = kmeans(X, 30, seed=7, n_init=2, return_seeds=True)
    b = kmeans(X, 30, seed=7, n_init=2, return_seeds=True)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def test_fixture_values():
    Z, meta = load_cell_lines(False)
    r = nmi_ari_cluster_labels_kmeans(Z, meta, "cell_type")
    assert r["nmi"] == pytest.approx(0.9909829259, abs=1e-9) and r["ari"] == pytest.approx(0.9966258397, abs=1e-9)
    Z, meta = load_cell_lines(True)
    r = nmi_ari_cluster_labels_kmeans(Z, Frame(meta), "cell_type")
    assert r == {"nmi": 1.0, "ari": 1.0}


def test_end_to_end_synthetic():
    """The 8-type, 4-batch draw of the PCR test (20k cells, d = 20): the raw embedding scores NMI / ARI 1.0 / 1.0 (the
    types at scale 6 outweigh the batch shifts at scale 2).  The CPU oracle's fp64 integration (make_Y0 centroids,
    seeds 0 and 1), clustered by the restatement from its seeds 0 and 1, also scores 1.0 / 1.0 in all four runs.
    RunHarmony on the GPU runs in fp32 from its own initialisation and is held to 0.01 of the oracle's."""
    import torch
    N, d = 20000, 20
    rng = np.random.default_rng(0)
    M = rng.standard_normal((8, d)) * 6
    S = rng.standard_normal((4, d)) * 2
    t = rng.integers(0, 8, N)
    b = rng.integers(0, 4, N)
    Z = M[t] + S[b] + rng.standard_normal((N, d))
    meta = {"batch": b, "cell_type": t}
    raw = nmi_ari_cluster_labels_kmeans(Z, meta, "cell_type")
    Zc = RunHarmony(torch.as_tensor(Z, device="cuda:0"), meta, "batch", verbose=False, seed=1)
    after = nmi_ari_cluster_labels_kmeans(Zc, {"cell_type": torch.as_tensor(t, device="cuda:0")}, "cell_type")
    print(f"[nmi/ari synthetic] raw {raw}, after {after}")
    assert raw == {"nmi": 1.0, "ari": 1.0}
    assert after["nmi"] >= 0.99 and after["ari"] >= 0.99


def test_string_labels_with_device_rows():
    """Host labels of any values (strings, objects) go with a CUDA embedding and CUDA predictions: they are factorised
    on the host and only their codes uploaded, with the host path's scores."""
    import torch
    rng = np.random.default_rng(6)
    X, t = _data(20000, 16, 5, rng, spread=1.5)
    names = np.array(["B cell", "T cell", "NK", "mono", "DC"])[t]
    for labels in (names, names.astype(object)):
        host = nmi_ari_cluster_labels_kmeans(X, {"cell_type": labels}, "cell_type", seed=2)
        dev = nmi_ari_cluster_labels_kmeans(torch.as_tensor(X, device="cuda:0"), Frame({"cell_type": labels}),
                                            "cell_type", seed=2)
        assert dev == host
        pred = kmeans(X, 5, seed=2)[0]
        want = nmi_ari(labels, pred)
        assert nmi_ari(labels, torch.as_tensor(pred, device="cuda:0")) == pytest.approx(want, abs=1e-12)
        assert nmi_ari(torch.as_tensor(pred, device="cuda:0"), labels) == pytest.approx(nmi_ari(pred, labels), abs=1e-12)


def test_handle_state_untouched():
    def call(h, phase, data):
        out = h.kmeans(data.probe, 10, seed=1)
        assert (out[0] >= 0).all()
    handle_state_untouched(call)


def _call(L, g, a):
    return L.hb_kmeans(g._h, a["X"], a["dtype"], a["ld"], a["N"], a["d"], a["K"], 0, a["n_init"], a["max_iter"],
                       a["tol"], a["labels"], a["centres"], a["inertia"], a["n_iter"], a["seeds"], None)


def test_refusals_launch_nothing():
    import torch
    from harmony_b200 import _lib
    L = _lib.lib()
    g = gpu_harmony()
    X = torch.zeros((100, 8), device="cuda:0")
    b = lambda n, t=torch.int32: torch.zeros(n, dtype=t, device="cuda:0")  # noqa: E731
    good = dict(X=ptr(X), dtype=0, ld=8, N=100, d=8, K=5, n_init=1, max_iter=10, tol=1e-4, labels=ptr(b(100)),
                centres=ptr(b(40, torch.float64)), inertia=ptr(b(1, torch.float64)), n_iter=ptr(b(1)), seeds=ptr(None))
    host = np.zeros(100, np.int32)
    bad = [dict(N=0), dict(d=0), dict(d=129), dict(K=0), dict(K=101), dict(N=2000, K=1025), dict(n_init=0),
           dict(max_iter=-1), dict(tol=-1.0), dict(tol=float("nan")), dict(tol=float("inf")), dict(dtype=2),
           dict(ld=7), dict(X=ptr(None)), dict(labels=ptr(None)), dict(centres=ptr(None)), dict(inertia=ptr(None)),
           dict(n_iter=ptr(None)), dict(labels=ctypes.c_void_p(host.ctypes.data)), dict(N=2 ** 31)]
    refusals_launch_nothing(g, lambda a: _call(L, g, a), good, bad)
    assert _call(L, g, good) == 0
    torch.cuda.synchronize()
    assert g.kernel_launches > 0


def test_launch_count_and_stream_order():
    """The launches of an iteration: the centres' preparation, the sweep, the merge, the labels, the tuple index of
    the labels (keys, scan, table, ids, one radix pass of hist + scan + scatter, starts), the segment sums and the
    means: 14 for 2 <= present codes <= 256."""
    import torch
    rng = np.random.default_rng(3)
    X = torch.as_tensor(_data(30000, 16, 10, rng, spread=1.0)[0].astype(np.float32), device="cuda:0")
    counts = []
    for it in (1, 2, 3):
        g = gpu_harmony()
        out = g.kmeans(X, 10, seed=1, max_iter=it, tol=0.0)
        assert int(out[3][0]) == it
        counts.append(g.kernel_launches)
        assert g.region_time("kmeans")[1] == g.kernel_launches
    assert counts[2] - counts[1] == counts[1] - counts[0] == 14
    lab = after_late_write(X, None, 20_000_000, lambda Y: kmeans(Y, 10, seed=1)[0])
    torch.cuda.synchronize()
    np.testing.assert_array_equal(lab.cpu().numpy(), kmeans(X, 10, seed=1)[0].cpu().numpy())


def test_nmi_ari_on_device_matches_host():
    import torch
    rng = np.random.default_rng(5)
    t, p = rng.integers(0, 6, 10000), rng.integers(-1, 9, 10000)
    assert nmi_ari(torch.as_tensor(t, device="cuda:0"), torch.as_tensor(p, device="cuda:0")) == \
        pytest.approx(nmi_ari(t, p), abs=1e-12)
