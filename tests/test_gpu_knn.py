"""hb_knn on the GPU against the fp64 restatement (knn_restatement.py): a table of shapes, each row naming the limit it
straddles, data that stress the selection, the handle's state left untouched, label transfer end to end, the refusals."""
import ctypes

import numpy as np
import pytest

import knn_restatement as kr
from harmony_b200 import MapQuery, RunHarmony, TransferLabels, knn
from harmony_b200._arrays import ptr
from helpers import gpu_harmony
from score_helpers import check_band, generic, geometry, handle_state_untouched, refusals_launch_nothing, strided

pytestmark = pytest.mark.gpu

EPS32 = 2.0 ** -24


def check(Q, X, k, metric, exclude_self, idx, dist, max_set_diff=0.001, block=1000):
    """The bar of DESIGN §9 for every query row; returns the share of rows whose index set differs from fp64's."""
    Q64, X64 = np.asarray(Q, np.float64), np.asarray(X, np.float64)
    qn, xn = kr.centred_norms(Q64, X64, metric)
    d = Q64.shape[1]
    assert idx.shape == dist.shape == (len(Q64), k) and idx.dtype == np.int32 and dist.dtype == np.float32
    assert (idx >= 0).all() and (idx < len(X64)).all(), "indices out of range"
    s = np.sort(idx, axis=1)
    assert (s[:, 1:] != s[:, :-1]).all(), "a reference row twice in a row"
    assert (np.diff(dist.astype(np.float64), axis=1) >= 0).all(), "dist does not ascend"
    differ = 0
    for r0 in range(0, len(Q64), block):
        r1 = min(len(Q64), r0 + block)
        D = kr.distances(Q64[r0:r1], X64, metric)
        if exclude_self:
            D[np.arange(r1 - r0), np.arange(r0, r1)] = np.inf
        got = np.take_along_axis(D, idx[r0:r1].astype(np.int64), 1)
        check_band(D, got, k, kr.band(qn[r0:r1], xn, d, metric))
        want = got if metric == "cosine" else np.sqrt(got)
        floor = 16 * EPS32 * (1.0 if metric == "cosine" else (qn[r0:r1, None] + xn))
        err = np.abs(dist[r0:r1] - want)
        assert (err <= 1e-5 * want + floor).all(), f"dist off by {float((err - 1e-5 * want - floor).max()):.3e}"
        exact = np.sort(np.argpartition(D, k - 1, axis=1)[:, :k], axis=1) if k < D.shape[1] else None
        if exact is not None:
            differ += int((np.sort(idx[r0:r1], axis=1) != exact).any(axis=1).sum())
    share = differ / len(Q64)
    if max_set_diff is not None:
        assert share <= max_set_diff, f"{share:.4%} of the rows differ from fp64's neighbours"
    return share


ROWS = [
    # name, d, k, Nq, Nx, metric, dtype, options
    ("d1_k1_one_query", 1, 1, 1, 127, "euclidean", np.float32, {}),
    ("d3_nx_equals_k", 3, 5, 129, 5, "euclidean", np.float64, {}),
    ("d8_one_full_tile", 8, 15, 129, 64, "cosine", np.float32, {}),
    ("d8_tile_plus_one", 8, 15, 129, 65, "euclidean", np.float32, {}),
    ("d50_nx127", 50, 5, 129, 127, "euclidean", np.float32, {}),
    ("d50_nx128", 50, 15, 20000, 128, "cosine", np.float64, {}),
    ("d50_nx129_k64", 50, 64, 129, 129, "euclidean", np.float32, {}),
    ("d50_split_merge", 50, 5, 1000, 50000, "euclidean", np.float32, dict(splits=True)),
    ("d50_no_split", 50, 15, 20000, 50000, "euclidean", np.float32, dict(splits=False)),
    ("d50_cosine_f64", 50, 15, 20000, 50000, "cosine", np.float64, dict(splits=False)),
    ("d56_kd_exact", 56, 5, 3000, 50000, "cosine", np.float32, dict(splits=True)),
    ("d64_k64", 64, 64, 1000, 50000, "euclidean", np.float32, dict(stages=2)),
    ("d100_k15", 100, 15, 20000, 50000, "euclidean", np.float32, dict(stages=2)),
    ("d100_k32_one_stage", 100, 32, 3000, 50000, "euclidean", np.float32, dict(stages=1)),
    # 64 boundaries per row 3e-5 apart in 1 - cos: rounding reorders the last place of 0.2 % of the rows
    ("d127_k64_small_tile", 127, 64, 3000, 50000, "cosine", np.float32, dict(tq=64, set_diff=0.005)),
    ("d128_k64_small_tile", 128, 64, 3000, 50000, "euclidean", np.float64, dict(tq=64)),
    ("d128_k1_one_stage", 128, 1, 129, 50000, "euclidean", np.float32, dict(stages=1)),
    ("self_search", 50, 15, 20000, 20000, "euclidean", np.float32, dict(self_search=True)),
    ("self_search_cosine_split", 50, 5, 5000, 5000, "cosine", np.float64, dict(self_search=True, splits=True)),
    ("strided_views", 50, 5, 3000, 20000, "euclidean", np.float32, dict(strided=True)),
    ("duplicates", 50, 5, 2000, 20000, "euclidean", np.float32, dict(duplicates=True)),
    ("far_from_origin", 50, 15, 5000, 50000, "euclidean", np.float32, dict(offset=1e3)),
    ("far_from_origin_f64", 50, 15, 5000, 50000, "euclidean", np.float64, dict(offset=1e3)),
    ("nearest_in_last_partial_tile", 50, 5, 2000, 50001 - 64 + 7, "euclidean", np.float32, dict(near="last")),
    ("nearest_in_first_tile", 50, 5, 2000, 50000, "euclidean", np.float32, dict(near="first")),
    ("cosine_special_rows", 50, 5, 3000, 20000, "cosine", np.float32, dict(special=True)),
]


@pytest.mark.parametrize("row", ROWS, ids=[r[0] for r in ROWS])
def test_knn_table(row):
    import torch
    name, d, k, Nq, Nx, metric, dtype, o = row
    rng = np.random.default_rng(sum(map(ord, name)))
    X = generic(rng, Nx, d)[0]
    if o.get("offset"):
        X += o["offset"]
    if o.get("duplicates"):
        X[Nx // 2:Nx // 2 + 4000] = X[:4000]
    if o.get("special"):
        X[:3] = 0.0
        X[3:6] *= 1e-25 / np.abs(X[3:6]).max(axis=1, keepdims=True)
        X[6:9] *= 1e20 / np.abs(X[6:9]).max(axis=1, keepdims=True)
    self_search = bool(o.get("self_search"))
    if self_search:
        Q = X
    else:
        Q = X[rng.integers(0, Nx, Nq)] + 0.5 * rng.standard_normal((Nq, d))
        if o.get("special"):
            Q[:2] = 0.0
            Q[2:4] = X[3:5]
            Q[4:6] = X[6:8]
    if o.get("near"):      # every query's neighbours sit in one tile of the reference: far rows elsewhere
        X += 50.0 * np.sign(rng.standard_normal((Nx, 1)))
        block = slice(Nx - 7, Nx) if o["near"] == "last" else slice(0, 40)
        X[block] = rng.standard_normal((block.stop - block.start, d)) * 0.5
        Q = rng.standard_normal((Nq, d)) * 0.5
    X, Q = X.astype(dtype), (X if self_search else Q).astype(dtype)
    if self_search:
        Q = X
    tq, tn, stages, splits, smem, per, KD, threads = geometry("hb_debug_knn_geometry", d, k, len(Q), Nx)
    if "splits" in o:
        assert (splits > 1) == o["splits"], (splits, o)
    if "stages" in o:
        assert stages == o["stages"]
    assert tq == o.get("tq", 128)
    dev = torch.device("cuda", 0)
    if o.get("strided"):
        xt, qt = strided(X), strided(Q)
    else:
        xt = torch.as_tensor(X, device=dev)
        qt = xt if self_search else torch.as_tensor(Q, device=dev)
    g = gpu_harmony()
    idx, dist = g.knn(qt, None if self_search else xt, k=k, metric=metric)
    assert idx.is_cuda and dist.is_cuda
    launches = g.region_time("knn")[1]
    # column sums (Euclidean), one or two preparations, the sweep, the merge
    assert launches == (metric == "euclidean") + (1 if self_search else 2) + 2 == g.kernel_launches
    loose = o.get("duplicates") or o.get("near") or o.get("special") or Nx <= k + 1
    share = check(Q, X, k, metric, self_search, idx.cpu().numpy(), dist.cpu().numpy(), None if loose else o.get("set_diff", 0.001))
    print(f"[knn {name}] tq={tq} stages={stages} splits={splits} smem={smem} set-diff rows {share:.5%}")


def test_non_finite_rows():
    """A NaN or infinite reference row is nobody's neighbour; such a query row has none (idx -1, dist inf)."""
    rng = np.random.default_rng(5)
    X, Q = generic(rng, 3000, 20)[0].astype(np.float32), generic(rng, 300, 20)[0].astype(np.float32)
    X[7, 3], X[100, 0], Q[5, 1], Q[9, 19] = np.nan, np.inf, np.nan, -np.inf
    for metric in ("euclidean", "cosine"):
        idx, dist = knn(Q, X, k=5, metric=metric)
        assert (idx[[5, 9]] == -1).all() and np.isinf(dist[[5, 9]]).all()
        ok = np.setdiff1d(np.arange(300), [5, 9])
        keep = np.setdiff1d(np.arange(3000), [7, 100])
        assert not np.isin(idx[ok], [7, 100]).any()
        back = np.full(3000, -1)
        back[keep] = np.arange(len(keep))
        check(Q[ok], X[keep], 5, metric, False, back[idx[ok]].astype(np.int32), dist[ok], None)
    few = X[:6].copy()
    few[[1, 4]] = np.nan
    idx, dist = knn(Q[:3], few, k=6)
    assert (np.sort(idx, axis=1) == [-1, -1, 0, 2, 3, 5]).all() and (idx[:, 4:] == -1).all() and np.isinf(dist[:, 4:]).all()


def test_numpy_and_tensor_paths_agree():
    import torch
    rng = np.random.default_rng(2)
    X, Q = generic(rng, 20000, 30)[0], generic(rng, 500, 30)[0]
    i0, d0 = knn(Q, X, k=10)
    i1, d1 = knn(torch.as_tensor(Q, device="cuda:0"), torch.as_tensor(X, device="cuda:0"), k=10)
    assert isinstance(i0, np.ndarray) and i1.is_cuda
    np.testing.assert_array_equal(i0, i1.cpu().numpy())
    np.testing.assert_array_equal(d0, d1.cpu().numpy())


def test_single_strided_query_row():
    """One query row taken as X.T[:1] of a [d, N] tensor (column stride N) is read as that row, not as the first d
    values of its memory: the same lists as the row made contiguous."""
    import torch
    X = torch.as_tensor(generic(np.random.default_rng(8), 40, 3000)[0], device="cuda:0")   # [d, N]
    q, ref = X.T[:1], X.T.contiguous()
    i0, d0 = knn(q, ref, k=10)
    i1, d1 = knn(q.contiguous(), ref, k=10)
    assert q.stride(1) == 3000 and int(i0[0, 0]) == 0
    np.testing.assert_array_equal(i0.cpu().numpy(), i1.cpu().numpy())
    np.testing.assert_array_equal(d0.cpu().numpy(), d1.cpu().numpy())


def test_handle_state_untouched():
    """hb_knn between cluster_cpp and moe_correct_ridge_cpp, and on a mapping handle before and after hb_map: Z_corr, R
    and Y read bit for bit the same before and after the call, and the run ends where a run without it ends (to the
    run-to-run noise of the atomics' order)."""

    def call(h, phase, data):
        if phase == "run":
            idx, _ = h.knn(data.probe, k=15)
            assert int(idx.min()) >= 0
        elif phase == "setup":
            h.knn(data.probe, k=5, metric="cosine")
        else:
            h.knn(h.get_tensor("Z_corr"), data.probe, k=5)

    handle_state_untouched(call, baseline=True)


def test_label_transfer_end_to_end():
    """RunHarmony on a reference, MapQuery of held-out cells with their own batch shifts, TransferLabels from CUDA
    tensors: the restatement's labels wherever no neighbour lies inside the band, and the planted types."""
    import torch
    rng = np.random.default_rng(8)
    n_types, d, Nr, Nq = 8, 30, 30000, 8000
    M = rng.standard_normal((n_types, d)) * 4.0
    types = rng.integers(0, n_types, Nr + Nq)
    batch = np.concatenate([rng.integers(0, 3, Nr), rng.integers(0, 2, Nq)])
    shifts = np.concatenate([rng.standard_normal((3, d)), rng.standard_normal((2, d))]) * 1.0
    Z = M[types] + 0.8 * rng.standard_normal((Nr + Nq, d)) + shifts[np.concatenate([batch[:Nr], 3 + batch[Nr:]])]
    obj = RunHarmony(Z[:Nr], {"b": batch[:Nr]}, "b", nclust=40, max_iter=5, return_object=True, verbose=False, seed=1)
    zr = obj.get_tensor("Z_corr")
    zq = MapQuery(torch.as_tensor(Z[Nr:], dtype=torch.float32, device="cuda:0"), {"b": batch[Nr:]}, "b",
                  obj.reference(), verbose=False)
    names = np.array([f"type{t}" for t in range(n_types)])
    pred, share = TransferLabels(zq, zr, names[types[:Nr]], k=5, return_prob=True)
    assert pred.dtype == names.dtype and ((share > 0) & (share <= 1)).all()
    assert (pred == names[types[Nr:]]).mean() >= 0.97
    zq_h, zr_h = zq.cpu().numpy(), zr.cpu().numpy()
    idx, dist = kr.brute_force(zq_h, zr_h, 6)
    qn, xn = kr.centred_norms(zq_h, zr_h, "euclidean")
    clear = dist[:, 5] ** 2 - dist[:, 4] ** 2 > kr.band(qn, xn, d)       # the 5th and 6th neighbours are told apart
    code, _ = kr.vote(idx[:, :5], dist[:, :5], types[:Nr], n_types)
    tally = np.stack([np.bincount(types[:Nr][r], minlength=n_types) for r in idx[:, :5]])
    ties_free = (tally == tally.max(axis=1, keepdims=True)).sum(axis=1) == 1
    sel = clear & ties_free
    assert sel.mean() > 0.9
    np.testing.assert_array_equal(pred[sel], names[code[sel]])
    pred_h = TransferLabels(zq_h, zr_h, names[types[:Nr]], k=5)
    np.testing.assert_array_equal(pred_h, pred)
    lab_d = torch.as_tensor(types[:Nr], device="cuda:0")
    pred_d = TransferLabels(zq, zr, lab_d, k=5)
    assert pred_d.is_cuda and (names[pred_d.cpu().numpy()] == pred).all()


def test_refusals_launch_nothing():
    import torch
    from harmony_b200 import _lib
    L = _lib.lib()
    g = gpu_harmony()
    dev = torch.device("cuda", 0)
    X, Q = torch.zeros((100, 8), device=dev), torch.zeros((10, 8), device=dev)
    idx, dist = torch.zeros((10, 5), dtype=torch.int32, device=dev), torch.zeros((10, 5), device=dev)
    host = np.zeros((100, 8), np.float32)
    good = dict(Q=ptr(Q), qt=0, qld=8, Nq=10, X=ptr(X), xt=0, xld=8, Nx=100, d=8, k=5, metric=0, excl=0, idx=ptr(idx),
                dist=ptr(dist))
    bad = [dict(k=0), dict(k=65), dict(k=101, Nx=100), dict(k=5, Nx=5, excl=1), dict(d=0), dict(d=129, qld=129, xld=129),
           dict(Nq=0), dict(Nx=0), dict(Nx=2 ** 31), dict(metric=2), dict(qt=2), dict(xt=-1), dict(qld=7), dict(xld=7),
           dict(Q=None), dict(X=None), dict(idx=None), dict(X=host.ctypes.data_as(ctypes.c_void_p)),
           dict(dist=host.ctypes.data_as(ctypes.c_void_p))]
    refusals_launch_nothing(g, lambda a: L.hb_knn(g._h, a["Q"], a["qt"], a["qld"], a["Nq"], a["X"], a["xt"], a["xld"],
                                                  a["Nx"], a["d"], a["k"], a["metric"], a["excl"], a["idx"], a["dist"],
                                                  None), good, bad)
    a = good
    assert L.hb_knn(g._h, a["Q"], 0, 8, 10, a["X"], 0, 8, 100, 8, 5, 0, 0, a["idx"], None, None) == 0   # dist may be NULL
    assert g.kernel_launches > 0
