"""hb_lisi on the GPU against the fp64 restatement (lisi_restatement.py): a table of shapes, each row naming the limit it
straddles, the handle's state left untouched, the refusals, and iLISI / cLISI of an integration end to end."""
import ctypes

import numpy as np
import pytest

import knn_restatement as kr
import lisi_restatement as lr
from harmony_b200 import RunHarmony, compute_lisi, knn
from harmony_b200._arrays import ptr
from helpers import gpu_harmony, load_cell_lines
from score_helpers import Frame, generic, geometry, handle_state_untouched, refusals_launch_nothing, strided
from score_helpers import check_band as in_band

pytestmark = pytest.mark.gpu

REL_OWN = 1e-9      # bar (a): the call's own neighbours through the restatement
REL_FP64 = 1e-4     # bar (b): the restatement from scratch, rows with fp64's neighbour set (DESIGN §10)
SET_DIFF = 0.001    # bar (b): rows whose neighbour set differs from fp64's (DESIGN §9's bar for the sweep)


def same_lisi(got, want, rel):
    """Equal markers (-1, NaN) and values within rel elsewhere; returns the largest relative difference."""
    assert (np.isnan(got) == np.isnan(want)).all(), "NaN rows differ"
    assert ((got == -1) == (want == -1)).all(), "-1 rows differ"
    ok = ~np.isnan(want) & (want != -1)
    err = np.abs(got[ok] - want[ok]) / np.abs(want[ok])
    worst = float(err.max()) if err.size else 0.0
    assert worst <= rel, f"LISI off by {worst:.3e} relative"
    return worst


def check_band(X, k, idx, block=2000):
    """Every row's neighbours against fp64 (DESIGN §9): all rows closer than the k-th distance minus the band are
    returned and none beyond it plus the band, so a set that differs from fp64's differs inside the band only."""
    rows = np.nonzero(np.isfinite(X).all(axis=1))[0]
    if len(rows) - 1 < k:
        return
    F = np.asarray(X[rows], np.float64)
    back = np.full(len(X), -1)
    back[rows] = np.arange(len(rows))
    qn, xn = kr.centred_norms(F, F, "euclidean")
    for r0 in range(0, len(F), block):
        r1 = min(len(F), r0 + block)
        D = kr.distances(F[r0:r1], F, "euclidean")
        D[np.arange(r1 - r0), np.arange(r0, r1)] = np.inf
        in_band(D, np.take_along_axis(D, back[idx[rows[r0:r1]]], 1), k, kr.band(qn[r0:r1], xn, F.shape[1]))


ROWS = [
    # name, perplexity, d, N, dtype, options
    ("p1_k2_n_equals_k_plus_1", 1, 3, 3, np.float64, {}),
    # one dimension: 5000 values on a line, the 2nd and 3rd neighbours within rounding of each other in 2 % of the rows
    ("p1_k2_d1", 1, 1, 5000, np.float32, dict(splits=True, set_diff=0.03)),
    ("p21_k62_split", 21, 50, 5000, np.float32, dict(splits=True)),
    ("p21_k62_no_split", 21, 50, 20000, np.float32, dict(splits=False)),
    ("p21_67_k64_last_2_entry_fold", 21.67, 64, 3000, np.float32, {}),
    ("p22_k65_first_4_entry_fold", 22, 50, 5000, np.float32, dict(splits=True)),
    ("p22_n_equals_k_plus_1", 22, 8, 66, np.float32, {}),
    ("p30_default_no_split", 30, 50, 20000, np.float32, dict(splits=False)),
    ("p30_n_one_past_a_tile", 30, 20, 64 * 40 + 1, np.float32, {}),
    # d >= 100 and k >= 89: the k-th and (k+1)-th distances of 0.1 % of the rows lie inside the band
    ("p30_d100_f64_strided_small_tile", 30, 100, 5000, np.float64, dict(strided=True, tq=64, stages=2, set_diff=0.003)),
    ("p30_d64_f32_strided_one_stage", 30, 64, 3000, np.float32, dict(strided=True, stages=1, splits=True)),
    ("p36_k107_d128_geometry_64_1", 36, 128, 5000, np.float32, dict(tq=64, stages=1, set_diff=0.003)),
    ("p43_k128_split_small_tile", 43, 50, 3000, np.float32, dict(splits=True, tq=64, stages=2)),
    ("p43_k128_no_split", 43, 30, 20000, np.float32, dict(splits=False)),
    ("p43_k128_d120_geometry_64_1", 43, 120, 3000, np.float64, dict(tq=64, stages=1)),
    ("p43_n_equals_k_plus_1", 43, 16, 129, np.float32, {}),
    ("one_set", 30, 50, 8000, np.float32, dict(sets="one")),
    ("five_sets_one_level_thousands_arbitrary", 30, 50, 8000, np.float32, dict(sets="five")),
    ("duplicates", 30, 50, 8000, np.float32, dict(duplicates=True)),
    ("offset_1e3", 30, 50, 8000, np.float32, dict(offset=1e3)),
    ("offset_1e3_f64", 30, 50, 8000, np.float64, dict(offset=1e3)),
    ("nan_rows", 30, 20, 5000, np.float32, dict(nan=True)),
]


def _labels(rng, n, t, kind):
    batch = rng.integers(0, 3, n)
    if kind == "one":
        return batch[None]
    if kind == "five":
        arbitrary = np.array([-2 ** 31, -7, 0, 99, 2 ** 31 - 1])[rng.integers(0, 5, n)]
        return np.stack([batch, t, np.zeros(n, np.int64) + 5, rng.integers(0, 3000, n), arbitrary])
    return np.stack([batch, t])


@pytest.mark.parametrize("row", ROWS, ids=[r[0] for r in ROWS])
def test_lisi_table(row):
    import torch
    name, p, d, N, dtype, o = row
    rng = np.random.default_rng(sum(map(ord, name)))
    X, t = generic(rng, N, d)
    if o.get("offset"):
        X += o["offset"]
    if o.get("duplicates"):
        X[N // 2:N // 2 + 2000] = X[:2000]
    if o.get("nan"):
        X[[3, 700, 4000]] = np.nan
        X[[11, 2500], 5] = np.inf
    X = X.astype(dtype)
    codes = _labels(rng, N, t, o.get("sets")).astype(np.int32)
    k = lr.neighbours_for(p)
    tq, tn, stages, splits, smem, per, KD, threads = geometry("hb_debug_lisi_geometry", d, p, N)
    if "splits" in o:
        assert (splits > 1) == o["splits"], (splits, o)
    if "stages" in o:
        assert stages == o["stages"]
    assert tq == o.get("tq", 128)
    dev = torch.device("cuda", 0)
    if o.get("strided"):
        xt = strided(X)
        cbuf = torch.zeros((codes.shape[0], N + 5), dtype=torch.int32, device=dev)
        ct = cbuf[:, :N]
        ct.copy_(torch.as_tensor(codes, device=dev))
    else:
        xt = torch.as_tensor(X, device=dev)
        ct = torch.as_tensor(codes, device=dev)
    g = gpu_harmony()
    out, idx, dist = g.lisi(xt, ct, p, return_neighbors=True)
    assert out.is_cuda and out.dtype == torch.float64 and out.shape == (N, codes.shape[0])
    # column sums, one preparation, the sweep, the merge, k_lisi
    assert g.region_time("lisi")[1] == 5 == g.kernel_launches
    out, idx, dist = out.cpu().numpy(), idx.cpu().numpy(), dist.cpu().numpy()
    # (a) the call's own neighbours through the restatement
    own, own_flag = lr.lisi(X, codes, p, idx, dist)
    keep = ~own_flag
    worst_a = same_lisi(out[keep], own[keep], REL_OWN)
    # (b) the restatement from scratch: rows with fp64's neighbour set
    ref_idx, ref_dist = lr.neighbours(X, p)
    want, flag = lr.lisi(X, codes, p, ref_idx, ref_dist)
    same_set = (np.sort(idx, axis=1) == np.sort(ref_idx, axis=1)).all(axis=1)
    share = float((~same_set).mean())
    check_band(X, k, idx)
    if not (o.get("duplicates") or N == k + 1):
        assert share <= o.get("set_diff", SET_DIFF), f"{share:.4%} of the rows differ from fp64's neighbours"
    sel = same_set & ~flag & ~own_flag
    worst_b = same_lisi(out[sel], want[sel], REL_FP64)
    # (c) up to k = 64 the neighbours are hb_knn's, bit for bit
    if k <= 64:
        i2, d2 = g.knn(xt, k=k)
        np.testing.assert_array_equal(idx, i2.cpu().numpy())
        np.testing.assert_array_equal(dist, d2.cpu().numpy())
    if o.get("nan"):
        bad = [3, 11, 700, 2500, 4000]
        assert np.isnan(out[bad]).all() and (idx[bad] == -1).all() and not np.isin(idx, bad).any()
    print(f"[lisi {name}] k={k} tq={tq} stages={stages} splits={splits} (a) {worst_a:.2e} (b) {worst_b:.2e} "
          f"set-diff {share:.4%} flagged {int((flag | own_flag).sum())}")


def test_compute_lisi_inputs_agree():
    """Host arrays, CUDA tensors, a DataFrame, CUDA integer labels and a default stream: one result."""
    import torch
    rng = np.random.default_rng(4)
    X, t = generic(rng, 6000, 30)
    batch = np.array(["b1", "b0", "b2"])[rng.integers(0, 3, len(X))]
    meta = Frame({"batch": batch, "type": t, "other": np.full(len(X), 1.5)})
    host = compute_lisi(X, meta, ["batch", "type"])
    assert isinstance(host, np.ndarray) and host.shape == (len(X), 2) and host.dtype == np.float64
    Xd = torch.as_tensor(X, device="cuda:0")
    dev = compute_lisi(Xd, {"batch": batch, "type": torch.as_tensor(t * 1000 - 7, device="cuda:0")}, ["batch", "type"])
    assert dev.is_cuda and dev.dtype == torch.float64
    np.testing.assert_array_equal(host, dev.cpu().numpy())
    one = compute_lisi(X, {"type": t}, "type", perplexity=30)
    np.testing.assert_array_equal(one[:, 0], host[:, 1])
    want, _ = lr.lisi(X, np.stack([np.unique(batch, return_inverse=True)[1], t]), 30)
    assert np.median(np.abs(host - want) / want) < 1e-6
    lisi, idx, dist = compute_lisi(X, meta, "batch", perplexity=10, return_neighbors=True)
    assert idx.shape == dist.shape == (len(X), 29) and lisi.shape == (len(X), 1)
    with pytest.raises(ValueError):
        compute_lisi(X, {"batch": torch.as_tensor(t, device="cuda:0")}, "batch")   # device labels, host X


def test_handle_state_untouched():
    """hb_lisi between cluster_cpp and moe_correct_ridge_cpp and on a mapping handle before and after hb_map: Z_corr, R
    and Y read bit for bit the same before and after the call."""
    import torch

    def call(h, phase, data):
        if phase == "run":
            assert not torch.isnan(h.lisi(data.probe, data.codes, 30)).any()
        elif phase == "setup":
            h.lisi(data.probe, data.codes, 10)
        else:
            h.lisi(h.get_tensor("Z_corr"), data.mapped_codes, 30)

    handle_state_untouched(call)


def test_refusals_launch_nothing():
    import torch
    from harmony_b200 import _lib
    L = _lib.lib()
    g = gpu_harmony()
    dev = torch.device("cuda", 0)
    N, d = 200, 8
    X = torch.zeros((N, d), device=dev)
    lab = torch.zeros((2, N), dtype=torch.int32, device=dev)
    out = torch.zeros((N, 2), dtype=torch.float64, device=dev)
    idx, dist = torch.zeros((N, 89), dtype=torch.int32, device=dev), torch.zeros((N, 89), device=dev)
    host = np.zeros((N, 89), np.float64)
    H = host.ctypes.data_as(ctypes.c_void_p)
    good = dict(X=ptr(X), xt=0, xld=d, N=N, d=d, lab=ptr(lab), lld=N, sets=2, p=30.0, out=ptr(out), idx=ptr(idx),
                dist=ptr(dist))
    bad = [dict(p=0.5), dict(p=float("nan")), dict(p=float("inf")), dict(p=-30.0), dict(p=43.34), dict(N=89),
           dict(N=2 ** 31), dict(d=0), dict(d=129, xld=129), dict(sets=0), dict(lld=N - 1), dict(xt=2), dict(xt=-1),
           dict(xld=d - 1), dict(X=None), dict(lab=None), dict(out=None), dict(X=H), dict(lab=H), dict(out=H),
           dict(idx=H), dict(dist=H)]
    refusals_launch_nothing(g, lambda a: L.hb_lisi(g._h, a["X"], a["xt"], a["xld"], a["N"], a["d"], a["lab"], a["lld"],
                                                   a["sets"], a["p"], a["out"], a["idx"], a["dist"], None), good, bad)
    a = good
    assert L.hb_lisi(g._h, a["X"], 0, d, N, d, a["lab"], N, 2, 30.0, a["out"], None, None, None) == 0   # no idx / dist
    assert g.kernel_launches > 0


def test_integration_scores_end_to_end():
    """iLISI over `dataset` rises from the input PCs to RunHarmony's Z_corr, and cLISI over `cell_type` stays near 1.
    The CPU oracle's integration of the same fixture (default parameters, 7-8 rounds, two seeds), scored with the
    restatement: median iLISI 1.018 on the PCs and 1.765 / 1.767 on Z_corr, median cLISI 1.0000 (mean 1.0015,
    largest 1.99).  The bound on the median cLISI is that 1.0000 plus a margin of 0.05."""
    import torch
    Z, meta = load_cell_lines(False)
    labels = ["dataset", "cell_type"]
    before = compute_lisi(Z, meta, labels)
    Zc = RunHarmony(torch.as_tensor(Z, device="cuda:0"), meta, "dataset", verbose=False, seed=1)
    after = compute_lisi(Zc, meta, labels).cpu().numpy()
    i0, i1, c1 = np.median(before[:, 0]), np.median(after[:, 0]), np.median(after[:, 1])
    print(f"[lisi cell_lines] median iLISI {i0:.4f} -> {i1:.4f}, median cLISI {c1:.4f}")
    assert i1 > i0
    assert c1 < 1.05
