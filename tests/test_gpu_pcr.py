"""hb_pcr on the GPU against the fp64 restatement (pcr_restatement.py) on the same values: a table of shapes, the inputs
Python takes, repeatability, the handle's state left untouched, the refusals, stream order, the launch count and the
scores of integrations end to end.

Bars (DESIGN §14): the score within 1e-10; each variance within 1e-10 lambda_1 / (n - 1); the R^2 and the component of
a PC whose eigenvalue is at least 1e-3 lambda_1 away from its neighbours' within 1e-9."""
import ctypes

import numpy as np
import pytest

import pcr_restatement as pr
from harmony_b200 import RunHarmony, pcr, pcr_comparison
from harmony_b200._arrays import ptr
from helpers import gpu_harmony, load_cell_lines
from score_helpers import (Frame, after_late_write, handle_state_untouched, non_finite_rows, refusals_launch_nothing,
                           strided, unwritten)

pytestmark = pytest.mark.gpu

SCORE_TOL, VAR_TOL, VEC_TOL, GAP = 1e-10, 1e-10, 1e-9, 1e-3

ROWS = [
    # name, N, d, dtype, batches (0: one per row), n_comps, options
    ("N2_d7", 2, 7, np.float32, 2, 50, {}),
    ("N3_d1_f64", 3, 1, np.float64, 2, 5, {}),
    ("N17_d8_one_row_per_batch", 17, 8, np.float32, 0, 8, {}),
    ("N1000_d16_f64_strided", 1000, 16, np.float64, 4, 16, dict(strided=True)),
    ("N100k_d50_comps_below_d", 100000, 50, np.float32, 4, 20, {}),
    ("N100k_d64_B1000_comps_at_d", 100000, 64, np.float32, 1000, 64, {}),
    ("N100k_d100_non_finite_rows", 100000, 100, np.float32, 4, 50, dict(nan=True)),
    ("N100k_d127_f64_offset_1e4_comps_above_d", 100000, 127, np.float64, 2, 200, dict(offset=1e4)),
    ("N100k_d128_one_batch", 100000, 128, np.float32, 1, 50, {}),
    ("N100k_d128_f32_strided_offset_1e3", 100000, 128, np.float32, 4, 128, dict(strided=True, offset=1e3)),
    ("N50k_d7_one_row_per_batch", 50000, 7, np.float32, 0, 7, {}),
    ("N2^20+5_d50", 2 ** 20 + 5, 50, np.float32, 4, 50, {}),
    ("N4M_d20", 4 * 2 ** 20, 20, np.float32, 4, 50, {}),
]


def _case(name, N, d, B, o):
    rng = np.random.default_rng(sum(map(ord, name)))
    b = np.arange(N) if B == 0 else rng.integers(0, B, N)
    X = rng.standard_normal((N, d)) * np.linspace(3.0, 0.5, d)
    X += rng.standard_normal((max(B, 1) if B else N, d))[b] * 0.5
    if o.get("offset"):
        X += o["offset"]
    if o.get("nan"):
        non_finite_rows(X)
    return X, b.astype(np.int32), (N if B == 0 else B)


def check(got, want):
    """The bars of the module's docstring on (var, r2, components, score) against the restatement's."""
    var, r2, comps, score = got
    m = len(want.var)
    assert len(var) == m and comps.shape == want.components.shape
    if np.isnan(want.score):
        assert np.isnan(score)
        return
    assert abs(score - want.score) <= SCORE_TOL, (score, want.score)
    lam1 = want.lam[0]
    assert (np.abs(var - want.var) <= VAR_TOL * lam1 / (want.n - 1)).all()
    lam = want.lam
    gap = np.abs(np.diff(lam)) / lam1
    iso = np.ones(m, bool)
    iso[:min(m, len(gap))] &= gap[:m] >= GAP
    iso[1:] &= gap[:m - 1] >= GAP
    iso &= lam[:m] > 1e-10 * lam1
    assert (np.abs(r2[iso] - want.r2[iso]) <= VEC_TOL).all()
    assert (np.abs(comps[iso] - want.components[iso]) <= VEC_TOL).all()
    assert ((r2 >= 0) & (r2 <= 1)).all()
    return iso.sum()


@pytest.mark.parametrize("row", ROWS, ids=[r[0] for r in ROWS])
def test_pcr_table(row):
    import torch
    name, N, d, dtype, B, n_comps, o = row
    X, b, n_batches = _case(name, N, d, B, o)
    X = X.astype(dtype)
    xt = strided(X) if o.get("strided") else torch.as_tensor(X, device="cuda:0")
    h = gpu_harmony()
    var, r2, comps, score = h.pcr(xt, torch.as_tensor(b, device="cuda:0"), n_comps)
    assert var.is_cuda and var.dtype == torch.float64 and comps.dtype == torch.float64
    got = (var.cpu().numpy(), r2.cpu().numpy(), comps.cpu().numpy(), score)
    want = pr.pcr(X.astype(np.float64), b, n_comps)
    iso = check(got, want)
    if B == 1:
        assert score == 0 and (got[1] == 0).all()
    full = len(want.var) >= min(want.n - 1, d)
    if full:
        assert abs(score - np.trace(want.M) / np.trace(want.C)) <= SCORE_TOL
    print(f"[pcr {name}] score {score:.10f}, restatement {want.score:.10f}, isolated PCs {iso}, full rank {full}")


def test_degenerate_spectrum_trace_identity():
    """Repeated eigenvalues at full rank: the score is tr(M) / tr(C) whatever basis each eigenspace gets."""
    import torch
    rng = np.random.default_rng(3)
    Q = np.linalg.qr(rng.standard_normal((10, 10)))[0]
    X = rng.standard_normal((20000, 10)) @ np.diag([2, 2, 2, 1, 1, 1, 1, 0.5, 0.5, 0.5]) @ Q
    b = rng.integers(0, 3, 20000).astype(np.int32)
    X += rng.standard_normal((3, 10))[b] * 0.3
    var, r2, comps, score = gpu_harmony().pcr(torch.as_tensor(X, device="cuda:0"), b, 10)
    assert abs(score - pr.trace_score(X, b)) <= SCORE_TOL
    comps = comps.cpu().numpy()
    np.testing.assert_allclose(comps @ comps.T, np.eye(10), rtol=0, atol=1e-12)


def test_inputs_agree_and_repeat():
    """Host arrays, CUDA tensors, a DataFrame and CUDA integer labels give one score; two calls are bit-identical."""
    import torch
    rng = np.random.default_rng(4)
    X = rng.standard_normal((30000, 30))
    bcode = rng.integers(0, 3, len(X))
    X += rng.standard_normal((3, 30))[bcode]
    batch = np.array(["b1", "b0", "b2"])[bcode]
    s_host, var, r2, comps = pcr(X, Frame({"batch": batch}), "batch", 10, return_all=True)
    assert isinstance(var, np.ndarray) and var.shape == (10,) and comps.shape == (10, 30)
    Xd = torch.as_tensor(X, device="cuda:0")
    codes = np.unique(batch, return_inverse=True)[1]     # the host's codes: the same sort, the same sums
    s_dev, vd, _, _ = pcr(Xd, {"batch": torch.as_tensor(codes, device="cuda:0")}, "batch", 10, return_all=True)
    assert vd.is_cuda and s_dev == s_host
    np.testing.assert_array_equal(vd.cpu().numpy(), var)
    assert s_host == pytest.approx(pr.pcr(X, bcode, 10).score, abs=SCORE_TOL)
    h = gpu_harmony()
    bt = torch.as_tensor(bcode.astype(np.int32), device="cuda:0")
    first = h.pcr(Xd.float(), bt, 30)
    second = h.pcr(Xd.float(), bt, 30)
    for u, v in zip(first[:3], second[:3]):
        np.testing.assert_array_equal(u.cpu().numpy(), v.cpu().numpy())
    assert first[3] == second[3]
    assert np.isnan(pcr(np.full((5, 3), np.nan), {"batch": batch[:5]}, "batch"))      # no finite row: NaN
    with pytest.raises(ValueError):
        pcr(X, {"batch": torch.as_tensor(bcode, device="cuda:0")}, "batch")   # device labels, host X


def test_handle_state_untouched():
    """hb_pcr between cluster_cpp and moe_correct_ridge_cpp and on a mapping handle: Z_corr, R and Y read bit for bit
    the same before and after the call."""
    def call(h, phase, data):
        if phase == "mapped":
            score = h.pcr(h.get_tensor("Z_corr"), data.mapped_codes)[3]
        else:
            score = h.pcr(data.probe, data.codes)[3]
        assert 0 <= score <= 1

    handle_state_untouched(call)


def _call(L, g, a):
    return L.hb_pcr(g._h, a["X"], a["xt"], a["xld"], a["N"], a["d"], a["bat"], a["nb"], a["nc"], a["var"], a["r2"],
                    a["comp"], a["score"], a.get("stream"))


def _buffers(N, d):
    import torch
    dev = torch.device("cuda", 0)
    X = torch.as_tensor(np.random.default_rng(0).standard_normal((N, d)).astype(np.float32), device=dev)
    bat = torch.as_tensor(np.arange(N, dtype=np.int32) % 2, device=dev)
    outs = [torch.full(s, -9.0, dtype=torch.float64, device=dev) for s in ((d,), (d,), (d, d), (1,))]
    return X, bat, outs


def test_refusals_launch_nothing():
    from harmony_b200 import _lib
    L = _lib.lib()
    g = gpu_harmony()
    N, d = 200, 8
    X, bat, (var, r2, comp, score) = _buffers(N, d)
    host = np.zeros(N, np.float64)
    H = host.ctypes.data_as(ctypes.c_void_p)
    good = dict(X=ptr(X), xt=0, xld=d, N=N, d=d, bat=ptr(bat), nb=2, nc=8, var=ptr(var), r2=ptr(r2), comp=ptr(comp),
                score=ptr(score))
    bad = [dict(N=1), dict(N=0), dict(N=2 ** 31), dict(d=0), dict(d=129, xld=129), dict(nb=0), dict(nb=N + 1),
           dict(nc=0), dict(nc=-1), dict(xt=2), dict(xt=-1), dict(xld=d - 1), dict(X=None), dict(bat=None),
           dict(var=None), dict(r2=None), dict(score=None), dict(X=H), dict(bat=H), dict(var=H), dict(r2=H),
           dict(comp=H), dict(score=H)]
    refusals_launch_nothing(g, lambda a: _call(L, g, a), good, bad)
    assert _call(L, g, dict(good, comp=None)) == 0     # the components are optional
    assert g.kernel_launches > 0
    unwritten(-9, comp)


@pytest.mark.parametrize("case", ["batch_past_n_batches", "batch_negative"])
def test_range_refusal_writes_nothing(case):
    from harmony_b200 import _lib
    L = _lib.lib()
    g = gpu_harmony()
    N, d = 2000, 8
    X, bat, outs = _buffers(N, d)
    if case == "batch_past_n_batches":
        bat[17] = 2
        msg = "hb_pcr: batches of cell 17 is not a code in 0..1"
    else:
        bat[5] = -1
        msg = "hb_pcr: batches of cell 5 is not a code in 0..1"
    a = dict(X=ptr(X), xt=0, xld=d, N=N, d=d, bat=ptr(bat), nb=2, nc=8, var=ptr(outs[0]), r2=ptr(outs[1]),
             comp=ptr(outs[2]), score=ptr(outs[3]))
    assert _call(L, g, a) == 2 and L.hb_last_error(g._h).decode() == msg
    unwritten(-9, *outs)


def test_launch_count_and_stream_order():
    """The batch index's eight launches (keys, scan, dictionary, tuple ids, one radix pass of histogram, scan and
    scatter, starts; with one batch no radix pass but the identity permutation), then sums, mean, combine and two Grams
    with their reductions.  The call reads X after the work queued on the caller's stream."""
    import torch
    rng = np.random.default_rng(9)
    X = rng.standard_normal((30000, 20)).astype(np.float32)
    b = rng.integers(0, 3, len(X)).astype(np.int32)
    xt, bt = torch.as_tensor(X, device="cuda:0"), torch.as_tensor(b, device="cuda:0")
    g = gpu_harmony()
    want = g.pcr(xt, bt, 20)
    assert g.kernel_launches == g.region_time("pcr")[1] == 8 + 7
    g = gpu_harmony()
    g.pcr(xt, torch.zeros_like(bt), 20)
    assert g.kernel_launches == 6 + 7
    g = gpu_harmony()
    got = after_late_write(xt, float("nan"), 200_000_000, lambda dst: g.pcr(dst, bt, 20))
    for u, v in zip(want[:3], got[:3]):
        np.testing.assert_array_equal(u.cpu().numpy(), v.cpu().numpy())
    assert want[3] == got[3]


def test_integration_cell_lines():
    """The raw PCs of cell_lines score 0.4686 by dataset.  The CPU oracle's fp64 integration (make_Y0 centroids, seeds 0
    and 1) scores 0.3944 and 0.3932, a comparison of 0.158 / 0.161: cell type and dataset are confounded there, so the
    drop is small.  RunHarmony on the GPU runs in fp32 from its own initialisation; its score is held to 0.03 of the
    oracle's, twenty times the spread of the oracle's two seeds."""
    import torch
    Z, meta = load_cell_lines(False)
    s0 = pcr(Z, meta, "dataset")
    assert s0 == pytest.approx(0.4685829545, abs=SCORE_TOL)
    Zc = RunHarmony(torch.as_tensor(Z, device="cuda:0"), meta, "dataset", verbose=False, seed=1)
    s1 = pcr(Zc, meta, "dataset")
    c = pcr_comparison(torch.as_tensor(Z, device="cuda:0"), Zc, meta, "dataset")
    print(f"[pcr cell_lines] {s0:.4f} -> {s1:.4f}, comparison {c:.4f}")
    assert s1 == pytest.approx(0.394, abs=0.03)
    assert c == pytest.approx((s0 - s1) / s0, abs=1e-12) and 0.09 <= c <= 0.23
    assert pcr_comparison(Z, Zc, meta, "dataset", scale=False) == pytest.approx(s1 - s0, abs=1e-10)


def test_integration_synthetic():
    """20k cells of 8 types and 4 batch shifts, d = 20: the raw embedding scores 0.0977 and the CPU oracle's fp64
    integration 0.0032, a comparison of 0.967.  RunHarmony on the GPU must remove most of the batch variance too."""
    import torch
    N, d = 20000, 20
    rng = np.random.default_rng(0)
    M = rng.standard_normal((8, d)) * 6
    S = rng.standard_normal((4, d)) * 2
    t = rng.integers(0, 8, N)
    b = rng.integers(0, 4, N)
    Z = M[t] + S[b] + rng.standard_normal((N, d))
    meta = {"batch": b}
    s0 = pcr(Z, meta, "batch")
    assert s0 == pytest.approx(pr.pcr(Z, b).score, abs=SCORE_TOL) and s0 == pytest.approx(0.0977, abs=5e-5)
    Zc = RunHarmony(torch.as_tensor(Z, device="cuda:0"), meta, "batch", verbose=False, seed=1)
    s1 = pcr(Zc, meta, "batch")
    c = pcr_comparison(Z, Zc, meta, "batch")
    print(f"[pcr synthetic] {s0:.4f} -> {s1:.4f}, comparison {c:.4f}")
    assert s1 <= 0.01 and c >= 0.9
