"""Shapes past the FFMA kernels' shared-memory limits: wide embeddings (d > 120 for the logits, d > 256 for the apply) and
large K (K x d beyond the FFMA assignment and k-means kernels).  They run on the d-chunked logits kernel with softmax
passes, the column-range ridge apply and the k-means initialisation from those logits (hb_debug_wide_paths).

The CPU tests restate today's fit tests of the FFMA kernels in Python and check, over every K in 2..1024 and d in
1..1024, that each stage keeps its kernel where that kernel fits and takes the new one everywhere else.  The GPU tests run
the four stages of test_gpu_kernel_edges.py on rows that straddle each new limit, against the fp64 numpy restatement.
"""
import ctypes

import numpy as np
import pytest

from harmony_b200 import _lib
from helpers import free_port, make_perms, num_sms, rel_l2
from stages import (ALPHA, BLOCK, CUTOFF, NB, SIGMA, T, TOL_OBJ, TOL_OE, TOL_R, TOL_R1, TOL_Y, TOL_Y_FIXED, TOL_Z,
                    TOL_ZN, _launches, _mix64, _nested, _obj_err, _one_cov, _set_zcorr, _sizes, _table_err, f32,
                    kernel_paths, make_Y0, native_order, numpy_model, planted_R, tables_of)

PER_STEP, TWO_PASS, SINGLE_PASS = 0, 1, 2
HB_KS_WIDE = 16
SMEM = 227 * 1024


# ---- today's fit tests (harmony_b200/csrc), restated --------------------------------------------------------------------
def up(x, m):
    return (x + m - 1) // m * m


def assign_ffma_fits(K, d):      # k_assign: Ys, Zs, Ls, sig, part
    KP, DP4 = up(K, 64), up(d, 4)
    return 4 * (DP4 * KP + 64 * DP4 + 64 * (KP + 4) + 9 * KP) <= SMEM


def logits_tc_fits(d):           # k_logits_tc: A hi/lo, B hi/lo, U stage, 2/sigma, norms
    KD = up(d, 8)
    return d <= 128 and 4 * (2 * 128 * KD + 2 * 64 * KD + 128 * 68 + 64 + 4 * 128) + 256 <= SMEM - 256


def apply_ffma_fits(K, d):       # k_ridge_apply: d / 4 x 16 threads, V_q and the R tile
    DP, KP4 = up(d, 4), up(K, 4)
    return DP // 4 * 16 <= 1024 and 4 * (KP4 * DP + 64 * KP4) <= SMEM


def kmeans_ffma_fits(K, d):      # k_kmeans_race / k_kmeans_assign: all centroids
    return 4 * K * d <= 200 * 1024


def wide_paths(K, d, J, n, num_sms, kernel_set=0):
    out = (ctypes.c_int64 * 4)()
    _lib.lib().hb_debug_wide_paths(K, d, J, n, NB, num_sms, kernel_set, out)
    return tuple(out)


# hb_debug_wide_paths values
A_FUSED, A_FFMA, A_LOGITS, A_WIDE = 1, 2, 3, 4            # natural-order assignment
C_NATURAL, C_FUSED, C_LOGITS, C_WIDE = 0, 1, 2, 3         # plan-order cold start
P_TC, P_FFMA, P_COLS = 1, 2, 3                            # ridge apply
M_FFMA, M_TC, M_LOGITS, M_WIDE = 1, 2, 3, 4               # k-means initialisation


def test_every_shape_has_a_kernel_and_keeps_the_one_that_fits():
    """K in 2..1024, d in 1..1024 (20 tuples, 1M cells, 132 SMs): the old kernel wherever it fits, the new one elsewhere."""
    L = _lib.lib()
    old, new = (ctypes.c_int64 * 8)(), (ctypes.c_int64 * 4)()
    for K in range(2, 1025):
        for d in range(1, 1025):
            L.hb_debug_kernel_paths(K, d, 20, 1000000, NB, 132, 0, old)
            L.hb_debug_wide_paths(K, d, 20, 1000000, NB, 132, 0, new)
            lw = 0 if logits_tc_fits(d) else 1
            fused, logits, apply_tc, km_tc, plan = old[1] > 0, old[2], old[3], old[4], old[5]
            # natural-order assignment
            if fused:
                want = A_FUSED
            elif assign_ffma_fits(K, d):
                want = A_FFMA
            else:
                want = A_LOGITS + lw
            assert new[0] == want, (K, d, tuple(new))
            # plan-order cold start: today's where it exists, the new logits where k_assign does not fit and the call
            # runs single-pass; natural order otherwise
            if old[0] == SINGLE_PASS and not fused and not logits and not assign_ffma_fits(K, d):
                assert plan == 1 and new[1] == C_LOGITS + lw, (K, d, tuple(new))
            else:
                assert new[1] == (C_NATURAL if not plan else C_FUSED if fused else C_LOGITS), (K, d, tuple(new))
            # ridge apply
            assert apply_tc == (d <= 128)
            assert new[2] == (P_TC if apply_tc else P_FFMA if apply_ffma_fits(K, d) else P_COLS), (K, d, tuple(new))
            # k-means initialisation
            want = M_TC if km_tc else M_FFMA if kmeans_ffma_fits(K, d) else M_LOGITS + lw
            assert new[3] == want, (K, d, tuple(new))
            assert min(new[0], new[2], new[3]) > 0


def test_wide_hook_forces_the_new_kernels():
    """HB_KS_WIDE puts every stage on the new kernels, c3 included."""
    assert wide_paths(100, 50, 20, 1000000, 132, HB_KS_WIDE) == (A_WIDE, C_WIDE, P_COLS, M_WIDE)
    assert kernel_paths(100, 50, 20, 1000000, 132)[1:5] == (2, 0, 1, 1)   # unchanged without the bit


# ---- rows -------------------------------------------------------------------------------------------------------------
def _apply_launches(K, d, wide):
    """Launches of the ridge apply: cluster ranges (x column ranges for the column-range kernel)."""
    KS, DS = up(K, 4), up(d, 4)
    fixed = 4 * 2 * (128 if (wide or d > 64) else 64) * 112 + 32

    def passes(DC):
        npass = (K + 111) // 112
        while True:
            Kp = up((K + npass - 1) // npass, 8)
            RS = min(KS, Kp)
            st = 4 * 64 * (RS + DC)
            n = (SMEM - 256 - fixed) // st if fixed < SMEM - 256 else 0
            if (min(n, 4) & ~1) >= 2:
                return len(range(0, K, Kp))
            npass += 1
    if not wide:
        return passes(DS)
    return sum(passes(min(128, DS - c)) for c in range(0, DS, 128))


# name -> (K, d, covariate builder(num_sms), hb_debug_wide_paths, update path, kernel_set)
ROWS = {
    # logits past k_logits_tc (d = 127 > 120), k_assign past its shared memory at K = 200
    "d127_K200": (200, 127, lambda s: _one_cov(_sizes(5, 6000)), (A_WIDE, C_WIDE, P_TC, M_FFMA), SINGLE_PASS, 0),
    # k_assign one column past its limit (d = 252 runs on it)
    "d253_K100": (100, 253, lambda s: _one_cov(_sizes(6, 6000)), (A_WIDE, C_WIDE, P_FFMA, M_FFMA), SINGLE_PASS, 0),
    # the FFMA apply's block is 1040 threads: column ranges 128 + 128 + 4
    "d257_K64": (64, 257, lambda s: _one_cov(_sizes(6, 6000)), (A_FFMA, C_NATURAL, P_COLS, M_FFMA), SINGLE_PASS, 0),
    "d300_K100": (100, 300, lambda s: _nested(_sizes(8, 8000), 4), (A_WIDE, C_WIDE, P_COLS, M_FFMA), SINGLE_PASS, 0),
    # 2 J = #SMs + 2: two-pass update, natural-order cold start from the d-chunked logits
    "d300_K100_two_pass": (100, 300, lambda s: _nested(_sizes(s // 2 + 1, 12000), 6), (A_WIDE, C_NATURAL, P_COLS, M_FFMA),
                           TWO_PASS, 0),
    # two 128-cluster logits ranges, four column ranges x three cluster ranges of the apply, k-means from wide logits
    "d512_K200": (200, 512, lambda s: _one_cov(_sizes(5, 6000)), (A_WIDE, C_WIDE, P_COLS, M_WIDE), SINGLE_PASS, 0),
    # k_assign one cluster past its limit at d = 8 (K = 704 runs on it); per-step update
    "K705_d8": (705, 8, lambda s: _one_cov(_sizes(4, 4000)), (A_LOGITS, C_NATURAL, P_TC, M_FFMA), PER_STEP, 0),
    # K = 1024: softmax with 8 pieces per lane, k-means from k_logits_tc logits
    "K1024_d64": (1024, 64, lambda s: _one_cov(_sizes(4, 4000)), (A_LOGITS, C_NATURAL, P_TC, M_LOGITS), PER_STEP, 0),
    # config 3's shape with every new kernel forced
    "c3_shape_wide": (100, 50, lambda s: _one_cov(_sizes(20, 20000)), (A_WIDE, C_WIDE, P_COLS, M_WIDE), SINGLE_PASS,
                      HB_KS_WIDE),
}


def build_case(name, num_sms, seed=0):
    """Inputs of a row, built like test_gpu_kernel_edges.build_case: three zero rows and three rows at 1e-25."""
    K, d, cov, _, _, _ = ROWS[name]
    tuples, B_vec, sizes = cov(num_sms)
    rng = np.random.default_rng(2000 + seed + sum(map(ord, name)))
    phi = np.concatenate([np.tile(np.asarray(t, dtype=np.int64), (s, 1)) for t, s in zip(tuples, sizes)])
    phi = phi[rng.permutation(len(phi))]
    N = len(phi)
    n_types = max(4, min(K, 30))
    centers = rng.standard_normal((n_types, d)) * 2.0
    Z = centers[rng.integers(0, n_types, N)] + 0.7 * rng.standard_normal((N, d))
    Z += 0.5 * rng.standard_normal((sum(B_vec), d))[phi].sum(axis=1)
    Z *= (10.0 / np.sqrt(1.0 + np.arange(d)))[None, :]
    special = rng.choice(N, 6, replace=False)
    Z[special[:3]] = 0.0
    Z[special[3:]] *= 1e-25 / np.abs(Z[special[3:]]).max(axis=1, keepdims=True)
    return dict(Z=Z, phi=phi, B_vec=B_vec, K=K, d=d, N=N, sizes=sizes, tuples=tuples)


@pytest.mark.parametrize("name", list(ROWS))
def test_wide_rows_reach_their_kernels(name):
    c = build_case(name, 132)
    K, d, _, want, update, ks = ROWS[name]
    J = len(c["sizes"])
    assert wide_paths(K, d, J, c["N"], 132, ks) == want
    assert kernel_paths(K, d, J, c["N"], 132)[0] == update


# ---- GPU ----------------------------------------------------------------------------------------------------------------
def _prenormalised(Z):
    """Z with the rows whose fp32 sum of squares under- or overflows (|v| ~ 1e-25 or 1e20) divided by their norm in fp64:
    the reference's fp32 arithmetic does not rescale such rows, so the fp32 oracle would measure that, not the stage."""
    Z = np.array(Z, dtype=np.float64)
    m = np.abs(Z).max(axis=1)
    x = (m > 0) & ((m < 1e-10) | (m > 1e10))
    Z[x] /= np.linalg.norm(Z[x] / m[x, None], axis=1, keepdims=True) * m[x, None]
    return Z


def _oracle(c, Z, dbl):
    from oracle.oracle import OracleHarmony
    B = sum(c["B_vec"])
    o = OracleHarmony(double=dbl)
    o.setup(Z=Z, phi_i=c["phi"], B_vec=np.asarray(c["B_vec"]), sigma=np.full(c["K"], SIGMA), theta=np.full(B, 2.0),
            lambda_=None, alpha=ALPHA, max_iter_kmeans=T, epsilon_kmeans=-np.inf, epsilon_harmony=-np.inf, K=c["K"],
            block_size=BLOCK, batch_proportion_cutoff=CUTOFF)
    return o


def _fp32_errors(c, Y0, R2, O2, E2, perms2, Zp, Yp, perms3):
    """max |R32 - R64| of the fp32 and fp64 oracles after each stage, each on that stage's inputs: S1 setup +
    init_cluster_cpp(Y0); S2 R, O, E written, then cluster_cpp; S3 Z_corr = Zp and Y = Yp, then cluster_cpp.  The R
    error of these stages comes from fp32 dot products over d columns amplified 2 / sigma = 20 times; where fp32 itself
    cannot hold the edge file's bar (d = 512), twice this error is the stage's bar."""
    R = {}
    for dbl in (False, True):
        o = _oracle(c, _prenormalised(c["Z"]), dbl)
        o.init_cluster_cpp(Y0)
        r1 = o.get("R")
        o.set("R", R2)
        o.set("O", O2.T)
        o.set("E", E2.T)
        o.cluster_cpp(perms2)
        r2 = o.get("R")
        o = _oracle(c, _prenormalised(Zp), dbl)
        o.init_cluster_cpp(Yp)
        o.cluster_cpp(perms3)
        R[dbl] = (r1, r2, o.get("R"))
    return [float(np.abs(a - b).max()) for a, b in zip(R[False], R[True])]


def _report(name, stage, errs, bars, ratios):
    print(f"[wide {name} {stage}] " + " ".join(f"{k}={v:.2e}(bar {bars[k]:.1e}, {v / bars[k]:.2f})" for k, v in errs.items()))
    for k, v in errs.items():
        ratios.append(v / bars[k])
        assert v <= bars[k], (name, stage, k, v, bars[k])


def _assign_launches(K, wide_logits, plan, normalise):
    lg = 1 + (K + 127) // 128 if wide_logits else (K + 63) // 64
    return lg + 2 + (1 if normalise and not plan else 0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ROWS))
def test_wide_row_stages(name):
    from harmony_b200.harmony import harmony
    sms = num_sms()
    c = build_case(name, sms)
    K, d, _, want, update, ks = ROWS[name]
    N, B, J = c["N"], sum(c["B_vec"]), len(c["sizes"])
    paths = wide_paths(K, d, J, N, sms, ks)
    assert paths == want
    rng = np.random.default_rng(11)
    Zf = f32(c["Z"])
    Y0 = f32(make_Y0(c["Z"], K, rng))
    # the inputs of S2 and S3 (drawn here, in the order the stages use them), then the fp32 oracle's R error per stage
    R2, _, _ = planted_R(c, rng)
    R4, kz, _ = planted_R(c, rng, special=True)
    Zp = rng.standard_normal((N, d)) * rng.uniform(0.1, 30.0, (N, 1))
    special = rng.choice(N, 8, replace=False)
    Zp[special[:2]] = 0.0
    Zp[special[2:5]] *= 1e-25 / np.abs(Zp[special[2:5]]).max(axis=1, keepdims=True)
    Zp[special[5:]] *= 1e20 / np.abs(Zp[special[5:]]).max(axis=1, keepdims=True)
    Zp = f32(Zp)
    Yp = rng.standard_normal((K, d))
    Yp = f32(Yp / np.linalg.norm(Yp, axis=1, keepdims=True))
    perms2, perms3 = make_perms(N, T, 5), make_perms(N, T, 6)
    npy = numpy_model(c, Zf)
    O2, E2 = tables_of(R2, c, npy.Pr_b)
    e32 = _fp32_errors(c, Y0, R2, O2, E2, perms2, Zp, Yp, perms3)
    bar_R1, bar_R2, bar_R3 = max(TOL_R1, 2 * e32[0]), max(TOL_R, 2 * e32[1]), max(TOL_R, 2 * e32[2])
    print(f"[wide {name}] fp32 oracle max|dR| per stage {e32[0]:.2e} {e32[1]:.2e} {e32[2]:.2e} -> R bars "
          f"{bar_R1:.2e} {bar_R2:.2e} {bar_R3:.2e}")
    ratios = []

    # ---- S1: setup + init_cluster_cpp(Y0)
    g = harmony()
    g.kernel_set = ks
    g.setup(c["Z"], c["phi"], SIGMA, np.full(B, 2.0), None, ALPHA, T, -np.inf, -np.inf, K, BLOCK, c["B_vec"], CUTOFF)
    errs = dict(Zn=float(np.abs(g.getZcorr().T - npy.Z_corr).max()))
    as0 = _launches(g, "assign")
    g.init_cluster_cpp(Y0)
    npy.init_cluster(Y0)
    if paths[0] in (A_LOGITS, A_WIDE):
        assert _launches(g, "assign") - as0 == _assign_launches(K, paths[0] == A_WIDE, False, False)
    errs.update(R=float(np.abs(g.R.T - npy.R).max()), O=_table_err(g.O, npy.O), E=_table_err(g.E, npy.E),
                obj=_obj_err(g, npy, 1))
    _report(name, "S1 assign", errs, dict(Zn=TOL_ZN, R=bar_R1, O=TOL_OE, E=TOL_OE, obj=TOL_OBJ),
            ratios)

    # ---- S2: R, O, E written through the fields, then one cluster_cpp call from them
    g.R, g.O, g.E = R2.T, O2, E2
    npy.R, npy.O, npy.E = R2, O2, E2
    assert g.cluster_cpp(perms2) == 0
    npy.cluster(perms2)
    errs = dict(R=float(np.abs(g.R.T - npy.R).max()), O=_table_err(g.O, npy.O), E=_table_err(g.E, npy.E),
                obj=_obj_err(g, npy, T))
    _report(name, "S2 update from written R", errs, dict(R=bar_R2, O=TOL_OE, E=TOL_OE, obj=TOL_OBJ), ratios)

    # ---- S4: ridge step from planted R, O, E, estimated then fixed lambda
    O, E = tables_of(R4, c, npy.Pr_b)
    g.R, g.O, g.E = R4.T, O, E
    npy.R, npy.O, npy.E = R4, O, E
    for lam in (None, np.concatenate([[0.0], np.linspace(0.5, 2.0, B)])):
        if lam is not None:
            g.lambda_ = lam
            npy.lam = lam
        Yb = g.Y.T.astype(np.float64)
        npy.Y = Yb
        ap0 = _launches(g, "ridge_apply")
        g.moe_correct_ridge_cpp()
        npy.moe_correct_ridge()
        if paths[2] != P_FFMA:
            assert _launches(g, "ridge_apply") - ap0 == _apply_launches(K, d, paths[2] == P_COLS)
        Yg = g.Y.T
        errs = dict(Z=rel_l2(g.getZcorr().T, npy.Z_corr), Y=float(np.abs(Yg - npy.Y).max()))
        _report(name, f"S4 ridge {'fixed' if lam is not None else 'estimated'} lambda", errs,
                dict(Z=TOL_Z, Y=TOL_Y if lam is None else TOL_Y_FIXED), ratios)
        np.testing.assert_array_equal(Yg[kz], np.float32(Yb[kz]))

    # ---- S3: planted Z_corr and Y, cold-start cluster_cpp
    _set_zcorr(g, Zp)
    g.Y = Yp.T
    npy.Z_corr, npy.Y = Zp, Yp
    as0 = _launches(g, "assign")
    assert g.cluster_cpp(perms3) == 0
    npy.cluster(perms3)
    if paths[1] == C_WIDE:
        assert _launches(g, "assign") - as0 == _assign_launches(K, True, True, True)
    elif paths[1] == C_NATURAL and paths[0] in (A_LOGITS, A_WIDE):
        assert _launches(g, "assign") - as0 == _assign_launches(K, paths[0] == A_WIDE, False, True)
    errs = dict(R=float(np.abs(g.R.T - npy.R).max()), O=_table_err(g.O, npy.O), E=_table_err(g.E, npy.E),
                obj=_obj_err(g, npy, T), Zn=float(np.abs(g.getZcorr().T - npy.Z_corr).max()))
    _report(name, "S3 cold start", errs, dict(R=bar_R3, O=TOL_OE, E=TOL_OE, obj=TOL_OBJ, Zn=TOL_ZN), ratios)
    assert int(g.kmeans_rounds[-1]) == T
    print(f"[wide {name}] largest ratio to a bar: {max(ratios):.2f}")


@pytest.mark.gpu
def test_parity_d300_K100():
    """A whole run at d = 300, K = 100 (50k cells, 3 iterations, injected centroids and orders) meets the parity bars of
    test_gpu_parity.py against the fp32 and fp64 oracles."""
    from harmony_b200 import prepare_inputs
    from helpers import make_Y0 as make_Y0_h, run_oracle, synthetic
    from test_gpu_parity import compare, run_gpu
    Z, meta = synthetic(50000, 300, [8], n_types=20, seed=41)
    a = prepare_inputs(Z, meta, "cov0", nclust=100, early_stop=False)
    N, T_ = Z.shape[0], a["max_iter_kmeans"]
    n_iter = 3
    Y0 = make_Y0_h(Z, a["K"], 17)
    perms = make_perms(N, n_iter * T_, 23).reshape(n_iter, T_, N)
    o32, _, _ = run_oracle(a, Y0, n_iter, perms=perms)
    o64, _, _ = run_oracle(a, Y0, n_iter, perms=perms, double=True)
    g, iters = run_gpu(a, Y0, n_iter, perms)
    assert iters == n_iter
    compare(g, o32, o64, "d300_K100")


# ---- RunHarmony on a CUDA tensor against the oracles, with the library's native update orders replayed ----------------
def test_native_order_replay_matches_the_library():
    """native_order restates hb_permute_inv exactly (checked through hb_debug_permute, host only)."""
    L = _lib.lib()
    for n, rc in [(50000, 0), (50000, 37), (1000003, 5)]:
        order = native_order(n, 123, rc)
        key = int(_mix64(np.array([123 ^ int(_mix64(np.array([rc + 0x1234567], dtype=np.uint64))[0])],
                                  dtype=np.uint64))[0])
        for p in list(range(50)) + list(range(n - 50, n)):
            assert L.hb_debug_permute(p, n, key, 1) == order[p]
        if n < 100000:
            assert np.array_equal(np.sort(order), np.arange(n))


@pytest.mark.gpu
def test_runharmony_cuda_tensor_d300(monkeypatch):
    """RunHarmony on a CUDA tensor (d = 300, K = 100, 50k cells, seeded native k-means initialisation and update orders,
    10 iterations) meets test_gpu_parity.py's bars against the fp32 and fp64 oracles: the oracles start from the
    centroids the library's initialisation produced and replay its native update orders."""
    import torch
    from harmony_b200 import harmony_options, prepare_inputs, ui
    from helpers import run_oracle, synthetic
    from test_gpu_parity import compare
    SEED, ITERS = 20261015, 10
    # one cell type per cluster: with 20 types for K = 100 many clusters end up as near-duplicates after 10 iterations,
    # and their exact ties (top-2 gaps <= 3e-6) flip the hard index of ~0.2 % of the cells in any fp32 evaluation (the fp32
    # oracle itself flips 264 of 50k cells there, this path 98; DESIGN.md §4), more than assert_argmax_bounded's 0.05 %
    Z, meta = synthetic(50000, 300, [8], n_types=100, seed=41)
    opts = harmony_options(epsilon_cluster=-np.inf)   # every call runs all its rounds: round i T + t is call i's round t
    seen = {}
    real = ui.harmonize

    def harmonize(obj, it, verbose):
        seen["Y0"] = np.asarray(obj.Y).T.copy()       # the normalised centroids of the native initialisation
        return real(obj, it, verbose)
    monkeypatch.setattr(ui, "harmonize", harmonize)
    Zt = torch.from_numpy(Z).cuda()
    g = ui.RunHarmony(Zt, meta, "cov0", nclust=100, max_iter=ITERS, early_stop=False, options=opts, seed=SEED,
                      return_object=True, verbose=False)
    zt = ui.RunHarmony(Zt, meta, "cov0", nclust=100, max_iter=ITERS, early_stop=False, options=opts, seed=SEED,
                       verbose=False)
    assert zt.is_cuda and zt.dtype == torch.float64 and zt.shape == Zt.shape
    a = prepare_inputs(Z, meta, "cov0", nclust=100, early_stop=False, options=opts)
    N, T_ = Z.shape[0], a["max_iter_kmeans"]
    perms = np.stack([native_order(N, SEED, r) for r in range(ITERS * T_)]).reshape(ITERS, T_, N)
    o32, _, _ = run_oracle(a, seen["Y0"], ITERS, perms=perms)
    o64, _, _ = run_oracle(a, seen["Y0"], ITERS, perms=perms, double=True)
    compare(g, o32, o64, "RunHarmony d300_K100 cuda")
    # the tensor result of the same seeded run is the object's Z_corr up to fp32 atomics
    assert rel_l2(zt.cpu().numpy(), g.getZcorr().T) < 1e-5


# ---- two GPUs: a wide row sharded over the cells ------------------------------------------------------------------------
def _run_sharded(rank, world, port, q):
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import torch
    import torch.distributed as dist
    from harmony_b200 import prepare_inputs
    from harmony_b200.dist import make_comm, shard_bounds
    from harmony_b200.harmony import harmony
    from helpers import make_perms, make_Y0, synthetic
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        Z, meta = synthetic(30011, 300, [8], n_types=20, seed=13)   # d = 300, K = 100: d-chunked logits, column ranges
        a = prepare_inputs(Z, meta, "cov0", nclust=100, early_stop=False)
        N, T_ = Z.shape[0], a["max_iter_kmeans"]
        Y0 = make_Y0(Z, a["K"], 5)
        perms = make_perms(N, 2 * T_, 6).reshape(2, T_, N)
        lo, hi = shard_bounds(N, world, rank)
        res = {}
        for name, comm, rows in (("sharded", make_comm(N), slice(lo, hi)), ("single", None, slice(0, N))):
            if name == "single" and rank != 0:
                break
            g = harmony(device=rank, comm=comm) if comm is not None else harmony(device=rank)
            g.setup(a["Z"][rows], a["phi_i"][rows], a["sigma"], a["theta"], a["lambda_"], a["alpha"], T_,
                    a["epsilon_kmeans"], a["epsilon_harmony"], a["K"], a["block_size"], a["B_vec"],
                    a["batch_proportion_cutoff"])
            g.init_cluster_cpp(Y0)
            r = dict(O0=g.O.copy(), E0=g.E.copy())
            for it in range(2):
                assert g.cluster_cpp(perms[it]) == 0
                g.moe_correct_ridge_cpp()
                g.check_convergence(1)
            r.update(lo=lo, hi=hi, Z=g.getZcorr().T.copy(), R=g.R.T.copy(), O=g.O.copy(), E=g.E.copy(), Y=g.Y.copy(),
                     obj=g.objective_kmeans.copy())
            res[name] = r
        dist.barrier()
        q.put((rank, res))
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, "ERR " + traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_two_gpu_wide_row_equals_one_gpu():
    """The wide kernels with sharded cells (the natural-order assignment's O / row-sum all-reduce, the plan-order cold
    start's removal-sum all-reduce, the column-range apply) give the single-GPU result up to fp32 reassociation."""
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    assert wide_paths(100, 300, 8, 15006, torch.cuda.get_device_properties(0).multi_processor_count)[:3] == \
        (A_WIDE, C_WIDE, P_COLS)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_run_sharded, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=600) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    for r in res.values():
        assert not isinstance(r, str), r
    single, s0, s1 = res[0]["single"], res[0]["sharded"], res[1]["sharded"]
    Zs, Rs = np.concatenate([s0["Z"], s1["Z"]]), np.concatenate([s0["R"], s1["R"]])
    relz = np.linalg.norm(Zs - single["Z"]) / np.linalg.norm(single["Z"])
    print(f"[2gpu wide d300_K100] relL2 Z = {relz:.2e}, max|dR| = {np.abs(Rs - single['R']).max():.2e}")
    assert relz < 2e-5
    assert np.abs(Rs - single["R"]).max() < 1e-4
    for f in ("O0", "E0", "O", "E", "Y"):
        np.testing.assert_allclose(s0[f], s1[f], rtol=0, atol=0)            # replicated state identical
        np.testing.assert_allclose(s0[f], single[f], rtol=2e-4, atol=2e-3)
    np.testing.assert_allclose(s0["obj"], single["obj"], rtol=1e-4)
