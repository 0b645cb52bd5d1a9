"""Stage tests of the legacy centroid step (HB_LEGACY_CENTROID_STEP: STEP 1 of harmony.cpp:235-238, commented out in
2.0.4 but run by the package version that rendered the reference's vignette) against the fp64 numpy restatement.

The step is legacy_centroid_step (assign_host.cuh): the ridge statistics kernel K3 run on the normalised Z_corr, the
centroids Y_k = normalise(sum_q S[q][k][0..d)) of k_centroids_from_stats, and the natural-order assignment on the new
centroids, after which R, O, E and the objective sums are put back.  Every legacy call runs update_R per step and drops
a prebuilt plan.  Each row of LEGACY_ROWS is a shape of the edge or wide table that sends the step through one kernel:
the fused wgmma assignment, the FFMA k_assign, k_logits_tc or k_logits_wide with k_softmax_tiles, and K3's cluster and
column launches; two rows have a two-pass default, one runs per-cluster sigma and per-level theta.

Each row runs three stages on both sides from the same fp32 state:
  L1  setup + init_cluster_cpp(Y0), one legacy call (not a cold start: Z_corr is setup's normalised Z_orig)
  L2  R, O, E written on a fresh handle after init, with an exactly empty cluster and a cluster of mass ~1e-22,
      one legacy call
  L3  Z_corr and Y planted (stages.planted_zy), a cold-start legacy call
Compared: R, O, E, the call's objective terms and rounds (stages.py's bars), Y (the centroids of the call's last round)
and, after L3, the normalised Z_corr.
"""
import numpy as np
import pytest

from helpers import make_perms, num_sms
from stages import (A_FFMA, A_FUSED, A_LOGITS, A_WIDE, EDGE_ROWS, HB_KS_FFMA_CONTRACTIONS, HB_KS_WIDE, PER_STEP,
                    SINGLE_PASS, TOL_OBJ, TOL_OE, TOL_R, TWO_PASS, RunParams, _nested, _report, _set_zcorr, _sizes,
                    build_case, case_of, cluster_and_compare, f32, kernel_paths, make_Y0, native_order, numpy_model,
                    oracle, planted_zy, prenormalised, setup_gpu, sigma_vec, state_errs, tables_of, theta_levels,
                    wide_paths)

TAG = "legacy"
# Y, the centroids of the call's last round, max |d|.  New bar: Y comes from the 3xTF32 statistics of K3 (relative
# error of a product <= 2^-20) summed over the cells and normalised in fp32, from the R of the round before; measured
# at most 1.0e-5 (d300_K100 after L1) and otherwise <= 7e-6 on an H100 80GB HBM3 (700 W)
TOL_Y_LEGACY = 2e-5
# The rows on the d-chunked 3xTF32 logits at d = 300 and 512 exceed twice the fp32 oracle's error where the call's
# centroids are loosely pinned: after L3 (random planted Z_corr) and, at d = 300, after L2, whose emptied clusters are
# refilled in round 0 from the cells far from every centroid.  Bars at about twice the error measured on an H100 80GB
# HBM3 (700 W): d300_K100 L2 R 9.8e-5, Y 6.7e-5, L3 R 2.9e-5 (fp32 oracle 1.3e-5); d512_K200 L3 R 2.26e-4 (fp32
# oracle 6.1e-5).  At d = 512 the objective terms after L1 and L2 are 1.54e-4 off (relative; 3xTF32 distances over
# 512 columns): bar 3e-4
WIDE_LOGITS_BARS = {"d300_K100": {"L2": dict(R=2e-4, Y=1.5e-4), "L3": dict(R=6e-5)},
                    "d512_K200": {"L1": dict(obj=3e-4), "L2": dict(obj=3e-4), "L3": dict(R=5e-4)}}

# name -> (shape row of the edge or wide table, HB_KERNEL_SET, per-cluster sigma and per-level theta,
#          hb_debug_kernel_paths at 132 SMs, natural-order assignment of hb_debug_wide_paths)
LEGACY_ROWS = {
    # nested covariates; fused K1 with two operand stages
    "k1_K33_d63": ("k1_K33_d63", 0, False, (SINGLE_PASS, 2, 0, 1, 1, 1, SINGLE_PASS, PER_STEP), A_FUSED),
    # fused K1 at both limits (one stage); K3 one 128-column launch
    "k1_limit_K128_d64": ("k1_limit_K128_d64", 0, False, (SINGLE_PASS, 1, 0, 1, 1, 1, SINGLE_PASS, PER_STEP), A_FUSED),
    # FFMA k_assign; K3's second column launch (d + 1 = 130)
    "ffma_d129_K64": ("ffma_d129_K64", 0, False, (SINGLE_PASS, 0, 0, 0, 0, 0, SINGLE_PASS, PER_STEP), A_FFMA),
    # FFMA k_assign; K3's second column launch holds only the ones column, two cluster ranges (128 + 8)
    "stats_d128_K136": ("stats_d128_K136", 0, False, (SINGLE_PASS, 0, 0, 1, 0, 0, SINGLE_PASS, PER_STEP), A_FFMA),
    # k_logits_tc in natural order (12 ranges of 64) + k_softmax_tiles; per-step default
    "K705_d8": ("K705_d8", 0, False, (PER_STEP, 0, 1, 1, 0, 0, PER_STEP, PER_STEP), A_LOGITS),
    # k_logits_tc over 16 ranges, softmax with 8 pieces per lane; K3 eight cluster ranges
    "K1024_d64": ("K1024_d64", 0, False, (PER_STEP, 0, 1, 1, 0, 0, PER_STEP, PER_STEP), A_LOGITS),
    # k_logits_wide (d chunks) + k_softmax_tiles; K3 three column ranges; nested covariates
    "d300_K100": ("d300_K100", 0, False, (SINGLE_PASS, 0, 0, 0, 0, 1, SINGLE_PASS, PER_STEP), A_WIDE),
    # k_logits_wide over two 128-cluster ranges; K3 five column ranges x two cluster ranges
    "d512_K200": ("d512_K200", 0, False, (SINGLE_PASS, 0, 0, 0, 0, 1, SINGLE_PASS, PER_STEP), A_WIDE),
    # config 3's shape (K = 100, d = 50, 20 tuples) with the FFMA contractions forced
    "c3_shape_ffma": ("c3_shape_wide", HB_KS_FFMA_CONTRACTIONS, False, (SINGLE_PASS, 0, 0, 0, 0, 0, SINGLE_PASS, PER_STEP),
                      A_FFMA),
    # config 3's shape with the wide kernels forced
    "c3_shape_wide": ("c3_shape_wide", HB_KS_WIDE, False, (SINGLE_PASS, 0, 0, 0, 0, 1, SINGLE_PASS, PER_STEP), A_WIDE),
    # two-pass default (2 J = #SMs + 2), run per step
    "two_pass_Jmax+1": ("two_pass_Jmax+1", 0, False, (TWO_PASS, 2, 0, 1, 1, 0, PER_STEP, PER_STEP), A_FUSED),
    # two-pass default, 140 tuples of 1-11 cells over three covariates
    "tiny_blocks": ("tiny_blocks", 0, False, (TWO_PASS, 2, 0, 1, 1, 0, PER_STEP, PER_STEP), A_FUSED),
    # per-cluster sigma and per-level theta; nested covariates, fused K1 with one stage
    "sigma_theta_K113_d50": ("apply_K113_d50", 0, True, (SINGLE_PASS, 1, 0, 1, 1, 1, SINGLE_PASS, PER_STEP), A_FUSED),
}


def params_of(name, c, **kw):
    if not LEGACY_ROWS[name][2]:
        return RunParams(**kw)
    return RunParams(sigma=sigma_vec(c["K"]), theta=theta_levels(sum(c["B_vec"])), **kw)


def planted_R_legacy(R0, rng):
    """R written for L2: the fp32 R of the assignment from Y0 (so the centroids keep the data's structure), with
    cluster 1 exactly empty and cluster 0 given a total mass of 1e-22 spread over every cell: its fp32 centroid sums
    (~1e-23) square below the smallest float.  Returns R and the two clusters."""
    R = np.array(R0, dtype=np.float64)
    kt, kz = 0, 1
    R[:, [kt, kz]] = 0.0
    R /= R.sum(axis=1, keepdims=True)
    w = rng.random(len(R)) + 0.5
    R[:, kt] = 1e-22 * w / w.sum()
    return f32(R), kz, kt


def pair(c, p, kernel_set, Y0):
    """A library handle and the numpy model, both with the legacy step on, after setup and init_cluster_cpp(Y0)."""
    g = setup_gpu(c, p, kernel_set)
    g.legacy_centroid_step = 1
    assert g.legacy_centroid_step == 1
    npy = numpy_model(c, f32(c["Z"]), None, p)
    npy.legacy_centroid_step = True
    g.init_cluster_cpp(Y0)
    npy.init_cluster(Y0)
    return g, npy


def legacy_call(name, stage, g, npy, perms, ratios, bars=None, Zn=False):
    """One cluster_cpp call on both sides (stages.cluster_and_compare), then the centroids of its last round."""
    b = dict(Y=TOL_Y_LEGACY)
    b.update(bars or {})
    n = cluster_and_compare(name, stage, g, npy, perms, TAG, bars=b, ratios=ratios, Zn=Zn)
    _report(name, stage, dict(Y=float(np.abs(g.Y.T - npy.Y).max())), b, TAG, ratios)
    return n


def fp32_bars(c, p, Y0, perms1, Zp, Yp, perms3):
    """The wide file's rule for the stages whose inputs the oracle takes (L1: setup + init_cluster_cpp(Y0); L3: Z_corr =
    Zp, Y = Yp): the R and Y bars are at least twice the fp32 oracle's error against the fp64 oracle after the same
    legacy call.  Each round's centroids are means under the last round's R, so an error in R moves the next centroids,
    and the call's error grows the more loosely the data pins them; the fp32 oracle measures that growth on the stage's
    own inputs.  The objective keeps stages.py's bar (the oracle sums it in fp32; its error is printed).  Returns the
    bars of L1 and of L3."""
    got = {}
    for dbl in (False, True):
        got[dbl] = []
        for Z, Y, perms in ((c["Z"], Y0, perms1), (Zp, Yp, perms3)):
            o = oracle(c, p, dbl, prenormalised(Z), legacy=True)
            o.init_cluster_cpp(Y)
            o.cluster_cpp(perms)
            got[dbl].append((o.get("R"), o.get("Y"), o.trace("objective_kmeans")[-p.T:]))
    bars = []
    for a, b in zip(got[False], got[True]):
        e = dict(R=np.abs(a[0] - b[0]).max(), Y=np.abs(a[1] - b[1]).max(),
                 obj=(np.abs(a[2] - b[2]) / np.abs(b[2])).max())
        bars.append(dict(R=max(TOL_R, 2 * e["R"]), Y=max(TOL_Y_LEGACY, 2 * e["Y"])))
        print(f"[{TAG}] fp32 oracle: max|dR| {e['R']:.2e} max|dY| {e['Y']:.2e} objective {e['obj']:.2e}")
    return bars


# ---- CPU tests --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(LEGACY_ROWS))
def test_legacy_rows_reach_their_kernels(name):
    """Each row's kernels on a 132-SM H100 with 20 update blocks; the last value of hb_debug_kernel_paths is the update
    path of a call with the legacy step (per step on every row)."""
    c = case_of(LEGACY_ROWS[name][0], 132)
    _, ks, _, paths, assign = LEGACY_ROWS[name]
    J = len(c["sizes"])
    assert kernel_paths(c["K"], c["d"], J, c["N"], 132, kernel_set=ks) == paths
    assert wide_paths(c["K"], c["d"], J, c["N"], 132, kernel_set=ks)[0] == assign


def test_legacy_rows_cover_every_natural_order_assignment():
    assert {r[4] for r in LEGACY_ROWS.values()} == {A_FUSED, A_FFMA, A_LOGITS, A_WIDE}


@pytest.mark.parametrize("name,stage", [("tiny_blocks", "L1"), ("tiny_blocks", "L2"), ("sigma_theta_K113_d50", "L2")])
def test_numpy_legacy_step_matches_oracle(name, stage):
    """The numpy legacy step and the fp64 oracle's agree on three covariates (L1, L2), on the empty and the 1e-22 mass
    clusters (L2), and under per-cluster sigma and per-level theta on nested covariates: this pins the restatement the
    GPU stages compare against, without a GPU."""
    c = case_of(LEGACY_ROWS[name][0], 132)
    if name != "tiny_blocks":   # a smaller instance of the row's shape, for the oracle's plain loops
        K, d, _ = EDGE_ROWS[LEGACY_ROWS[name][0]][:3]
        c = build_case(name, K, d, lambda s: _nested(_sizes(10, 2000), 5), 132)
    p = params_of(name, c)
    rng = np.random.default_rng(11)
    Y0 = f32(make_Y0(c["Z"], c["K"], rng))
    o = oracle(c, p, legacy=True)
    npy = numpy_model(c, c["Z"], None, p)
    npy.legacy_centroid_step = True
    o.init_cluster_cpp(Y0)
    npy.init_cluster(Y0)
    kz = kt = None
    if stage == "L2":
        R, kz, kt = planted_R_legacy(npy.R, rng)
        O, E = tables_of(R, c, npy.Pr_b)
        o.set("R", R)
        o.set("O", O.T)
        o.set("E", E.T)
        npy.R, npy.O, npy.E = R, O, E
        assert 5e-23 < R[:, kt].sum() < 2e-22 and not R[:, kz].any()
    perms = make_perms(c["N"], p.T, 5)
    o.cluster_cpp(perms)
    npy.cluster(perms)
    assert np.abs(o.get("R") - npy.R).max() < 1e-9
    assert np.abs(o.get("Y") - npy.Y).max() < 1e-9
    np.testing.assert_allclose(o.get("O").T, npy.O, rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(o.get("E").T, npy.E, rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(o.trace("objective_kmeans"), npy.obj_kmeans, rtol=1e-6)   # the traces hold floats
    assert int(o.trace("kmeans_rounds")[-1]) == p.T
    np.testing.assert_allclose(np.linalg.norm(npy.Y, axis=1), 1.0, atol=1e-12)


def early_stop_epsilon(c, p, Y0, perms):
    """An epsilon_kmeans at which a legacy call stops at round s >= 5 with a clear margin: the geometric mean of the
    smallest convergence ratio before s and the one at s, as numpy measures them.  Returns (epsilon, s + 1 rounds,
    margin)."""
    npy = numpy_model(c, f32(c["Z"]), None, p)
    npy.legacy_centroid_step = True
    npy.init_cluster(Y0)
    npy.cluster(perms)
    o, w = npy.obj_kmeans, npy.window_size
    ratio = {t: abs(sum(o[t - i] for i in range(w)) - sum(o[t + 1 - i] for i in range(w))) / abs(sum(o[t - i] for i in range(w)))
             for t in range(w + 1, p.T)}
    best = max(range(w + 2, p.T), key=lambda s: min(ratio[t] for t in range(w + 1, s)) / ratio[s])
    above = min(ratio[t] for t in range(w + 1, best))
    return float(np.sqrt(above * ratio[best])), best + 1, above / ratio[best]


def test_early_stop_fixture_has_a_margin():
    """The early-stop test's epsilon stops the numpy call at a round after the first check, with a factor >= 2 between
    the ratios on either side of it (so fp32 objective sums cannot move the stop)."""
    c = case_of("k1_K33_d63", 132)
    p = RunParams(T=12)
    Y0 = f32(make_Y0(c["Z"], c["K"], np.random.default_rng(11)))
    eps, n, margin = early_stop_epsilon(c, p, Y0, make_perms(c["N"], p.T, 5))
    assert 6 <= n < p.T and margin >= 2.0, (eps, n, margin)


# ---- GPU tests --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(LEGACY_ROWS))
def test_legacy_row_stages(name):
    sms = num_sms()
    c = case_of(LEGACY_ROWS[name][0], sms)
    _, ks, _, paths, assign = LEGACY_ROWS[name]
    J = len(c["sizes"])
    if sms == 132:
        assert kernel_paths(c["K"], c["d"], J, c["N"], sms, kernel_set=ks) == paths
    assert wide_paths(c["K"], c["d"], J, c["N"], sms, kernel_set=ks)[0] == assign
    p = params_of(name, c)
    rng = np.random.default_rng(11)
    Y0 = f32(make_Y0(c["Z"], c["K"], rng))
    Zp, Yp = planted_zy(c, np.random.default_rng(13))
    perms1, perms2, perms3 = (make_perms(c["N"], p.T, s) for s in (4, 5, 6))
    bars1, bars3 = fp32_bars(c, p, Y0, perms1, Zp, Yp, perms3)
    wide = WIDE_LOGITS_BARS.get(name, {})
    bars2 = dict(bars1, **wide.get("L2", {}))
    bars1.update(wide.get("L1", {}))
    bars3.update(wide.get("L3", {}))
    ratios = []

    # L1: setup + init_cluster_cpp(Y0), one legacy call
    g, npy = pair(c, p, ks, Y0)
    assert legacy_call(name, "L1 after init", g, npy, perms1, ratios, bars1) == p.T

    # L2: R, O, E written (an empty cluster, a cluster of mass 1e-22), one legacy call.  The written R is L1's first R
    # with two clusters taken out, so the call runs on L1's data and centroids: L1's bars
    g, npy = pair(c, p, ks, Y0)
    R, _, _ = planted_R_legacy(npy.R, rng)
    O, E = tables_of(R, c, npy.Pr_b)
    g.R, g.O, g.E = R.T, O, E
    npy.R, npy.O, npy.E = R, O, E
    assert legacy_call(name, "L2 written R", g, npy, perms2, ratios, bars2) == p.T

    # L3: Z_corr and Y planted, a cold-start legacy call
    _set_zcorr(g, Zp)
    g.Y = Yp.T
    npy.Z_corr, npy.Y = Zp, Yp
    assert legacy_call(name, "L3 cold start", g, npy, perms3, ratios, bars3, Zn=True) == p.T
    print(f"[{TAG} {name}] largest ratio to a bar: {max(ratios):.2f}")


@pytest.mark.gpu
def test_legacy_early_stop():
    """A finite epsilon_kmeans stops a legacy call at the round numpy stops at (after the first check)."""
    c = case_of("k1_K33_d63", num_sms())
    rng = np.random.default_rng(11)
    Y0 = f32(make_Y0(c["Z"], c["K"], rng))
    perms = make_perms(c["N"], 12, 5)
    eps, n, margin = early_stop_epsilon(c, RunParams(T=12), Y0, perms)
    print(f"[{TAG} early stop] epsilon_kmeans {eps:.3e}: {n} rounds, margin {margin:.1f}")
    g, npy = pair(c, RunParams(T=12, epsilon_kmeans=eps), 0, Y0)
    ratios = []
    assert legacy_call("k1_K33_d63", "early stop", g, npy, perms, ratios) == n < 12


@pytest.mark.gpu
def test_native_orders_across_legacy_toggles():
    """Native update orders (no injected ones) over four calls: single-pass with the step off (it prebuilds the next
    call's plan), with the step on (per step: the prebuilt plan is dropped and its rounds drawn again), off, on.  Call i
    runs the native rounds 6 i .. 6 i + 5 of the seed, as numpy replays them."""
    SEED = 20261017
    c = case_of("k1_K33_d63", num_sms())
    p = RunParams()
    rng = np.random.default_rng(11)
    Y0 = f32(make_Y0(c["Z"], c["K"], rng))
    g = setup_gpu(c, p)
    g.set_seed(SEED)
    npy = numpy_model(c, f32(c["Z"]), None, p)
    g.init_cluster_cpp(Y0)
    npy.init_cluster(Y0)
    ratios = []
    for call, legacy in enumerate((False, True, False, True)):
        g.legacy_centroid_step = int(legacy)
        npy.legacy_centroid_step = legacy
        perms = np.stack([native_order(c["N"], SEED, p.T * call + t) for t in range(p.T)])
        before = len(npy.obj_kmeans)
        assert g.cluster_cpp() == 0
        npy.cluster(perms)
        n = len(npy.obj_kmeans) - before
        assert n == p.T and int(g.kmeans_rounds[-1]) == n
        errs = state_errs(g, npy, n)
        errs["Y"] = float(np.abs(g.Y.T - npy.Y).max())
        bars = dict(R=TOL_R, O=TOL_OE, E=TOL_OE, obj=TOL_OBJ, Y=TOL_Y_LEGACY)
        _report("native toggles", f"call {call} legacy={int(legacy)}", errs, bars, TAG, ratios)
    print(f"[{TAG} native toggles] largest ratio to a bar: {max(ratios):.2f}")
