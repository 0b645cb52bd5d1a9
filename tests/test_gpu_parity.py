"""GPU parity tests: the CUDA path (through the C ABI / the ``harmony`` class) against the CPU oracle on
the same inputs, with the k-means centroids and the per-round update orders injected into both
(SURVEY.md §0.3: parity is only definable that way).

Tolerances (BASELINE.json north_star; helpers.compare applies them): corrected embedding within 1e-4 rel-L2 of the
reference-order fp32 oracle; hard cluster index argmax_k R identical except for cells whose top-2 gap is inside the
fp32 noise band.  We additionally require the GPU to be no further from the fp64 oracle than
2x the fp32 oracle is (+ a small floor).

Where the reference-order fp32 arithmetic is itself further than the bar from exact arithmetic (measured:
rel-L2(oracle32, oracle64) = 2e-4 .. 3e-4 on the two- and three-covariate shapes of BASELINE.json configs 4
and 5 — fp32 `arma::inv` plus sequential fp32 sums over 40k cells), "within 1e-4 of the reference" cannot be
told apart from the reference's own rounding noise.  There the GPU must be within 1e-4 of the fp64 evaluation
of the same algorithm AND no further from the fp32 oracle than that oracle is from fp64 (+1e-5).

Hard cluster indices, explicitly (VERDICT r1 "weak" 2): against BOTH oracles every cell whose hard index
differs must be a near-tie of that oracle (top-2 gap <= ARGMAX_GAP_MAX), and the number of such cells is
bounded by ARGMAX_FRAC_MAX of the cells.  Calibration on the CPU: the fp32 oracle itself differs from the
fp64 one in 0 / 4 / 5 cells of 20k / 40k / 30k with gaps up to 1.8e-4.  Against the fp32 oracle both bounds
widen by that oracle's own deviation from fp64 (its flips are added to the count, twice its max |dR| bounds the
gap): with 200k cells per block its sequential sums drift to max |dR| 4e-2 and ~740 flips of 600k cells
(`synthetic_big_blocks`) while the GPU path stays at 2e-4 / 6 cells of the fp64 truth.
"""
import numpy as np
import pytest

from harmony_b200 import harmony_options, prepare_inputs
from helpers import (TOL_Z, assert_argmax_bounded, compare, gpu_setup, load_cell_lines, load_pbmc, make_perms, make_Y0,
                     oracle_setup, rel_l2, run_gpu, run_oracle, synthetic)

pytestmark = pytest.mark.gpu

CASES = {
    # config 1 of BASELINE.json: cell_lines_small, 1 covariate, K=5
    "cell_lines_small_K5": lambda: (load_cell_lines(True), "dataset", dict(nclust=5)),
    # test_integration.R:5-7
    "cell_lines_small_K50_T10": lambda: (load_cell_lines(True), "dataset",
                                         dict(theta=1, nclust=50, options=harmony_options(max_iter_cluster=10))),
    # test_two_variable.R:5-11 (arma::inv branch)
    "cell_lines_2cov_K50": lambda: (load_cell_lines(False), ["cell_type", "dataset"],
                                    dict(theta=[1, 1], nclust=50, options=harmony_options(max_iter_cluster=10))),
    "cell_lines_1cov_default": lambda: (load_cell_lines(False), "dataset", dict()),
    # config 2 of BASELINE.json: pbmc_stim, 50 PCs, covariate stim, K=50
    "pbmc_stim_K50": lambda: (load_pbmc(), "stim", dict(nclust=50)),
    "synthetic_3cov_nested": lambda: (synthetic(6000, 30, [4, 12, 3], seed=3), ["cov0", "cov1", "cov2"],
                                      dict(nclust=40, theta=[2, 1, 0.5])),
    "synthetic_fixed_lambda": lambda: (synthetic(5000, 16, [5], seed=4), "cov0", dict(nclust=24, lambda_=1.0)),
    "synthetic_theta0_sigma_vec": lambda: (synthetic(4000, 10, [3], seed=5), "cov0",
                                           dict(nclust=7, theta=0, sigma=np.linspace(0.08, 0.15, 7))),
    "synthetic_blocksize_odd": lambda: (synthetic(3001, 9, [2, 4], seed=6, nested=False), ["cov0", "cov1"],
                                        dict(nclust=33, options=harmony_options(block_size=0.07, max_iter_cluster=6))),
    "synthetic_K100_d50": lambda: (synthetic(20000, 50, [20], n_types=30, seed=7), "cov0", dict(nclust=100)),
    # the shape of BASELINE.json config 4 (dataset + donor nested, J = 40 tuples, arma::inv branch), K=100, d=50
    "config4_shape_2cov_J40": lambda: (synthetic(40000, 50, [10, 40], n_types=30, seed=8), ["cov0", "cov1"],
                                       dict(nclust=100)),
    # the shape of BASELINE.json config 5: K=200, d=100, 3 covariates (10 / 40 / 6 levels)
    "config5_shape_K200_d100_3cov": lambda: (synthetic(30000, 100, [10, 40, 6], n_types=30, seed=9),
                                             ["cov0", "cov1", "cov2"], dict(nclust=200)),
    # ADVICE r1: shapes that used to overflow the persistent update kernel's shared memory
    "synthetic_K128": lambda: (synthetic(12000, 24, [6], n_types=20, seed=10), "cov0", dict(nclust=128)),
    "synthetic_blocksize_001": lambda: (synthetic(20000, 20, [4], n_types=12, seed=11), "cov0",
                                        dict(nclust=100, options=harmony_options(block_size=0.01))),
    # few, large blocks: 600k cells in 3 blocks -> ~1380 rows per CTA and block step, 86 per warp: the prefetch cursor
    # of the update kernel walks several 32-row plan windows per step (config 3 has 21 rows per warp: one window)
    "synthetic_big_blocks": lambda: (synthetic(600000, 8, [3], n_types=6, seed=13), "cov0",
                                     dict(nclust=12, options=harmony_options(block_size=0.34, max_iter_cluster=3))),
    # legacy usage: many clustering rounds per call (max.iter.cluster = 40 > 31)
    "synthetic_T40": lambda: (synthetic(3000, 12, [3], seed=12), "cov0",
                              dict(nclust=10, options=harmony_options(max_iter_cluster=40, epsilon_cluster=-np.inf))),
}


@pytest.mark.parametrize("case", list(CASES))
def test_parity_full_run(case):
    (Z, meta), vars_use, kw = CASES[case]()
    a = prepare_inputs(Z, meta, vars_use, early_stop=False, **kw)
    N, T = Z.shape[0], a["max_iter_kmeans"]
    n_iter = 3
    Y0 = make_Y0(Z, a["K"], 17)
    perms = make_perms(N, n_iter * T, 23).reshape(n_iter, T, N)
    o32, _, _ = run_oracle(a, Y0, n_iter, perms=perms)
    o64, _, _ = run_oracle(a, Y0, n_iter, perms=perms, double=True)
    g, iters = run_gpu(a, Y0, n_iter, perms)
    assert iters == n_iter
    compare(g, o32, o64, case)


@pytest.mark.parametrize("N,n_iter,with32", [(200000, 2, True), (1000000, 1, False)])
def test_parity_large(N, n_iter, with32):
    """BASELINE.json config 3's shape (50 PCs, 20 batches, K=100) at 200k cells against both oracles and at the
    full 1M cells against the fp64 oracle (one Harmony iteration: ~40 s of CPU) — fp32 atomics over 1M cells are
    where drift would show (VERDICT r1 weak 3)."""
    Z, meta = synthetic(N, 50, [20], n_types=30, seed=21)
    a = prepare_inputs(Z, meta, "cov0", nclust=100, early_stop=False)
    T = a["max_iter_kmeans"]
    Y0 = make_Y0(Z[:50000], a["K"], 5)
    perms = make_perms(N, n_iter * T, 29).reshape(n_iter, T, N)
    o64, _, _ = run_oracle(a, Y0, n_iter, perms=perms, double=True)
    g, iters = run_gpu(a, Y0, n_iter, perms)
    assert iters == n_iter
    if with32:
        o32, _, _ = run_oracle(a, Y0, n_iter, perms=perms)
        compare(g, o32, o64, f"large_{N}")
        return
    Zg, Z64 = g.getZcorr().T, o64.get("Z_corr")
    Rg, R64 = g.R.T, o64.get("R")
    e = rel_l2(Zg, Z64)
    dR = float(np.abs(Rg - R64).max())
    print(f"[large_{N}] relL2(Z gpu,o64)={e:.2e} max|dR|={dR:.2e}")
    assert e <= TOL_Z
    assert dR <= 2e-4
    assert_argmax_bounded(Rg, R64, f"large_{N} vs oracle64")
    np.testing.assert_allclose(g.O.T, o64.get("O"), rtol=2e-4, atol=0.5)
    np.testing.assert_allclose(g.objective_kmeans, o64.trace("objective_kmeans"), rtol=2e-4)
    np.testing.assert_allclose(g.Y.T, o64.get("Y"), atol=5e-5)


@pytest.mark.parametrize("case", ["cell_lines_2cov_K50", "synthetic_K100_d50", "config4_shape_2cov_J40"])
def test_ridge_step_against_plain_formulas(case):
    """moe_correct_ridge_cpp against an INDEPENDENT restatement (tests/numpy_restatement.py: the plain-R
    formulas of vignettes/detailedWalkthrough.Rmd:637-649, 817-822 + the level filter of harmony.cpp:358-410,
    fp64, no code shared with oracle/): the GPU's own R, O, E after cluster_cpp() are handed to the numpy
    code, both run the ridge step, Z_corr and Y must agree.  The reference holds no number for this step
    (DESIGN.md section 4: this row stays unpinned by reference-produced values)."""
    from numpy_restatement import NumpyHarmony
    (Z, meta), vars_use, kw = CASES[case]()
    a = prepare_inputs(Z, meta, vars_use, early_stop=False, **kw)
    N, T = Z.shape[0], a["max_iter_kmeans"]
    Y0 = make_Y0(Z, a["K"], 17)
    perms = make_perms(N, T, 31)
    g = gpu_setup(a)
    g.init_cluster_cpp(Y0)
    assert g.cluster_cpp(perms) == 0
    npy = NumpyHarmony(a["Z"], a["phi_i"], a["B_vec"], a["sigma"], a["theta"], a["lambda_"], a["alpha"], T, a["K"],
                       a["block_size"], a["batch_proportion_cutoff"])
    npy.Y = g.Y.T.astype(np.float64)
    npy.R, npy.O, npy.E = g.R.T.astype(np.float64), g.O.astype(np.float64), g.E.astype(np.float64)
    g.moe_correct_ridge_cpp()
    npy.moe_correct_ridge()
    e = rel_l2(g.getZcorr().T, npy.Z_corr)
    dY = float(np.abs(g.Y.T - npy.Y).max())
    print(f"[ridge vs plain formulas, {case}] relL2(Z)={e:.2e} max|dY|={dY:.2e}")
    assert e <= 2e-5
    assert dY <= 5e-5


def test_parity_stepwise():
    """After init, after one clustering, after one correction: every exposed field against the oracle."""
    (Z, meta) = load_cell_lines(False)
    a = prepare_inputs(Z, meta, ["cell_type", "dataset"], nclust=30)
    N, T = Z.shape[0], a["max_iter_kmeans"]
    Y0 = make_Y0(Z, a["K"], 3)
    perms = make_perms(N, T, 1)
    o = oracle_setup(a)
    g = gpu_setup(a)
    assert (g.N, g.K, g.d, g.B) == (N, 30, 20, 5)
    np.testing.assert_allclose(g.getZorig().T, Z.astype(np.float32), rtol=0, atol=0)
    np.testing.assert_allclose(g.getZcorr().T, o.get("Z_corr"), atol=1e-6)
    np.testing.assert_allclose(g.Pr_b, o.get("Pr_b"), rtol=1e-6)
    o.init_cluster_cpp(Y0)
    g.init_cluster_cpp(Y0)
    np.testing.assert_allclose(g.R.T, o.get("R"), atol=5e-6)   # 3xTF32 contraction + ex2.approx softmax
    np.testing.assert_allclose(g.O.T, o.get("O"), rtol=1e-4, atol=1e-3)
    np.testing.assert_allclose(g.E.T, o.get("E"), rtol=1e-4, atol=1e-3)
    np.testing.assert_allclose(g.objective_kmeans, o.trace("objective_kmeans"), rtol=1e-4)
    o.cluster_cpp(perms)
    g.cluster_cpp(perms)
    np.testing.assert_allclose(g.R.T, o.get("R"), atol=1e-5)
    np.testing.assert_allclose(g.O.T, o.get("O"), rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(g.E.T, o.get("E"), rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(g.objective_kmeans, o.trace("objective_kmeans"), rtol=2e-4)
    o.moe_correct_ridge_cpp()
    g.moe_correct_ridge_cpp()
    assert rel_l2(g.getZcorr().T, o.get("Z_corr")) < 2e-5
    np.testing.assert_allclose(g.Y.T, o.get("Y"), atol=2e-5)
    np.testing.assert_allclose(g.getLambda().T, o.get("lambda"), rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(g.W.T, o.get("W"), rtol=1e-3, atol=1e-5)
    g.compute_objective()   # standalone objective == the fused one of the last round
    ok = g.objective_kmeans
    np.testing.assert_allclose(ok[-1], ok[-2], rtol=1e-5)


def test_small_n_guards_and_errors():
    # harmony.cpp:83-91 and the error conventions of the C ABI
    from harmony_b200.harmony import HarmonyError, harmony
    Z, meta = synthetic(5, 4, [2], seed=1)
    a = prepare_inputs(Z, meta, "cov0", nclust=2)
    g = harmony()
    with pytest.raises(HarmonyError, match="less than 6 cells"):
        g.setup(a["Z"], a["phi_i"], a["sigma"], a["theta"], None, 0.2, 4, 1e-3, 1e-2, 2, 0.05, a["B_vec"], 1e-5)
    Z, meta = synthetic(30, 4, [2], seed=1)
    a = prepare_inputs(Z, meta, "cov0", nclust=2)
    g = harmony()
    with pytest.warns(UserWarning, match="Too few cells"):
        g.setup(a["Z"], a["phi_i"], a["sigma"], a["theta"], None, 0.2, 4, 1e-3, 1e-2, 2, 0.05, a["B_vec"], 1e-5)
    Y0, perms = make_Y0(Z, 2, 0), make_perms(30, 4, 0)
    g.init_cluster_cpp(Y0)
    g.cluster_cpp(perms)
    g.moe_correct_ridge_cpp()
    o, _, _ = run_oracle(dict(a, epsilon_harmony=-np.inf), Y0, 1, perms=perms.reshape(1, 4, 30))
    assert rel_l2(g.getZcorr().T, o.get("Z_corr")) < 1e-4
    g2 = harmony()
    with pytest.raises(HarmonyError):
        g2.init_cluster_cpp(Y0)          # before setup
    bad = perms.copy()
    bad[0, 0] = 10 ** 6
    with pytest.raises(HarmonyError, match="outside"):
        g.cluster_cpp(bad)


def test_field_writes_and_resume():
    """Fields are read-write like the Rcpp module's (.field); the object survives across harmonize calls
    (vignettes/detailedWalkthrough.Rmd:364, 891-893)."""
    from harmony_b200.harmony import harmony
    Z, meta = load_cell_lines(True)
    a = prepare_inputs(Z, meta, "dataset", nclust=5)
    g = harmony()
    g.setup(a["Z"], a["phi_i"], a["sigma"], a["theta"], None, a["alpha"], 4, 1e-3, 1e-2, 5, 0.05, a["B_vec"], 1e-5)
    g.init_cluster_cpp(make_Y0(Z, 5, 0))
    g.max_iter_kmeans = 10
    assert g.max_iter_kmeans == 10
    g.cluster_cpp(make_perms(300, 10, 0))
    assert 5 <= int(g.kmeans_rounds[-1]) <= 10
    Y = g.Y.copy()
    g.Y = Y * 1.0
    np.testing.assert_array_equal(g.Y, Y.astype(np.float32))
    g.moe_correct_ridge_cpp()
    g.cluster_cpp(make_perms(300, 10, 1))
    assert len(g.objective_harmony) == 3


@pytest.mark.parametrize("kernel_set", [
    1,    # HB_KS_FFMA_CONTRACTIONS: fp32 FFMA assignment / apply / k-means initialisation instead of wgmma
    2,    # HB_KS_UPDATE_PER_STEP: three launches per block step
    4,    # HB_KS_UPDATE_TWO_PASS: two-pass persistent update_R kernel
])
def test_fallback_kernels_match_oracle(kernel_set):
    """The FFMA / per-step / two-pass kernels that serve shapes outside the default kernels' limits (d > 64, K > 128,
    too many tuples for tuple-aligned CTA slices) are forced onto a shape the default kernels would take through the
    HB_KERNEL_SET test hook of the handle (include/harmony_b200.h) and held to the same parity bar."""
    (Z, meta), vars_use, kw = CASES["synthetic_3cov_nested"]()
    a = prepare_inputs(Z, meta, vars_use, early_stop=False, **kw)
    N, T = Z.shape[0], a["max_iter_kmeans"]
    Y0 = make_Y0(Z, a["K"], 17)
    perms = make_perms(N, 2 * T, 23).reshape(2, T, N)
    o32, _, _ = run_oracle(a, Y0, 2, perms=perms)
    o64, _, _ = run_oracle(a, Y0, 2, perms=perms, double=True)
    g, iters = run_gpu(a, Y0, 2, perms, kernel_set=kernel_set)
    compare(g, o32, o64, f"kernel_set {kernel_set}")
