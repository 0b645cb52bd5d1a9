"""Stage tests of the hot-path kernels at every kernel-selection boundary, against the fp64 numpy restatement.

Each row of EDGE_ROWS (stages.py) is a shape that straddles one limit of select_kernels (select.cuh) or of a kernel's
tiling: the fused assignment kernel at d = 64 and K = 128 and its m64n16 tail, the logits + softmax cold start past
them, the cluster ranges of the ridge apply (K > 112 runs as several launches), the cluster and column launches of the
ridge statistics (K > 128, d + 1 > 128), the FFMA kernels past d = 128, the per-step update past KS = 256, the
single-pass / two-pass switch at 2 J = #SMs, tuples whose sizes put short tiles at every tile edge, and blocks with
fewer cells than CTAs. Covariates are built so that the tuple sizes are exact.

Every row runs the four stages of stages.py (S1 assignment, S2 update from written R, S4 ridge, S3 cold start) on one
handle, with the default run parameters; each stage starts both sides from the same fp32 state, so a comparison
measures that stage's error alone, not drift accumulated over a run.
A CPU test pins which kernels each row reaches (hb_debug_kernel_paths at 132 SMs), and each GPU test asserts the same
with the device's SM count and counts the launches of the multi-launch ranges.
"""
import numpy as np
import pytest

from helpers import num_sms, rel_l2
from stages import (CUTOFF, EDGE_ROWS, T, TOL_R1, TOL_ZN, case_of, f32, kernel_paths, level_of_single_cluster, make_Y0,
                    numpy_model, oracle, planted_R, setup_gpu, stage_s1, stage_s2, stage_s3, stage_s4, tables_of)


# ---- CPU tests --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(EDGE_ROWS))
def test_edge_rows_reach_their_kernels(name):
    """Each row reaches the kernels it names, on a 132-SM H100 with 20 update blocks."""
    c = case_of(name, 132)
    J = len(c["sizes"])
    assert kernel_paths(c["K"], c["d"], J, c["N"], 132) == EDGE_ROWS[name][3]


@pytest.mark.parametrize("name", list(EDGE_ROWS))
def test_edge_row_builders(name):
    """Tuple sizes are exact, planted R rows sum to 1, the empty and the single-level clusters are there, and their
    levels' means stay clear of the cutoff."""
    c = case_of(name, 132)
    tup, counts = np.unique(c["phi"], axis=0, return_counts=True)
    want = {tuple(t): s for t, s in zip(c["tuples"], c["sizes"])}
    assert len(tup) == len(want)
    for t, n in zip(tup, counts):
        assert want[tuple(int(x) for x in t)] == n
    rng = np.random.default_rng(3)
    R, kz, ks = planted_R(c, rng, special=True)
    np.testing.assert_allclose(R.sum(axis=1), 1.0, atol=1e-6)
    assert (R[:, kz] == 0).all()
    b0 = level_of_single_cluster(c)
    assert (R[c["phi"][:, 0] != b0, ks] == 0).all() and (R[c["phi"][:, 0] == b0, ks] > 0).all()
    B = sum(c["B_vec"])
    N_b = np.bincount(c["phi"].ravel(), minlength=B)
    O, _ = tables_of(R, c, N_b / c["N"])
    avg = O / N_b[None, :]
    assert ((avg == 0) | (avg > 4 * CUTOFF)).all()
    if len(c["B_vec"]) > 1:   # the single-level cluster keeps >= 2 levels of another covariate (Gauss-Jordan branch)
        second = avg[ks, c["B_vec"][0]:c["B_vec"][0] + c["B_vec"][1]]
        assert (second > 0).sum() >= 2


@pytest.mark.parametrize("name", ["k1_tail_K17_d3", "tiny_blocks"])
@pytest.mark.parametrize("fixed_lambda", [False, True])
def test_planted_ridge_inputs_numpy_matches_oracle(name, fixed_lambda):
    """On the S4 inputs (one-hot rows, an empty cluster, a single-level cluster) the numpy restatement and the fp64
    oracle give the same ridge step: this pins the restatement on these edge inputs without a GPU."""
    c = case_of(name, 132)
    B = sum(c["B_vec"])
    lam = np.concatenate([[0.0], np.linspace(0.5, 2.0, B)]) if fixed_lambda else None
    rng = np.random.default_rng(7)
    Y0 = make_Y0(c["Z"], c["K"], rng)
    o = oracle(c, lambda_=lam)
    o.init_cluster_cpp(Y0)
    npy = numpy_model(c, c["Z"], lam)
    npy.init_cluster(Y0)
    R, kz, ks = planted_R(c, rng, special=True)
    O, E = tables_of(R, c, npy.Pr_b)
    o.set("R", R)
    o.set("O", O.T)
    o.set("E", E.T)
    npy.R, npy.O, npy.E = R, O, E
    npy.Y = o.get("Y")
    Ybefore = npy.Y.copy()
    o.moe_correct_ridge_cpp()
    npy.moe_correct_ridge()
    assert rel_l2(o.get("Z_corr"), npy.Z_corr) < 1e-9
    assert np.abs(o.get("Y") - npy.Y).max() < 1e-9
    np.testing.assert_allclose(o.get("lambda").T, npy.lambda_mat, rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(o.get("W").T, npy.W, rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(npy.Y[kz], Ybefore[kz] / np.linalg.norm(Ybefore[kz]), atol=1e-12)   # empty: skipped
    if len(c["B_vec"]) == 1:   # one covariate: the single-level cluster is skipped as well
        np.testing.assert_allclose(npy.Y[ks], Ybefore[ks] / np.linalg.norm(Ybefore[ks]), atol=1e-12)


# ---- GPU tests --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(EDGE_ROWS))
def test_edge_row_stages(name):
    sms = num_sms()
    c = case_of(name, sms)
    K, d, N = c["K"], c["d"], c["N"]
    J = len(c["sizes"])
    paths = EDGE_ROWS[name][3]
    assert kernel_paths(K, d, J, N, sms) == paths
    rng = np.random.default_rng(11)
    Zf = f32(c["Z"])
    Y0 = f32(make_Y0(c["Z"], K, rng))
    g = setup_gpu(c)
    npy = numpy_model(c, Zf)
    stage_s1(name, g, npy, Y0)
    assert stage_s2(name, g, npy, c, rng) == T
    stage_s4(name, g, npy, c, rng, EDGE_ROWS[name][4], EDGE_ROWS[name][5])
    # the logits cold start: one launch per 64-cluster range, the softmax pass and the finalize
    assign = (K + 63) // 64 + 2 if paths[2] and paths[5] else None
    assert stage_s3(name, g, npy, c, rng, assign_launches=assign) == T


@pytest.mark.gpu
@pytest.mark.parametrize("kernel_set", [0, 1])
def test_setup_normalises_rows_at_extreme_scales(kernel_set):
    """Rows whose fp32 sum of squares overflows (|v| ~ 1e20) or underflows (|v| <= 1e-25) are normalised like any
    other row at setup, and the assignment sees them so; a zero row stays zero."""
    c = case_of("k1_tail_K17_d3", num_sms())
    Z = c["Z"].copy()
    rng = np.random.default_rng(2)
    rows = rng.choice(c["N"], 12, replace=False)
    for i, s in zip(rows, [1e20, 3e25, 1e30, 1e-20, 1e-25, 1e-30, 1e-35, 0.0, 1e19, 1e-19, 1e-22, 1e-36]):
        Z[i] = 0.0 if s == 0 else Z[i] * s / np.abs(Z[i]).max()
    g = setup_gpu(dict(c, Z=Z), kernel_set=kernel_set)
    npy = numpy_model(c, f32(Z))
    Zn = g.getZcorr().T
    dz = float(np.abs(Zn - npy.Z_corr).max())
    Y0 = f32(make_Y0(c["Z"], c["K"], rng))
    g.init_cluster_cpp(Y0)
    npy.init_cluster(Y0)
    dR = float(np.abs(g.R.T - npy.R).max())
    print(f"[extreme rows kernel_set={kernel_set}] max|dZn|={dz:.2e} max|dR|={dR:.2e}")
    assert np.isfinite(Zn).all()
    assert dz <= TOL_ZN and dR <= TOL_R1
