"""Stage tests of the hot-path kernels at every kernel-selection boundary, against the fp64 numpy restatement.

Each row of EDGE_ROWS is a shape that straddles one limit of select_kernels (select.cuh) or of a kernel's tiling:
the fused assignment kernel at d = 64 and K = 128 and its m64n16 tail, the logits + softmax cold start past them, the
cluster ranges of the ridge apply (K > 112 runs as several launches), the cluster and column launches of the ridge
statistics (K > 128, d + 1 > 128), the FFMA kernels past d = 128, the per-step update past KS = 256, the single-pass /
two-pass switch at 2 J = #SMs, tuples whose sizes put short tiles at every tile edge, and blocks with fewer cells than
CTAs.  Covariates are built so that the tuple sizes are exact.

Every row runs the four stages of stages.py (S1 assignment, S2 update from written R, S4 ridge, S3 cold start) on one
handle, with the default run parameters; each stage starts both sides from the same fp32 state, so a comparison
measures that stage's error alone, not drift accumulated over a run.
A CPU test pins which kernels each row reaches (hb_debug_kernel_paths at 132 SMs), and each GPU test asserts the same
with the device's SM count and counts the launches of the multi-launch ranges.
"""
import numpy as np
import pytest

from helpers import num_sms, rel_l2
from stages import (ALPHA, BLOCK, CUTOFF, NB, PER_STEP, SIGMA, SINGLE_PASS, T, TOL_OBJ, TOL_OE, TOL_R, TOL_R1,  # noqa: F401
                    TOL_Y, TOL_Y_FIXED, TOL_Z, TOL_ZN, TWO_PASS, _grid, _launches, _nested, _obj_err, _one_cov,
                    _set_zcorr, _sizes, _table_err, f32, kernel_paths, level_of_single_cluster, make_Y0, numpy_model,
                    planted_R, setup_gpu, stage_s1, stage_s2, stage_s3, stage_s4, tables_of)
from stages import build_case as _build_case


# ---- rows ------------------------------------------------------------------------------------------------------------
# name -> (K, d, covariate builder(num_sms), expected hb_debug_kernel_paths tuple, ridge_stats launches,
#          ridge_apply launches).  Paths tuple: (update path, fused K1 stages, logits, wgmma apply, tensor-core k-means,
#          plan-order cold start, path of a 40-round call, path with the legacy centroid step).
EDGE_ROWS = {
    # fused K1 with the m64n16 tail only (NP = 32: K mod 32 = 17), smallest DS / KD
    "k1_tail_K17_d3": (17, 3, lambda s: _one_cov(_sizes(6, 6000)), (SINGLE_PASS, 2, 0, 1, 1, 1, SINGLE_PASS, PER_STEP), 1, 1),
    # fused K1: one n32 MMA plus the n16 tail (NP = 48)
    "k1_K33_d63": (33, 63, lambda s: _nested(_sizes(9, 8000), 3), (SINGLE_PASS, 2, 0, 1, 1, 1, SINGLE_PASS, PER_STEP), 1, 1),
    # fused K1 at both limits (one operand stage fits); K3 one 128-column launch (d + 1 = 65); K5 two ranges of 64
    "k1_limit_K128_d64": (128, 64, lambda s: _nested(_sizes(12, 10000), 4), (SINGLE_PASS, 1, 0, 1, 1, 1, SINGLE_PASS, PER_STEP), 1, 2),
    # d = 65: logits + softmax cold start
    "logits_K100_d65": (100, 65, lambda s: _one_cov(_sizes(8, 8000)), (SINGLE_PASS, 0, 1, 1, 1, 1, SINGLE_PASS, PER_STEP), 1, 1),
    # K = 129: logits; K3 second cluster launch k_off = 128 with 4 rows; apply 72 + 57; single-pass nv = 2
    "logits_K129_d64": (129, 64, lambda s: _one_cov(_sizes(7, 8000)), (SINGLE_PASS, 0, 1, 1, 1, 1, SINGLE_PASS, PER_STEP), 2, 2),
    # apply 64 + 49: the last range's stage row (52) is narrower than its KD (56); fused K1 with one stage
    "apply_K113_d50": (113, 50, lambda s: _nested(_sizes(10, 8000), 5), (SINGLE_PASS, 1, 0, 1, 1, 1, SINGLE_PASS, PER_STEP), 1, 2),
    # d + 1 = 128: the ones column is the last column of a full launch; K3 two cluster ranges (the second of 8 rows);
    # apply 72 + 64.  The logits kernel's operands do not fit shared memory at KD = 128: FFMA assignment.  (The FFMA
    # assignment kernel holds K x d up to about 136 x 128: larger K at this d is rejected by init_cluster_cpp.)
    "stats_d127_K136": (136, 127, lambda s: _one_cov(_sizes(5, 6000)), (SINGLE_PASS, 0, 0, 1, 0, 0, SINGLE_PASS, PER_STEP), 2, 2),
    # d + 1 = 129: the second column launch holds only the ones column (RC = 0)
    "stats_d128_K136": (136, 128, lambda s: _one_cov(_sizes(5, 6000)), (SINGLE_PASS, 0, 0, 1, 0, 0, SINGLE_PASS, PER_STEP), 4, 2),
    # KS = 256: the widest single-pass row (nv = 2) and tensor-core k-means; apply 88 + 88 + 80
    "single_pass_K256_d16": (256, 16, lambda s: _one_cov(_sizes(6, 8000)), (SINGLE_PASS, 0, 1, 1, 1, 1, SINGLE_PASS, PER_STEP), 2, 3),
    # d = 129: FFMA assignment and apply; K3 second column launch with 4 columns
    "ffma_d129_K64": (64, 129, lambda s: _one_cov(_sizes(6, 6000)), (SINGLE_PASS, 0, 0, 0, 0, 0, SINGLE_PASS, PER_STEP), 2, 1),
    # K = 257: per-step update, FFMA k_assign<16>
    "per_step_K257": (257, 8, lambda s: _one_cov(_sizes(6, 8000)), (PER_STEP, 0, 1, 1, 0, 0, PER_STEP, PER_STEP), 3, 3),
    # K = 520: k_assign<32>
    "per_step_K520": (520, 8, lambda s: _one_cov(_sizes(4, 3000)), (PER_STEP, 0, 1, 1, 0, 0, PER_STEP, PER_STEP), 5, 5),
    # 2 J = #SMs: the last J of the single-pass kernel
    "single_pass_Jmax": (40, 20, lambda s: _nested(_sizes(s // 2, 12000), 6), (SINGLE_PASS, 2, 0, 1, 1, 1, SINGLE_PASS, PER_STEP), 1, 1),
    # 2 J = #SMs + 2: the two-pass kernel (round 0 of a call after a written R reads that R)
    "two_pass_Jmax+1": (40, 20, lambda s: _nested(_sizes(s // 2 + 1, 12000), 6), (TWO_PASS, 2, 0, 1, 1, 0, PER_STEP, PER_STEP), 1, 1),
    # 64-row (K3 / K5 / update) and 128-row (K1) tiles never cross a tuple: short tiles at every edge
    "tuple_edges": (100, 50, lambda s: _one_cov([1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 8000]),
                    (SINGLE_PASS, 2, 0, 1, 1, 1, SINGLE_PASS, PER_STEP), 1, 1),
    # ~840 cells in 140 tuples of 1-11 cells: blocks of ~42 cells over the persistent CTAs, most of them idle
    "tiny_blocks": (24, 10, lambda s: _grid([5, 7, 4], lambda q: 1 + (7 * q) % 11),
                    (TWO_PASS, 2, 0, 1, 1, 0, PER_STEP, PER_STEP), 1, 1),
}


def build_case(name, num_sms, seed=0):
    """Inputs of a row (stages.build_case)."""
    K, d, cov, _, _, _ = EDGE_ROWS[name]
    return _build_case(name, K, d, cov, num_sms, seed)


# ---- CPU tests --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(EDGE_ROWS))
def test_edge_rows_reach_their_kernels(name):
    """Each row reaches the kernels it names, on a 132-SM H100 with 20 update blocks."""
    c = build_case(name, 132)
    J = len(c["sizes"])
    assert kernel_paths(c["K"], c["d"], J, c["N"], 132) == EDGE_ROWS[name][3]


@pytest.mark.parametrize("name", list(EDGE_ROWS))
def test_edge_row_builders(name):
    """Tuple sizes are exact, planted R rows sum to 1, the empty and the single-level clusters are there, and their
    levels' means stay clear of the cutoff."""
    c = build_case(name, 132)
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
    from oracle.oracle import OracleHarmony
    c = build_case(name, 132)
    B = sum(c["B_vec"])
    lam = np.concatenate([[0.0], np.linspace(0.5, 2.0, B)]) if fixed_lambda else None
    rng = np.random.default_rng(7)
    Y0 = make_Y0(c["Z"], c["K"], rng)
    o = OracleHarmony(double=True)
    o.setup(Z=c["Z"], phi_i=c["phi"], B_vec=np.asarray(c["B_vec"]), sigma=np.full(c["K"], SIGMA), theta=np.full(B, 2.0),
            lambda_=lam, alpha=ALPHA, max_iter_kmeans=T, epsilon_kmeans=-np.inf, epsilon_harmony=-np.inf, K=c["K"],
            block_size=BLOCK, batch_proportion_cutoff=CUTOFF)
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
    c = build_case(name, sms)
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
    # logits per 64-cluster range + softmax pass + finalize
    assert stage_s3(name, g, npy, c, rng, logits_launches=bool(paths[2] and paths[5])) == T


@pytest.mark.gpu
@pytest.mark.parametrize("kernel_set", [0, 1])
def test_setup_normalises_rows_at_extreme_scales(kernel_set):
    """Rows whose fp32 sum of squares overflows (|v| ~ 1e20) or underflows (|v| <= 1e-25) are normalised like any
    other row at setup, and the assignment sees them so; a zero row stays zero."""
    from harmony_b200.harmony import harmony
    c = build_case("k1_tail_K17_d3", num_sms())
    Z = c["Z"].copy()
    rng = np.random.default_rng(2)
    rows = rng.choice(c["N"], 12, replace=False)
    for i, s in zip(rows, [1e20, 3e25, 1e30, 1e-20, 1e-25, 1e-30, 1e-35, 0.0, 1e19, 1e-19, 1e-22, 1e-36]):
        Z[i] = 0.0 if s == 0 else Z[i] * s / np.abs(Z[i]).max()
    K, B = c["K"], sum(c["B_vec"])
    g = harmony()
    g.kernel_set = kernel_set
    g.setup(Z, c["phi"], SIGMA, np.full(B, 2.0), None, ALPHA, T, -np.inf, -np.inf, K, BLOCK, c["B_vec"], CUTOFF)
    npy = numpy_model(c, f32(Z))
    Zn = g.getZcorr().T
    dz = float(np.abs(Zn - npy.Z_corr).max())
    Y0 = f32(make_Y0(c["Z"], K, rng))
    g.init_cluster_cpp(Y0)
    npy.init_cluster(Y0)
    dR = float(np.abs(g.R.T - npy.R).max())
    print(f"[extreme rows kernel_set={kernel_set}] max|dZn|={dz:.2e} max|dR|={dR:.2e}")
    assert np.isfinite(Zn).all()
    assert dz <= TOL_ZN and dR <= TOL_R1
