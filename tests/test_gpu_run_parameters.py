"""Stage tests of the hot-path kernels under run parameters other than the edge table's (scalar sigma = 0.1, theta = 2
on every level, block size 0.05, 6 rounds per call, no early stop), against the fp64 numpy restatement.

Each row pairs a shape of test_gpu_kernel_edges.py (or, for d127_K200, of test_gpu_wide_shapes.py) with one run
parameter, and names the code that parameter reaches:
- sigma per cluster (fp32-distinct values in [0.1, 0.3], not monotone in k, sigma_0 not the smallest): the
  <NV, false> instances of the single-pass kernel and their objective sums, the two-pass kernel's sig_u = 0 branch,
  sigma[n_off + k] of the logits kernels past cluster 64 / 128, the softmax passes and the per-step sig table;
  stages S1, S2, a standalone compute_objective and S3;
- theta per level (0, 0.5, 1, 2, 3 cycled over the global levels): derive()'s theta[b], both ways the two-pass kernel
  finds b, the objective's cross-entropy term; stages S1, S2 and S3;
- sigma written through the field after init_cluster_cpp: the next update_R and compute_objective divide the distances
  of the last assignment by the new sigma, as the reference does;
- block counts (nb = 1, 3, 100, a last block larger than the others, one-cell blocks, the largest nb at which the
  two-pass kernel fits and one more); stages S2 and S3;
- call lengths T = 0, 1, 2, 5 (and 31 / 32 on the two-pass row): which rounds store R and file the next round's
  removal sums; stages S2 (warm) and S3 (cold);
- early stop (epsilon_kmeans = +inf: every convergence check passes, so a call stops after window_size + 2 = 5
  rounds), and the native update orders of three such calls on each update path.
The bars are the edge file's, except R in two places.  Where fp32 cannot hold the R bar on a row's inputs (the wide
row; nb = 1, where round 0 removes every cell and O, E fall to fp32 noise), the bar is the wide file's: twice the fp32
oracle's error on the same inputs, computed in the test and printed.  The wide row's R bars after S1 and S2 are 2e-5
(measured reason at the row).
"""
import numpy as np
import pytest

from helpers import make_perms
from numpy_restatement import my_ceil
from stages import (ALPHA, CUTOFF, PER_STEP, SINGLE_PASS, TOL_OBJ, TOL_OE, TOL_R, TOL_R1, TWO_PASS, RunParams,
                    _nested, _obj_err, _one_cov, _sizes, build_case, cluster_and_compare, f32, kernel_paths, make_Y0,
                    native_order, numpy_model, planted_R, planted_zy, setup_gpu, stage_s1, stage_s2, stage_s3,
                    state_errs, tables_of, _report, _table_err)
from test_gpu_kernel_edges import EDGE_ROWS
from test_gpu_wide_shapes import ROWS as WIDE_ROWS

HB_KS_UPDATE_PER_STEP, HB_KS_UPDATE_TWO_PASS = 2, 4
TAG = "runparam"


def sigma_vec(K):
    """0.1 (1 + 2 frac(0.618 (k + 3))): in [0.1, 0.3], not monotone, sigma_0 = 0.171 is not the smallest."""
    k = np.arange(K)
    return f32(0.1 * (1.0 + 2.0 * np.modf(0.618 * (k + 3))[0]))


def theta_levels(B):
    return np.array([(0.0, 0.5, 1.0, 2.0, 3.0)[b % 5] for b in range(B)])


def block_for(nb):
    """A block size that gives exactly nb blocks under the reference's my_ceil(1 / block_size)."""
    for x in (nb, nb - 0.5):
        bs = float(np.float32(1.0 / x))
        if my_ceil(np.float32(1.0) / np.float32(bs)) == nb:
            return bs
    raise AssertionError(nb)


# ---- rows ---------------------------------------------------------------------------------------------------------------
def _shape(row):
    if row in EDGE_ROWS:
        return EDGE_ROWS[row][0], EDGE_ROWS[row][1], EDGE_ROWS[row][2]
    return WIDE_ROWS[row][0], WIDE_ROWS[row][1], WIDE_ROWS[row][2]


SIGMA_ROWS = {
    "k1_K33_d63": "fused K1 with per-cluster sigma, single-pass <1, false>",
    "logits_K129_d64": "k_logits_tc ranges at n_off 64 and 128, single-pass <2, false>",
    "single_pass_K256_d16": "single-pass <2, false> at KS = 256",
    "two_pass_Jmax+1": "two-pass sig_u = 0",
    "per_step_K257": "per-step sig table, FFMA k_assign<16>",
    "ffma_d129_K64": "FFMA k_assign and single-pass <1, false>",
    "d127_K200": "k_logits_wide range n_off = 128, k_softmax_tiles",
}
THETA_ROWS = {
    "k1_tail_K17_d3": "derive() with theta per level, C = 1",
    "apply_K113_d50": "nested covariates, C = 2",
    "two_pass_Jmax+1": "both ways the two-pass kernel finds b",
    "per_step_K257": "per-step penalty table",
    "tiny_blocks": "three covariates, C = 3",
}
# name -> (table row, covariates override(num_sms) or None, nb)
BLOCK_ROWS = {
    "nb1_single_pass": ("k1_K33_d63", None, 1),
    "nb1_two_pass": ("two_pass_Jmax+1", None, 1),
    "nb3_single_pass": ("single_pass_K256_d16", None, 3),
    "nb3_two_pass": ("two_pass_Jmax+1", None, 3),
    # N = 1199 at 20 blocks: 19 blocks of 59 and a last block of 78
    "last_block_large": ("k1_tail_K17_d3", lambda s: _one_cov([200, 200, 200, 200, 199, 200]), 20),
    "nb100_single_pass": ("k1_K33_d63", None, 100),
    "nb100_two_pass": ("two_pass_Jmax+1", None, 100),
    # one-cell blocks (cells_per_block = 1, the last block takes the rest): 1400 blocks over 1601 cells, 1000 over 1292
    "one_cell_blocks_single_pass": ("k1_tail_K17_d3", lambda s: _one_cov(_sizes(6, 1800)), 1400),
    "one_cell_blocks_two_pass": ("two_pass_Jmax+1", lambda s: _nested(_sizes(s // 2 + 1, 1500), 6), 1000),
    # the largest nb at which the two-pass kernel's shared tables fit (132 SMs), then per step
    "two_pass_nb_max": ("two_pass_Jmax+1", None, 412),
    "two_pass_nb_max+1": ("two_pass_Jmax+1", None, 413),
}
BLOCK_PATHS = {
    "nb1_single_pass": SINGLE_PASS, "nb1_two_pass": TWO_PASS, "nb3_single_pass": SINGLE_PASS, "nb3_two_pass": TWO_PASS,
    "last_block_large": SINGLE_PASS, "nb100_single_pass": SINGLE_PASS, "nb100_two_pass": TWO_PASS,
    "one_cell_blocks_single_pass": SINGLE_PASS, "one_cell_blocks_two_pass": PER_STEP,
    "two_pass_nb_max": TWO_PASS, "two_pass_nb_max+1": PER_STEP,
}
LENGTH_ROWS = [(row, T) for row in ("k1_K33_d63", "two_pass_Jmax+1", "per_step_K257") for T in (0, 1, 2, 5)] + \
              [("two_pass_Jmax+1", 31), ("two_pass_Jmax+1", 32)]
EARLY_ROWS = [("k1_K33_d63", 6), ("k1_K33_d63", 8), ("two_pass_Jmax+1", 6), ("two_pass_Jmax+1", 8),
              ("two_pass_Jmax+1", 40)]


def case_of(row, num_sms, cov=None):
    K, d, c0 = _shape(row)
    base = 1000 if row in EDGE_ROWS else 2000
    return build_case(row, K, d, cov or c0, num_sms, base=base)


def update_path(c, num_sms, p, T=None, kernel_set=0):
    """The update path a call of T rounds takes (call_path: two-pass calls of more than 31 rounds run per step)."""
    path = kernel_paths(c["K"], c["d"], len(c["sizes"]), c["N"], num_sms, p.nb(), kernel_set)[0]
    T = p.T if T is None else T
    return PER_STEP if path == TWO_PASS and T > 31 else path


# ---- CPU tests --------------------------------------------------------------------------------------------------------
def test_rows_reach_their_paths():
    """Each row's update path on a 132-SM H100, with the row's block count."""
    for row in set(SIGMA_ROWS) | set(THETA_ROWS):
        c = case_of(row, 132)
        want = EDGE_ROWS[row][3][0] if row in EDGE_ROWS else WIDE_ROWS[row][4]
        assert update_path(c, 132, RunParams()) == want, row
    for name, (row, cov, nb) in BLOCK_ROWS.items():
        c = case_of(row, 132, cov)
        assert update_path(c, 132, RunParams(block_size=block_for(nb))) == BLOCK_PATHS[name], name
    c = case_of("two_pass_Jmax+1", 132)
    assert update_path(c, 132, RunParams(T=31)) == TWO_PASS and update_path(c, 132, RunParams(T=32)) == PER_STEP
    assert kernel_paths(c["K"], c["d"], len(c["sizes"]), c["N"], 132)[6] == PER_STEP       # the 40-round call
    c = case_of("k1_K33_d63", 132)
    for ks, want in ((0, SINGLE_PASS), (HB_KS_UPDATE_TWO_PASS, TWO_PASS), (HB_KS_UPDATE_PER_STEP, PER_STEP)):
        assert update_path(c, 132, RunParams(T=8), kernel_set=ks) == want


def test_block_rows_geometry():
    """The block rows have the block counts and block sizes they name (numpy's update_R rule)."""
    for name, (row, cov, nb) in BLOCK_ROWS.items():
        c = case_of(row, 132, cov)
        bs = np.float32(block_for(nb))
        cpb = int(np.float32(c["N"]) * bs)
        last = c["N"] - (nb - 1) * cpb
        assert cpb >= 1 and last >= 1, name
        if name == "last_block_large":
            assert (c["N"], cpb, last) == (1199, 59, 78)
        if name.startswith("one_cell"):
            assert cpb == 1 and 1200 <= c["N"] <= 1700


def _oracle_numpy_pair(c, p, Y0):
    from oracle.oracle import OracleHarmony
    B = sum(c["B_vec"])
    o = OracleHarmony(double=True)
    o.setup(Z=c["Z"], phi_i=c["phi"], B_vec=np.asarray(c["B_vec"]), sigma=p.sigma_of(c["K"]), theta=p.theta_of(B),
            lambda_=None, alpha=ALPHA, max_iter_kmeans=p.T, epsilon_kmeans=p.epsilon_kmeans, epsilon_harmony=-np.inf,
            K=c["K"], block_size=p.block_size, batch_proportion_cutoff=CUTOFF)
    npy = numpy_model(c, c["Z"], None, p)
    return o, npy


def _agree(o, npy, n):
    assert np.abs(o.get("R") - npy.R).max() < 1e-9
    np.testing.assert_allclose(o.get("O").T, npy.O, rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(o.get("E").T, npy.E, rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(o.trace("objective_kmeans"), npy.obj_kmeans, rtol=1e-6)   # the traces hold floats
    assert int(o.trace("kmeans_rounds")[-1]) == n


@pytest.mark.parametrize("what", ["sigma_vec", "theta_levels", "sigma_written", "T0", "T1", "nb1", "early_stop"])
def test_numpy_matches_oracle_on_run_parameters(what):
    """The numpy restatement and the fp64 oracle agree on the run parameters the GPU rows use: this pins the
    restatement's semantics (a written sigma divides the kept distances; T = 0; early stop at +inf) without a GPU."""
    row = "tiny_blocks" if what == "theta_levels" else "k1_tail_K17_d3"
    c = case_of(row, 132, None if row == "tiny_blocks" else (lambda s: _one_cov(_sizes(6, 1500))))
    K, B = c["K"], sum(c["B_vec"])
    p = dict(sigma_vec=RunParams(sigma=sigma_vec(K)), theta_levels=RunParams(theta=theta_levels(B)),
             sigma_written=RunParams(), T0=RunParams(T=0), T1=RunParams(T=1), nb1=RunParams(block_size=1.0),
             early_stop=RunParams(T=8, epsilon_kmeans=np.inf))[what]
    rng = np.random.default_rng(3)
    Y0 = make_Y0(c["Z"], K, rng)
    o, npy = _oracle_numpy_pair(c, p, Y0)
    o.init_cluster_cpp(Y0)
    npy.init_cluster(Y0)
    if what == "sigma_written":
        s = sigma_vec(K)
        o.set("sigma", s)
        npy.sigma = s.copy()
        o.compute_objective()
        npy.compute_objective()
    perms = make_perms(c["N"], max(p.T, 1), 5)
    o.cluster_cpp(perms)
    npy.cluster(perms)
    n = 5 if what == "early_stop" else p.T
    _agree(o, npy, n)
    o.cluster_cpp(perms)     # a cold start
    npy.cluster(perms)
    _agree(o, npy, n)


# ---- GPU tests --------------------------------------------------------------------------------------------------------
def _num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _fp32_r_errors(c, p, Y0, R2, perms2, Zp, Yp, perms3, tables=False):
    """max |R32 - R64| of the fp32 and fp64 oracles after S1, S2 and S3 on the stages' inputs (the wide file's rule);
    tables: also the O and E errors (as _table_err measures them) after S2 and S3."""
    from oracle.oracle import OracleHarmony
    from test_gpu_wide_shapes import _prenormalised
    B = sum(c["B_vec"])
    R = {}
    for dbl in (False, True):
        def fresh(Z):
            o = OracleHarmony(double=dbl)
            o.setup(Z=Z, phi_i=c["phi"], B_vec=np.asarray(c["B_vec"]), sigma=p.sigma_of(c["K"]), theta=p.theta_of(B),
                    lambda_=None, alpha=ALPHA, max_iter_kmeans=p.T, epsilon_kmeans=p.epsilon_kmeans,
                    epsilon_harmony=-np.inf, K=c["K"], block_size=p.block_size, batch_proportion_cutoff=CUTOFF)
            return o
        o = fresh(_prenormalised(c["Z"]))
        o.init_cluster_cpp(Y0)
        r1 = o.get("R")
        O2, E2 = tables_of(R2, c, o.get("Pr_b"))
        o.set("R", R2)
        o.set("O", O2.T)
        o.set("E", E2.T)
        o.cluster_cpp(perms2)
        r2, t2 = o.get("R"), (o.get("O"), o.get("E"))
        o = fresh(_prenormalised(Zp))
        o.init_cluster_cpp(Yp)
        o.cluster_cpp(perms3)
        R[dbl] = (r1, r2, o.get("R"), t2, (o.get("O"), o.get("E")))
    err = [float(np.abs(a - b).max()) for a, b in zip(R[False][:3], R[True][:3])]
    if tables:
        err += [max(_table_err(a, b) for a, b in zip(R[False][i], R[True][i])) for i in (3, 4)]
    return err


def _run_stages(name, c, p, stages, kernel_set=0, r_bars=None, objective=False, oe_bars=None):
    sms = _num_sms()
    rng = np.random.default_rng(11)
    Y0 = f32(make_Y0(c["Z"], c["K"], rng))
    g = setup_gpu(c, p, kernel_set)
    npy = numpy_model(c, f32(c["Z"]), None, p)
    ratios = []
    rb = r_bars or (TOL_R1, TOL_R, TOL_R)
    ob = oe_bars or (TOL_OE, TOL_OE)
    if "S1" in stages:
        stage_s1(name, g, npy, Y0, TAG, dict(R=rb[0]), ratios)
    else:
        g.init_cluster_cpp(Y0)
        npy.init_cluster(Y0)
    n2 = n3 = None
    if "S2" in stages:
        n2 = stage_s2(name, g, npy, c, rng, tag=TAG, bars=dict(R=rb[1], O=ob[0], E=ob[0]), ratios=ratios)
        if objective:   # k_objective_cells: R and the kept distances, term by term
            g.compute_objective()
            npy.compute_objective()
            _report(name, "compute_objective", dict(obj=_obj_err(g, npy, 1)), dict(obj=TOL_OBJ), TAG, ratios)
    if "S3" in stages:
        n3 = stage_s3(name, g, npy, c, rng, tag=TAG, bars=dict(R=rb[2], O=ob[1], E=ob[1]), ratios=ratios)
    print(f"[{TAG} {name}] path {update_path(c, sms, p, kernel_set=kernel_set)}, largest ratio to a bar: "
          f"{max(ratios):.2f}")
    return g, npy, n2, n3


@pytest.mark.gpu
@pytest.mark.parametrize("row", list(SIGMA_ROWS))
def test_sigma_per_cluster(row):
    c = case_of(row, _num_sms())
    p = RunParams(sigma=sigma_vec(c["K"]))
    r_bars = None
    if row in WIDE_ROWS:
        rng = np.random.default_rng(11)
        Y0 = f32(make_Y0(c["Z"], c["K"], rng))
        R2, _, _ = planted_R(c, rng)
        Zp, Yp = planted_zy(c, rng)
        e32 = _fp32_r_errors(c, p, Y0, R2, make_perms(c["N"], p.T, 5), Zp, Yp, make_perms(c["N"], p.T, 6))
        # S1 and S2: 2e-5.  U from the d-chunked 3xTF32 logits over d = 127, amplified by 2 / sigma_k (up to 20), gave
        # max|dR| 1.12e-5 after S1 and 1.003e-5 after S2 on an H100 80GB HBM3 (400 W); the fp32 oracle's FFMA dot products
        # give 2.7e-6 and 2.6e-6 on the same inputs
        r_bars = (2e-5, 2e-5, max(TOL_R, 2 * e32[2]))
        print(f"[{TAG} sigma {row}] fp32 oracle max|dR| per stage {e32[0]:.2e} {e32[1]:.2e} {e32[2]:.2e}")
    _run_stages(f"sigma {row}", c, p, ("S1", "S2", "S3"), r_bars=r_bars, objective=True)


@pytest.mark.gpu
@pytest.mark.parametrize("row", list(THETA_ROWS))
def test_theta_per_level(row):
    c = case_of(row, _num_sms())
    _run_stages(f"theta {row}", c, RunParams(theta=theta_levels(sum(c["B_vec"]))), ("S1", "S2", "S3"))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BLOCK_ROWS))
def test_block_counts(name):
    row, cov, nb = BLOCK_ROWS[name]
    sms = _num_sms()
    c = case_of(row, sms, cov)
    p = RunParams(block_size=block_for(nb))
    if sms == 132:
        assert update_path(c, sms, p) == BLOCK_PATHS[name]
    r_bars = oe_bars = None
    if nb == 1:
        # one block: round 0 removes every cell, so O and E fall to fp32 noise before the penalty is formed.  fp32 cannot
        # hold the edge bar here (the fp32 oracle's max|dR| after S2 / S3: 2.4e-4 / 3.1e-4 single-pass row, 1.3e-4 /
        # 1.5e-4 two-pass row); the wide file's rule applies, twice the fp32 oracle's error on the same inputs, to R and
        # (measured 1.06e-4 against 1e-4 after S3 on the single-pass row) to O and E
        rng = np.random.default_rng(11)
        Y0 = f32(make_Y0(c["Z"], c["K"], rng))
        R2, _, _ = planted_R(c, rng)
        Zp, Yp = planted_zy(c, rng)
        e32 = _fp32_r_errors(c, p, Y0, R2, make_perms(c["N"], p.T, 5), Zp, Yp, make_perms(c["N"], p.T, 6), tables=True)
        r_bars = (TOL_R1, max(TOL_R, 2 * e32[1]), max(TOL_R, 2 * e32[2]))
        oe_bars = (max(TOL_OE, 2 * e32[3]), max(TOL_OE, 2 * e32[4]))
        print(f"[{TAG} blocks {name}] fp32 oracle after S2, S3: max|dR| {e32[1]:.2e} {e32[2]:.2e}, O / E {e32[3]:.2e} "
              f"{e32[4]:.2e}")
    _run_stages(f"blocks {name}", c, p, ("S2", "S3"), r_bars=r_bars, oe_bars=oe_bars)


@pytest.mark.gpu
@pytest.mark.parametrize("row,T", LENGTH_ROWS)
def test_call_length(row, T):
    """S2 (warm, from written R) and S3 (cold) with T rounds.  T = 0: the warm call changes nothing; the cold call leaves
    the natural-order assignment's R, O, E and the normalised Z_corr."""
    c = case_of(row, _num_sms())
    p = RunParams(T=T)
    if T == 0:
        rng = np.random.default_rng(11)
        Y0 = f32(make_Y0(c["Z"], c["K"], rng))
        g = setup_gpu(c, p)
        npy = numpy_model(c, f32(c["Z"]), None, p)
        g.init_cluster_cpp(Y0)
        npy.init_cluster(Y0)
        R, _, _ = planted_R(c, rng)
        O, E = tables_of(R, c, npy.Pr_b)
        g.R, g.O, g.E = R.T, O, E
        npy.R, npy.O, npy.E = R, O, E
        n_obj = len(g.objective_kmeans)
        assert g.cluster_cpp(make_perms(c["N"], 1, 5)) == 0
        np.testing.assert_array_equal(g.R.T, R)
        np.testing.assert_array_equal(g.O, O)
        np.testing.assert_array_equal(g.E, E)
        assert int(g.kmeans_rounds[-1]) == 0 and len(g.objective_kmeans) == n_obj
        npy.cluster(make_perms(c["N"], 1, 5))
        stage_s3(f"length {row} T=0", g, npy, c, rng, tag=TAG)
        assert int(g.kmeans_rounds[-1]) == 0
        return
    _, _, n2, n3 = _run_stages(f"length {row} T={T}", c, p, ("S2", "S3"))
    assert n2 == n3 == T


@pytest.mark.gpu
@pytest.mark.parametrize("row,T", EARLY_ROWS)
def test_early_stop(row, T):
    """epsilon_kmeans = +inf: both calls stop after 5 rounds, like numpy; the second (cold) call starts from the state
    the first one left when it stopped."""
    c = case_of(row, _num_sms())
    _, _, n2, n3 = _run_stages(f"early {row} T={T}", c, RunParams(T=T, epsilon_kmeans=np.inf), ("S2", "S3"))
    assert n2 == n3 == 5


@pytest.mark.gpu
@pytest.mark.parametrize("path,kernel_set", [("single_pass", 0), ("two_pass", HB_KS_UPDATE_TWO_PASS),
                                             ("per_step", HB_KS_UPDATE_PER_STEP)])
def test_native_orders_after_early_stop(path, kernel_set):
    """Three 8-round calls with native update orders that each stop after 5 rounds: call i runs the native rounds
    5 i .. 5 i + 4 of the seed on every update path (the reference draws one shuffle per executed update_R)."""
    SEED = 20261016
    c = case_of("k1_K33_d63", _num_sms())
    p = RunParams(T=8, epsilon_kmeans=np.inf)
    rng = np.random.default_rng(11)
    Y0 = f32(make_Y0(c["Z"], c["K"], rng))
    g = setup_gpu(c, p, kernel_set)
    g.set_seed(SEED)
    npy = numpy_model(c, f32(c["Z"]), None, p)
    g.init_cluster_cpp(Y0)
    npy.init_cluster(Y0)
    counter, ratios = 0, []
    for call in range(3):
        before = len(npy.obj_kmeans)
        assert g.cluster_cpp() == 0
        perms = np.stack([native_order(c["N"], SEED, counter + t) for t in range(p.T)])
        npy.cluster(perms)
        n = len(npy.obj_kmeans) - before
        assert n == 5 and int(g.kmeans_rounds[-1]) == 5
        _report(f"native {path}", f"call {call}", state_errs(g, npy, n),
                dict(R=TOL_R, O=1e-4, E=1e-4, obj=TOL_OBJ), TAG, ratios)
        counter += n
    print(f"[{TAG} native {path}] largest ratio to a bar: {max(ratios):.2f}")


@pytest.mark.gpu
@pytest.mark.parametrize("row", ["k1_K33_d63", "two_pass_Jmax+1", "per_step_K257"])
def test_written_sigma(row):
    """setup with scalar sigma, init_cluster_cpp(Y0), sigma written per cluster, then a warm cluster_cpp and a
    standalone compute_objective; then a uniform sigma written, compute_objective and a (cold) cluster_cpp.  The
    library must divide the distances of the last assignment by the sigma written since, as the reference does."""
    c = case_of(row, _num_sms())
    K = c["K"]
    p = RunParams()
    rng = np.random.default_rng(11)
    Y0 = f32(make_Y0(c["Z"], K, rng))
    g = setup_gpu(c, p)
    npy = numpy_model(c, f32(c["Z"]), None, p)
    g.init_cluster_cpp(Y0)
    npy.init_cluster(Y0)
    ratios = []
    s1, s2 = sigma_vec(K), np.full(K, 0.15)
    for step, s in enumerate((s1, s2)):
        g.sigma = s
        npy.sigma = f32(s)
        np.testing.assert_array_equal(g.sigma, np.float32(s))
        g.compute_objective()
        npy.compute_objective()
        _report(f"written sigma {row}", f"compute_objective after write {step}", dict(obj=_obj_err(g, npy, 1)),
                dict(obj=TOL_OBJ), TAG, ratios)
        if step == 0:
            R, _, _ = planted_R(c, rng)
            O, E = tables_of(R, c, npy.Pr_b)
            g.R, g.O, g.E = R.T, O, E
            npy.R, npy.O, npy.E = R, O, E
        cluster_and_compare(f"written sigma {row}", f"cluster_cpp after write {step}", g, npy,
                            make_perms(c["N"], p.T, 5 + step), TAG, ratios=ratios)
        g.compute_objective()
        npy.compute_objective()
        _report(f"written sigma {row}", f"compute_objective after call {step}", dict(obj=_obj_err(g, npy, 1)),
                dict(obj=TOL_OBJ), TAG, ratios)
    print(f"[{TAG} written sigma {row}] largest ratio to a bar: {max(ratios):.2f}")


@pytest.mark.gpu
def test_sigma_written_before_init():
    """A sigma written between setup and init_cluster_cpp is the sigma of the first assignment."""
    c = case_of("k1_K33_d63", _num_sms())
    s = sigma_vec(c["K"])
    rng = np.random.default_rng(11)
    Y0 = f32(make_Y0(c["Z"], c["K"], rng))
    g = setup_gpu(c, RunParams())
    g.sigma = s
    npy = numpy_model(c, f32(c["Z"]), None, RunParams(sigma=s))
    stage_s1("written sigma before init", g, npy, Y0, TAG)
    stage_s2("written sigma before init", g, npy, c, rng, tag=TAG)


@pytest.mark.gpu
def test_vector_setters_check_lengths():
    """sigma takes K values or one (broadcast, as in setup), theta B and lambda_ B + 1; any other length raises
    ValueError before the library reads the buffer.  A sigma that is not finite and positive is rejected."""
    from harmony_b200.harmony import HarmonyError
    c = case_of("k1_tail_K17_d3", _num_sms())
    K, B = c["K"], sum(c["B_vec"])
    g = setup_gpu(c, RunParams())
    g.sigma = 0.2
    np.testing.assert_array_equal(g.sigma, np.float32(np.full(K, 0.2)))
    for name, bad in (("sigma", K - 1), ("sigma", K + 1), ("theta", B - 1), ("theta", B + 1), ("lambda_", B),
                      ("lambda_", B + 2), ("theta", 1)):
        with pytest.raises(ValueError):
            setattr(g, name, np.full(bad, 0.5))
    np.testing.assert_array_equal(g.sigma, np.float32(np.full(K, 0.2)))
    g.theta = np.full(B, 1.0)
    g.lambda_ = np.full(B + 1, 1.0)
    for v in (0.0, -0.1, np.nan, np.inf):
        s = np.full(K, 0.2)
        s[K // 2] = v
        with pytest.raises(HarmonyError):
            g.sigma = s
    np.testing.assert_array_equal(g.sigma, np.float32(np.full(K, 0.2)))
