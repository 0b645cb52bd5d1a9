"""Stage tests of the hot-path kernels at every kernel-selection boundary, against the fp64 numpy restatement.

Each row of EDGE_ROWS is a shape that straddles one limit of select_kernels (harmony_b200.cu) or of a kernel's tiling:
the fused assignment kernel at d = 64 and K = 128 and its m64n16 tail, the logits + softmax cold start past them, the
cluster ranges of the ridge apply (K > 112 runs as several launches), the cluster and column launches of the ridge
statistics (K > 128, d + 1 > 128), the FFMA kernels past d = 128, the per-step update past KS = 256, the single-pass /
two-pass switch at 2 J = #SMs, tuples whose sizes put short tiles at every tile edge, and blocks with fewer cells than
CTAs.  Covariates are built so that the tuple sizes are exact.

Every row runs four stages on one handle, and each stage starts both sides from the same fp32 state, so a comparison
measures that stage's error alone, not drift accumulated over a run:
  S1  setup + init_cluster_cpp(Y0)                         Z_corr after setup, R, O, E, objective terms
  S2  R, O, E written through the fields, cluster_cpp       R, O, E, objective terms, kmeans_rounds
      (round 0 takes its removal sums from the written R)
  S4  R, O, E planted with one-hot rows, an empty cluster   Z_corr, Y, getLambda, W
      and a cluster whose mass lies in one level; ridge
      with estimated and with fixed lambda
  S3  Z_corr and Y planted (zero rows, rows at 1e-25 and    R, O, E, objective terms, normalised Z_corr
      1e20), cold-start cluster_cpp
A CPU test pins which kernels each row reaches (hb_debug_kernel_paths at 132 SMs), and each GPU test asserts the same
with the device's SM count and counts the launches of the multi-launch ranges.
"""
import ctypes

import numpy as np
import pytest

from harmony_b200 import _lib
from helpers import make_perms, rel_l2
from numpy_restatement import NumpyHarmony

PER_STEP, TWO_PASS, SINGLE_PASS = 0, 1, 2
NB = 20          # update blocks at the default block size 0.05
T = 6            # clustering rounds per call: one launch of rounds 0-4, then one of round 5
SIGMA, ALPHA, CUTOFF, BLOCK = 0.1, 0.2, 1e-5, 0.05

# bars: those of test_parity_stepwise and the ridge tests, except where noted
TOL_ZN = 1e-6    # normalised rows, max |d|
# R after the assignment, max |d|: 1e-5 instead of 5e-6.  The error of the fp32 dot products grows with d and is
# amplified 2 / sigma = 20 times in the logits: measured 3.0-3.5e-6 at d = 63-64 (fused kernel) and 4.5e-6 at d = 129
# (FFMA kernel) on an H100
TOL_R1 = 1e-5
TOL_R = 1e-5     # R after a cluster_cpp call, max |d|
TOL_OE = 1e-4    # O, E: rtol (atol = TOL_OE * max |table|)
TOL_OBJ = 1e-4   # objective terms: |d| / max(|total|, |term|)
TOL_Z = 2e-5     # Z_corr after the ridge step, rel-L2
TOL_Y = 5e-5     # Y after the ridge step, max |d|
# Y after the ridge step with the fixed lambda (0.5 .. 2): far less regularised than with the estimated alpha E, so the
# fp32 solve of a small cluster loses more; measured 4.2e-5 (two_pass_Jmax+1) on an H100
TOL_Y_FIXED = 1e-4


# ---- rows ------------------------------------------------------------------------------------------------------------
def _one_cov(sizes):
    return [(b,) for b in range(len(sizes))], [len(sizes)], list(sizes)


def _nested(sizes, B0):
    """Two covariates: tuple q = (level q % B0 of the first, level q of the second)."""
    J = len(sizes)
    return [(q % B0, B0 + q) for q in range(J)], [B0, J], list(sizes)


def _grid(B_vec, size_of):
    """Every combination of the covariates' levels is a tuple; tuple q holds size_of(q) cells."""
    tuples = []
    for a in range(B_vec[0]):
        for b in range(B_vec[1]):
            for c in range(B_vec[2]):
                tuples.append((a, B_vec[0] + b, B_vec[0] + B_vec[1] + c))
    return tuples, list(B_vec), [size_of(q) for q in range(len(tuples))]


def _sizes(J, n):
    """J tuple sizes summing to about n, uneven (every fifth tuple is short)."""
    base = n // J
    return [base // 3 + 1 if q % 5 == 4 else base for q in range(J)]


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


def kernel_paths(K, d, J, n, num_sms):
    L = _lib.lib()
    out = (ctypes.c_int64 * 8)()
    L.hb_debug_kernel_paths(K, d, J, n, NB, num_sms, 0, out)
    return tuple(out)


def build_case(name, num_sms, seed=0):
    """Inputs of a row: Z [N, d] (three zero rows, three rows at 1e-25), phi [N, C] (global level ids), B_vec, K and
    the tuples with their sizes.  Cells are shuffled, so the library's tuple sort is exercised."""
    K, d, cov, _, _, _ = EDGE_ROWS[name]
    tuples, B_vec, sizes = cov(num_sms)
    rng = np.random.default_rng(1000 + seed + sum(map(ord, name)))
    phi = np.concatenate([np.tile(np.asarray(t, dtype=np.int64), (s, 1)) for t, s in zip(tuples, sizes)])
    perm = rng.permutation(len(phi))
    phi = phi[perm]
    N = len(phi)
    n_types = max(4, min(K, 30))
    centers = rng.standard_normal((n_types, d)) * 2.0
    Z = centers[rng.integers(0, n_types, N)] + 0.7 * rng.standard_normal((N, d))
    B = sum(B_vec)
    Z += 0.5 * rng.standard_normal((B, d))[phi].sum(axis=1)
    Z *= (10.0 / np.sqrt(1.0 + np.arange(d)))[None, :]
    # a few zero rows and rows at 1e-25 (their squares underflow fp32)
    special = rng.choice(N, 6, replace=False)
    Z[special[:3]] = 0.0
    Z[special[3:]] *= 1e-25 / np.abs(Z[special[3:]]).max(axis=1, keepdims=True)
    return dict(Z=Z, phi=phi, B_vec=B_vec, K=K, d=d, N=N, sizes=sizes, tuples=tuples)


def make_Y0(Z, K, rng):
    nz = np.flatnonzero(np.abs(Z).max(axis=1) > 1e-10)
    Y = Z[rng.choice(nz, K, replace=False)]
    return Y / np.linalg.norm(Y, axis=1, keepdims=True)


def f32(x):
    return np.asarray(x, dtype=np.float32).astype(np.float64)


def level_of_single_cluster(c):
    """The level of the first covariate that holds the single-level cluster's mass: one with >= 2 tuples, so that
    another covariate keeps >= 2 levels for that cluster when there is one."""
    first = c["phi"][:, 0]
    key = {int(b): (len({t for t in c["tuples"] if t[0] == b}), int((first == b).sum())) for b in np.unique(first)}
    return max(key, key=key.get)


def planted_R(c, rng, special=False):
    """Row-stochastic fp32 R: softmax rows mixed with the uniform row (every entry >= 0.1 / K, so a level's mean stays
    far above the cutoff), 10 % one-hot rows.  special: cluster 1 is empty (all-zero column) and cluster 2 only holds
    cells of one level of the first covariate."""
    N, K = c["N"], c["K"]
    L = rng.standard_normal((N, K))
    A = np.exp(L - L.max(axis=1, keepdims=True))
    R = 0.9 * A / A.sum(axis=1, keepdims=True) + 0.1 / K
    hot = rng.random(N) < 0.1
    R[hot] = 0.0
    R[hot, rng.choice(np.arange(3, K) if special else np.arange(K), hot.sum())] = 1.0
    kz = ks = None
    if special:
        kz, ks = 1, 2
        R[:, kz] = 0.0
        b0 = level_of_single_cluster(c)
        in_b0 = c["phi"][:, 0] == b0
        R[:, ks] = 0.0
        R[in_b0, ks] = 0.3
        R /= R.sum(axis=1, keepdims=True)
    R = f32(R)
    return R, kz, ks


def tables_of(R, c, Pr_b):
    """O = R Phi^T and E = R's column sums x Pr_b, [K, B], rounded to fp32."""
    B = sum(c["B_vec"])
    Phi = np.zeros((B, c["N"]))
    for col in range(c["phi"].shape[1]):
        Phi[c["phi"][:, col], np.arange(c["N"])] = 1.0
    return f32(R.T @ Phi.T), f32(np.outer(R.sum(axis=0), Pr_b))


def numpy_model(c, Zf, lambda_=None):
    B = sum(c["B_vec"])
    return NumpyHarmony(Zf, c["phi"], c["B_vec"], SIGMA, np.full(B, 2.0), lambda_, ALPHA, T, c["K"], BLOCK, CUTOFF,
                        epsilon_kmeans=-np.inf)


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
def _num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _set_zcorr(g, Z):
    """Z_corr is writable through the C ABI (HB_Z_CORR) though not through the Python class."""
    v = np.ascontiguousarray(Z, dtype=np.float64)
    g._check(g._L.hb_set_field(g._h, 0, v.ctypes.data_as(ctypes.c_void_p)))


def _launches(g, region):
    return g.region_time(region)[1]


def _obj_terms(g, n):
    return np.stack([np.asarray(getattr(g, t))[-n:] for t in
                     ("objective_kmeans_dist", "objective_kmeans_entropy", "objective_kmeans_cross")], axis=1)


def _obj_err(g, npy, n):
    tg = _obj_terms(g, n)
    tn = np.asarray(npy.obj_parts[-n:])
    tot = np.asarray(npy.obj_kmeans[-n:])
    scale = np.maximum(np.abs(tot)[:, None], np.abs(tn))
    return float((np.abs(tg - tn) / scale).max())


def _table_err(a, b):
    return float(np.abs(a - b).max() / max(1.0, np.abs(b).max()))


def _report(name, stage, errs, bars):
    txt = " ".join(f"{k}={v:.2e}(bar {bars[k]:.0e})" for k, v in errs.items())
    print(f"[edge {name} {stage}] {txt}")
    for k, v in errs.items():
        assert v <= bars[k], (name, stage, k, v, bars[k])


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(EDGE_ROWS))
def test_edge_row_stages(name):
    from harmony_b200.harmony import harmony
    sms = _num_sms()
    c = build_case(name, sms)
    K, d, N, B = c["K"], c["d"], c["N"], sum(c["B_vec"])
    J = len(c["sizes"])
    assert kernel_paths(K, d, J, N, sms) == EDGE_ROWS[name][3]
    rng = np.random.default_rng(11)
    Zf = f32(c["Z"])
    Y0 = f32(make_Y0(c["Z"], K, rng))

    # ---- S1: setup + init_cluster_cpp
    g = harmony()
    g.setup(c["Z"], c["phi"], SIGMA, np.full(B, 2.0), None, ALPHA, T, -np.inf, -np.inf, K, BLOCK, c["B_vec"], CUTOFF)
    npy = numpy_model(c, Zf)
    errs = dict(Zn=float(np.abs(g.getZcorr().T - npy.Z_corr).max()))
    g.init_cluster_cpp(Y0)
    npy.init_cluster(Y0)
    errs.update(R=float(np.abs(g.R.T - npy.R).max()), O=_table_err(g.O, npy.O), E=_table_err(g.E, npy.E),
                obj=_obj_err(g, npy, 1))
    _report(name, "S1 assign", errs, dict(Zn=TOL_ZN, R=TOL_R1, O=TOL_OE, E=TOL_OE, obj=TOL_OBJ))

    # ---- S2: R, O, E written through the fields, then one cluster_cpp call from them
    R, _, _ = planted_R(c, rng)
    O, E = tables_of(R, c, npy.Pr_b)
    g.R, g.O, g.E = R.T, O, E
    npy.R, npy.O, npy.E = R, O, E
    perms = make_perms(N, T, 5)
    assert g.cluster_cpp(perms) == 0
    npy.cluster(perms)
    errs = dict(R=float(np.abs(g.R.T - npy.R).max()), O=_table_err(g.O, npy.O), E=_table_err(g.E, npy.E),
                obj=_obj_err(g, npy, T))
    _report(name, "S2 update from written R", errs, dict(R=TOL_R, O=TOL_OE, E=TOL_OE, obj=TOL_OBJ))
    assert int(g.kmeans_rounds[-1]) == T

    # ---- S4: ridge step from planted R, O, E, estimated then fixed lambda
    R, kz, ks = planted_R(c, rng, special=True)
    O, E = tables_of(R, c, npy.Pr_b)
    g.R, g.O, g.E = R.T, O, E
    npy.R, npy.O, npy.E = R, O, E
    for lam in (None, np.concatenate([[0.0], np.linspace(0.5, 2.0, B)])):
        if lam is not None:
            g.lambda_ = lam
            npy.lam = lam
        Yb = g.Y.T.astype(np.float64)
        npy.Y = Yb
        st0, ap0 = _launches(g, "ridge_stats"), _launches(g, "ridge_apply")
        g.moe_correct_ridge_cpp()
        npy.moe_correct_ridge()
        assert _launches(g, "ridge_stats") - st0 == EDGE_ROWS[name][4]
        assert _launches(g, "ridge_apply") - ap0 == EDGE_ROWS[name][5]
        Yg = g.Y.T
        errs = dict(Z=rel_l2(g.getZcorr().T, npy.Z_corr), Y=float(np.abs(Yg - npy.Y).max()),
                    lam=float(np.abs(g.getLambda() - npy.lambda_mat).max() / max(1.0, np.abs(npy.lambda_mat).max())),
                    W=float(np.abs(g.W - npy.W).max() / max(1e-3, np.abs(npy.W).max())))
        _report(name, f"S4 ridge {'fixed' if lam is not None else 'estimated'} lambda", errs,
                dict(Z=TOL_Z, Y=TOL_Y if lam is None else TOL_Y_FIXED, lam=1e-6, W=1e-3))
        np.testing.assert_array_equal(Yg[kz], np.float32(Yb[kz]))          # empty cluster: skipped, Y unchanged
        if len(c["B_vec"]) == 1:
            np.testing.assert_array_equal(Yg[ks], np.float32(Yb[ks]))      # single level, one covariate: skipped

    # ---- S3: planted Z_corr and Y, cold-start cluster_cpp
    Zp = rng.standard_normal((N, d)) * rng.uniform(0.1, 30.0, (N, 1))
    special = rng.choice(N, 8, replace=False)
    Zp[special[:2]] = 0.0
    Zp[special[2:5]] *= 1e-25 / np.abs(Zp[special[2:5]]).max(axis=1, keepdims=True)
    Zp[special[5:]] *= 1e20 / np.abs(Zp[special[5:]]).max(axis=1, keepdims=True)
    Zp = f32(Zp)
    Yp = rng.standard_normal((K, d))
    Yp = f32(Yp / np.linalg.norm(Yp, axis=1, keepdims=True))
    _set_zcorr(g, Zp)
    g.Y = Yp.T
    npy.Z_corr, npy.Y = Zp, Yp
    as0 = _launches(g, "assign")
    perms = make_perms(N, T, 6)
    assert g.cluster_cpp(perms) == 0
    npy.cluster(perms)
    if EDGE_ROWS[name][3][2] and EDGE_ROWS[name][3][5]:   # logits per 64-cluster range + softmax pass + finalize
        assert _launches(g, "assign") - as0 == (K + 63) // 64 + 2
    errs = dict(R=float(np.abs(g.R.T - npy.R).max()), O=_table_err(g.O, npy.O), E=_table_err(g.E, npy.E),
                obj=_obj_err(g, npy, T), Zn=float(np.abs(g.getZcorr().T - npy.Z_corr).max()))
    _report(name, "S3 cold start", errs, dict(R=TOL_R, O=TOL_OE, E=TOL_OE, obj=TOL_OBJ, Zn=TOL_ZN))
    assert int(g.kmeans_rounds[-1]) == T


@pytest.mark.gpu
@pytest.mark.parametrize("kernel_set", [0, 1])
def test_setup_normalises_rows_at_extreme_scales(kernel_set):
    """Rows whose fp32 sum of squares overflows (|v| ~ 1e20) or underflows (|v| <= 1e-25) are normalised like any
    other row at setup, and the assignment sees them so; a zero row stays zero."""
    from harmony_b200.harmony import harmony
    c = build_case("k1_tail_K17_d3", _num_sms())
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
