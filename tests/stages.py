"""The stage rows of the kernel stage tests (test_gpu_kernel_edges.py, test_gpu_wide_shapes.py,
test_gpu_run_parameters.py, test_gpu_legacy_centroid.py) and everything they share: the edge and wide row tables, the
kernel-selection hooks and their values, the run parameters, the row builders, planted inputs, the fp64 numpy model, the
CPU oracle and its fp32 bars, and the stages with their bars.

Every stage starts the library and the numpy restatement from the same fp32 state, so a comparison measures that
stage's error alone, not drift accumulated over a run:
  S1  setup + init_cluster_cpp(Y0)                         Z_corr after setup, R, O, E, objective terms
  S2  R, O, E written through the fields, cluster_cpp       R, O, E, objective terms, kmeans_rounds
      (round 0 takes its removal sums from the written R)
  S4  R, O, E planted with one-hot rows, an empty cluster   Z_corr, Y, getLambda, W
      and a cluster whose mass lies in one level; ridge
      with estimated and with fixed lambda
  S3  Z_corr and Y planted (zero rows, rows at 1e-25 and    R, O, E, objective terms, normalised Z_corr
      1e20), cold-start cluster_cpp
The run parameters (sigma, theta, block size, rounds per call, epsilon_kmeans) are a RunParams; the defaults are the
ones the edge and wide tables run with.
"""
import ctypes
from dataclasses import dataclass

import numpy as np

from harmony_b200 import _lib
from helpers import make_perms, rel_l2
from numpy_restatement import NumpyHarmony, my_ceil

# hb_debug_kernel_paths: update path
PER_STEP, TWO_PASS, SINGLE_PASS = 0, 1, 2
# hb_debug_wide_paths
A_FUSED, A_FFMA, A_LOGITS, A_WIDE = 1, 2, 3, 4            # natural-order assignment
C_NATURAL, C_FUSED, C_LOGITS, C_WIDE = 0, 1, 2, 3         # plan-order cold start
P_TC, P_FFMA, P_COLS = 1, 2, 3                            # ridge apply
M_FFMA, M_TC, M_LOGITS, M_WIDE = 1, 2, 3, 4               # k-means initialisation
# HB_KERNEL_SET bits (include/harmony_b200.h)
HB_KS_FFMA_CONTRACTIONS, HB_KS_UPDATE_PER_STEP, HB_KS_UPDATE_TWO_PASS, HB_KS_WIDE = 1, 2, 4, 16

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


@dataclass
class RunParams:
    sigma: object = SIGMA            # a scalar or K values
    theta: object = None             # B values; None: 2 on every level
    block_size: float = BLOCK
    T: int = T
    epsilon_kmeans: float = -np.inf

    def sigma_of(self, K):
        return np.broadcast_to(np.asarray(self.sigma, dtype=np.float64), (K,)).copy()

    def theta_of(self, B):
        return np.full(B, 2.0) if self.theta is None else np.asarray(self.theta, dtype=np.float64)

    def nb(self):
        return my_ceil(np.float32(1.0) / np.float32(self.block_size))


DEFAULT = RunParams()


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


# ---- row builders ----------------------------------------------------------------------------------------------------
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


def kernel_paths(K, d, J, n, num_sms, nb=NB, kernel_set=0):
    out = (ctypes.c_int64 * 8)()
    _lib.lib().hb_debug_kernel_paths(K, d, J, n, nb, num_sms, kernel_set, out)
    return tuple(out)


def wide_paths(K, d, J, n, num_sms, nb=NB, kernel_set=0):
    out = (ctypes.c_int64 * 4)()
    _lib.lib().hb_debug_wide_paths(K, d, J, n, nb, num_sms, kernel_set, out)
    return tuple(out)


# ---- rows ------------------------------------------------------------------------------------------------------------
# Edge rows: shapes that straddle one limit of select_kernels (select.cuh) or of a kernel's tiling.
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

# Wide rows: shapes past the FFMA kernels' shared-memory limits.
# name -> (K, d, covariate builder(num_sms), hb_debug_wide_paths, update path, kernel_set)
WIDE_ROWS = {
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


def case_of(row, num_sms, cov=None):
    """Inputs of an edge or wide row (build_case, seeded from base 1000 for an edge row and 2000 for a wide one); cov
    replaces the row's covariate builder."""
    if row in EDGE_ROWS:
        K, d, c0 = EDGE_ROWS[row][:3]
        return build_case(row, K, d, cov or c0, num_sms, base=1000)
    K, d, c0 = WIDE_ROWS[row][:3]
    return build_case(row, K, d, cov or c0, num_sms, base=2000)


def build_case(name, K, d, cov, num_sms, seed=0, base=1000):
    """Inputs of a row: Z [N, d] (three zero rows, three rows at 1e-25), phi [N, C] (global level ids), B_vec, K and
    the tuples with their sizes.  Cells are shuffled, so the library's tuple sort is exercised."""
    tuples, B_vec, sizes = cov(num_sms)
    rng = np.random.default_rng(base + seed + sum(map(ord, name)))
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


def numpy_model(c, Zf, lambda_=None, p=DEFAULT):
    B = sum(c["B_vec"])
    return NumpyHarmony(Zf, c["phi"], c["B_vec"], p.sigma_of(c["K"]), p.theta_of(B), lambda_, ALPHA, p.T, c["K"],
                        p.block_size, CUTOFF, epsilon_kmeans=p.epsilon_kmeans)


def setup_gpu(c, p=DEFAULT, kernel_set=0):
    """A library handle set up on a row with the run parameters p (sigma passed as K values when it is a vector)."""
    from harmony_b200.harmony import harmony
    B = sum(c["B_vec"])
    g = harmony()
    if kernel_set:
        g.kernel_set = kernel_set
    sigma = p.sigma if np.ndim(p.sigma) == 0 else p.sigma_of(c["K"])
    g.setup(c["Z"], c["phi"], sigma, p.theta_of(B), None, ALPHA, p.T, p.epsilon_kmeans, -np.inf, c["K"],
            p.block_size, c["B_vec"], CUTOFF)
    return g


# ---- the CPU oracle and the bars derived from it ---------------------------------------------------------------------
def oracle(c, p=DEFAULT, double=True, Z=None, lambda_=None, legacy=False):
    """The CPU oracle (fp64, or the reference's fp32 arithmetic) set up on a row with the run parameters p; Z replaces
    the row's embedding, lambda_ the estimated ridge penalty, and legacy switches the legacy centroid step on."""
    from oracle.oracle import OracleHarmony
    o = OracleHarmony(double=double)
    o.setup(Z=c["Z"] if Z is None else Z, phi_i=c["phi"], B_vec=np.asarray(c["B_vec"]), sigma=p.sigma_of(c["K"]),
            theta=p.theta_of(sum(c["B_vec"])), lambda_=lambda_, alpha=ALPHA, max_iter_kmeans=p.T,
            epsilon_kmeans=p.epsilon_kmeans, epsilon_harmony=-np.inf, K=c["K"], block_size=p.block_size,
            batch_proportion_cutoff=CUTOFF)
    if legacy:
        o.set_legacy_centroid_step(True)
    return o


def prenormalised(Z):
    """Z with the rows whose fp32 sum of squares under- or overflows (|v| ~ 1e-25 or 1e20) divided by their norm in fp64:
    the reference's fp32 arithmetic does not rescale such rows, so the fp32 oracle would measure that, not the stage."""
    Z = np.array(Z, dtype=np.float64)
    m = np.abs(Z).max(axis=1)
    x = (m > 0) & ((m < 1e-10) | (m > 1e10))
    Z[x] /= np.linalg.norm(Z[x] / m[x, None], axis=1, keepdims=True) * m[x, None]
    return Z


def fp32_errors(c, p, Y0, R2, perms2, Zp, Yp, perms3, tables=False, own_pr_b=False):
    """max |R32 - R64| of the fp32 and fp64 oracles after S1, S2 and S3, each on that stage's inputs: S1 setup +
    init_cluster_cpp(Y0); S2 R2 and its O, E written, then cluster_cpp(perms2); S3 Z_corr = Zp and Y = Yp, then
    cluster_cpp(perms3).  O and E are built from the fp64 level proportions, as the stages write them, or with own_pr_b
    from each oracle's own (fp32 in the fp32 oracle; at nb = 1 this moves the S2 error by up to 30 %).  tables: also the
    O and E errors (as _table_err measures them) after S2 and S3.
    The R error of these stages comes from fp32 dot products over d columns amplified 2 / sigma times; where fp32 itself
    cannot hold a stage's bar, twice this error is the bar."""
    Pr_b = np.bincount(c["phi"].ravel(), minlength=sum(c["B_vec"])) / c["N"]
    got = {}
    for dbl in (False, True):
        o = oracle(c, p, dbl, prenormalised(c["Z"]))
        o.init_cluster_cpp(Y0)
        r1 = o.get("R")
        O2, E2 = tables_of(R2, c, o.get("Pr_b") if own_pr_b else Pr_b)
        o.set("R", R2)
        o.set("O", O2.T)
        o.set("E", E2.T)
        o.cluster_cpp(perms2)
        r2, t2 = o.get("R"), (o.get("O"), o.get("E"))
        o = oracle(c, p, dbl, prenormalised(Zp))
        o.init_cluster_cpp(Yp)
        o.cluster_cpp(perms3)
        got[dbl] = (r1, r2, o.get("R"), t2, (o.get("O"), o.get("E")))
    err = [float(np.abs(a - b).max()) for a, b in zip(got[False][:3], got[True][:3])]
    if tables:
        err += [max(_table_err(a, b) for a, b in zip(got[False][i], got[True][i])) for i in (3, 4)]
    return err


# ---- measures --------------------------------------------------------------------------------------------------------
def _set_zcorr(g, Z):
    """Z_corr is writable through the C ABI (HB_Z_CORR) though not through the Python class."""
    v = np.ascontiguousarray(Z, dtype=np.float64)
    g._check(g._L.hb_set_field(g._h, 0, v.ctypes.data_as(ctypes.c_void_p)))


def _launches(g, region):
    return g.region_time(region)[1]


def _obj_terms(g, n):
    return np.stack([np.asarray(getattr(g, t))[len(g.objective_kmeans) - n:] for t in
                     ("objective_kmeans_dist", "objective_kmeans_entropy", "objective_kmeans_cross")], axis=1)


def _obj_err(g, npy, n):
    """Largest relative error of the last n objective entries, term by term (0 for n = 0)."""
    if n == 0:
        return 0.0
    tg = _obj_terms(g, n)
    tn = np.asarray(npy.obj_parts[-n:])
    tot = np.asarray(npy.obj_kmeans[-n:])
    scale = np.maximum(np.abs(tot)[:, None], np.abs(tn))
    return float((np.abs(tg - tn) / scale).max())


def _table_err(a, b):
    return float(np.abs(a - b).max() / max(1.0, np.abs(b).max()))


def _report(name, stage, errs, bars, tag="edge", ratios=None):
    txt = " ".join(f"{k}={v:.2e}(bar {bars[k]:.1e}, {v / bars[k]:.2f})" for k, v in errs.items())
    print(f"[{tag} {name} {stage}] {txt}")
    for k, v in errs.items():
        if ratios is not None:
            ratios.append(v / bars[k])
        assert v <= bars[k], (name, stage, k, v, bars[k])


def state_errs(g, npy, n_obj):
    """R, O, E and the last n_obj objective entries against numpy."""
    return dict(R=float(np.abs(g.R.T - npy.R).max()), O=_table_err(g.O, npy.O), E=_table_err(g.E, npy.E),
                obj=_obj_err(g, npy, n_obj))


def rounds_of(npy, before):
    """Rounds the numpy model ran in its last cluster call (objective entries appended since `before`)."""
    return len(npy.obj_kmeans) - before


# ---- stages ----------------------------------------------------------------------------------------------------------
def _assert_launches(g, region, before, want):
    if want is not None:
        assert _launches(g, region) - before == want, (region, _launches(g, region) - before, want)


def stage_s1(name, g, npy, Y0, tag="edge", bars=None, ratios=None, assign_launches=None):
    """setup (already run) + init_cluster_cpp(Y0).  assign_launches: the launches the assignment must take."""
    errs = dict(Zn=float(np.abs(g.getZcorr().T - npy.Z_corr).max()))
    as0 = _launches(g, "assign")
    g.init_cluster_cpp(Y0)
    npy.init_cluster(Y0)
    _assert_launches(g, "assign", as0, assign_launches)
    errs.update(state_errs(g, npy, 1))
    b = dict(Zn=TOL_ZN, R=TOL_R1, O=TOL_OE, E=TOL_OE, obj=TOL_OBJ)
    b.update(bars or {})
    _report(name, "S1 assign", errs, b, tag, ratios)


def stage_s2(name, g, npy, c, rng, perm_seed=5, tag="edge", bars=None, ratios=None, R=None):
    """R, O, E written through the fields (planted from rng unless given), then one cluster_cpp call from them.
    Returns the rounds the call ran (asserted equal on both sides)."""
    if R is None:
        R, _, _ = planted_R(c, rng)
    O, E = tables_of(R, c, npy.Pr_b)
    g.R, g.O, g.E = R.T, O, E
    npy.R, npy.O, npy.E = R, O, E
    return cluster_and_compare(name, "S2 update from written R", g, npy, make_perms(c["N"], max(npy.T, 1), perm_seed),
                               tag, bars, ratios)


def cluster_and_compare(name, stage, g, npy, perms, tag="edge", bars=None, ratios=None, Zn=False):
    """One cluster_cpp call on both sides from their current state; R, O, E, the call's objective entries and the
    rounds it ran (and the normalised Z_corr when Zn) against numpy."""
    before = len(npy.obj_kmeans)
    assert g.cluster_cpp(perms) == 0
    npy.cluster(perms)
    n = rounds_of(npy, before)
    errs = state_errs(g, npy, n)
    b = dict(R=TOL_R, O=TOL_OE, E=TOL_OE, obj=TOL_OBJ)
    if Zn:
        errs["Zn"] = float(np.abs(g.getZcorr().T - npy.Z_corr).max())
        b["Zn"] = TOL_ZN
    b.update(bars or {})
    _report(name, stage, errs, b, tag, ratios)
    assert int(g.kmeans_rounds[-1]) == n, (int(g.kmeans_rounds[-1]), n)
    assert len(g.objective_kmeans) == len(npy.obj_kmeans)
    return n


def stage_s4(name, g, npy, c, rng, stats_launches=None, apply_launches=None, tag="edge", ratios=None, R=None):
    """Ridge step from planted R, O, E, estimated then fixed lambda.  R: planted_R(c, rng, special=True)'s result,
    drawn here unless given."""
    B = sum(c["B_vec"])
    R, kz, ks = planted_R(c, rng, special=True) if R is None else R
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
        _assert_launches(g, "ridge_stats", st0, stats_launches)
        _assert_launches(g, "ridge_apply", ap0, apply_launches)
        Yg = g.Y.T
        errs = dict(Z=rel_l2(g.getZcorr().T, npy.Z_corr), Y=float(np.abs(Yg - npy.Y).max()),
                    lam=float(np.abs(g.getLambda() - npy.lambda_mat).max() / max(1.0, np.abs(npy.lambda_mat).max())),
                    W=float(np.abs(g.W - npy.W).max() / max(1e-3, np.abs(npy.W).max())))
        _report(name, f"S4 ridge {'fixed' if lam is not None else 'estimated'} lambda", errs,
                dict(Z=TOL_Z, Y=TOL_Y if lam is None else TOL_Y_FIXED, lam=1e-6, W=1e-3), tag, ratios)
        np.testing.assert_array_equal(Yg[kz], np.float32(Yb[kz]))          # empty cluster: skipped, Y unchanged
        if len(c["B_vec"]) == 1:
            np.testing.assert_array_equal(Yg[ks], np.float32(Yb[ks]))      # single level, one covariate: skipped


def planted_zy(c, rng):
    """S3's planted Z_corr (zero rows, rows at 1e-25 and 1e20) and Y, in fp32."""
    N, K, d = c["N"], c["K"], c["d"]
    Zp = rng.standard_normal((N, d)) * rng.uniform(0.1, 30.0, (N, 1))
    special = rng.choice(N, 8, replace=False)
    Zp[special[:2]] = 0.0
    Zp[special[2:5]] *= 1e-25 / np.abs(Zp[special[2:5]]).max(axis=1, keepdims=True)
    Zp[special[5:]] *= 1e20 / np.abs(Zp[special[5:]]).max(axis=1, keepdims=True)
    Yp = rng.standard_normal((K, d))
    return f32(Zp), f32(Yp / np.linalg.norm(Yp, axis=1, keepdims=True))


def stage_s3(name, g, npy, c, rng, perm_seed=6, tag="edge", bars=None, ratios=None, assign_launches=None, Zp=None,
             Yp=None):
    """Planted Z_corr and Y (planted_zy(c, rng) unless given), then a cold-start cluster_cpp.  assign_launches: the
    launches the cold start must take.  Returns the rounds the call ran."""
    if Zp is None:
        Zp, Yp = planted_zy(c, rng)
    _set_zcorr(g, Zp)
    g.Y = Yp.T
    npy.Z_corr, npy.Y = Zp, Yp
    as0 = _launches(g, "assign")
    n = cluster_and_compare(name, "S3 cold start", g, npy, make_perms(c["N"], max(npy.T, 1), perm_seed), tag, bars,
                            ratios, Zn=True)
    _assert_launches(g, "assign", as0, assign_launches)
    return n


# ---- native update orders --------------------------------------------------------------------------------------------
_M64 = (1 << 64) - 1


def _mix64(x):
    """hb_mix64 (common.cuh) on uint64 arrays."""
    with np.errstate(over="ignore"):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return x ^ (x >> np.uint64(31))


def _half_bits(n):
    bits = 1
    while (1 << bits) < n:
        bits += 1
    return (bits + 1) // 2


def native_order(n, seed, round_counter):
    """Cells in update order of a native round (plan.cuh: key = plan_round_key(seed, counter), the cell at position p is
    hb_permute_inv(p)): the Feistel network of common.cuh, inverted, with cycle walking, in numpy."""
    key = int(_mix64(np.array([seed ^ int(_mix64(np.array([round_counter + 0x1234567], dtype=np.uint64))[0])],
                              dtype=np.uint64))[0])
    hb = _half_bits(n)
    mask = np.uint64((1 << hb) - 1)
    rk = [np.uint64((key + 0x632BE59BD9B4E019 * (r + 1)) & _M64) for r in range(6)]
    x = np.arange(n, dtype=np.uint64)
    todo = np.ones(n, dtype=bool)
    while todo.any():
        v = x[todo]
        l, r = v >> np.uint64(hb), v & mask
        for rnd in range(5, -1, -1):
            f = _mix64(l ^ rk[rnd]) & mask
            l, r = r ^ f, l
        v = (l << np.uint64(hb)) | r
        x[todo] = v
        todo[todo] = v >= np.uint64(n)
    return x.astype(np.int64)
