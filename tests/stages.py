"""The four-stage driver of the kernel stage tests (test_gpu_kernel_edges.py, test_gpu_wide_shapes.py,
test_gpu_run_parameters.py): row builders, planted inputs, the fp64 numpy model and the stages with their bars.

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


# ---- row builders -----------------------------------------------------------------------------------------------------
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
    L = _lib.lib()
    out = (ctypes.c_int64 * 8)()
    L.hb_debug_kernel_paths(K, d, J, n, nb, num_sms, kernel_set, out)
    return tuple(out)


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


# ---- measures -----------------------------------------------------------------------------------------------------------
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


# ---- stages ---------------------------------------------------------------------------------------------------------------
def stage_s1(name, g, npy, Y0, tag="edge", bars=None, ratios=None):
    """setup (already run) + init_cluster_cpp(Y0)."""
    errs = dict(Zn=float(np.abs(g.getZcorr().T - npy.Z_corr).max()))
    g.init_cluster_cpp(Y0)
    npy.init_cluster(Y0)
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


def stage_s4(name, g, npy, c, rng, stats_launches=None, apply_launches=None, tag="edge", ratios=None):
    """Ridge step from planted R, O, E, estimated then fixed lambda."""
    B = sum(c["B_vec"])
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
        if stats_launches is not None:
            assert _launches(g, "ridge_stats") - st0 == stats_launches
        if apply_launches is not None:
            assert _launches(g, "ridge_apply") - ap0 == apply_launches
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


def stage_s3(name, g, npy, c, rng, perm_seed=6, tag="edge", bars=None, ratios=None, logits_launches=False):
    """Planted Z_corr and Y, then a cold-start cluster_cpp.  logits_launches: assert the launches of the logits cold
    start (one per 64-cluster range, the softmax pass and the finalize).  Returns the rounds the call ran."""
    Zp, Yp = planted_zy(c, rng)
    _set_zcorr(g, Zp)
    g.Y = Yp.T
    npy.Z_corr, npy.Y = Zp, Yp
    as0 = _launches(g, "assign")
    n = cluster_and_compare(name, "S3 cold start", g, npy, make_perms(c["N"], max(npy.T, 1), perm_seed), tag, bars,
                            ratios, Zn=True)
    if logits_launches:
        assert _launches(g, "assign") - as0 == (c["K"] + 63) // 64 + 2
    return n


# ---- native update orders ---------------------------------------------------------------------------------------------------
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
