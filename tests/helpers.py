"""Shared helpers for the test-suite (test infrastructure; may use oracle/)."""
import os
import socket

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def load_cell_lines(small=True):
    f = np.load(os.path.join(GOLDEN, "cell_lines_small.npz" if small else "cell_lines.npz"))
    meta = {"dataset": f["dataset_levels"][f["dataset"]], "cell_type": f["cell_type_levels"][f["cell_type"]]}
    return f["scaled_pcs"], meta


def load_pbmc():
    f = np.load(os.path.join(GOLDEN, "pbmc_stim_pcs.npz"))
    return f["pcs"], {"stim": f["stim_levels"][f["stim"]]}


def synthetic(N, d, B_vec, n_types=8, seed=0, nested=True):
    """Small synthetic embedding following SURVEY.md §8d's generator (numpy, test sizes)."""
    rng = np.random.default_rng(seed)
    t = rng.integers(0, n_types, N)
    M = rng.standard_normal((n_types, d))
    sd = 10.0 / np.sqrt(1.0 + np.arange(d))
    Z = M[t] + 0.6 * rng.standard_normal((N, d))
    meta = {}
    prev = None
    for c, Bc in enumerate(B_vec):
        if c == 0 or not nested:
            lv = rng.integers(0, Bc, N)
        else:  # nested: each level of this covariate belongs to one level of the first
            parent = np.arange(Bc) % B_vec[0]
            lv = np.empty(N, dtype=np.int64)
            for p in range(B_vec[0]):
                cand = np.flatnonzero(parent == p)
                sel = prev == p
                lv[sel] = rng.choice(cand, sel.sum()) if len(cand) else 0
        if c == 0:
            prev = lv
        S = rng.standard_normal((Bc, d))
        Z = Z + 0.5 * S[lv]
        meta[f"cov{c}"] = lv
    return Z * sd[None, :], meta


def make_Y0(Z, K, seed=0):
    """K distinct random cells, cosine-normalised (stand-in for kmeans_centers, injected on both sides)."""
    rng = np.random.default_rng(seed)
    Zn = Z / np.maximum(np.linalg.norm(Z, axis=1, keepdims=True), 1e-30)
    idx = rng.choice(Z.shape[0], K, replace=False)
    Y = Zn[idx].copy()
    for _ in range(2):  # two Lloyd iterations on the cosine-normalised data
        a = np.argmax(Zn @ Y.T, axis=1)
        for k in range(K):
            if np.any(a == k):
                Y[k] = Zn[a == k].mean(axis=0)
    return Y


def make_perms(N, n, seed=0):
    rng = np.random.default_rng(seed)
    return np.stack([rng.permutation(N) for _ in range(n)]).astype(np.int64)


def setup_args(a):
    """prepare_inputs() dict -> positional args of OracleHarmony.setup / harmony.setup order differs; keep dict."""
    return dict(Z=a["Z"], phi_i=a["phi_i"], B_vec=a["B_vec"], sigma=a["sigma"], theta=a["theta"],
                lambda_=a["lambda_"], alpha=a["alpha"], max_iter_kmeans=a["max_iter_kmeans"],
                epsilon_kmeans=a["epsilon_kmeans"], epsilon_harmony=a["epsilon_harmony"], K=a["K"],
                block_size=a["block_size"], batch_proportion_cutoff=a["batch_proportion_cutoff"])


def oracle_setup(a, double=False):
    """The CPU oracle set up on a prepare_inputs() dict."""
    from oracle.oracle import OracleHarmony
    o = OracleHarmony(double=double)
    o.setup(**setup_args(a))
    return o


def run_oracle(a, Y0, n_iter, perm_seed=0, double=False, perms=None):
    """Drive the CPU oracle exactly like RunHarmony.default + harmonize (R/ui.R:269-283, R/utils.R:15-46)
    with injected centroids / update orders.  Returns the OracleHarmony object and the perms used."""
    o = oracle_setup(a, double)
    o.init_cluster_cpp(Y0)
    T = a["max_iter_kmeans"]
    N = a["Z"].shape[0]
    if perms is None:
        perms = make_perms(N, n_iter * T, perm_seed).reshape(n_iter, T, N)
    iters = 0
    for it in range(n_iter):
        o.cluster_cpp(perms[it])
        o.moe_correct_ridge_cpp()
        iters += 1
        if o.check_convergence(1):
            break
    return o, perms, iters


def gpu_setup(a, Z=None, T=None, K=None, kernel_set=0, device=None):
    """The library's counterpart of setup_args: a harmony object (harmony(), or harmony(device=device)) set up on a
    prepare_inputs() dict.  Z, T (max_iter_kmeans) and K replace what `a` gives; kernel_set is the HB_KERNEL_SET test
    hook (read by setup)."""
    from harmony_b200.harmony import harmony
    g = harmony() if device is None else harmony(device=device)
    if kernel_set:
        g.kernel_set = kernel_set
    g.setup(a["Z"] if Z is None else Z, a["phi_i"], a["sigma"], a["theta"], a["lambda_"], a["alpha"],
            a["max_iter_kmeans"] if T is None else T, a["epsilon_kmeans"], a["epsilon_harmony"],
            a["K"] if K is None else K, a["block_size"], a["B_vec"], a["batch_proportion_cutoff"])
    return g


def run_gpu(a, Y0, n_iter, perms, kernel_set=0):
    """Drive the library like run_oracle drives the oracle.  Returns the harmony object and the iterations run."""
    g = gpu_setup(a, kernel_set=kernel_set)
    g.init_cluster_cpp(Y0)
    iters = 0
    for it in range(n_iter):
        assert g.cluster_cpp(perms[it]) == 0
        g.moe_correct_ridge_cpp()
        iters += 1
        if g.check_convergence(1):
            break
    return g, iters


# ---- the parity bars of a whole run against the fp32 and fp64 oracles (test_gpu_parity.py's docstring) ---------------
TOL_Z = 1e-4
TIE_BAND = 1e-5
ARGMAX_GAP_MAX = 1e-3     # a differing hard index is only tolerated on cells this close to a tie ...
ARGMAX_FRAC_MAX = 5e-4    # ... and on at most this fraction of the cells


def argmax_mismatch_outside_band(Rg, Ro, band=TIE_BAND):
    """#cells whose hard assignment differs although the oracle's top-2 gap exceeds the noise band."""
    ag, ao = Rg.argmax(axis=1), Ro.argmax(axis=1)
    part = np.partition(Ro, -2, axis=1)
    gap = part[:, -1] - part[:, -2]
    bad = (ag != ao) & (gap > band)
    return int(bad.sum()), int((ag != ao).sum())


def argmax_report(Rg, Ro):
    """(#cells with a different hard index, largest top-2 gap of the oracle among them)."""
    ag, ao = Rg.argmax(axis=1), Ro.argmax(axis=1)
    m = ag != ao
    if not m.any():
        return 0, 0.0
    part = np.partition(Ro[m], -2, axis=1)
    return int(m.sum()), float((part[:, -1] - part[:, -2]).max())


def assert_argmax_bounded(Rg, Ro, label, own_flips=0, own_dev=0.0):
    """`own_flips` / `own_dev`: hard-index flips and max |dR| of the oracle instance `Ro` against the fp64 truth;
    they widen the bounds, so that an fp32 oracle that has drifted itself (long sequential sums at several
    100k cells per block) is not held against the GPU path."""
    n, gap = argmax_report(Rg, Ro)
    limit = max(1, int(np.ceil(ARGMAX_FRAC_MAX * Rg.shape[0]))) + own_flips
    gap_max = max(ARGMAX_GAP_MAX, 2 * own_dev)
    print(f"[{label}] hard-index mismatches: {n} of {Rg.shape[0]} (limit {limit}), largest oracle top-2 gap among them {gap:.2e} (limit {gap_max:.2e})")
    assert n <= limit, (label, n, limit)
    assert gap <= gap_max, (label, gap, gap_max)
    return n


def compare(g, o32, o64, label):
    Zg, Z32, Z64 = g.getZcorr().T, o32.get("Z_corr"), o64.get("Z_corr")
    Rg, R32, R64 = g.R.T, o32.get("R"), o64.get("R")
    e_g32, e_g64, e_3264 = rel_l2(Zg, Z32), rel_l2(Zg, Z64), rel_l2(Z32, Z64)
    dR = float(np.abs(Rg - R32).max())
    dR64, dR3264 = float(np.abs(Rg - R64).max()), float(np.abs(R32 - R64).max())
    # hard cluster index: identical to the fp64 truth wherever fp32 arithmetic can resolve it at all, i.e.
    # outside a tie band of the fp32 oracle's own deviation from fp64 (>= 1e-5); the count against the
    # fp32 oracle itself is reported as well (it flips with that oracle's sequential-sum noise)
    bad, anydiff = argmax_mismatch_outside_band(Rg, R64, band=max(TIE_BAND, 2 * dR3264))
    bad32, anydiff32 = argmax_mismatch_outside_band(Rg, R32)
    dY = float(np.abs(g.Y.T - o32.get("Y")).max())
    dO = float(np.abs(g.O.T - o32.get("O")).max() / max(1.0, np.abs(o32.get("O")).max()))
    print(f"[{label}] relL2(Z gpu,o32)={e_g32:.2e} (gpu,o64)={e_g64:.2e} (o32,o64)={e_3264:.2e} "
          f"max|dR|={dR:.2e} (vs o64 {dR64:.2e}; o32 vs o64 {dR3264:.2e}) max|dY|={dY:.2e} rel|dO|={dO:.2e} argmax diff={anydiff} outside band={bad}")
    assert np.all(np.isfinite(Zg))
    if e_3264 <= 0.5 * TOL_Z:
        assert e_g32 <= TOL_Z
    else:   # the reference-order fp32 arithmetic is itself outside the bar (module docstring)
        assert e_g64 <= TOL_Z and e_g32 <= e_3264 + 1e-5, (e_g64, e_g32, e_3264)
    assert e_g64 <= 2 * e_3264 + 2e-5
    assert bad == 0
    assert_argmax_bounded(Rg, R32, label + " vs oracle32", own_flips=argmax_report(R32, R64)[0], own_dev=dR3264)
    assert_argmax_bounded(Rg, R64, label + " vs oracle64")
    # the fp32 oracle carries the reference's own sequential-sum noise: judge R against the fp64 truth
    assert dR64 <= 2 * dR3264 + 1e-5, (dR64, dR3264)
    np.testing.assert_allclose(Rg.sum(axis=1), 1.0, atol=1e-5)
    # traces: same lengths, values within fp32 summation noise of the fp64 truth
    for name in ("objective_kmeans", "objective_harmony", "objective_kmeans_dist", "objective_kmeans_entropy",
                 "objective_kmeans_cross"):
        tg, t64 = getattr(g, name), o64.trace(name)
        assert len(tg) == len(t64), name
        np.testing.assert_allclose(tg, t64, rtol=2e-4, atol=2e-4, err_msg=name)
    assert list(g.kmeans_rounds) == [int(x) for x in o32.trace("kmeans_rounds")]


def rel_l2(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(np.asarray(b)), 1e-300))


def num_sms():
    """The SM count of GPU 0, which the geometry and kernel-path hooks take."""
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def gpu_harmony():
    """A fresh harmony object on GPU 0."""
    from harmony_b200.harmony import harmony
    return harmony(device=0)


def free_port():
    """A TCP port on 127.0.0.1 that was free a moment ago, for a test's process group."""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p
