"""Stage tests of the native k-means initialisation (hb_init_cluster(h, NULL), kmeans_init.cuh) against the fp64
restatement of kmeans_restatement.py, on every kernel path: FFMA (k_kmeans_race, k_kmeans_assign, k_kmeans_update),
and k_logits_tc or k_logits_wide logits feeding k_kmeans_race_u<NV>, k_kmeans_norms, k_kmeans_pick<NV>, K3 and
k_kmeans_means_from_stats, at NV = 1, 2, 4 and 8.

Each step is checked from the GPU's own previous state (the recorded winners and means, hb_debug_kmeans_means), so a
comparison measures that step alone:
  race     centroid i, taken = the GPU's cells[:i]: its winner is free, and its key interval (race_intervals) reaches
           down to the smallest upper end over the free cells; when every free key is +inf, the smallest free cell
  step 0   Y_0 = the winners' rows, copied bit for bit
  Lloyd    from Y_{t-1}: a cluster with definite members has their mean (TOL_KM_MEAN, widened by 2 / |D_k| per
           ambiguous cell that may join it); a cluster no cell may join keeps its mean bit for bit
  result   g.Y = the row-normalised Y_10
Every row asserts the premise it is named for (its kernel path, and re-runs, exact ties or infinite keys where named).
"""
import ctypes

import numpy as np
import pytest

from harmony_b200 import _lib
from helpers import num_sms
from kmeans_restatement import (LLOYD_STEPS, canonical_clusters, exact_rows, kmeans_uniform, lloyd_eps,
                                lloyd_step_model, race_delta, race_intervals, start_cells)
from kmeans_rows import CASES, ROWS, Row
from stages import ALPHA, BLOCK, CUTOFF, SIGMA, T, TOL_ZN, wide_paths

SEED = 77
# a Lloyd mean against the fp64 mean of its definite members, max |d|.  The fp32 sums of m unit rows (atomics on the
# FFMA path, 3xTF32 K3 on the logits path) err by ~sqrt(m) 2^-24 on the mean for m <= 2000 members (~1e-7); one
# member dropped or added moves the mean by ~1 / m >= 5e-4.  Measured on an H100: at most 0.24 of the bar (tc_K12).
TOL_KM_MEAN = 1e-5
# cells within 2 eps of two means, per Lloyd step, at most max(3, AMB_RATE N): eps is a worst-case bound (up to
# (5 d + 80) 2^-24, 1.6e-4 at d = 512), so the rows' data are separated blobs; measured at most 1.2 % (wide_K200_d512)
# in the fp64 restatement
AMB_RATE = 0.02

N_DUP = 40      # antipodal: exact copies of -e_0


def make_row(name):
    """Raw cells Z [N, d] and one covariate of J levels; every level is present."""
    r = ROWS[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    K, d, N, J = r.K, r.d, r.N, r.J
    phi = (np.arange(N) % J)[rng.permutation(N)].reshape(N, 1)
    e0 = np.eye(d)[0]
    if r.kind in ("blobs", "special"):
        # separated blobs, more of them than centroids: few Lloyd boundaries cut through a blob, so few cells lie
        # within the score band of two means
        n_types = max(4, min(4 * K, N // 20))
        centers = rng.standard_normal((n_types, d))
        centers /= np.linalg.norm(centers, axis=1, keepdims=True)
        Z = (centers[rng.integers(0, n_types, N)] + 0.1 * rng.standard_normal((N, d)) / np.sqrt(d)) * \
            rng.uniform(0.5, 20.0, (N, 1))
        if r.kind == "special":     # zero rows, rows at 1e-25 (their squares underflow fp32) and at 1e20; a zero start
            sp = np.concatenate([start_cells(SEED, K, N)[:2], rng.choice(N, 13, replace=False)])
            Z[sp[:7]] = 0.0
            Z[sp[7:11]] *= 1e-25 / np.abs(Z[sp[7:11]]).max(axis=1, keepdims=True)
            Z[sp[11:]] *= 1e20 / np.abs(Z[sp[11:]]).max(axis=1, keepdims=True)
    elif r.kind == "d1":            # every normalised cell is +-1
        Z = rng.uniform(0.5, 3.0, (N, 1)) * np.where(rng.random((N, 1)) < 0.5, -1.0, 1.0)
    elif r.kind == "antipodal":     # cells near +e_0, N_DUP exact copies of -e_0, three of them start cells
        Z = e0 + 0.03 * rng.standard_normal((N, d))
        st = np.unique(start_cells(SEED, K, N))
        dup = np.concatenate([st[:3], rng.choice(np.setdiff1d(np.arange(N), st), N_DUP - 3, replace=False)])
        Z[dup] = -2.0 * e0
    else:                           # n_equals_k: 10 scattered cells and 30 copies of e_0 (exact rows)
        Z = np.tile(4.0 * e0, (N, 1))
        Z[rng.choice(N, 10, replace=False)] = rng.standard_normal((10, d))
    return Z, phi


def new_model(r, Z, phi, ks, block=BLOCK):
    from harmony_b200.harmony import harmony
    g = harmony()
    if ks:
        g.kernel_set = ks
    g.setup(Z, phi, SIGMA, np.full(r.J, 2.0), None, ALPHA, T, -np.inf, -np.inf, r.K, block, [r.J], CUTOFF)
    return g


def check_race(X, cells, K, d, N, exact):
    """The race of every centroid from the GPU's earlier winners.  Returns (largest ratio of a winner's deviation from
    the fp64 minimum to the deviation its band allows, largest relative deviation, fp64 re-runs, centroids whose free
    keys were all +inf)."""
    start = start_cells(SEED, K, N)
    delta = race_delta(d)
    taken = np.zeros(N, dtype=bool)
    worst = dev_max = 0.0
    reruns = all_inf = 0
    g = np.arange(N)
    for i0 in range(0, K, 32):
        i1 = min(K, i0 + 32)
        U = kmeans_uniform(SEED, np.arange(i0, i1)[:, None], g[None, :])
        for i in range(i0, i1):
            w = int(cells[i])
            assert 0 <= w < N and not taken[w], (i, w)
            u = U[i - i0]
            lo, hi = race_intervals(X, start[i], np.flatnonzero(taken), u, delta, exact)
            with np.errstate(divide="ignore"):
                key = -np.log(u.astype(np.float64)) / np.abs(2.0 * (1.0 - X @ X[start[i]]))
            first = int(np.argmin(key))
            if taken[first]:
                reruns += 1
            free = ~taken
            hmin = hi[free].min()
            assert lo[w] <= hmin, (i, w, lo[w], hmin)
            if np.isinf(lo[free]).all():          # every free key +inf: the key packing takes the smallest free cell
                all_inf += 1
                assert w == int(np.flatnonzero(free)[0]), (i, w)
            kmin = key[free].min()
            if np.isfinite(kmin) and key[w] > kmin:
                dev = key[w] / kmin - 1.0
                allowed = (hmin / kmin) * (key[w] / lo[w]) - 1.0
                dev_max = max(dev_max, dev)
                worst = max(worst, dev / allowed)
            taken[w] = True
    return worst, dev_max, reruns, all_inf


def check_lloyd(X, means, K, d, N):
    """Every Lloyd step from the GPU's previous means.  Returns (largest ratio to a bar, steps x exact ties,
    largest number of ambiguous cells in a step, clusters with only ambiguous candidates)."""
    eps = lloyd_eps(d)
    worst = 0.0
    ties = max_amb = unchecked = 0
    for t in range(1, LLOYD_STEPS + 1):
        Yp, Yt = means[t - 1].astype(np.float64), means[t].astype(np.float64)
        ties += int((canonical_clusters(Yp) != np.arange(K)).sum())
        D, A, mean, admitted, n_amb = lloyd_step_model(X, Yp, eps)
        max_amb = max(max_amb, n_amb)
        assert n_amb <= max(3, AMB_RATE * N), (t, n_amb)
        kept = ~admitted
        np.testing.assert_array_equal(means[t][kept].view(np.uint32), means[t - 1][kept].view(np.uint32))
        chk = admitted & (D > 0)
        unchecked += int((admitted & (D == 0)).sum())
        err = np.abs(Yt[chk] - mean[chk]).max(axis=1)
        bar = TOL_KM_MEAN + 2.0 * A[chk] / D[chk]
        bad = np.flatnonzero(err > bar)
        assert bad.size == 0, (t, np.flatnonzero(chk)[bad][:5], err[bad][:5], bar[bad][:5])
        if chk.any():
            worst = max(worst, float((err / bar).max()))
    return worst, ties, max_amb, unchecked


@pytest.mark.gpu
@pytest.mark.parametrize("name, ks, path, nv", CASES, ids=[f"{c[0]}-ks{c[1]}" for c in CASES])
def test_native_kmeans_init_step_by_step(name, ks, path, nv):
    r = ROWS[name]
    K, d, N = r.K, r.d, r.N
    assert wide_paths(r.K, r.d, r.J, r.N, num_sms(), kernel_set=ks)[3] == path
    Z, phi = make_row(name)
    g = new_model(r, Z, phi, ks)
    X32 = np.ascontiguousarray(g.getZcorr().T, dtype=np.float32)     # the library's normalised cells
    X = X32.astype(np.float64)
    Zf = np.float32(Z).astype(np.float64)
    nrm = np.linalg.norm(Zf, axis=1, keepdims=True)
    assert np.abs(X - Zf / np.where(nrm == 0, 1.0, nrm)).max() <= TOL_ZN
    g.set_seed(SEED)
    L = _lib.lib()
    for i, j in [(0, 0), (K, N - 1), (K - 1, N // 2), (3 % K, 12345 % N)]:
        assert L.hb_debug_kmeans_uniform(g._h, i, j) == float(kmeans_uniform(SEED, i, j))
    assert L.hb_debug_kmeans_keep_means(g._h, 1) == 0
    g.init_cluster_cpp()
    cells = (ctypes.c_int64 * K)()
    assert L.hb_debug_kmeans_cells(g._h, cells) == K
    cells = np.array(list(cells))
    means = np.zeros((LLOYD_STEPS + 1) * K * d, dtype=np.float32)
    assert L.hb_debug_kmeans_means(g._h, means.ctypes.data_as(ctypes.c_void_p)) == means.size
    means = means.reshape(LLOYD_STEPS + 1, K, d)

    # race, centroid by centroid
    assert len(np.unique(cells)) == K
    race_ratio, dev, reruns, all_inf = check_race(X, cells, K, d, N, exact_rows(X))
    # step 0: the winners' rows, bit for bit
    np.testing.assert_array_equal(means[0].view(np.uint32), X32[cells].view(np.uint32))
    # Lloyd steps
    lloyd_ratio, ties, max_amb, unchecked = check_lloyd(X, means, K, d, N)
    # result
    Y10 = means[LLOYD_STEPS].astype(np.float64)
    n10 = np.linalg.norm(Y10, axis=1, keepdims=True)
    dy = float(np.abs(g.Y.T - Y10 / np.where(n10 == 0, 1.0, n10)).max())
    assert dy <= TOL_ZN
    print(f"[kmeans {name} ks={ks}] race: largest deviation {dev:.2e} (ratio to band {race_ratio:.2f}), "
          f"{reruns} re-runs, {all_inf} all-inf; Lloyd: ratio to bar {lloyd_ratio:.2f}, {ties} tied means, "
          f"<= {max_amb} ambiguous cells/step, {unchecked} clusters of ambiguous cells only; "
          f"Y {dy:.1e} (ratio {dy / TOL_ZN:.2f}); largest ratio to a bar: {max(race_ratio, lloyd_ratio, dy / TOL_ZN):.2f}")

    # the premise each row is named for
    if name == "c3like":            # several grid-stride passes of the race and pick kernels (8 warps, <= 8 CTAs/SM)
        assert N > 2 * num_sms() * 8 * 8 and N > 2 * num_sms() * 4 * 128
    if name == "d1":
        assert ties >= 1
    if name == "antipodal":
        dup = np.flatnonzero((X32 == X32[np.argmin(X32[:, 0])]).all(axis=1))
        assert len(dup) == N_DUP and np.isin(start_cells(SEED, K, N), dup).any()    # start-cell duplicates: +inf keys
        assert reruns >= 10
        tied = np.isin(cells, dup).sum()
        assert tied >= 2 and ties >= LLOYD_STEPS * (tied - 1)       # equal centroids stay tied, all but one empty
    if name == "N_equals_K":
        assert np.array_equal(np.sort(cells), np.arange(N)) and all_inf >= 1
    if name.startswith("special_rows"):
        zero = np.flatnonzero(np.abs(X).max(axis=1) == 0)
        assert len(zero) == 7 and np.isin(start_cells(SEED, K, N), zero).any()     # a race from a zero row


@pytest.mark.gpu
def test_native_kmeans_init_refuses_more_clusters_than_cells():
    """K > N: centroid N finds no free cell; the call reports it (status 3), launches nothing past the cells, and the
    handle takes injected centroids afterwards."""
    from harmony_b200.harmony import HarmonyError
    r = Row(24, 8, 20, 1, "blobs", None)
    rng = np.random.default_rng(5)
    Z = rng.standard_normal((r.N, r.d))
    g = new_model(r, Z, np.zeros((r.N, 1), dtype=np.int64), 0, block=0.2)
    g.set_seed(SEED)
    assert _lib.lib().hb_init_cluster(g._h, None) == 3
    assert "no free cell for centroid 20" in _lib.lib().hb_last_error(g._h).decode()
    with pytest.raises(HarmonyError, match="no free cell for centroid 20"):
        g.init_cluster_cpp()
    Y0 = rng.standard_normal((r.K, r.d))
    g.init_cluster_cpp(Y0)
    np.testing.assert_allclose(g.Y.T, Y0 / np.linalg.norm(Y0, axis=1, keepdims=True), atol=TOL_ZN)
