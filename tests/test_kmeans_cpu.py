"""The k-means restatement (kmeans_restatement.py) against a literal one-draw-at-a-time statement of the same rule, its
race intervals and Lloyd admissible sets on planted cases, and the kernels every row of kmeans_rows.py
reaches on a 132-SM H100 (host-only hooks, no GPU needed)."""
import numpy as np
import pytest

from kmeans_restatement import (KEY_REL, canonical_clusters, exact_rows, kmeans_centers, kmeans_centers_fast,
                                kmeans_uniform, lloyd_admissible, lloyd_eps, race_delta, race_intervals, start_cells)
from kmeans_rows import CASES, ROWS
from stages import M_FFMA, M_LOGITS, M_TC, wide_paths

M64 = (1 << 64) - 1


def mix64_int(x):
    """hb_mix64 (common.cuh) on one Python int."""
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def uniform_int(seed, i, g):
    """kmeans_uniform (kernels.cuh) of one (centroid, cell), written literally in Python ints and float32 scalars."""
    s = mix64_int(seed ^ 0x6b6d65616e73)
    h = mix64_int(s ^ mix64_int((((i << 40) & M64) ^ g ^ 0x6b6d2b2b00000000) & M64))
    u = (np.float32(h >> 40) + np.float32(0.5)) * np.float32(1.0 / 16777216.0)
    return float(min(u, np.float32(1.0 - 2.0 ** -24)))


def test_uniform_stays_below_one():
    """The top 24-bit value plus one half rounds to 2^24 in float32; the draw is held just below 1 so that its race key
    -log(u) / dist stays positive (a -0.0 key would order after every other)."""
    assert np.float32(2 ** 24 - 1) + np.float32(0.5) == np.float32(2 ** 24)
    seed = 77
    g = np.arange(1 << 24, dtype=np.uint64)
    u = kmeans_uniform(seed, 9, g)
    top = np.flatnonzero(u == np.float32(1.0 - 2.0 ** -24))
    assert len(top) >= 1 and u.max() < 1.0
    assert uniform_int(seed, 9, int(top[0])) == 1.0 - 2.0 ** -24


@pytest.mark.parametrize("seed", [0, 77, 2 ** 63 + 12345])
def test_vectorised_uniform_matches_the_literal_hash(seed):
    i = np.array([0, 1, 5, 40, 1023, 1024])
    g = np.array([0, 1, 2, 999, 2 ** 24 - 1, 2 ** 31 + 7, 2 ** 32 - 1])
    u = kmeans_uniform(seed, i[:, None], g[None, :])
    assert u.dtype == np.float32
    for a, ii in enumerate(i):
        for b, gg in enumerate(g):
            assert float(u[a, b]) == uniform_int(seed, int(ii), int(gg))
    assert 0.0 < u.min() and u.max() < 1.0


def _cells(rng, N, d):
    X = rng.standard_normal((N, d)) + 2.0 * rng.standard_normal((6, d))[rng.integers(0, 6, N)]
    return X / np.linalg.norm(X, axis=1, keepdims=True)


@pytest.mark.parametrize("N, d, K, ndup, seed", [(300, 5, 8, 0, 3), (400, 3, 24, 0, 9), (250, 4, 20, 10, 11)])
def test_fast_restatement_matches_the_literal_loop(N, d, K, ndup, seed):
    """Vectorised draws, race and Lloyd steps against the per-centroid loop with one hash call per (centroid, cell).
    The duplicated case makes centroids re-run their race without the taken cells."""
    rng = np.random.default_rng(N + K)
    X = _cells(rng, N, d)
    if ndup:                             # cells near +e_0 and ndup copies of -e_0, which win most races
        X = np.eye(d)[0] + 0.2 * rng.standard_normal((N, d))
        X /= np.linalg.norm(X, axis=1, keepdims=True)
        X[rng.choice(N, ndup, replace=False)] = -np.eye(d)[0]
    Yl, cells_l = kmeans_centers(X, K, lambda i, j: uniform_int(seed, i, j))
    Yf, cells_f, reruns = kmeans_centers_fast(X, K, seed, chunk=7)
    np.testing.assert_array_equal(cells_f, cells_l)
    np.testing.assert_allclose(Yf, Yl, rtol=0, atol=1e-12)
    assert np.array_equal(start_cells(seed, K, N),
                          [int(np.floor(uniform_int(seed, K, k) * (N - 1))) for k in range(K)])
    if ndup:
        assert reruns >= 3


def test_race_intervals_on_planted_cells():
    d = 8
    rng = np.random.default_rng(1)
    X = _cells(rng, 50, d)
    X[7] = X[3]                          # a duplicate of the start cell 3
    X[9] = X[11]                         # two identical free cells ...
    u = rng.uniform(0.01, 0.99, 50).astype(np.float32)
    u[9] = u[11]                         # ... with the same draw: an exact tie of their keys
    delta = race_delta(d)
    lo, hi = race_intervals(X, 3, [20, 21], u, delta)
    with np.errstate(divide="ignore"):
        key = -np.log(u.astype(np.float64)) / np.abs(2.0 * (1.0 - X @ X[3]))
    free = np.setdiff1d(np.arange(50), [3, 7, 20, 21])
    assert (lo[free] <= key[free]).all() and (key[free] <= hi[free]).all()
    assert np.isinf(lo[[20, 21]]).all() and np.isinf(hi[[20, 21]]).all()        # taken: never the winner
    for j in (3, 7):                      # dist64 <= delta: dist32 may be 0, the key +inf
        assert np.isfinite(lo[j]) and np.isinf(hi[j])
    assert lo[9] == lo[11] and hi[9] == hi[11]
    # the width: the key's relative band is KEY_REL plus delta / dist
    dist = np.abs(2.0 * (1.0 - X[free] @ X[3]))
    np.testing.assert_allclose(hi[free] / key[free], (1 + KEY_REL) / (1 - delta / dist), rtol=1e-12)
    np.testing.assert_allclose(lo[free] / key[free], (1 - KEY_REL) / (1 + delta / dist), rtol=1e-12)
    # a near-tie inside the band: both cells' intervals overlap, either may win
    X2 = X.copy()
    X2[12] = X2[13] * (1 + 1e-7)
    u2 = u.copy()
    u2[12] = u2[13]
    lo2, hi2 = race_intervals(X2, 3, [], u2, delta)
    assert lo2[12] <= hi2[13] and lo2[13] <= hi2[12]


def test_race_intervals_all_infinite():
    """Exact rows (one +-1 entry) carry no distance error: duplicates of an exact start cell have the key +inf exactly,
    and when every free cell is such a duplicate, all intervals are [+inf, +inf] (the library then takes the smallest
    free cell)."""
    X = np.zeros((12, 4))
    X[:, 0] = 1.0
    X[[2, 5], 0] = 0.0
    X[2, 1], X[5, 3] = -1.0, 1.0
    ex = exact_rows(X)
    assert ex.all()
    u = np.full(12, 0.5, dtype=np.float32)
    lo, hi = race_intervals(X, 0, [2, 5], u, race_delta(4), exact=ex)
    assert np.isinf(lo).all() and np.isinf(hi).all()
    lo, hi = race_intervals(X, 0, [], u, race_delta(4), exact=ex)
    L2 = -np.log(0.5) / 2.0                                      # dist 2 exactly: only logf and the division err
    assert lo[2] == pytest.approx(L2 * (1 - KEY_REL), rel=1e-15) and hi[2] == pytest.approx(L2 * (1 + KEY_REL), rel=1e-15)
    assert np.isinf(lo[[0, 1, 3, 4]]).all()


def test_lloyd_admissible_on_planted_means():
    d = 6
    eps = lloyd_eps(d)
    rng = np.random.default_rng(2)
    Y = rng.standard_normal((5, d))
    Y /= 2.0 * np.linalg.norm(Y, axis=1, keepdims=True)
    Y = np.float32(Y).astype(np.float64)
    Y[3] = Y[1]                          # equal rows: an exact tie, the lower k takes the cell
    X = np.float32(rng.standard_normal((40, d))).astype(np.float64)
    X /= np.linalg.norm(X, axis=1, keepdims=True)
    X[0] = 0.0                           # a zero row scores -|y_k|^2
    X[1] = Y[1] / np.linalg.norm(Y[1])   # nearest to the tied pair
    assert list(canonical_clusters(Y)) == [0, 1, 2, 1, 4]
    adm = lloyd_admissible(X, Y, eps)
    assert not adm[:, 3].any()
    assert adm[1, 1] and adm[1].sum() == 1
    assert adm[0, np.argmin((Y * Y).sum(1))]
    assert (adm.sum(axis=1) >= 1).all()
    # a near-tie inside 2 eps: y_4 = y_2 + t x with t chosen so that x scores eps / 2 less with y_4 than with y_2
    x = Y[2] / np.linalg.norm(Y[2])
    c = 2.0 - 2.0 * x @ Y[2]             # score(y_2 + t x) - score(y_2) = t (c - t)
    t = (c - np.sqrt(c * c + 2.0 * eps)) / 2.0
    Y2 = Y.copy()
    Y2[4] = Y[2] + t * x
    sc = 2.0 * Y2 @ x - (Y2 * Y2).sum(1)
    assert sc[2] == sc.max() and sc[2] - sc[4] == pytest.approx(eps / 2, rel=1e-6)
    assert lloyd_admissible(x[None, :], Y2, eps)[0].tolist() == [False, False, True, False, True]
    Y2[4] = Y[2] + 8.0 * t * x            # 4 eps below: out
    assert lloyd_admissible(x[None, :], Y2, eps)[0].tolist() == [False, False, True, False, False]
    # +0 and -0 give the same scores: still a tie (a mean of -0 entries sums to +0)
    Y3 = Y.copy()
    Y3[1, 0], Y3[3, 0] = 0.0, -0.0
    assert list(canonical_clusters(Y3)) == [0, 1, 2, 1, 4]
    Y3[3, 1] = np.nextafter(np.float32(Y3[1, 1]), np.float32(2.0))
    assert list(canonical_clusters(Y3)) == [0, 1, 2, 3, 4]


# ---- the kernels of the GPU rows ------------------------------------------------------------------------------------------
def _sp_nv(KS):
    nv = 1
    while 128 * nv < KS:
        nv <<= 1
    return nv


def test_gpu_rows_reach_their_kernels():
    """Every row of test_gpu_kmeans_init.py on a 132-SM H100: the k-means path of hb_debug_wide_paths, NV = sp_nv(KS)
    of the race and pick kernels, and ceil(K / 64) k_logits_tc launches per logits pass."""
    for name, ks, path, nv in CASES:
        r = ROWS[name]
        got = wide_paths(r.K, r.d, r.J, r.N, 132, kernel_set=ks)[3]
        assert got == path, (name, ks, got, path)
        if path != M_FFMA:
            assert _sp_nv((r.K + 3) & ~3) == nv, (name, nv)
        if path in (M_TC, M_LOGITS):              # k_logits_tc: 64 clusters per launch
            assert (r.K + 63) // 64 == r.launches, name
