"""The native k-means initialisation (kmeans_init.cuh, the library's kmeans_centers of utils.cpp:10-64) restated in
float64 numpy, with the error bands its stage tests (test_gpu_kmeans_init.py) hold each step of the kernels to.

  kmeans_centers        the rule written literally, one centroid at a time, with the uniforms injected
  kmeans_uniform        the keyed-hash uniforms of kernels.cuh (kmeans_uniform) in vectorised uint64 numpy
  kmeans_centers_fast   the same rule, vectorised over cells and centroids (the GPU rows' premises)
  race_intervals        the interval each cell's fp32 race key must lie in
  lloyd_admissible      the clusters each cell may join in an fp32 Lloyd step
"""
import numpy as np

from stages import _mix64

U24 = 2.0 ** -24
SEED_TAG = 0x6b6d65616e73          # kmeans_centers: seed = hb_mix64(h->seed ^ SEED_TAG)
CELL_TAG = 0x6b6d2b2b00000000      # kmeans_uniform: hb_mix64(seed ^ hb_mix64((i << 40) ^ g ^ CELL_TAG))
LLOYD_STEPS = 10


def kmeans_centers(X, K, uniform):
    """kmeans_centers of the reference (src/utils.cpp:10-64) in float64, with the uniforms injected:
    ``uniform(i, j)`` stands in for arma::randu at (centroid i, cell j); i = K addresses the K start-cell draws.

    initialize_centroids (:10-49): K start cells floor(u (N - 1)); then centroid i becomes the cell that minimises
    -log(u_ij) / |2 (1 - y_i . x_j)| with y_i its START cell, cells taken earlier skipped.  Then 10 x
    arma::kmeans(Y, X, K, keep_existing, 1): one Lloyd iteration each — nearest mean in Euclidean distance, mean of
    the members; a mean without members is left where it is (Armadillo's own dead-mean heuristic is not restated:
    Armadillo is not vendored in the reference; documented deviation).  X: [N, d] rows = cosine-normalised cells.
    Returns (Y [K, d] un-normalised means, chosen cells [K])."""
    X = np.asarray(X, dtype=np.float64)
    N = X.shape[0]
    start = np.array([int(np.floor(uniform(K, k) * (N - 1))) for k in range(K)])
    Y = X[start].copy()
    taken = []
    cells = np.empty(K, dtype=np.int64)
    U = np.array([[uniform(i, j) for j in range(N)] for i in range(K)])
    for i in range(K):
        dist = np.abs(2.0 * (1.0 - X @ Y[i]))
        with np.errstate(divide="ignore"):
            prob = -np.log(U[i]) / dist
        if taken:
            prob[np.array(taken)] = np.inf
        cells[i] = int(np.argmin(prob))
        taken.append(int(cells[i]))
    Y = X[cells].copy()
    for _ in range(LLOYD_STEPS):
        d2 = (X * X).sum(1)[:, None] - 2.0 * X @ Y.T + (Y * Y).sum(1)[None, :]
        a = np.argmin(d2, axis=1)
        for k in range(K):
            m = a == k
            if m.any():
                Y[k] = X[m].mean(axis=0)
    return Y, cells


# ---- the draws ------------------------------------------------------------------------------------------------------------
def kmeans_seed(seed):
    """The key of a native initialisation under the handle's seed (kmeans_init.cuh)."""
    return _mix64(np.array([int(seed) ^ SEED_TAG], dtype=np.uint64))[0]


def kmeans_uniform(seed, i, g):
    """kmeans_uniform (kernels.cuh) of centroid(s) i and global cell(s) g under the handle's seed, broadcast, as float32:
    24 hash bits h, then (float(h) + 0.5f) * 2^-24 in float32 (the + 0.5f rounds to even above 2^23, as on the GPU),
    the top value, which rounds to 1, held at 1 - 2^-24."""
    i = np.asarray(i, dtype=np.uint64)
    g = np.asarray(g, dtype=np.uint64)
    h = _mix64(kmeans_seed(seed) ^ _mix64((i << np.uint64(40)) ^ g ^ np.uint64(CELL_TAG)))
    u = ((h >> np.uint64(40)).astype(np.float32) + np.float32(0.5)) * np.float32(U24)
    return np.minimum(u, np.float32(1.0 - U24))


def start_cells(seed, K, N):
    """floor(u (N - 1)) of the K start-cell draws (centroid index K), in double like the host code."""
    u = kmeans_uniform(seed, K, np.arange(K)).astype(np.float64)
    return np.floor(u * (N - 1)).astype(np.int64)


# ---- the race -------------------------------------------------------------------------------------------------------------
def race_delta(d):
    """Bound on |dist32 - dist64|, dist = |2 (1 - z.y)|, for the fp32 rows z, y of the library's normalised cells
    (|z|, |y| = 1 to within d 2^-24).
      FFMA k_kmeans_race: a chain of d fmaf, |error| <= d 2^-24 sum|z_c y_c| <= d 2^-24.
      3xTF32 (k_logits_tc, k_logits_wide): z = hi + lo with hi the tf32 truncation (|z - hi| < 2^-10 |z|) and lo
      rounded to tf32 (error < 2^-21 |z|); the dropped lo.lo product (< 2^-20 |z y|) and the two lo roundings cost
      < 32 2^-24 sum|z_c y_c|; the fp32 accumulation of the tensor cores, which need not round to nearest, < 2 d 2^-24.
      Then 1 - acc (exact by Sterbenz near acc = 1, else < 2 2^-24) and the exact doubling.
    So |dist32 - dist64| <= 2 (2 d + 32 + 2) 2^-24 < 4 (d + 16) 2^-24 on every path."""
    return 4.0 * (d + 16) * U24


# -log(u) by logf (1 ulp) and the correctly rounded division: the key of an exact distance is within 2 ulp
KEY_REL = 4.0 * U24


def exact_rows(X):
    """Rows with one entry of +-1 and zeros elsewhere: their dot products with each other are exact on every path
    (integers in fp32, tf32 hi = the value, lo = 0), so their distances carry no error."""
    X = np.asarray(X)
    return (np.abs(X) == 1.0).sum(axis=1) + (X == 0.0).sum(axis=1) == X.shape[1]


def race_intervals(X, start, taken, u, delta, exact=None):
    """[lo, hi] per cell of the fp32 race key -log(u_j) / |2 (1 - x_j . x_start)| of one centroid.  X: [N, d] the
    library's fp32 normalised cells (float64 copies), start: its start cell, taken: cells taken earlier (their
    interval is [+inf, +inf]: they never win), u: [N] float32 uniforms of this centroid, delta: race_delta(d).
    The centre is the fp64 key; the width comes from |dist32 - dist64| <= delta and KEY_REL.  A cell with
    dist64 <= delta may have dist32 = 0, so its upper end is +inf (duplicates of the start cell).  Pairs of exact rows
    (exact_rows) have delta = 0: a duplicate of such a start cell has the key +inf exactly ([+inf, +inf])."""
    X = np.asarray(X, dtype=np.float64)
    dist = np.abs(2.0 * (1.0 - X @ X[start]))
    L = -np.log(np.asarray(u, dtype=np.float64))
    dl = np.full(len(X), float(delta))
    if exact is not None and exact[start]:
        dl[exact] = 0.0
    with np.errstate(divide="ignore", invalid="ignore"):
        lo = L * (1.0 - KEY_REL) / (dist + dl)
        hi = np.where(dist > dl, L * (1.0 + KEY_REL) / (dist - dl), np.inf)
    lo = np.where((dist == 0.0) & (dl == 0.0), np.inf, lo)
    if len(taken):
        t = np.asarray(taken, dtype=np.int64)
        lo[t] = np.inf
        hi[t] = np.inf
    return lo, hi


# ---- a Lloyd step ---------------------------------------------------------------------------------------------------------
def lloyd_eps(d):
    """Bound on the fp32 error of a score 2 x.y_k - |y_k|^2 (|x| <= 1, |y_k| <= 1: means of unit rows).
      FFMA k_kmeans_assign: x.y and |y|^2 by d fmaf each (< d 2^-24 apiece), the doubling exact, the difference
      rounded (< 3 2^-24): < (3 d + 3) 2^-24.
      Logits (k_kmeans_pick): U = 2 (x.y - 1) by 3xTF32 as in race_delta (< 2 (2 d + 32) + 4 units), |y|^2 by
      k_kmeans_norms (< d), U - |y|^2 rounded at |U - |y|^2| <= 5 (< 5): < (5 d + 73) 2^-24.
    Both are < (5 d + 80) 2^-24."""
    return (5.0 * d + 80.0) * U24


def canonical_clusters(Y):
    """canon[k] = the lowest k' whose row of Y equals row k (+0 and -0 alike): both kernels compute the same score for
    such rows, and their tie rules (score > best; equal scores: the lower k) give the cell to the lowest of them."""
    bits = np.ascontiguousarray(np.asarray(Y, dtype=np.float32) + np.float32(0.0)).view(np.uint32)
    _, first, inv = np.unique(bits, axis=0, return_index=True, return_inverse=True)
    return first[inv.reshape(-1)]


def lloyd_admissible(X, Y, eps):
    """[N, K] bool: the clusters cell j may join in one fp32 Lloyd step from the means Y — those whose fp64 score
    2 x_j.y_k - |y_k|^2 lies within 2 eps of the best.  Equal rows of Y are one cluster, the lowest k
    (canonical_clusters).  A zero row of X scores -|y_k|^2 and joins like any other cell: it adds 0 to the sum and 1
    to the count."""
    X = np.asarray(X, dtype=np.float64)
    Y = np.asarray(Y, dtype=np.float64)
    s = 2.0 * X @ Y.T - (Y * Y).sum(axis=1)[None, :]
    s[:, canonical_clusters(Y) != np.arange(len(Y))] = -np.inf
    return s >= s.max(axis=1, keepdims=True) - 2.0 * eps


def lloyd_step_model(X, Y, eps):
    """What one Lloyd step from Y may give, per cluster: (definite members D_k, ambiguous cells admitting k A_k,
    fp64 mean of the definite members, cells admitting k at all).  The GPU's members of k are D_k plus some subset of
    A_k, so its mean lies within 2 |A_k| / |D_k| of the definite mean (each such cell moves it by < 2 / |D_k| per
    coordinate), and a cluster no cell admits keeps its mean."""
    adm = lloyd_admissible(X, Y, eps)
    K, d = Y.shape
    amb = adm.sum(axis=1) > 1
    a = np.argmax(adm, axis=1)
    defn = ~amb
    D = np.bincount(a[defn], minlength=K)
    A = adm[amb].sum(axis=0)
    S = np.stack([np.bincount(a[defn], weights=X[defn, c], minlength=K) for c in range(d)], axis=1)
    with np.errstate(invalid="ignore", divide="ignore"):
        mean = S / D[:, None]
    return D, A, mean, adm.any(axis=0), int(amb.sum())


# ---- the whole rule, vectorised -------------------------------------------------------------------------------------------
def kmeans_centers_fast(X, K, seed, chunk=16):
    """kmeans_centers with the library's draws, vectorised: the race keys of `chunk` centroids at a time, one matrix
    product per Lloyd step.  Returns (Y, cells, re-runs): a re-run is a centroid whose winner over all cells was
    taken earlier (the retake loop of utils.cpp:38-45).  Ties of the keys go to the smaller cell (the library's key
    packing), also when every free cell's key is +inf."""
    X = np.asarray(X, dtype=np.float64)
    N = X.shape[0]
    start = start_cells(seed, K, N)
    cells = np.empty(K, dtype=np.int64)
    taken = np.zeros(N, dtype=bool)
    reruns = 0
    g = np.arange(N)
    for i0 in range(0, K, chunk):
        i1 = min(K, i0 + chunk)
        u = kmeans_uniform(seed, np.arange(i0, i1)[:, None], g[None, :]).astype(np.float64)
        dist = np.abs(2.0 * (1.0 - X[start[i0:i1]] @ X.T))
        with np.errstate(divide="ignore"):
            key = -np.log(u) / dist
        for r in range(i1 - i0):
            w = int(np.argmin(key[r]))
            if taken[w]:
                reruns += 1
                kr = np.where(taken, np.nan, key[r])
                w = int(np.flatnonzero(~taken)[np.argmin(kr[~taken])])
            cells[i0 + r] = w
            taken[w] = True
    Y = X[cells].copy()
    for _ in range(LLOYD_STEPS):
        s = 2.0 * X @ Y.T - (Y * Y).sum(axis=1)[None, :]
        a = np.argmax(s, axis=1)
        cnt = np.bincount(a, minlength=K)
        S = np.stack([np.bincount(a, weights=X[:, c], minlength=K) for c in range(X.shape[1])], axis=1)
        live = cnt > 0
        Y[live] = S[live] / cnt[live, None]
    return Y, cells, reruns
