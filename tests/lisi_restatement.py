"""fp64 restatement of hb_lisi (DESIGN.md §10): the neighbours (knn_restatement's brute force without the row itself),
the calibration of the weights to the perplexity, the Simpson fold per label set, and the geometry of the search."""
import math

import numpy as np

import knn_restatement as kr

TOL, MAX_EVALS = 1e-5, 50
FLAG = 1e-12          # an evaluation whose |H - ln p| lies this close to TOL takes the branch rounding picks


def neighbours_for(p):
    return math.floor(3 * p) - 1


def neighbours(X, p):
    """(idx [N, k], dist [N, k]) of every row's k = floor(3 p) - 1 nearest other rows, fp64, ascending (ties: smaller
    row).  A row with a non-finite value is nobody's neighbour and has none: idx = -1, dist = +inf fill the lists."""
    X = np.asarray(X, dtype=np.float64)
    k = neighbours_for(p)
    idx, dist = np.full((len(X), k), -1, np.int64), np.full((len(X), k), np.inf)
    rows = np.nonzero(np.isfinite(X).all(axis=1))[0]
    kk = min(k, len(rows) - 1)
    if kk > 0:
        i, d = kr.brute_force(X[rows], X[rows], kk, exclude_self=True)
        idx[rows, :kk], dist[rows, :kk] = rows[i], d
    return idx, dist


def calibrate(dist, p):
    """Per row of dist [N, k] (+inf: no neighbour): the bisection of beta in P_j ~ exp(-beta D_j) until |H - ln p| <
    TOL or MAX_EVALS evaluations, H on distances shifted by the row's smallest -> (P [N, k], H [N], flag [N], beta
    [N]) of the last evaluation, flag: some evaluation lay within FLAG of the tolerance.  Rows without a neighbour keep
    P = 0, H = 0."""
    dist = np.asarray(dist, dtype=np.float64)
    valid = np.isfinite(dist)
    has = valid.any(axis=1)
    lo = np.where(has, np.where(valid, dist, np.inf).min(axis=1, initial=np.inf), 0.0)
    D = np.where(valid, dist - lo[:, None], 0.0)
    n = len(dist)
    beta, bmin, bmax = np.ones(n), np.full(n, -np.inf), np.full(n, np.inf)
    P, H, flag = np.zeros(dist.shape), np.zeros(n), np.zeros(n, bool)
    last_beta = np.ones(n)
    active = has.copy()
    log_p = math.log(p)
    for _ in range(MAX_EVALS):
        a = np.nonzero(active)[0]
        if len(a) == 0:
            break
        b = beta[a]
        E = np.where(valid[a], np.exp(-b[:, None] * D[a]), 0.0)
        s = E.sum(axis=1)
        Ha = np.log(s) + b * (D[a] * E).sum(axis=1) / s
        H[a], P[a], last_beta[a] = Ha, E / s[:, None], b
        diff = Ha - log_p
        flag[a] |= np.abs(np.abs(diff) - TOL) <= FLAG
        done = np.abs(diff) < TOL
        up, down = ~done & (diff > 0), ~done & ~(diff > 0)
        u, w = a[up], a[down]
        bmin[u] = beta[u]
        beta[u] = np.where(np.isinf(bmax[u]), 2.0 * beta[u], (beta[u] + bmax[u]) / 2)
        bmax[w] = beta[w]
        beta[w] = np.where(np.isinf(bmin[w]), beta[w] / 2, (beta[w] + bmin[w]) / 2)
        active[a[done]] = False
    return P, H, flag, last_beta


def simpson(P, labels, block=1024):
    """sum over labels of (sum of P over the entries with that label)^2, per row of P [N, k] and labels [N, k]."""
    S = np.empty(len(P))
    for r0 in range(0, len(P), block):
        p, lab = P[r0:r0 + block], labels[r0:r0 + block]
        same = lab[:, :, None] == lab[:, None, :]
        S[r0:r0 + block] = (p * (same * p[:, None, :]).sum(axis=2)).sum(axis=1)
    return S


def lisi(X, label_sets, p, idx=None, dist=None):
    """LISI [N, n_sets] of the rows of X for label_sets [n_sets, N] (any codes), and the rows' flags.  idx / dist: the
    neighbours to use (e.g. the ones hb_lisi returned); by default neighbours(X, p)."""
    if idx is None:
        idx, dist = neighbours(X, p)
    idx = np.asarray(idx, dtype=np.int64)
    dist = np.where(idx >= 0, np.asarray(dist, dtype=np.float64), np.inf)
    P, H, flag, _ = calibrate(dist, p)
    has = (idx >= 0).any(axis=1)
    out = np.empty((len(idx), len(label_sets)))
    for s, codes in enumerate(np.atleast_2d(label_sets)):
        lab = np.asarray(codes)[np.clip(idx, 0, None)]
        with np.errstate(divide="ignore"):   # rows without neighbours: S = 0, NaN below
            out[:, s] = 1.0 / simpson(P, lab)
    out[H == 0] = -1.0
    out[~has] = np.nan
    return out, flag


def geometry(d, p, N, num_sms):
    """hb_debug_lisi_geometry's eight values: knn_restatement's geometry with the (64, 1) fallback, for a self-search
    of N rows at k = floor(3 p) - 1."""
    k = neighbours_for(p)
    KD = (d + 7) // 8 * 8
    tq, stages = next((t, s) for t, s in ((128, 2), (128, 1), (64, 2), (64, 1))
                      if kr.smem_bytes(t, s, KD, k) <= kr.SMEM_LIMIT)
    qtiles, xtiles = -(-N // tq), -(-N // kr.TN)
    splits = max(1, min(num_sms // qtiles, xtiles, kr.MERGE_MAX // k)) if qtiles < num_sms else 1
    per = -(-xtiles // splits)
    return [tq, kr.TN, stages, -(-xtiles // per), kr.smem_bytes(tq, stages, KD, k), per, KD, 2 * tq]
