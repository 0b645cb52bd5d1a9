"""fp64 restatement of hb_knn (DESIGN.md §9): blocked brute force, the selection band, the vote rule, the geometry."""
import numpy as np

SMEM_LIMIT = 227 * 1024 - 256
CAP, SS, TN, MERGE_MAX = 16, 18, 64, 1024


def unit_rows(A):
    """Rows divided by their norm; a zero row divides by 1."""
    A = np.asarray(A, dtype=np.float64)
    with np.errstate(over="ignore", under="ignore"):
        m = np.abs(A).max(axis=1, keepdims=True)
        m = np.where(m == 0, 1.0, m)
        n = m * np.sqrt(((A / m) ** 2).sum(axis=1, keepdims=True))
    return A / np.where(n == 0, 1.0, n)


def distances(Q, X, metric):
    """[Nq, Nx] fp64: squared Euclidean distances, or 1 - cosine."""
    Q, X = np.asarray(Q, dtype=np.float64), np.asarray(X, dtype=np.float64)
    if metric == "cosine":
        return 1.0 - unit_rows(Q) @ unit_rows(X).T
    c = X.mean(axis=0)
    Q, X = Q - c, X - c
    return np.maximum((Q * Q).sum(1)[:, None] - 2.0 * Q @ X.T + (X * X).sum(1)[None, :], 0.0)


def brute_force(Q, X, k, metric="euclidean", exclude_self=False, block=2048):
    """(idx [Nq, k], dist [Nq, k]) by ascending distance (ties: smaller row), in blocks of query rows."""
    Q = np.asarray(Q, dtype=np.float64)
    idx, dist = np.empty((len(Q), k), np.int64), np.empty((len(Q), k))
    for r0 in range(0, len(Q), block):
        D = distances(Q[r0:r0 + block], X, metric)
        if exclude_self:
            D[np.arange(len(D)), r0 + np.arange(len(D))] = np.inf
        part = np.argpartition(D, k - 1, axis=1)[:, :k] if k < D.shape[1] else np.broadcast_to(np.arange(D.shape[1]), D.shape)
        dk = np.take_along_axis(D, part, 1)
        o = np.lexsort((part, dk), axis=1)
        idx[r0:r0 + block] = np.take_along_axis(part, o, 1)
        dist[r0:r0 + block] = np.take_along_axis(dk, o, 1)
    return idx, (dist if metric == "cosine" else np.sqrt(dist))


def band(qn, xn, d, metric="euclidean"):
    """Width of the band around the k-th distance inside which membership is the selection's: on SQUARED Euclidean
    distances for rows of norm qn (query) and at most xn (reference) after centring on the reference's mean, on
    1 - cosine with qn = xn = 1 (half the squared distance of unit rows)."""
    b = 2.0 ** -18 * (1.0 + d / 16.0) * qn * xn + 2.0 ** -20 * xn * xn
    return 0.5 * b if metric == "cosine" else b


def centred_norms(Q, X, metric):
    if metric == "cosine":
        return np.ones(len(Q)), 1.0
    c = np.asarray(X, dtype=np.float64).mean(axis=0)
    return np.linalg.norm(np.asarray(Q, np.float64) - c, axis=1), float(np.linalg.norm(np.asarray(X, np.float64) - c, axis=1).max())


def vote(idx, dist, codes, n_labels):
    """Plain loops: the most frequent code among a row's neighbours; ties -> nearest member, then the smaller code."""
    code, share = np.full(len(idx), -1), np.zeros(len(idx))
    for i, (row, dr) in enumerate(zip(idx, dist)):
        tally = {}
        for j, dj in zip(row, dr):
            if j < 0:
                continue
            c = int(codes[j])
            n, near = tally.get(c, (0, np.inf))
            tally[c] = (n + 1, min(near, float(dj)))
        if tally:
            code[i] = min(tally, key=lambda c: (-tally[c][0], tally[c][1], c))
            share[i] = tally[code[i]][0] / sum(v[0] for v in tally.values())
    return code, share


def smem_bytes(tq, stages, KD, k):
    return 4 * (2 * tq * KD + (stages + 1) * TN * KD + 2 * TN + 2 * tq + 2 * tq * k + 2 * tq * CAP + tq * SS) + 256


def geometry(d, k, Nq, Nx, num_sms):
    """hb_debug_knn_geometry's eight values."""
    KD = (d + 7) // 8 * 8
    tq, stages = next((t, s) for t, s in ((128, 2), (128, 1), (64, 2)) if smem_bytes(t, s, KD, k) <= SMEM_LIMIT)
    qtiles, xtiles = -(-Nq // tq), -(-Nx // TN)
    splits = max(1, min(num_sms // qtiles, xtiles, MERGE_MAX // k)) if qtiles < num_sms else 1
    per = -(-xtiles // splits)
    return [tq, TN, stages, -(-xtiles // per), smem_bytes(tq, stages, KD, k), per, KD, 2 * tq]
