"""fp64 restatement of hb_silhouette (DESIGN.md §11): chunked pairwise distances and per-(group, label) sums, the
per-row error bound of the GPU's 3xTF32 distances, and the launch geometry."""
import numpy as np

import knn_restatement as kr

TN = 64
SUM_REL = 32 * 2.0 ** -24   # sqrt rounding, the per-thread fp32 sum of 16 columns and the quad's two adds, per distance


def finite_rows(X):
    """The rows that take part, and their norms after centring on the column sums of the finite entries / N (the
    library's centre): a row with a NaN or an infinity, or whose centred squared norm overflows fp32, does not."""
    X = np.asarray(X, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        c = np.where(np.isfinite(X), X, 0.0).sum(0) / len(X)
        ss = ((X - c) ** 2).sum(1)
    fin = np.isfinite(X).all(1) & (ss <= np.finfo(np.float32).max)
    return fin, c, np.sqrt(np.where(fin, ss, 0.0))


def silhouette(X, labels, groups=None, bound=False, block=1024):
    """s [N] by the definition of DESIGN §11; with bound also the per-row bound on the GPU's error (0 where s is exact
    by rule, inf where max(a, b) = 0)."""
    X = np.asarray(X, dtype=np.float64)
    N, d = X.shape
    labels = np.asarray(labels)
    groups = np.zeros(N, np.int64) if groups is None else np.asarray(groups)
    fin, c, norm = finite_rows(X)
    s, err = np.full(N, np.nan), np.zeros(N)
    for g in np.unique(groups):
        rows = np.nonzero((groups == g) & fin)[0]
        if len(rows) == 0:
            continue
        levels, lab = np.unique(labels[rows], return_inverse=True)
        L = len(levels)
        if L < 2:
            continue
        onehot = np.zeros((len(rows), L))
        onehot[np.arange(len(rows)), lab] = 1.0
        n = onehot.sum(0)
        F = X[rows] - c
        sq = (F * F).sum(1)
        sums, dsums = np.empty((len(rows), L)), np.empty((len(rows), L))
        for r0 in range(0, len(rows), block):
            r1 = min(len(rows), r0 + block)
            D2 = np.maximum(sq[r0:r1, None] + sq[None, :] - 2.0 * F[r0:r1] @ F.T, 0.0)
            near = np.nonzero(D2 <= 1e-8 * (sq[r0:r1, None] + sq[None, :]))   # cancelled: directly, duplicates exact
            D2[near] = ((X[rows[r0 + near[0]]] - X[rows[near[1]]]) ** 2).sum(1)
            D = np.sqrt(D2)
            D[np.arange(r1 - r0), np.arange(r0, r1)] = 0.0
            sums[r0:r1] = D @ onehot
            if bound:
                qn, xn = norm[rows[r0:r1]][:, None], norm[rows][None, :]
                eps = kr.band(qn, xn, d) + 2.0 ** -20 * qn * qn    # the row's own |q|^2 / 2 rounds like |x|^2 / 2
                with np.errstate(divide="ignore", invalid="ignore"):
                    dD = np.minimum(np.where(D > 0, eps / D, np.inf), np.sqrt(eps))
                dD += SUM_REL * D + 2.0 ** -24 * (qn + xn)          # + the rounding of the centred rows to fp32
                dD[np.arange(r1 - r0), np.arange(r0, r1)] = 0.0
                dsums[r0:r1] = dD @ onehot
        own = n[lab]
        i = np.arange(len(rows))
        with np.errstate(divide="ignore", invalid="ignore"):
            a = np.where(own > 1, sums[i, lab] / (own - 1), 0.0)
            means = sums / n
            means[i, lab] = np.inf
            b = means.min(1)
            m = np.maximum(a, b)
            sg = np.where(m > 0, (b - a) / m, 0.0)
        sg[own == 1] = 0.0
        s[rows] = sg
        if bound:
            with np.errstate(divide="ignore", invalid="ignore"):
                da = np.where(own > 1, dsums[i, lab] / (own - 1), 0.0)
                dm = dsums / n
                dm[i, lab] = 0.0
                e = (da + dm.max(1)) / m
            e[m == 0] = np.inf
            e[own == 1] = 0.0
            err[rows] = e
    return (s, err) if bound else s


def smem_bytes(tq, stages, KD):
    return 4 * (2 * tq * KD + (stages + 1) * TN * KD + 2 * TN) + 256


def geometry(d, N, num_sms):
    """hb_debug_silhouette_geometry's eight values."""
    KD = (d + 7) // 8 * 8
    tq, stages = next((t, s) for t, s in ((128, 2), (128, 1), (64, 2), (64, 1)) if smem_bytes(t, s, KD) <= kr.SMEM_LIMIT)
    tiles = -(-N // tq)
    return [tq, TN, stages, smem_bytes(tq, stages, KD), KD, 2 * tq, tiles, -(-tiles // num_sms)]
