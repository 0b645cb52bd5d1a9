"""fp64 numpy restatement of mapping a query onto a reference (DESIGN.md §8), steps 1-4, in two forms of the solve:
the tuple-folded one the library computes (per-tuple sums -> G_k, s_k) and a dense-design np.linalg.solve one.

Cells are rows: Z [N, d], R [N, K]; phi [N, C] holds global level ids (covariate c's levels follow those of c - 1).
"""
import numpy as np


def l2_rows(X):
    """Rows divided by their norm; a zero row stays zero."""
    n = np.linalg.norm(X, axis=1, keepdims=True)
    return X / np.where(n == 0, 1.0, n)


def reference_stats(Zc, R):
    """Nr [K], Cref [K, d] and the centroids Cref / |Cref| [K, d] of an integration's Z_corr and R."""
    Nr = R.sum(axis=0)
    Cref = R.T @ Zc
    return Nr, Cref, l2_rows(Cref)


def assign(Zq, Y, sigma):
    """R_q = softmax_k(-2 (1 - Y_k . z / |z|) / sigma_k), [N, K]."""
    D = 2.0 * (1.0 - l2_rows(Zq) @ Y.T)
    L = -D / np.asarray(sigma, dtype=np.float64)[None, :]
    A = np.exp(L - L.max(axis=1, keepdims=True))
    return A / A.sum(axis=1, keepdims=True)


def lambda_levels(lambda_, B_vec):
    """A scalar or one value per covariate -> one value per level (RunHarmony's broadcast)."""
    lam = np.atleast_1d(np.asarray(lambda_, dtype=np.float64))
    return np.repeat(lam, B_vec) if len(lam) > 1 else np.repeat(lam, int(np.sum(B_vec)))


def _design(phi, B):
    """x_n = [1; one-hot levels of n], [N, B + 1]."""
    X = np.zeros((phi.shape[0], B + 1))
    X[:, 0] = 1.0
    for c in range(phi.shape[1]):
        X[np.arange(phi.shape[0]), phi[:, c] + 1] = 1.0
    return X


def weights_dense(R, Zq, phi, B, lam, Nr, Cref):
    """W [K, B + 1, d] from the dense design: G_k = X^T diag(R_k) X + diag(0, lam), G_k[0,0] += Nr_k,
    s_k = X^T diag(R_k) Z, s_k[0] += Cref_k, W_k = G_k^-1 s_k with row 0 zeroed (0 where G_k[0,0] == 0)."""
    X = _design(phi, B)
    K, d = R.shape[1], Zq.shape[1]
    W = np.zeros((K, B + 1, d))
    for k in range(K):
        XR = X * R[:, k:k + 1]
        G = XR.T @ X + np.diag(np.r_[0.0, lam])
        G[0, 0] += Nr[k]
        if G[0, 0] == 0:
            continue
        s = XR.T @ Zq
        s[0] += Cref[k]
        W[k] = np.linalg.solve(G, s)
        W[k, 0] = 0.0
    return W


def weights_folded(R, Zq, phi, B, lam, Nr, Cref):
    """The same W from the per-tuple sums S[q][k] = sum over tuple q's cells of R_k [z | 1], as the library's solve
    folds them (every level kept, no filter)."""
    tuples, inv = np.unique(phi, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    J, K, d = len(tuples), R.shape[1], Zq.shape[1]
    S = np.zeros((J, K, d + 1))
    Z1 = np.concatenate([Zq, np.ones((len(Zq), 1))], axis=1)
    for q in range(J):
        S[q] = R[inv == q].T @ Z1[inv == q]
    W = np.zeros((K, B + 1, d))
    for k in range(K):
        G = np.zeros((B + 1, B + 1))
        s = np.zeros((B + 1, d))
        for q in range(J):
            rows = np.r_[0, tuples[q] + 1]
            G[np.ix_(rows, rows)] += S[q, k, d]
            s[rows] += S[q, k, :d]
        G[np.arange(1, B + 1), np.arange(1, B + 1)] += lam
        G[0, 0] += Nr[k]
        s[0] += Cref[k]
        if G[0, 0] == 0:
            continue
        W[k] = np.linalg.solve(G, s)
        W[k, 0] = 0.0
    return W


def correct(Zq, R, phi, W):
    """z'_n = z_n - sum_k R_kn W_k^T x_n."""
    X = _design(phi, W.shape[1] - 1)
    return Zq - np.einsum("nk,nb,kbd->nd", R, X, W)


def map_query(Zq, phi, B_vec, lam, centroids, Nr, Cref, sigma, R=None):
    """Steps 1-4 with lam one value per query level (R: a given assignment, else computed from the centroids).
    Returns (mapped Z, R)."""
    if R is None:
        R = assign(Zq, centroids, sigma)
    W = weights_folded(R, Zq, phi, int(np.sum(B_vec)), np.asarray(lam, dtype=np.float64), Nr, Cref)
    return correct(Zq, R, phi, W), R


def type_offset(Zq, tq, Zr, tr):
    """Mean over the cell types present in both of the distance between a type's query mean and its reference mean."""
    types = [t for t in np.unique(tq) if np.any(tr == t)]
    return float(np.mean([np.linalg.norm(Zq[tq == t].mean(0) - Zr[tr == t].mean(0)) for t in types]))
