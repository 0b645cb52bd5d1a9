"""PCR (DESIGN §14) restated in fp64 numpy: the covariance of the finite rows, its leading eigenpairs by
``numpy.linalg.eigh`` and each component's R^2 on the one-hot batches from the batches' centred sums; and a literal
transcription of scib's ``pc_regression`` (sklearn's full-SVD PCA, ``pd.get_dummies``, one ``LinearRegression`` per
component) that the restatement is checked against."""
from types import SimpleNamespace

import numpy as np


def finite(X):
    return np.isfinite(X).all(axis=1)


def sign_rule(V):
    """Each column of V with its entry of largest magnitude positive (the first such entry on a tie)."""
    big = np.argmax(np.abs(V), axis=0)
    return V * np.where(V[big, np.arange(V.shape[1])] < 0, -1.0, 1.0)


def pcr(X, b, n_comps=50):
    """-> var, r2, components [m, d], score, lam (all d eigenvalues of C, descending), C, and the between-batch
    scatter M = sum_b S_b S_b^T / n_b, with m = min(n_comps, N, d)."""
    X = np.asarray(X, np.float64)
    N, d = X.shape
    m = min(n_comps, N, d)
    keep = finite(X)
    F, bf = X[keep], np.asarray(b)[keep]
    n = len(F)
    mean = F.mean(0) if n else np.zeros(d)
    Y = F - mean
    C = Y.T @ Y
    levels, codes = np.unique(bf, return_inverse=True)
    S = np.zeros((len(levels), d))
    np.add.at(S, codes, Y)
    nb = np.bincount(codes, minlength=len(levels)).astype(np.float64)
    M = (S / np.sqrt(np.maximum(nb, 1))[:, None]).T @ (S / np.sqrt(np.maximum(nb, 1))[:, None])
    lam, V = np.linalg.eigh(C)
    lam, V = lam[::-1], sign_rule(V[:, ::-1])
    lam_m, V_m = lam[:m], V[:, :m]
    r2 = np.zeros(m)
    if len(levels) >= 2 and lam[0] > 0:
        live = lam_m > d * np.finfo(np.float64).eps * lam[0]
        q = np.einsum("im,ij,jm->m", V_m, M, V_m)
        r2[live] = np.clip(q[live] / lam_m[live], 0.0, 1.0)
    if n < 2:
        var, r2, score = np.full(m, np.nan), np.full(m, np.nan), np.nan
    else:
        var = lam_m / (n - 1)
        score = (r2 * lam_m).sum() / lam_m.sum() if lam_m.sum() != 0 else np.nan
    return SimpleNamespace(var=var, r2=r2, components=V_m.T, score=score, lam=lam, C=C, M=M, n=n)


def trace_score(X, b):
    """The score at full rank without eigenvectors: tr(M) / tr(C)."""
    r = pcr(X, b, X.shape[1])
    return np.trace(r.M) / np.trace(r.C)


def scib_pc_regression(X, b, n_comps=50):
    """scib's pc_regression on a categorical covariate, transcribed: n_comps capped at min(X.shape), PCA (sklearn, full
    SVD, the variance scanpy reports), R^2 of a LinearRegression of each PC on pd.get_dummies(covariate) clamped at 0,
    and R2Var = sum(r2 * Var) / 100 with Var = var / sum(var) * 100.  Returns (score, var, r2)."""
    import pandas as pd
    from sklearn.decomposition import PCA
    from sklearn.linear_model import LinearRegression
    X = np.asarray(X, np.float64)
    if n_comps is None or n_comps > min(X.shape):
        n_comps = min(X.shape)
    pca = PCA(n_components=n_comps, svd_solver="full")
    X_pca = pca.fit_transform(X)
    pca_var = pca.explained_variance_
    covariate = pd.get_dummies(pd.Series(np.asarray(b)).astype("category"))
    r2 = []
    for i in range(n_comps):
        pc = X_pca[:, [i]]
        lm = LinearRegression()
        lm.fit(covariate, pc)
        r2.append(np.maximum(0, lm.score(covariate, pc)))
    r2 = np.array(r2)
    Var = pca_var / sum(pca_var) * 100
    return sum(r2 * Var) / 100, pca_var, r2


def comparison(before, after, scale=True):
    """scib's pcr_comparison fold."""
    if scale:
        score = (before - after) / before
        return 0 if score < 0 else score
    return after - before
