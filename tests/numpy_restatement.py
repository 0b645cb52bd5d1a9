"""Independent float64 numpy restatement of the hot path, written in the *batched* form the
GPU computes (SURVEY.md §8a'), from the maths in the reference's plain-R walkthrough:

  * assignment / diversity statistics  vignettes/detailedWalkthrough.Rmd:320,346-348 (O = R Phi^T, E)
    with the penalty actually coded in src/harmony.cpp:322 ((2E+1)/(O+E+1))^theta (the vignette's
    snippet at :439-449 is illustrative and differs; the C++ wins)
  * ridge regression per cluster        vignettes/detailedWalkthrough.Rmd:637-649
    W_k = (Phi* diag(R_k) Phi*^T + diag(lambda_k))^-1 Phi* diag(R_k) Z^T
  * per-cell correction                 vignettes/detailedWalkthrough.Rmd:817-822
  * level filter                        src/harmony.cpp:358-410

It shares no code with oracle/harmony_oracle.cpp; tests/test_oracle.py checks the two against each
other, which is the strongest pin available (the reference holds no golden vectors for this path).
"""
import numpy as np


def my_ceil(x):
    i = int(np.float32(x))
    return i if np.float32(x) == np.float32(i) else i + 1


class NumpyHarmony:
    def __init__(self, Z, phi_i, B_vec, sigma, theta, lambda_, alpha, T, K, block_size, cutoff, epsilon_kmeans=1e-3):
        self.Z_orig = np.asarray(Z, dtype=np.float64)
        self.N, self.d = self.Z_orig.shape
        self.lev = np.asarray(phi_i, dtype=np.int64).reshape(self.N, -1)
        self.C = self.lev.shape[1]
        self.B_vec = list(B_vec)
        self.B = int(sum(B_vec))
        self.K = K
        self.sigma = np.broadcast_to(np.asarray(sigma, dtype=np.float64), (K,)).copy()
        self.theta = np.asarray(theta, dtype=np.float64)
        self.lam = None if lambda_ is None else np.asarray(lambda_, dtype=np.float64)
        # alpha and the cutoff are declared `float` in the reference (src/harmony.h:62)
        self.alpha, self.T, self.cutoff = float(np.float32(alpha)), T, cutoff
        self.block_size = np.float32(0.2) if self.N < 40 else np.float32(block_size)
        self.N_b = np.array([(self.lev == b).sum() for b in range(self.B)], dtype=np.float64)
        self.Pr_b = self.N_b / self.N
        self.cov_of = np.repeat(np.arange(self.C), self.B_vec)
        self.Phi = np.zeros((self.B, self.N))
        for c in range(self.C):
            self.Phi[self.lev[:, c], np.arange(self.N)] = 1.0
        self.Z_corr = self._l2(self.Z_orig)
        self.epsilon_kmeans = epsilon_kmeans
        self.obj_kmeans, self.obj_harmony = [], []
        self.obj_parts = []   # (distance, entropy, cross-entropy) terms of every objective_kmeans entry

    @staticmethod
    def _l2(X):
        n = np.sqrt((X * X).sum(axis=1, keepdims=True))
        return X / np.where(n == 0, 1.0, n)

    def _assign(self):
        self.D = 2.0 * (1.0 - self.Z_corr @ self.Y.T)            # [N, K]
        A = np.exp(-self.D / self.sigma[None, :])
        self.R = A / A.sum(axis=1, keepdims=True)
        self.E = np.outer(self.R.sum(axis=0), self.Pr_b)          # [K, B]
        self.O = self.R.T @ self.Phi.T                            # [K, B]

    def init_cluster(self, Y0):
        self.Y = self._l2(np.asarray(Y0, dtype=np.float64))
        self._assign()
        self.compute_objective()
        self.obj_harmony.append(self.obj_kmeans[-1])

    def compute_objective(self):
        R = self.R
        logR = np.log(np.where(R > 0, R, 1.0))
        kerr = (R * self.D).sum()
        ent = (R * logR * self.sigma[None, :]).sum()
        L = self.theta[None, :] * np.log((self.O + self.E + 1) / (2 * self.E + 1))    # [K, B]
        cross = ((R * self.sigma[None, :]) * (self.Phi.T @ L.T)).sum()
        self.obj_kmeans.append((kerr + ent + cross) * 2000.0 / self.N)
        self.obj_parts.append((kerr * 2000.0 / self.N, ent * 2000.0 / self.N, cross * 2000.0 / self.N))

    def update_R(self, order):
        N = self.N
        n_blocks = my_ceil(np.float32(1.0) / self.block_size)
        cpb = int(np.float32(N) * self.block_size)
        A = np.exp(-self.D / self.sigma[None, :])
        A = A / A.sum(axis=1, keepdims=True)
        for blk in range(n_blocks):
            lo = blk * cpb
            hi = N if blk == n_blocks - 1 else (blk + 1) * cpb
            cells = np.asarray(order[lo:hi], dtype=np.int64)
            if len(cells) == 0:
                continue
            Rb, Pb = self.R[cells], self.Phi[:, cells]
            self.E -= np.outer(Rb.sum(axis=0), self.Pr_b)
            self.O -= Rb.T @ Pb.T
            P = ((2 * self.E + 1) / (self.O + self.E + 1)) ** self.theta[None, :]         # [K, B]
            Rn = A[cells] * (Pb.T @ P.T)                                                 # sum over covariates
            s = np.abs(Rn).sum(axis=1, keepdims=True)
            Rn = Rn / np.where(s == 0, 1.0, s)
            self.R[cells] = Rn
            self.E += np.outer(Rn.sum(axis=0), self.Pr_b)
            self.O += Rn.T @ Pb.T

    legacy_centroid_step = False   # STEP 1 of harmony.cpp:235-238, commented out in 2.0.4
    window_size = 3

    def cluster(self, perms):
        if len(self.obj_harmony) != 1:
            self.Z_corr = self._l2(self.Z_corr)
            self._assign()
        for t in range(self.T):
            if self.legacy_centroid_step:
                self.Y = self._l2(self.R.T @ self.Z_corr)
                self.D = 2.0 * (1.0 - self.Z_corr @ self.Y.T)
            self.update_R(perms[t])
            self.compute_objective()
            if t > self.window_size:                                   # harmony.cpp:249-256 + :176-189
                o, w = self.obj_kmeans, self.window_size
                old, new = sum(o[-2 - i] for i in range(w)), sum(o[-1 - i] for i in range(w))
                if abs(old - new) / abs(old) < self.epsilon_kmeans:
                    break
        self.obj_harmony.append(self.obj_kmeans[-1])

    def moe_correct_ridge(self):
        """Batched: sufficient statistics per (cluster, level), then tiny solves, then one apply.  Also records
        ``lambda_mat`` (K x (B+1), getLambda of harmony.cpp:657-669) and ``W`` ((B+1) x d: the betas of the last
        corrected cluster, row 0 and the rows of dropped levels zero)."""
        K, B, d, N = self.K, self.B, self.d, self.N
        Zc = self.Z_orig.copy()
        Ynew = self.Y.copy()
        self.lambda_mat = np.zeros((K, B + 1))
        if self.lam is None:
            self.lambda_mat[:, 1:] = self.alpha * self.E
        else:
            self.lambda_mat[:] = self.lam[None, :]
        self.W = np.zeros((B + 1, d))
        avg = self.O / self.N_b[None, :]                                                 # [K, B]
        over = avg > np.float32(self.cutoff)
        for k in range(K):
            cov_levels = np.array([over[k, self.cov_of == c].sum() for c in range(self.C)])
            m = over[k] & (cov_levels[self.cov_of] > 1)
            keep = np.flatnonzero(m)
            if len(keep) == 0:
                continue
            part = (self.Phi[keep] > 0).any(axis=0)                                       # cells taking part
            Phis = np.vstack([np.ones((1, part.sum())), self.Phi[keep][:, part]])         # Phi* (B'+1 x n)
            Rk = self.R[part, k]
            lam = np.zeros(len(keep) + 1)
            lam[1:] = self.alpha * self.E[k, keep] if self.lam is None else self.lam[keep + 1]
            cov = (Phis * Rk[None, :]) @ Phis.T + np.diag(lam)
            Wk = np.linalg.solve(cov, (Phis * Rk[None, :]) @ self.Z_orig[part])           # [B'+1, d]
            Ynew[k] = Wk[0]
            Wk[0] = 0
            self.W = np.zeros((B + 1, d))
            self.W[keep + 1] = Wk[1:]
            Zc[part] -= (Phis * Rk[None, :]).T @ Wk
        self.Z_corr = Zc
        self.Y = self._l2(Ynew)

