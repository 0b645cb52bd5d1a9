"""``HarmonyReference``: an integration compressed for mapping new cells onto it (DESIGN.md §8).

Per cluster k of a finished integration: ``Nr[k] = sum_n R[k, n]``, ``Cref[k] = sum_n R[k, n] Z_corr[:, n]``, the
centroid ``Cref[k] / |Cref[k]|`` and sigma[k].  These K x (2 d + 2) numbers are all that mapping a query needs, so a
reference can be saved and mapped against later without the harmony object or its cells.  Host arrays only: loading and
saving a reference needs no GPU.
"""
import os

import numpy as np


class HarmonyReference:
    """``centroids`` [K, d], ``Nr`` [K], ``Cref`` [K, d], ``sigma`` [K] (float64 host arrays)."""

    FIELDS = ("centroids", "Nr", "Cref", "sigma")

    def __init__(self, centroids, Nr, Cref, sigma):
        self.centroids = np.ascontiguousarray(centroids, dtype=np.float64)
        self.Nr = np.ascontiguousarray(Nr, dtype=np.float64).reshape(-1)
        self.Cref = np.ascontiguousarray(Cref, dtype=np.float64)
        self.sigma = np.ascontiguousarray(sigma, dtype=np.float64).reshape(-1)
        K = len(self.Nr)
        if self.centroids.ndim != 2 or self.centroids.shape[0] != K or self.Cref.shape != self.centroids.shape:
            raise ValueError("centroids and Cref must be [K, d] with K = len(Nr)")
        if len(self.sigma) != K:
            raise ValueError("sigma must hold one value per cluster")

    @property
    def K(self):
        return len(self.Nr)

    @property
    def d(self):
        return self.centroids.shape[1]

    def save(self, path):
        """Writes the four arrays with ``np.savez``."""
        np.savez(path, **{f: getattr(self, f) for f in self.FIELDS})

    @classmethod
    def load(cls, path):
        """Reads what ``save`` wrote (``save`` appends ".npz" to a path without it; so may ``path`` leave it out)."""
        if isinstance(path, (str, os.PathLike)) and not os.path.exists(path) and os.path.exists(f"{os.fspath(path)}.npz"):
            path = f"{os.fspath(path)}.npz"
        with np.load(path) as f:
            return cls(*(f[name] for name in cls.FIELDS))

    def __repr__(self):
        return f"HarmonyReference(K={self.K}, d={self.d})"
