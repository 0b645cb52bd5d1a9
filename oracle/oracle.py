"""ctypes wrapper around oracle/libharmony_oracle.so (CPU restatement of the reference).

TEST INFRASTRUCTURE ONLY — imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs; never by harmony_b200/.
"""
import ctypes
import glob
import os
import subprocess
import sysconfig

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

FIELDS = {"Z_corr": 0, "Z_orig": 1, "R": 2, "Y": 3, "O": 4, "E": 5, "W": 6, "Pr_b": 7, "theta": 8, "sigma": 9,
          "lambda": 10, "dist_mat": 11}
TRACES = {"objective_kmeans": 0, "objective_kmeans_dist": 1, "objective_kmeans_entropy": 2,
          "objective_kmeans_cross": 3, "objective_harmony": 4, "kmeans_rounds": 5}


def build(force=False):
    so = os.path.join(_HERE, "libharmony_oracle.so")
    src = os.path.join(_HERE, "harmony_oracle.cpp")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-B", "libharmony_oracle.so"], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = ctypes.CDLL(build())
        L.ho_create.restype = ctypes.c_void_p
        L.ho_create.argtypes = [ctypes.c_int]
        L.ho_destroy.argtypes = [ctypes.c_void_p]
        L.ho_last_error.restype = ctypes.c_char_p
        L.ho_last_error.argtypes = [ctypes.c_void_p]
        L.ho_blas_name.restype = ctypes.c_char_p
        L.ho_load_blas.argtypes = [ctypes.c_char_p, ctypes.c_int]
        P = ctypes.c_void_p
        L.ho_setup.argtypes = [P, P, ctypes.c_int, ctypes.c_int64, P, P, ctypes.c_int, P, P, P, ctypes.c_double,
                               ctypes.c_int, ctypes.c_double, ctypes.c_double, ctypes.c_int, ctypes.c_double,
                               ctypes.c_double]
        L.ho_init_cluster.argtypes = [P, P]
        L.ho_cluster.argtypes = [P, P]
        L.ho_update_R.argtypes = [P, P]
        L.ho_moe_correct_ridge.argtypes = [P]
        L.ho_check_convergence.argtypes = [P, ctypes.c_int]
        L.ho_compute_objective.argtypes = [P]
        L.ho_warned_small.argtypes = [P]
        L.ho_set_max_iter_kmeans.argtypes = [P, ctypes.c_int]
        L.ho_set_legacy_centroid_step.argtypes = [P, ctypes.c_int]
        L.ho_get.argtypes = [P, ctypes.c_int, P]
        L.ho_set.argtypes = [P, ctypes.c_int, P]
        L.ho_trace.restype = ctypes.c_int64
        L.ho_trace.argtypes = [P, ctypes.c_int, P, ctypes.c_int64]
        _LIB = L
    return _LIB


def find_openblas():
    """Candidate OpenBLAS shared objects shipped inside this image's wheels (no system BLAS)."""
    sp = sysconfig.get_paths()["purelib"]
    pats = ["opencv_python_headless.libs/libopenblas*.so", "scipy.libs/libscipy_openblas*.so",
            "numpy.libs/libscipy_openblas*.so"]
    out = []
    for p in pats:
        out += sorted(glob.glob(os.path.join(sp, p)))
    return out


def load_blas(threads=0):
    """Try to give the oracle a real sgemm (what Armadillo would call).  Returns the name used."""
    L = lib()
    for cand in find_openblas():
        if L.ho_load_blas(cand.encode(), int(threads)) == 0:
            break
    return L.ho_blas_name().decode()


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


class OracleHarmony:
    """Mirror of the reference's ``harmony`` class (src/harmony.h:20-70) on the CPU oracle.

    Matrices cross this boundary in the reference's own layout (column-major, cells are columns),
    which numpy sees as C-contiguous [N, d] / [N, K] / [K, d] / [B, K] arrays.
    """

    def __init__(self, double=False):
        self.L = lib()
        self.h = self.L.ho_create(1 if double else 0)
        self.double = double

    def __del__(self):
        if getattr(self, "h", None):
            self.L.ho_destroy(self.h)
            self.h = None

    def _check(self, st):
        if st != 0:
            raise RuntimeError(f"oracle status {st}: {self.L.ho_last_error(self.h).decode()}")

    def setup(self, Z, phi_i, B_vec, sigma, theta, lambda_, alpha, max_iter_kmeans, epsilon_kmeans,
              epsilon_harmony, K, block_size, batch_proportion_cutoff):
        Z = np.ascontiguousarray(Z, dtype=np.float64)            # [N, d]
        self.N, self.d = Z.shape
        phi_i = np.ascontiguousarray(phi_i, dtype=np.int32).reshape(self.N, -1)
        self.C = phi_i.shape[1]
        B_vec = np.ascontiguousarray(B_vec, dtype=np.int32)
        self.B = int(B_vec.sum())
        self.K = int(K)
        sigma = np.ascontiguousarray(np.broadcast_to(np.asarray(sigma, dtype=np.float64), (self.K,)))
        theta = np.ascontiguousarray(theta, dtype=np.float64)
        lam = None if lambda_ is None else np.ascontiguousarray(lambda_, dtype=np.float64)
        self._check(self.L.ho_setup(self.h, _ptr(Z), self.d, self.N, _ptr(phi_i), _ptr(B_vec), self.C, _ptr(sigma),
                                    _ptr(theta), None if lam is None else _ptr(lam), float(alpha),
                                    int(max_iter_kmeans), float(epsilon_kmeans), float(epsilon_harmony), self.K,
                                    float(block_size), float(batch_proportion_cutoff)))
        self.max_iter_kmeans = int(max_iter_kmeans)

    def init_cluster_cpp(self, Y0):
        Y0 = np.ascontiguousarray(Y0, dtype=np.float64)          # [K, d]
        assert Y0.shape == (self.K, self.d)
        self._check(self.L.ho_init_cluster(self.h, _ptr(Y0)))

    def cluster_cpp(self, perms):
        perms = np.ascontiguousarray(perms, dtype=np.int64).reshape(-1, self.N)
        assert perms.shape[0] >= self.max_iter_kmeans
        st = self.L.ho_cluster(self.h, _ptr(perms))
        self._check(st)
        return st

    def update_R(self, perm):
        perm = np.ascontiguousarray(perm, dtype=np.int64)
        self._check(self.L.ho_update_R(self.h, _ptr(perm)))

    def moe_correct_ridge_cpp(self):
        self._check(self.L.ho_moe_correct_ridge(self.h))

    def check_convergence(self, type_):
        return bool(self.L.ho_check_convergence(self.h, int(type_)))

    def compute_objective(self):
        self.L.ho_compute_objective(self.h)

    def set_legacy_centroid_step(self, on=True):
        """Run STEP 1 of harmony.cpp:235-238 (centroid update, commented out in 2.0.4) in every clustering round."""
        self.L.ho_set_legacy_centroid_step(self.h, int(bool(on)))

    def set_max_iter_kmeans(self, v):
        self.L.ho_set_max_iter_kmeans(self.h, int(v))
        self.max_iter_kmeans = int(v)

    def get(self, name):
        shapes = {"Z_corr": (self.N, self.d), "Z_orig": (self.N, self.d), "R": (self.N, self.K),
                  "Y": (self.K, self.d), "O": (self.B, self.K), "E": (self.B, self.K), "W": (self.d, self.B + 1),
                  "Pr_b": (self.B,), "theta": (self.B,), "sigma": (self.K,), "lambda": (self.B + 1, self.K),
                  "dist_mat": (self.N, self.K)}
        out = np.empty(shapes[name], dtype=np.float64)
        st = self.L.ho_get(self.h, FIELDS[name], _ptr(out))
        assert st == 0
        return out

    def set(self, name, value):
        """Write R [N, K], Y [K, d], O or E [B, K], theta [B] or sigma [K] (the layouts get() returns)."""
        shapes = {"R": (self.N, self.K), "Y": (self.K, self.d), "O": (self.B, self.K), "E": (self.B, self.K),
                  "theta": (self.B,), "sigma": (self.K,)}
        v = np.ascontiguousarray(value, dtype=np.float64)
        assert v.shape == shapes[name], (name, v.shape)
        self._check(self.L.ho_set(self.h, FIELDS[name], _ptr(v)))

    def trace(self, name):
        n = self.L.ho_trace(self.h, TRACES[name], None, 0)
        out = np.empty(n, dtype=np.float64)
        self.L.ho_trace(self.h, TRACES[name], _ptr(out), n)
        return out
