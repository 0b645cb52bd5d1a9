"""The ``harmony`` class: Python mirror of the reference's Rcpp module class
(/root/reference/src/harmony.cpp:672-709 — same method and field names, same shapes), implemented
by calls into the C ABI of include/harmony_b200.h.  This is what the reference's R code would hold
as ``harmonyObj`` (R/ui.R:269); the parity tests drive it exactly like the reference's testthat files.

Shapes follow R (column-major, cells are columns): ``obj.R`` is [K, N], ``obj.getZcorr()`` [d, N],
``obj.Y`` [d, K], ``obj.O`` / ``obj.E`` [K, B].  They are Fortran-ordered views of the buffers the
C ABI fills, i.e. the bytes an R numeric matrix would hold.
"""
import ctypes
import warnings

import numpy as np

from . import _lib
from ._arrays import DTYPE, current_stream, device_rows
from .utils import is_cuda_tensor

FIELD = {"Z_corr": 0, "Z_orig": 1, "R": 2, "Y": 3, "O": 4, "E": 5, "W": 6, "Pr_b": 7, "theta": 8, "sigma": 9,
         "lambda_mat": 10, "lambda": 11}
SCALAR = {"N": 0, "B": 1, "K": 2, "d": 3, "C": 4, "alpha": 5, "max_iter_kmeans": 6, "block_size": 7,
          "epsilon_kmeans": 8, "epsilon_harmony": 9, "N_local": 10, "lambda_estimation": 11, "window_size": 12,
          "legacy_centroid_step": 13, "kernel_set": 14, "device": 15}
TRACE = {"objective_kmeans": 0, "objective_kmeans_dist": 1, "objective_kmeans_entropy": 2,
         "objective_kmeans_cross": 3, "objective_harmony": 4, "kmeans_rounds": 5}
_INT_SCALARS = ("N", "B", "K", "d", "C", "max_iter_kmeans", "N_local", "window_size", "legacy_centroid_step", "kernel_set",
                "device")


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


class HarmonyError(RuntimeError):
    pass


class harmony:
    """``new(harmony)`` — an opaque device-resident model; see module docstring."""

    def __init__(self, device=None, comm=None):
        object.__setattr__(self, "_h", None)
        L = _lib.lib()
        h = ctypes.c_void_p()
        st = L.hb_create(ctypes.byref(h), -1 if device is None else int(device))
        if st != 0 or not h:
            raise HarmonyError("hb_create failed: no usable CUDA device (harmony_b200 has no CPU fallback)")
        object.__setattr__(self, "_L", L)
        object.__setattr__(self, "_h", h)
        object.__setattr__(self, "_injected_orders", None)
        if comm is not None:
            self._init_comm(comm)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._L.hb_destroy(h)
            object.__setattr__(self, "_h", None)

    # ---- plumbing -------------------------------------------------------------------------------
    def _check(self, st):
        self._drain_warnings()
        if st != 0:
            raise HarmonyError(self._L.hb_last_error(self._h).decode())

    def _drain_warnings(self):
        buf = ctypes.create_string_buffer(512)
        while self._L.hb_pop_warning(self._h, buf, 512):
            warnings.warn(buf.value.decode())

    def _init_comm(self, comm):
        """comm = (rank, world_size, id_bytes or None, N_global, cell_offset); see harmony_b200.dist.
        ``id_bytes = None`` shares the process-wide communicator an earlier object created."""
        rank, world, uid, n_global, offset = comm
        self._check(self._L.hb_comm_init(self._h, int(rank), int(world), None if uid is None else bytes(uid)))
        self._check(self._L.hb_set_shard(self._h, int(n_global), int(offset)))

    def _scalar(self, name):
        v = ctypes.c_double()
        if self._L.hb_get_scalar(self._h, SCALAR[name], ctypes.byref(v)) != 0:
            raise HarmonyError(f"no scalar {name}")
        return int(v.value) if name in _INT_SCALARS else float(v.value)

    def _field(self, name, shape):
        n = self._L.hb_field_size(self._h, FIELD[name])
        out = np.empty(int(n), dtype=np.float64)
        self._check(self._L.hb_get_field(self._h, FIELD[name], _ptr(out)))
        return out.reshape(shape, order="F")

    # ---- methods of the Rcpp module (harmony.cpp:697-707) --------------------------------------
    def setup(self, Z, Phi, sigma, theta, lambda_, alpha, max_iter_kmeans, epsilon_kmeans, epsilon_harmony, K,
              block_size, B_vec, batch_proportion_cutoff, verbose=False):
        """harmony::setup (harmony.h:25-30).  ``Z``: [N, d] C-order (== the d x N column-major matrix
        of the reference) or [d, N] F-order; ``Phi``: the row-index slot of the B x N design matrix,
        int array [N, C]; ``lambda_``: B+1 values or None / -1 for automatic estimation.

        ``Z`` may also be a float32 / float64 CUDA tensor on the object's device, in either orientation: it is read
        where it lies (no host round trip), after the work queued on the device's current torch stream.  With such a
        ``Z``, ``Phi`` may be an int32 / int64 CUDA tensor ([N] or [N, C]) on the same device, read the same way."""
        dev, Z, z_args, phi_i, phi_ptr, n = self._cell_inputs(Z, Phi)
        B_vec = np.ascontiguousarray(np.atleast_1d(B_vec), dtype=np.int32)
        K = int(K)
        sigma = np.ascontiguousarray(np.broadcast_to(np.asarray(sigma, dtype=np.float64), (K,)))
        theta = np.ascontiguousarray(theta, dtype=np.float64)
        if len(theta) != int(B_vec.sum()):
            raise ValueError("theta must hold one value per covariate level")
        lam = None
        if lambda_ is not None and not (np.ndim(lambda_) == 0 and lambda_ == -1):
            lam = np.ascontiguousarray(np.atleast_1d(lambda_), dtype=np.float64)
            if len(lam) == 1 and lam[0] == -1:
                lam = None
            elif len(lam) != int(B_vec.sum()) + 1:
                raise ValueError("lambda must hold B+1 values")
        rest = (Z.shape[1], n, phi_ptr, _ptr(B_vec), len(B_vec), _ptr(sigma), _ptr(theta),
                None if lam is None else _ptr(lam), float(alpha), int(max_iter_kmeans), float(epsilon_kmeans),
                float(epsilon_harmony), K, float(block_size), float(batch_proportion_cutoff), int(bool(verbose)))
        if dev:
            self._check(self._L.hb_setup_device(self._h, *z_args, *rest))
        else:
            self._check(self._L.hb_setup(self._h, _ptr(Z), *rest))

    def _cell_inputs(self, Z, Phi):
        """The per-cell inputs of setup and map_setup: Z ([N, d] or [d, N], host array or CUDA tensor) and Phi ([N] or
        [N, C]) -> (Z on device, Z to read, its hb_*_device arguments (None for host Z), phi_i, phi_i's pointer, N).
        The returned arrays and tensors must stay alive until the library call returns."""
        dev = is_cuda_tensor(Z)
        if not dev:
            Z = np.asarray(Z)
        if is_cuda_tensor(Phi):
            if not dev:
                raise ValueError("Phi is a CUDA tensor but Z is not: device labels go with a device embedding")
            phi_i = self._device_Phi(Phi)
        else:
            phi_i = np.ascontiguousarray(Phi, dtype=np.int32)
            if phi_i.ndim == 1:
                phi_i = phi_i.reshape(-1, 1)
        n = phi_i.shape[0]
        if Z.ndim != 2:
            raise ValueError("Z must be a matrix")
        if Z.shape[0] != n and Z.shape[1] == n:
            Z = Z.T                                   # d x N given: its transpose view is the same memory order
        if Z.shape[0] != n:
            raise ValueError("number of cells in Z and Phi differ")
        z_args = None
        if dev:
            Z, ptr, dtype, ld = device_rows(self, Z, "Z")
            z_args = (ptr, dtype, ld, current_stream(Z.device))
        else:
            Z = np.ascontiguousarray(Z, dtype=np.float64)
        phi_ptr = ctypes.c_void_p(phi_i.data_ptr()) if is_cuda_tensor(phi_i) else _ptr(phi_i)
        return dev, Z, z_args, phi_i, phi_ptr, n

    # ---- mapping a query onto a finished integration (DESIGN.md §8) ----------------------------
    def reference(self):
        """The compression of this integration (any state after init_cluster_cpp; normally after harmonize) as a
        HarmonyReference: per cluster Nr = sum R, Cref = R Z_corr^T (the Z_corr getZcorr() returns), the normalised
        centroids Cref / |Cref| and sigma."""
        from .mapping import HarmonyReference
        K, d = self._scalar("K"), self._scalar("d")
        Y, Nr, Cref, sigma = np.empty((K, d)), np.empty(K), np.empty((K, d)), np.empty(K)
        self._check(self._L.hb_reference(self._h, _ptr(Y), _ptr(Nr), _ptr(Cref), _ptr(sigma)))
        return HarmonyReference(Y, Nr, Cref, sigma)

    def map_setup(self, Z, Phi, B_vec, lambda_, reference):
        """Sets this object up to map a query onto ``reference`` (a HarmonyReference), instead of ``setup``.  ``Z``
        and ``Phi`` take setup's forms (host arrays or CUDA tensors); ``Phi`` and ``B_vec`` describe the query's own
        covariates; ``lambda_``: a scalar or one value per query level, each finite and > 0."""
        K, d = reference.K, reference.d
        dev, Z, z_args, phi_i, phi_ptr, n = self._cell_inputs(Z, Phi)
        if Z.shape[1] != d:
            raise ValueError(f"the query has {Z.shape[1]} dimensions, the reference {d}")
        B_vec = np.ascontiguousarray(np.atleast_1d(B_vec), dtype=np.int32)
        lam = np.ascontiguousarray(np.broadcast_to(np.asarray(lambda_, dtype=np.float64).reshape(-1),
                                                   (int(B_vec.sum()),)))
        ref = [np.ascontiguousarray(a, dtype=np.float64) for a in
               (reference.centroids, reference.Nr, reference.Cref, reference.sigma)]
        rest = (d, n, phi_ptr, _ptr(B_vec), len(B_vec), _ptr(lam), K, *(_ptr(a) for a in ref))
        if dev:
            self._check(self._L.hb_map_setup_device(self._h, *z_args, *rest))
        else:
            self._check(self._L.hb_map_setup(self._h, _ptr(Z), *rest))

    def map(self):
        """Maps the query set up by map_setup: soft assignment to the reference's clusters, then one ridge correction
        anchored on the reference.  getZcorr() / get_tensor("Z_corr") then hold the mapped embedding, getR() the
        assignment."""
        self._check(self._L.hb_map(self._h))

    def knn(self, query, ref=None, k=15, metric="euclidean"):
        """``harmony_b200.knn`` on this object's device and stream, without a second handle: the exact k nearest rows
        of ``ref`` (``None``: of ``query`` itself, leaving each row out) for every row of ``query`` -> (idx, dist).
        Works in any state of the object and changes none of it, e.g. ``obj.knn(obj.get_tensor("Z_corr"))``."""
        from .neighbors import knn_on
        return knn_on(self, query, ref, k, metric)

    def lisi(self, X, codes, perplexity=30, return_neighbors=False):
        """LISI of every row of ``X`` [N, d] (host array or CUDA tensor) for the label sets ``codes`` (int32 [N] or
        [n_sets, N]; any codes, only equality counts) on this object's device and stream -> [N, n_sets] float64, with
        ``return_neighbors`` also ``(idx, dist)``.  ``harmony_b200.compute_lisi`` takes labels by column name.  Works
        in any state of the object and changes none of it, e.g. ``obj.lisi(obj.get_tensor("Z_corr"), batch_codes)``."""
        from .lisi import lisi_on
        return lisi_on(self, X, codes, perplexity, return_neighbors)

    def silhouette(self, X, labels, groups=None):
        """Silhouette width of every row of ``X`` [N, d] (host array or CUDA tensor) for the label codes ``labels``
        (dense codes 0..n-1, [N]; numpy or int32 CUDA tensor), only rows of one group interacting when ``groups`` (the
        same) are given, on this object's device and stream -> [N] float64.  ``harmony_b200.silhouette_samples`` takes
        any label values.  Works in any state of the object and changes none of it."""
        from .silhouette import silhouette_on
        return silhouette_on(self, X, labels, groups)

    def graph_components(self, idx, labels=None):
        """Connected components of the neighbour graph ``idx`` [N, k] (int32, -1 for no neighbour; host array or CUDA
        tensor), with edges only between rows of one label when ``labels`` (dense codes 0..n-1, [N]; numpy or int32 CUDA
        tensor) are given, on this object's device and stream -> ``(comp, largest)``: the smallest row of each row's
        component, and the largest component of each label.  ``harmony_b200.graph_components`` takes any label values.
        Works in any state of the object and changes none of it."""
        from .graph import components_on
        return components_on(self, idx, labels)

    def kbet(self, X, batches, labels=None, k0=0, return_neighbors=False):
        """kBET's per-cell test of every row of ``X`` [N, d] (host array or CUDA tensor) with the batch codes ``batches``
        and, within each label of ``labels`` (both dense codes 0..n-1, [N]; numpy or int32 CUDA tensors; no labels: one
        label), ``k0`` = 0 for scib's rule or a fixed 2..129, on this object's device and stream -> ``(stat, pval, k0)``,
        with ``return_neighbors`` also ``idx``.  ``harmony_b200.kbet`` takes labels by column name and folds the score.
        Works in any state of the object and changes none of it."""
        from .kbet import kbet_on
        return kbet_on(self, X, batches, labels, k0, return_neighbors)

    def pcr(self, X, batches, n_comps=50):
        """Principal component regression of ``X`` [N, d] (host array or CUDA tensor) on the batch codes ``batches``
        (dense codes 0..n-1, [N]; numpy or an int32 CUDA tensor) on this object's device and stream -> ``(var, r2,
        components, score)`` of the min(n_comps, N, d) leading components.  ``harmony_b200.pcr`` takes the batches by
        column name.  Works in any state of the object and changes none of it."""
        from .pcr import pcr_on
        return pcr_on(self, X, batches, n_comps)

    def kmeans(self, X, n_clusters, seed=0, n_init=1, max_iter=300, tol=1e-4, return_seeds=False):
        """k-means of ``X`` [N, d] (host array or CUDA tensor) into ``n_clusters`` clusters on this object's device and
        stream -> ``(labels, centres, inertia, n_iter)`` (and the seed rows with ``return_seeds``), as
        ``harmony_b200.kmeans`` returns them.  Works in any state of the object and changes none of it."""
        from .clustering import kmeans_on
        return kmeans_on(self, X, n_clusters, seed, n_init, max_iter, tol, return_seeds)

    def umap_connectivities(self, X, n_neighbors=15):
        """``hb_umap_graph`` of X's exact neighbour graph on this object's device, as
        ``harmony_b200.umap_connectivities`` returns it.  Works in any state of the object and changes none of it."""
        from .community import umap_on
        return umap_on(self, X, n_neighbors)

    def leiden(self, X_or_graph, resolution=1.0, n_neighbors=15, n_iterations=-1, return_info=False):
        """``hb_leiden`` on this object's device, as ``harmony_b200.leiden`` returns it.  Works in any state of the
        object and changes none of it."""
        from .community import leiden_on
        return leiden_on(self, X_or_graph, resolution, n_neighbors, n_iterations, return_info)

    def _device_Phi(self, Phi):
        """An [N] or [N, C] int32 / int64 CUDA tensor -> contiguous [N, C] int32 on the object's device (converted, if
        need be, on the current torch stream, which hb_setup_device orders its read after)."""
        import torch
        if Phi.dtype not in (torch.int32, torch.int64):
            raise TypeError(f"Phi must be int32 or int64, not {Phi.dtype}")
        if Phi.device.index != self._scalar("device"):
            raise ValueError(f"Phi is on {Phi.device}, the harmony object on cuda:{self._scalar('device')}")
        if Phi.ndim == 1:
            Phi = Phi.reshape(-1, 1)
        if Phi.ndim != 2:
            raise ValueError("Phi must be [N] or [N, C]")
        return Phi.to(torch.int32).contiguous()

    def set_seed(self, seed):
        self._check(self._L.hb_set_seed(self._h, int(seed) & 0xFFFFFFFFFFFFFFFF))

    def init_cluster_cpp(self, Y0=None):
        """harmony::init_cluster_cpp.  ``Y0`` ([d, K] like ``obj.Y`` or [K, d] C-order) injects the
        k-means centroids (what kmeans_centers returns, harmony.cpp:133)."""
        if Y0 is None:
            self._check(self._L.hb_init_cluster(self._h, None))
            return
        K, d = self._scalar("K"), self._scalar("d")
        if K == 0:                                    # setup has not run: let the library report it
            self._check(self._L.hb_init_cluster(self._h, None))
        Y0 = np.asarray(Y0, dtype=np.float64)
        if Y0.shape == (d, K) and not (K == d and Y0.flags.c_contiguous):
            Y0 = Y0.T
        Y0 = np.ascontiguousarray(Y0)
        if Y0.shape != (K, d):
            raise ValueError("Y0 must be d x K")
        self._check(self._L.hb_init_cluster(self._h, _ptr(Y0)))

    def set_abort_callback(self, fn):
        """Progress::check_abort of the reference (harmony.cpp:233, 355): ``fn()`` is polled before the clustering
        rounds of every cluster_cpp call (and between them); a true value makes cluster_cpp return -1, which
        harmonize() turns into "terminated by user" (R/utils.R:27-29).  ``None`` removes the callback."""
        import ctypes
        if fn is None:
            self._abort_cb = None
            self._check(self._L.hb_set_abort_callback(self._h, None, None))
            return
        proto = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p)
        self._abort_cb = proto(lambda _user: 1 if fn() else 0)   # keep the trampoline alive with the object
        self._check(self._L.hb_set_abort_callback(self._h, ctypes.cast(self._abort_cb, ctypes.c_void_p), None))

    def cluster_cpp(self, update_orders=None):
        """harmony::cluster_cpp -> 0 / -1 (aborted).  ``update_orders``: [max_iter_kmeans, N] int64,
        row t = the shuffled update order of the t-th update_R call (harmony.cpp:272-273)."""
        if update_orders is None:
            st = self._L.hb_cluster(self._h, None)
        else:
            T, N = self._scalar("max_iter_kmeans"), self._scalar("N")
            uo = np.ascontiguousarray(update_orders, dtype=np.int64).reshape(-1, N)
            if uo.shape[0] < T:
                raise ValueError("need one update order per clustering round")
            st = self._L.hb_cluster(self._h, _ptr(uo))
        if st == -1:
            return -1
        self._check(st)
        return 0

    def moe_correct_ridge_cpp(self):
        self._check(self._L.hb_moe_correct_ridge(self._h))

    def check_convergence(self, type_):
        r = self._L.hb_check_convergence(self._h, int(type_))
        if r < 0:
            raise HarmonyError(self._L.hb_last_error(self._h).decode())
        return bool(r)

    def compute_objective(self):
        self._check(self._L.hb_compute_objective(self._h))

    def getZcorr(self):
        return self._field("Z_corr", (self._scalar("d"), self._scalar("N_local")))

    def getZorig(self):
        return self._field("Z_orig", (self._scalar("d"), self._scalar("N_local")))

    def getR(self):
        return self._field("R", (self._scalar("K"), self._scalar("N_local")))

    def getCentroids(self):
        return self._field("Y", (self._scalar("d"), self._scalar("K")))

    def getLambda(self):
        return self._field("lambda_mat", (self._scalar("K"), self._scalar("B") + 1))

    def get_tensor(self, name, dtype=None):
        """``name`` ("Z_corr", "Z_orig" or "R") as a new [N_local, cols] CUDA tensor on the object's device: the bytes
        of the [cols, N_local] array getZcorr() / getZorig() / getR() return, without leaving the device.
        ``dtype``: torch.float32 (default) or torch.float64.  The copy is ordered on the device's current torch stream
        (work queued there afterwards sees it); the host is not blocked."""
        import torch
        dtype = torch.float32 if dtype is None else dtype
        if name not in ("Z_corr", "Z_orig", "R"):
            raise ValueError(f"get_tensor: no per-cell field {name!r} (Z_corr, Z_orig, R)")
        if dtype not in (torch.float32, torch.float64):
            raise TypeError(f"get_tensor: dtype must be torch.float32 or torch.float64, not {dtype}")
        cols = self._scalar("K" if name == "R" else "d")
        device = torch.device("cuda", self._scalar("device"))
        out = torch.empty((self._scalar("N_local"), cols), dtype=dtype, device=device)
        self._check(self._L.hb_get_field_device(self._h, FIELD[name], ctypes.c_void_p(out.data_ptr()),
                                                DTYPE[str(dtype)[6:]], cols, current_stream(device)))
        return out

    # ---- fields of the Rcpp module (harmony.cpp:675-696) ---------------------------------------
    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        if name in ("N", "B", "K", "d", "alpha", "max_iter_kmeans", "legacy_centroid_step", "kernel_set"):
            return self._scalar(name)
        if name == "R":
            return self.getR()
        if name == "Y":
            return self.getCentroids()
        if name in ("O", "E"):
            return self._field(name, (self._scalar("K"), self._scalar("B")))
        if name == "W":
            return self._field("W", (self._scalar("B") + 1, self._scalar("d")))
        if name in ("Pr_b", "theta"):
            return self._field(name, (self._scalar("B"),))
        if name == "sigma":
            return self._field(name, (self._scalar("K"),))
        if name == "lambda_":
            return self._field("lambda", (self._scalar("B") + 1,))
        if name == "B_vec":
            out = np.empty(self._scalar("C"), dtype=np.int32)
            self._L.hb_get_B_vec(self._h, _ptr(out))
            return out
        if name in TRACE:
            n = self._L.hb_trace(self._h, TRACE[name], None, 0)
            if n < 0:
                raise HarmonyError(self._L.hb_last_error(self._h).decode())
            out = np.empty(int(n), dtype=np.float64)
            self._L.hb_trace(self._h, TRACE[name], _ptr(out), n)
            return out.astype(np.int64) if name == "kmeans_rounds" else out
        raise AttributeError(name)

    def __setattr__(self, name, value):
        if name.startswith("_"):
            object.__setattr__(self, name, value)
            return
        if name in ("alpha", "max_iter_kmeans", "legacy_centroid_step", "kernel_set"):
            self._check(self._L.hb_set_scalar(self._h, SCALAR[name], float(value)))
            return
        shapes = {"Y": ("Y", "d", "K"), "R": ("R", "K", "N_local"), "O": ("O", "K", "B"), "E": ("E", "K", "B")}
        if name in shapes:
            f, r, c = shapes[name]
            v = np.asfortranarray(np.asarray(value, dtype=np.float64))
            if v.shape != (self._scalar(r), self._scalar(c)):
                raise ValueError(f"{name} must be {r} x {c}")
            self._check(self._L.hb_set_field(self._h, FIELD[f], _ptr(v)))
            return
        if name in ("theta", "sigma", "lambda_"):
            v = np.ascontiguousarray(value, dtype=np.float64).ravel()
            n = {"theta": self._scalar("B"), "sigma": self._scalar("K"), "lambda_": self._scalar("B") + 1}[name]
            if name == "sigma" and v.size == 1:
                v = np.full(n, v[0])   # a scalar sigma is broadcast to the K clusters, as in setup
            if v.size != n:
                raise ValueError(f"{name} must have {n} values, got {v.size}")
            self._check(self._L.hb_set_field(self._h, FIELD["lambda" if name == "lambda_" else name], _ptr(v)))
            return
        raise AttributeError(f"field {name} is not writable")

    # ---- instrumentation -----------------------------------------------------------------------
    def synchronize(self):
        self._check(self._L.hb_synchronize(self._h))

    @property
    def kernel_launches(self):
        return int(self._L.hb_kernel_launches(self._h))

    @property
    def cuda_stream(self):
        return int(self._L.hb_stream(self._h) or 0)

    def enable_timing(self, on=True):
        self._L.hb_enable_timing(self._h, int(bool(on)))

    def region_time(self, region):
        ms, n = ctypes.c_double(), ctypes.c_int64()
        if self._L.hb_region_time(self._h, region.encode(), ctypes.byref(ms), ctypes.byref(n)) != 0:
            return 0.0, 0
        return ms.value, int(n.value)
