"""Loader / builder of libharmony_b200.so (the C ABI declared in include/harmony_b200.h).

There is no CPU fallback: if the shared library is missing or no CUDA device is present the
constructors raise.  The library is built IN-TREE (harmony_b200/libharmony_b200.so) with
``nvcc -gencode arch=compute_90a,code=sm_90a`` (H100) by ``build()`` / ``__graft_entry__.build()``.
"""
import ctypes
import glob
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(_HERE)
SO_PATH = os.path.join(_HERE, "libharmony_b200.so")
# the translation unit build() compiles, then every header it may include: a new header cannot miss needs_build()
SOURCES = [os.path.join(_HERE, "csrc", "harmony_b200.cu")] + sorted(glob.glob(os.path.join(_HERE, "csrc", "*.cuh")))
HEADER = os.path.join(ROOT, "include", "harmony_b200.h")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-shared",
              "-Xcompiler", "-fPIC"]

_LIB = None


def needs_build():
    if not os.path.exists(SO_PATH):
        return True
    t = os.path.getmtime(SO_PATH)
    return any(os.path.exists(s) and os.path.getmtime(s) > t for s in SOURCES + [HEADER])


def build(force=False, verbose=False):
    """Compile the CUDA library for sm_90a (cross-compiles without a GPU)."""
    if not force and not needs_build():
        return SO_PATH
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc] + NVCC_FLAGS + ["-o", SO_PATH, SOURCES[0], "-ldl"]
    if verbose:
        print(" ".join(cmd))
    subprocess.check_call(cmd)
    return SO_PATH


def exported_symbols():
    """Function names declared in include/harmony_b200.h (used by the CPU-side ABI test)."""
    import re
    txt = open(HEADER).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(hb_[a-z_0-9A-Z]+)\s*\(", txt)))


def lib():
    """ctypes handle with argument types set; raises if the library is missing."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(SO_PATH):
        raise RuntimeError(
            f"{SO_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            f"(harmony_b200 has no CPU fallback)")
    L = ctypes.CDLL(SO_PATH)
    P, I, I64, D = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_double
    L.hb_create.argtypes = [ctypes.POINTER(P), I]
    L.hb_destroy.argtypes = [P]
    L.hb_last_error.restype = ctypes.c_char_p
    L.hb_last_error.argtypes = [P]
    L.hb_pop_warning.argtypes = [P, ctypes.c_char_p, ctypes.c_size_t]
    L.hb_comm_unique_id.argtypes = [ctypes.c_char_p]
    L.hb_comm_init.argtypes = [P, I, I, ctypes.c_char_p]
    L.hb_set_shard.argtypes = [P, I64, I64]
    L.hb_setup.argtypes = [P, P, I, I64, P, P, I, P, P, P, D, I, D, D, I, D, D, I]
    L.hb_setup_device.argtypes = [P, P, I, I64, P, I, I64, P, P, I, P, P, P, D, I, D, D, I, D, D, I]
    L.hb_set_seed.argtypes = [P, ctypes.c_uint64]
    L.hb_set_abort_callback.argtypes = [P, P, P]
    L.hb_reference.argtypes = [P, P, P, P, P]
    L.hb_map_setup.argtypes = [P, P, I, I64, P, P, I, P, I, P, P, P, P]
    L.hb_map_setup_device.argtypes = [P, P, I, I64, P, I, I64, P, P, I, P, I, P, P, P, P]
    L.hb_map.argtypes = [P]
    L.hb_knn.argtypes = [P, P, I, I64, I64, P, I, I64, I64, I, I, I, I, P, P, P]
    L.hb_debug_knn_geometry.argtypes = [I, I, I64, I64, I, ctypes.POINTER(I64)]
    L.hb_lisi.argtypes = [P, P, I, I64, I64, I, P, I64, I, D, P, P, P, P]
    L.hb_debug_lisi_geometry.argtypes = [I, D, I64, I, ctypes.POINTER(I64)]
    L.hb_silhouette.argtypes = [P, P, I, I64, I64, I, P, I, P, I, P, P]
    L.hb_debug_silhouette_geometry.argtypes = [I, I64, I, ctypes.POINTER(I64)]
    L.hb_graph_components.argtypes = [P, P, I64, I64, I, P, I, P, P, P]
    L.hb_kbet.argtypes = [P, P, I, I64, I64, I, P, I, P, I, I, P, P, P, P, I64, P]
    L.hb_debug_chi2_sf.argtypes = [D, I, ctypes.POINTER(D)]
    L.hb_pcr.argtypes = [P, P, I, I64, I64, I, P, I, I, P, P, P, P, P]
    L.hb_debug_sym_eig.argtypes = [I, P, P, P]
    L.hb_kmeans.argtypes = [P, P, I, I64, I64, I, I, ctypes.c_uint64, I, I, D, P, P, P, P, P, P]
    L.hb_umap_graph.argtypes = [P, P, I64, P, I64, I64, I, I, P, P, P, ctypes.POINTER(I64), P]
    L.hb_leiden.argtypes = [P, P, P, P, I, I64, I64, D, I, P, ctypes.POINTER(I), ctypes.POINTER(D), ctypes.POINTER(I),
                            P, P]
    L.hb_init_cluster.argtypes = [P, P]
    L.hb_cluster.argtypes = [P, P]
    L.hb_moe_correct_ridge.argtypes = [P]
    L.hb_check_convergence.argtypes = [P, I]
    L.hb_compute_objective.argtypes = [P]
    L.hb_field_size.restype = I64
    L.hb_field_size.argtypes = [P, I]
    L.hb_get_field.argtypes = [P, I, P]
    L.hb_get_field_device.argtypes = [P, I, P, I, I64, P]
    L.hb_set_field.argtypes = [P, I, P]
    L.hb_get_scalar.argtypes = [P, I, ctypes.POINTER(D)]
    L.hb_set_scalar.argtypes = [P, I, D]
    L.hb_get_B_vec.argtypes = [P, P]
    L.hb_trace.restype = I64
    L.hb_trace.argtypes = [P, I, P, I64]
    L.hb_kernel_launches.restype = I64
    L.hb_kernel_launches.argtypes = [P]
    L.hb_stream.restype = P
    L.hb_stream.argtypes = [P]
    L.hb_synchronize.argtypes = [P]
    L.hb_region_time.argtypes = [P, ctypes.c_char_p, ctypes.POINTER(D), ctypes.POINTER(I64)]
    L.hb_enable_timing.argtypes = [P, I]
    L.hb_debug_permute.restype = ctypes.c_uint64
    L.hb_debug_permute.argtypes = [ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint64, I]
    L.hb_debug_update_geometry.argtypes = [I, I, ctypes.POINTER(I64)]
    L.hb_debug_kernel_paths.argtypes = [I, I, I, I64, I, I, I, ctypes.POINTER(I64)]
    L.hb_debug_wide_paths.argtypes = [I, I, I, I64, I, I, I, ctypes.POINTER(I64)]
    L.hb_debug_kmeans_uniform.restype = D
    L.hb_debug_kmeans_uniform.argtypes = [P, ctypes.c_uint64, ctypes.c_uint64]
    L.hb_debug_kmeans_cells.argtypes = [P, P]
    L.hb_debug_kmeans_keep_means.argtypes = [P, I]
    L.hb_debug_kmeans_means.restype = I64
    L.hb_debug_kmeans_means.argtypes = [P, P]
    L.hb_debug_tuple_index.argtypes = [P, P, P, P]
    L.hb_debug_widen.argtypes = [P, P, I64, I]
    _LIB = L
    return L
