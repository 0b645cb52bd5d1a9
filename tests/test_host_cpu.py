"""CPU tests of the host-side logic and of the C-ABI library's surface (no compute calls: this box
has no GPU).  Mirrors the argument checks of /root/reference/tests/testthat/test_integration.R:43-55."""
import ctypes
import os

import numpy as np
import pytest

from harmony_b200 import _lib, harmony_options, prepare_inputs
from harmony_b200.harmony_option import check_legacy_args
from helpers import load_cell_lines


def test_library_exports_every_declared_symbol():
    _lib.build()
    L = ctypes.CDLL(_lib.SO_PATH)
    names = _lib.exported_symbols()
    assert len(names) >= 25
    for s in names:
        assert hasattr(L, s), s
    assert L.hb_version() >= 100


def test_no_cpu_fallback_without_device():
    """On a box without a CUDA device the product path fails loudly (no CPU fallback)."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from harmony_b200.harmony import HarmonyError, harmony
    with pytest.raises(HarmonyError, match="no usable CUDA device"):
        harmony()


def test_product_never_imports_oracle():
    root = os.path.dirname(_lib._HERE)
    for dp, _, files in os.walk(os.path.join(root, "harmony_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(dp, f)).read()
                assert "oracle" not in txt.replace("the CPU oracle", "").lower() or f == "__init__.py", (dp, f)


def test_prepare_inputs_defaults():
    Z, meta = load_cell_lines(True)
    a = prepare_inputs(Z, meta, "dataset")
    assert a["K"] == 10                       # min(round(300/30), 100), R/ui.R:192-194
    assert a["B_vec"].tolist() == [3]
    assert a["theta"].tolist() == [2, 2, 2]
    assert a["lambda_"] is None               # lambda = NULL -> estimation
    assert a["sigma"].shape == (10,) and np.all(a["sigma"] == 0.1)
    assert a["max_iter_kmeans"] == 4 and a["block_size"] == 0.05
    assert a["phi_i"].shape == (300, 1) and a["phi_i"].max() == 2
    a = prepare_inputs(Z.T, meta, "dataset")  # transposed input is detected (R/ui.R:178-183)
    assert a["Z"].shape == (300, 20)
    a2 = prepare_inputs(Z, meta, ["cell_type", "dataset"], theta=[1, 3], lambda_=[0.5, 2.0])
    assert a2["B_vec"].tolist() == [2, 3]
    assert a2["theta"].tolist() == [1, 1, 3, 3, 3]
    assert a2["lambda_"].tolist() == [0, 0.5, 0.5, 2, 2, 2]
    assert a2["phi_i"][:, 1].min() == 2        # second covariate's levels are offset by B_vec[0]
    a3 = prepare_inputs(Z, meta, "dataset", lambda_=1.5)
    assert a3["lambda_"].tolist() == [0, 1.5, 1.5, 1.5]
    a4 = prepare_inputs(Z, meta, "dataset", early_stop=False)
    assert a4["epsilon_harmony"] == -np.inf
    a5 = prepare_inputs(Z, np.asarray(meta["dataset"]), None)   # bare vector -> batch_variable
    assert a5["vars_use"] == ["batch_variable"]
    a6 = prepare_inputs(Z, meta, "dataset", options=harmony_options(tau=5), nclust=5)
    nb = 100.0
    assert np.allclose(a6["theta"], 2 * (1 - np.exp(-(nb / (5 * 5)) ** 2)))


def test_error_messages():
    # test_integration.R:43-55
    Z, meta = load_cell_lines(True)
    with pytest.raises(ValueError):
        prepare_inputs(Z, meta, "fake_variable")
    with pytest.raises(ValueError, match="mismatch"):
        prepare_inputs(Z, meta, "dataset", lambda_=[1, 2])
    short = {k: v[:-1] for k, v in meta.items()}
    with pytest.raises(ValueError, match="do not correspond"):
        prepare_inputs(Z, short, "dataset")
    with pytest.raises(ValueError, match="positive"):
        prepare_inputs(Z, meta, "dataset", lambda_=-1.0)
    with pytest.raises(ValueError, match="theta"):
        prepare_inputs(Z, meta, "dataset", theta=[1, 2])
    with pytest.raises(TypeError):
        prepare_inputs(Z, meta, "dataset", options={"alpha": 1})
    with pytest.raises(ValueError, match="block.size"):
        harmony_options(block_size=0)
    with pytest.raises(TypeError, match="dropped"):
        check_legacy_args(tau=1)
    with pytest.raises(TypeError, match="unhandled"):
        check_legacy_args(foo=1)


def test_harmonize_driver_contract():
    """R/utils.R:15-46 against a scripted stand-in object."""
    from harmony_b200 import harmonize

    class Fake:
        def __init__(self, conv_at, status=0):
            self.calls, self.conv_at, self.status, self.it = [], conv_at, status, 0

        def cluster_cpp(self):
            self.calls.append("cluster")
            return self.status

        def moe_correct_ridge_cpp(self):
            self.calls.append("moe")

        def check_convergence(self, t):
            assert t == 1
            self.it += 1
            return self.it >= self.conv_at

    f = Fake(3)
    assert harmonize(f, 10, verbose=False) == 0
    assert f.calls == ["cluster", "moe"] * 3
    f = Fake(99)
    assert harmonize(f, 2, verbose=False) is None
    assert len(f.calls) == 4
    assert harmonize(Fake(1), 0, verbose=False) == 0
    with pytest.raises(KeyboardInterrupt):
        harmonize(Fake(1, status=-1), 3, verbose=False)
    with pytest.raises(RuntimeError, match="non-zero exit status: 7"):
        harmonize(Fake(1, status=7), 3, verbose=False)


@pytest.mark.parametrize("n", [1, 2, 7, 300, 4096, 100003])
def test_native_update_order_is_a_permutation(n):
    """The keyed Feistel order that stands in for arma::shuffle (harmony.cpp:272-273) is a bijection of
    [0, n), its inverse inverts it, different keys give different orders, and blocks come out balanced."""
    L = _lib.lib()
    key = 0x1234ABCD
    pos = np.array([L.hb_debug_permute(i, n, key, 0) for i in range(min(n, 5000))], dtype=np.int64)
    if n <= 5000:
        assert sorted(pos.tolist()) == list(range(n))
    assert pos.min() >= 0 and pos.max() < n and len(set(pos.tolist())) == len(pos)
    for i in range(0, min(n, 200)):
        assert L.hb_debug_permute(int(pos[i]), n, key, 1) == i
    assert L.hb_debug_permute(n, n, key, 0) == 2 ** 64 - 1
    if n >= 4096:
        other = np.array([L.hb_debug_permute(i, n, key + 1, 0) for i in range(1000)])
        assert (other != pos[:1000]).mean() > 0.9
        blk = np.minimum(pos // (n // 20), 19)           # 20 update blocks as in harmony.cpp:280-300
        cnt = np.bincount(blk, minlength=20)
        assert cnt.min() > 0.5 * len(pos) / 20 and cnt.max() < 1.6 * len(pos) / 20


def test_update_kernel_ring_geometry():
    """Ring geometry of the persistent update kernel: for every padded row width the library either declines
    (the other update kernels serve the shape) or returns per-warp rings that fit shared memory, whose lanes cover
    the row and whose depth is a power of two (slot index = group counter & (depth - 1))."""
    import ctypes
    L = _lib.lib()
    out = (ctypes.c_int64 * 9)()
    supported = 0
    for KS in range(4, 1025, 4):
        if not L.hb_debug_update_geometry(KS, 20, out):
            continue
        supported += 1
        NV, DG, RU, smem, NW = list(out)[:5]
        assert NV in (1, 2) and 128 * NV >= KS and (NV == 1 or 128 < KS)   # lane l owns float4 l + 32 v
        assert DG >= 2 and DG & (DG - 1) == 0 and RU in (2, 4) and NW == 16
        assert smem <= 227 * 1024 - 256 and smem >= NW * DG * RU * KS * 4
    assert not L.hb_debug_update_geometry(6, 20, out)          # row widths are multiples of 4 floats
    assert L.hb_debug_update_geometry(100, 20, out) and out[0] == 1 and out[1] * out[2] >= 24   # K = 100: > 1 block step of a warp's rows at 1M cells
    assert L.hb_debug_update_geometry(200, 20, out) and out[0] == 2
    assert supported >= 50


PER_STEP, TWO_PASS, SINGLE_PASS = 0, 1, 2
C3 = dict(K=100, d=50, J=20, n=1_000_000)


# shape -> (update path, fused K1 operand stages (0: FFMA or logits), wgmma logits, wgmma apply, tensor-core k-means
#           init, cold start in plan order, path of a 40-round call, path of a call with the legacy centroid step)
@pytest.mark.parametrize("shape, kernel_set, expected", [
    (C3, 0, (SINGLE_PASS, 2, 0, 1, 1, 1, SINGLE_PASS, PER_STEP)),
    (dict(K=100, d=50, J=40, n=1_250_000), 0, (SINGLE_PASS, 2, 0, 1, 1, 1, SINGLE_PASS, PER_STEP)),    # c4
    (dict(K=200, d=100, J=40, n=6_250_000), 0, (SINGLE_PASS, 0, 1, 1, 1, 1, SINGLE_PASS, PER_STEP)),   # c5
    (dict(K=100, d=50, J=100, n=1_000_000), 0, (TWO_PASS, 2, 0, 1, 1, 0, PER_STEP, PER_STEP)),
    (dict(K=300, d=50, J=20, n=1_000_000), 0, (PER_STEP, 0, 1, 1, 0, 0, PER_STEP, PER_STEP)),
    (dict(K=50, d=150, J=20, n=1_000_000), 0, (SINGLE_PASS, 0, 0, 0, 0, 0, SINGLE_PASS, PER_STEP)),
    (C3, 1, (SINGLE_PASS, 0, 0, 0, 0, 0, SINGLE_PASS, PER_STEP)),    # HB_KS_FFMA_CONTRACTIONS
    (C3, 2, (PER_STEP, 2, 0, 1, 1, 0, PER_STEP, PER_STEP)),          # HB_KS_UPDATE_PER_STEP
    (C3, 4, (TWO_PASS, 2, 0, 1, 1, 0, PER_STEP, PER_STEP)),          # HB_KS_UPDATE_TWO_PASS
    (dict(K=100, d=50, J=20, n=50_000_000), 0, (TWO_PASS, 2, 0, 1, 1, 0, PER_STEP, PER_STEP)),   # n KS >= 2^32
])
def test_kernel_paths_per_shape(shape, kernel_set, expected):
    """The kernels hb_setup picks for a shape on a 132-SM H100 with 20 update blocks (the benchmark's c3 / c4 / c5 and
    one shape past each limit), and the per-call rule of cluster_cpp: the two-pass kernel keeps R-store rounds in a
    32-bit mask, so a 40-round call runs the per-step path, as does every call with the legacy centroid step."""
    L = _lib.lib()
    out = (ctypes.c_int64 * 8)()
    L.hb_debug_kernel_paths(shape["K"], shape["d"], shape["J"], shape["n"], 20, 132, kernel_set, out)
    assert tuple(out) == expected


PIN_SHAPES = {"c3": C3, "c5": dict(K=200, d=100, J=40, n=6_250_000), "K1024_d64": dict(K=1024, d=64, J=20, n=1_000_000),
              "K100_d300": dict(K=100, d=300, J=20, n=1_000_000), "K300_d50": dict(K=300, d=50, J=20, n=1_000_000)}


# shape, HB_KERNEL_SET, hb_debug_kernel_paths (as above), hb_debug_wide_paths (natural-order assignment, plan-order
# cold start, ridge apply, k-means initialisation; numbered as in tests/test_gpu_wide_shapes.py)
@pytest.mark.parametrize("shape, kernel_set, kernel_paths, wide_paths", [
    ("c3", 0, (2, 2, 0, 1, 1, 1, 2, 0), (1, 1, 1, 2)),
    ("c3", 1, (2, 0, 0, 0, 0, 0, 2, 0), (2, 0, 2, 1)),
    ("c3", 2, (0, 2, 0, 1, 1, 0, 0, 0), (1, 0, 1, 2)),
    ("c3", 4, (1, 2, 0, 1, 1, 0, 0, 0), (1, 0, 1, 2)),
    ("c3", 16, (2, 0, 0, 0, 0, 1, 2, 0), (4, 3, 3, 4)),
    ("c3", 17, (2, 0, 0, 0, 0, 1, 2, 0), (4, 3, 3, 4)),
    ("c3", 18, (0, 0, 0, 0, 0, 0, 0, 0), (4, 0, 3, 4)),
    ("c3", 20, (1, 0, 0, 0, 0, 0, 0, 0), (4, 0, 3, 4)),
    ("c5", 0, (2, 0, 1, 1, 1, 1, 2, 0), (2, 2, 1, 2)),
    ("c5", 1, (2, 0, 0, 0, 0, 0, 2, 0), (2, 0, 2, 1)),
    ("c5", 2, (0, 0, 1, 1, 1, 0, 0, 0), (2, 0, 1, 2)),
    ("c5", 4, (1, 0, 1, 1, 1, 0, 0, 0), (2, 0, 1, 2)),
    ("c5", 16, (2, 0, 0, 0, 0, 1, 2, 0), (4, 3, 3, 4)),
    ("c5", 17, (2, 0, 0, 0, 0, 1, 2, 0), (4, 3, 3, 4)),
    ("c5", 18, (0, 0, 0, 0, 0, 0, 0, 0), (4, 0, 3, 4)),
    ("c5", 20, (1, 0, 0, 0, 0, 0, 0, 0), (4, 0, 3, 4)),
    ("K1024_d64", 0, (0, 0, 1, 1, 0, 0, 0, 0), (3, 0, 1, 3)),
    ("K1024_d64", 1, (0, 0, 0, 0, 0, 0, 0, 0), (3, 0, 3, 3)),
    ("K1024_d64", 2, (0, 0, 1, 1, 0, 0, 0, 0), (3, 0, 1, 3)),
    ("K1024_d64", 4, (0, 0, 1, 1, 0, 0, 0, 0), (3, 0, 1, 3)),
    ("K1024_d64", 16, (0, 0, 0, 0, 0, 0, 0, 0), (4, 0, 3, 4)),
    ("K1024_d64", 17, (0, 0, 0, 0, 0, 0, 0, 0), (4, 0, 3, 4)),
    ("K1024_d64", 18, (0, 0, 0, 0, 0, 0, 0, 0), (4, 0, 3, 4)),
    ("K1024_d64", 20, (0, 0, 0, 0, 0, 0, 0, 0), (4, 0, 3, 4)),
    ("K100_d300", 0, (2, 0, 0, 0, 0, 1, 2, 0), (4, 3, 3, 1)),
    ("K100_d300", 1, (2, 0, 0, 0, 0, 1, 2, 0), (4, 3, 3, 1)),
    ("K100_d300", 2, (0, 0, 0, 0, 0, 0, 0, 0), (4, 0, 3, 1)),
    ("K100_d300", 4, (1, 0, 0, 0, 0, 0, 0, 0), (4, 0, 3, 1)),
    ("K100_d300", 16, (2, 0, 0, 0, 0, 1, 2, 0), (4, 3, 3, 4)),
    ("K100_d300", 17, (2, 0, 0, 0, 0, 1, 2, 0), (4, 3, 3, 4)),
    ("K100_d300", 18, (0, 0, 0, 0, 0, 0, 0, 0), (4, 0, 3, 4)),
    ("K100_d300", 20, (1, 0, 0, 0, 0, 0, 0, 0), (4, 0, 3, 4)),
    ("K300_d50", 0, (0, 0, 1, 1, 0, 0, 0, 0), (2, 0, 1, 1)),
    ("K300_d50", 1, (0, 0, 0, 0, 0, 0, 0, 0), (2, 0, 2, 1)),
    ("K300_d50", 2, (0, 0, 1, 1, 0, 0, 0, 0), (2, 0, 1, 1)),
    ("K300_d50", 4, (0, 0, 1, 1, 0, 0, 0, 0), (2, 0, 1, 1)),
    ("K300_d50", 16, (0, 0, 0, 0, 0, 0, 0, 0), (4, 0, 3, 4)),
    ("K300_d50", 17, (0, 0, 0, 0, 0, 0, 0, 0), (4, 0, 3, 4)),
    ("K300_d50", 18, (0, 0, 0, 0, 0, 0, 0, 0), (4, 0, 3, 4)),
    ("K300_d50", 20, (0, 0, 0, 0, 0, 0, 0, 0), (4, 0, 3, 4)),
])
def test_kernel_sets_per_shape(shape, kernel_set, kernel_paths, wide_paths):
    """Both selection hooks under kernel sets 0, 1, 2, 4 and 16 and under HB_KS_WIDE combined with 1, 2 or 4, at the
    benchmark's c3 / c5 and at three more rows of DESIGN §3's kernel-selection table."""
    L = _lib.lib()
    s = PIN_SHAPES[shape]
    kp, wp = (ctypes.c_int64 * 8)(), (ctypes.c_int64 * 4)()
    L.hb_debug_kernel_paths(s["K"], s["d"], s["J"], s["n"], 20, 132, kernel_set, kp)
    L.hb_debug_wide_paths(s["K"], s["d"], s["J"], s["n"], 20, 132, kernel_set, wp)
    assert (tuple(kp), tuple(wp)) == (kernel_paths, wide_paths)


def test_host_widen_pool_matches_numpy():
    """The worker pool of the download path widens float32 to float64 exactly, for
    sizes around its slice boundaries and repeatedly (the pool is persistent)."""
    import ctypes
    L = _lib.lib()
    rng = np.random.default_rng(5)
    nthreads = None
    for n in [0, 1, 7, (1 << 18) - 1, 1 << 18, (1 << 18) + 1, 3 * (1 << 18) + 12345, 5_000_000]:
        src = rng.standard_normal(n).astype(np.float32)
        out = np.full(n, np.nan)
        t = L.hb_debug_widen(out.ctypes.data_as(ctypes.c_void_p), src.ctypes.data_as(ctypes.c_void_p), n, 4)
        nthreads = nthreads or t
        assert t == nthreads and t >= 1
        assert np.array_equal(out, src.astype(np.float64))


def test_bench_workloads_are_well_formed():
    """bench.py's synthetic shards of BASELINE.json configs 3 / 4 / 5: level ids per covariate in range, further
    covariates nested in the first (J = number of donors), shards consistent for any split, setup arguments in the
    global level numbering of R/ui.R:219-231."""
    import bench
    saved = dict(bench.W)
    try:
        for cid, J_expected in (("c3", 20), ("c4", 40), ("c5", 40)):
            bench.W.clear()
            bench.W.update(bench.WORKLOADS[cid])
            B_vec = bench.W["B_vec"]
            Z, lv = bench.synth_shard(30000, 0, 7)
            assert Z.shape == (30000, bench.W["d"]) and lv.shape == (30000, len(B_vec))
            for c, b in enumerate(B_vec):
                assert lv[:, c].min() >= 0 and lv[:, c].max() < b
            assert len(np.unique(lv, axis=0)) == J_expected
            if len(B_vec) > 1:   # every donor belongs to one dataset; a third covariate is a property of the donor
                for donor in range(B_vec[1]):
                    assert len(np.unique(lv[lv[:, 1] == donor, 0])) <= 1
                    if len(B_vec) > 2:
                        assert len(np.unique(lv[lv[:, 1] == donor, 2])) <= 1
            Za, la = bench.synth_shard(10000, 0, 7)
            Zb, lb = bench.synth_shard(10000, 0, 7)
            np.testing.assert_array_equal(Za, Zb)                      # deterministic in (seed, offset)
            kw = bench.setup_kwargs(lv)
            assert kw["phi"].max() < sum(B_vec) and len(kw["theta"]) == sum(B_vec) and kw["K"] == bench.W["K"]
            assert bench.algo_bytes_per_cell_iter(100, 50) == 6224 and bench.algo_bytes_per_cell_iter(200, 100) == 12424
    finally:
        bench.W.clear()
        bench.W.update(saved)


def test_c_host_builds_against_the_header_and_fails_loudly_without_a_device(tmp_path):
    """`include/harmony_b200.h` is plain C99 and a C host (examples/harmonize.c: the reference's harmonize() loop
    on the C ABI alone) links against the in-tree library; without a CUDA device it stops at hb_create."""
    import shutil
    import subprocess
    import torch
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    _lib.lib()   # builds the library if it is missing
    exe = str(tmp_path / "harmonize_demo")
    cmd = ["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-O1", "-I", os.path.join(_lib.ROOT, "include"),
           os.path.join(_lib.ROOT, "examples", "harmonize.c"), "-L", _lib._HERE, "-lharmony_b200",
           "-Wl,-rpath," + _lib._HERE, "-lm", "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    if torch.cuda.is_available():   # with a device it runs the whole loop
        r = subprocess.run([exe, "20000"], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0 and "kernel launches" in r.stdout, (r.returncode, r.stderr[-2000:])
        return
    r = subprocess.run([exe, "1000"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 3, (r.returncode, r.stderr)
    assert "no usable CUDA device" in r.stderr


# names the reference's Rcpp module exposes (src/harmony.cpp:672-709: .field / .method of class `harmony`)
REFERENCE_MODULE_NAMES = """N B K d O E Y Pr_b B_vec alpha W R theta sigma lambda kmeans_rounds objective_kmeans
objective_kmeans_dist objective_kmeans_entropy objective_kmeans_cross objective_harmony max_iter_kmeans getZcorr getZorig
getLambda getR getCentroids check_convergence setup compute_objective init_cluster_cpp cluster_cpp
moe_correct_ridge_cpp""".split()


def test_rcpp_shim_type_checks_against_the_c_abi(tmp_path):
    """r/src/harmony_shim.cpp cannot be built as an R module here (no R / Rcpp); it is at least type-checked against
    include/harmony_b200.h through an API-shaped stand-in for the Rcpp types it uses (tests/stubs/Rcpp.h), linked to
    the in-tree library, its module registration run (same names as the reference's module) and its constructor
    driven to the library's no-device error."""
    import shutil
    import subprocess
    import torch
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    _lib.lib()
    exe = str(tmp_path / "shim_driver")
    root = _lib.ROOT
    cmd = ["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(root, "tests", "stubs"),
           "-I", os.path.join(root, "include"), "-I", os.path.join(root, "r", "src"),
           os.path.join(root, "tests", "stubs", "shim_driver.cpp"), "-L", _lib._HERE, "-lharmony_b200",
           "-Wl,-rpath," + _lib._HERE, "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    exposed = [ln.split()[-1] for ln in r.stdout.splitlines() if ln.startswith(("property", "method"))]
    assert sorted(exposed) == sorted(REFERENCE_MODULE_NAMES)
    if not torch.cuda.is_available():
        assert r.returncode == 3 and "no usable CUDA device" in r.stderr, (r.returncode, r.stderr)
