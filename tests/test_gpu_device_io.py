"""Embeddings in device memory: hb_setup_device / hb_get_field_device through harmony.setup(tensor), get_tensor and
RunHarmony(tensor).

The per-cell conversions are exact (fp32 -> fp32, fp32 <-> fp64 widening) or the same rounding as the host path
(fp64 -> fp32), so a handle set up from a CUDA tensor holds the same bits as one set up from the numpy array, and
get_tensor returns the bits of getZcorr() / getZorig() / getR()."""
import ctypes
import os
import sys

import numpy as np
import pytest

from harmony_b200 import RunHarmony, prepare_inputs
from helpers import free_port, gpu_setup, make_perms, make_Y0, rel_l2, synthetic

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

HB_Z_CORR, HB_Z_ORIG, HB_R, HB_Y = 0, 1, 2, 3
HB_FLOAT32, HB_FLOAT64 = 0, 1


def iterate(g, Y0, perms):
    g.init_cluster_cpp(Y0)
    for p in perms:
        assert g.cluster_cpp(p) == 0
        g.moe_correct_ridge_cpp()
        g.check_convergence(1)


def raw_setup(g, a, ptr, dtype, ld, stream=None, host=False, d=None, N=None, C=None, K=None, phi_ptr=None):
    """hb_setup_device through the ABI with an arbitrary pointer (only ever one the library must refuse), or hb_setup
    on the host array a["Z"] when `host`.  d, N, C, K and phi_ptr replace what `a` gives."""
    phi = np.ascontiguousarray(a["phi_i"], dtype=np.int32)
    B_vec = np.ascontiguousarray(a["B_vec"], dtype=np.int32)
    sigma = np.ascontiguousarray(a["sigma"], dtype=np.float64)
    theta = np.ascontiguousarray(a["theta"], dtype=np.float64)
    P = ctypes.c_void_p
    rest = (a["Z"].shape[1] if d is None else d, phi.shape[0] if N is None else N,
            P(phi.ctypes.data if phi_ptr is None else phi_ptr), P(B_vec.ctypes.data), len(B_vec) if C is None else C,
            P(sigma.ctypes.data), P(theta.ctypes.data), None, a["alpha"], a["max_iter_kmeans"], a["epsilon_kmeans"],
            a["epsilon_harmony"], a["K"] if K is None else K, a["block_size"], a["batch_proportion_cutoff"], 0)
    if host:
        Z = np.ascontiguousarray(a["Z"], dtype=np.float64)
        return g._L.hb_setup(g._h, P(Z.ctypes.data), *rest)
    return g._L.hb_setup_device(g._h, P(ptr), dtype, ld, P(stream), *rest)


@pytest.fixture(scope="module")
def small():
    Z, meta = synthetic(5000, 50, [4], seed=21)
    return prepare_inputs(Z, meta, "cov0", nclust=40, early_stop=False)


@pytest.fixture(scope="module")
def c3():
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from bench import synth_shard
    Z, b = synth_shard(1_000_000, 0, 123, d=50, B_vec=[20])
    return prepare_inputs(Z, {"batch": b[:, 0]}, "batch", nclust=100, early_stop=False)


@pytest.mark.parametrize("size", ["small", "c3"])
def test_setup_from_tensor_is_bit_identical(size, request):
    a = request.getfixturevalue(size)
    Z = a["Z"]
    host = gpu_setup(a, Z, device=0)
    dev = gpu_setup(a, torch.from_numpy(Z).cuda(), device=0)
    assert np.array_equal(dev.getZorig(), host.getZorig())
    assert np.array_equal(dev.getZcorr(), host.getZcorr())
    Z32 = Z.astype(np.float32)
    g32 = gpu_setup(a, torch.from_numpy(Z32).cuda(), device=0)
    assert np.array_equal(g32.getZorig().T, Z32.astype(np.float64))


def test_get_tensor_matches_host_getters(small):
    a = small
    N, T = a["Z"].shape[0], a["max_iter_kmeans"]
    g = gpu_setup(a, a["Z"], device=0)

    def check():
        for name, host in (("Z_corr", g.getZcorr), ("Z_orig", g.getZorig), ("R", g.getR)):
            t64, t32 = g.get_tensor(name, torch.float64), g.get_tensor(name)
            ref = host().T
            assert t64.dtype == torch.float64 and t32.dtype == torch.float32 and t64.shape == ref.shape
            assert t64.device == torch.device("cuda", 0)
            assert np.array_equal(t64.cpu().numpy(), ref), name
            assert np.array_equal(t32.cpu().numpy(), ref.astype(np.float32)), name

    check()
    iterate(g, make_Y0(a["Z"], a["K"], 1), make_perms(N, 2 * T, 2).reshape(2, T, N))
    # the device getter runs first here, so it is the one that applies the pending normalisation of Z_corr
    first = g.get_tensor("Z_corr", torch.float64).cpu().numpy()
    assert np.array_equal(first, g.getZcorr().T)
    check()


def test_strided_and_transposed_tensors(small):
    a = small
    Z = a["Z"]
    N, d = Z.shape
    ref = gpu_setup(a, Z, device=0).getZorig()
    wide = torch.zeros((N, d + 7), dtype=torch.float64, device="cuda")
    wide[:, :d] = torch.from_numpy(Z).cuda()
    view = wide[:, :d]                                   # row stride d + 7
    assert view.stride() == (d + 7, 1)
    assert np.array_equal(gpu_setup(a, view, device=0).getZorig(), ref)
    Zt = torch.from_numpy(np.ascontiguousarray(Z.T)).cuda()   # d x N, cells as columns
    assert np.array_equal(gpu_setup(a, Zt, device=0).getZorig(), ref)
    dxn = torch.from_numpy(Z).cuda().T                      # d x N view of N x d memory
    assert np.array_equal(gpu_setup(a, dxn, device=0).getZorig(), ref)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_unaligned_tensor_and_output(small, dtype):
    """A view one element past an allocation is only element-aligned: the copies take their scalar path."""
    a = small
    Z = a["Z"]
    N, d = Z.shape
    npdt = np.float32 if dtype == torch.float32 else np.float64
    buf = torch.empty(N * d + 1, dtype=dtype, device="cuda")
    view = buf[1:].view(N, d)
    view.copy_(torch.from_numpy(Z.astype(npdt)))
    assert view.data_ptr() % 16 != 0
    g = gpu_setup(a, view, device=0)
    aligned = gpu_setup(a, torch.from_numpy(Z.astype(npdt)).cuda(), device=0)
    assert np.array_equal(g.getZorig(), aligned.getZorig())
    assert np.array_equal(g.getZcorr(), aligned.getZcorr())
    # output one element off and with row stride d + 1: the extra column must stay untouched
    out = torch.full((N * (d + 1) + 1,), -7.0, dtype=dtype, device="cuda")
    st = g._L.hb_get_field_device(g._h, HB_Z_ORIG, ctypes.c_void_p(out.data_ptr() + out.element_size()),
                                  HB_FLOAT32 if dtype == torch.float32 else HB_FLOAT64, d + 1,
                                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert st == 0
    rows = out[1:].view(N, d + 1).cpu().numpy()
    assert np.array_equal(rows[:, :d].astype(np.float64), g.getZorig().T)
    assert np.all(rows[:, d] == -7.0) and out[0].item() == -7.0


def test_whole_runs_match_host_runs(small):
    a = small
    Z = a["Z"]
    N, T = Z.shape[0], a["max_iter_kmeans"]
    Y0 = make_Y0(Z, a["K"], 3)
    perms = make_perms(N, 2 * T, 4).reshape(2, T, N)

    def run(Zin):
        g = gpu_setup(a, Zin, device=0)
        iterate(g, Y0, perms)
        return g.getZcorr(), g.getR()

    h1, h2, dv = run(Z), run(Z), run(torch.from_numpy(Z).cuda())

    def dev(x, y):
        return float(np.abs(x[0] - y[0]).max()), float(np.abs(x[1] - y[1]).max())

    aa, ab = dev(h1, h2), dev(h1, dv)
    print(f"[device io] host/host max|dZ| {aa[0]:.2e} max|dR| {aa[1]:.2e}; host/device {ab[0]:.2e} {ab[1]:.2e}")
    for x, y in zip(ab, aa):
        assert x <= 2 * y + 1e-6, (ab, aa)


def test_runharmony_with_tensor():
    Z, meta = synthetic(5000, 20, [4], seed=9)
    ref = RunHarmony(Z, meta, "cov0", nclust=20, max_iter=3, verbose=False, seed=11)
    for dtype in (torch.float64, torch.float32):
        X = torch.from_numpy(Z).to("cuda", dtype)
        out = RunHarmony(X, meta, "cov0", nclust=20, max_iter=3, verbose=False, seed=11)
        assert isinstance(out, torch.Tensor) and out.dtype == dtype and out.device == X.device
        assert tuple(out.shape) == Z.shape
        assert rel_l2(out.double().cpu().numpy(), ref) < 1e-5
        # cells as columns: the reference's orientation rule, without leaving the device
        out_t = RunHarmony(X.T, meta, "cov0", nclust=20, max_iter=3, verbose=False, seed=11)
        assert tuple(out_t.shape) == Z.shape and rel_l2(out_t.double().cpu().numpy(), ref) < 1e-5
    obj = RunHarmony(torch.from_numpy(Z).cuda(), meta, "cov0", nclust=20, max_iter=1, verbose=False, seed=1,
                     return_object=True)
    assert obj.getZcorr().shape == (20, 5000)
    with pytest.raises(ValueError):
        RunHarmony(torch.from_numpy(Z).cuda(), meta, "cov0", nclust=20, verbose=False, device=1)


def test_side_stream_ordering(small):
    """Input written on a side stream and read by setup, result read on that stream: no explicit synchronisation."""
    a = small
    Z = a["Z"]
    ref = gpu_setup(a, Z, device=0)
    src = torch.from_numpy(Z).cuda()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        Zd = torch.empty_like(src)
        torch.cuda._sleep(50_000_000)      # keeps the stream busy well past the enqueue of setup's copy
        Zd.copy_(src)
        g = gpu_setup(a, Zd, device=0)
        assert np.array_equal(g.getZorig(), ref.getZorig())
        torch.cuda._sleep(50_000_000)      # the getter's copy must wait for this
        out = g.get_tensor("Z_orig", torch.float64)
        back = (out * 1.0).cpu()           # queued on s after the getter
    assert np.array_equal(back.numpy(), ref.getZorig().T)


def test_rejected_before_any_launch(small):
    from harmony_b200.harmony import HarmonyError, harmony
    a = small
    Z = a["Z"]
    N, d = Z.shape
    g = harmony(device=0)
    pageable = np.ascontiguousarray(Z)
    pinned = torch.from_numpy(Z).pin_memory()
    Zd = torch.from_numpy(Z).cuda()
    for ptr, dtype, ld, what in ((pageable.ctypes.data, HB_FLOAT64, d, "not device"),
                                 (pinned.data_ptr(), HB_FLOAT64, d, "not device"),
                                 (0, HB_FLOAT64, d, "null"),
                                 (Zd.data_ptr(), HB_FLOAT64, d - 1, "row stride"),
                                 (Zd.data_ptr(), 7, d, "dtype")):
        assert raw_setup(g, a, ptr, dtype, ld) == 2
        assert what in g._L.hb_last_error(g._h).decode()
    # the dimension checks of both entry points, and device labels given to the host one
    for host in (False, True):
        for bad in (dict(d=0), dict(N=0), dict(C=0), dict(K=0), dict(K=1025)):
            assert raw_setup(g, a, Zd.data_ptr(), HB_FLOAT64, d, host=host, **bad) == 2, (host, bad)
    phi_d = torch.from_numpy(np.ascontiguousarray(a["phi_i"], dtype=np.int32)).cuda()
    assert raw_setup(g, a, None, HB_FLOAT64, d, host=True, phi_ptr=phi_d.data_ptr()) == 2
    assert "hb_setup_device" in g._L.hb_last_error(g._h).decode()
    assert g.kernel_launches == 0
    with pytest.raises(TypeError):
        gpu_setup(a, Zd.half(), device=0)
    g = gpu_setup(a, Zd, device=0)
    n0 = g.kernel_launches
    for host in (False, True):   # a second setup
        assert raw_setup(g, a, Zd.data_ptr(), HB_FLOAT64, d, host=host) == 3, host
    out = torch.empty((N, d), dtype=torch.float64, device="cuda")
    P, s = ctypes.c_void_p, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for field, ptr, dtype, ld in ((HB_Z_CORR, pageable.ctypes.data, HB_FLOAT64, d),
                                  (HB_Z_CORR, pinned.data_ptr(), HB_FLOAT64, d),
                                  (HB_Z_CORR, out.data_ptr(), HB_FLOAT64, d - 1),
                                  (HB_Z_CORR, out.data_ptr(), 5, d),
                                  (HB_Y, out.data_ptr(), HB_FLOAT64, d),
                                  (99, out.data_ptr(), HB_FLOAT64, d)):
        assert g._L.hb_get_field_device(g._h, field, P(ptr), dtype, ld, s) == 2
    assert g.kernel_launches == n0
    with pytest.raises(ValueError):
        g.get_tensor("Y")
    with pytest.raises(TypeError):
        g.get_tensor("R", torch.float16)
    with pytest.raises(HarmonyError):
        g._check(g._L.hb_get_field_device(g._h, HB_R, P(out.data_ptr()), HB_FLOAT64, 1, s))
    if torch.cuda.device_count() < 2:
        return
    other = torch.from_numpy(Z).to("cuda:1")
    with pytest.raises(ValueError):
        gpu_setup(a, other, device=0)
    g2 = harmony(device=0)
    assert raw_setup(g2, a, other.data_ptr(), HB_FLOAT64, d) == 2
    assert "device 1" in g2._L.hb_last_error(g2._h).decode()
    assert g2.kernel_launches == 0


def _shard_run(rank, world, port, q):
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import torch
    import torch.distributed as dist
    from harmony_b200 import prepare_inputs
    from harmony_b200.dist import make_comm, shard_bounds
    from harmony_b200.harmony import harmony
    from helpers import make_perms, make_Y0, synthetic
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        Z, meta = synthetic(30011, 50, [20], n_types=30, seed=11)
        a = prepare_inputs(Z, meta, "cov0", nclust=100, early_stop=False)
        N, T = Z.shape[0], a["max_iter_kmeans"]
        Y0 = make_Y0(Z, a["K"], 5)
        perms = make_perms(N, 2 * T, 6).reshape(2, T, N)
        lo, hi = shard_bounds(N, world, rank)
        res = {}
        for name, Zs in (("host", a["Z"][lo:hi]), ("device", torch.from_numpy(a["Z"][lo:hi]).cuda(rank))):
            comm = make_comm(N) if name == "host" else (rank, world, None, N, lo)
            g = harmony(device=rank, comm=comm)
            g.setup(Zs, a["phi_i"][lo:hi], a["sigma"], a["theta"], a["lambda_"], a["alpha"], T, a["epsilon_kmeans"],
                    a["epsilon_harmony"], a["K"], a["block_size"], a["B_vec"], a["batch_proportion_cutoff"])
            Zo = g.getZorig().copy()
            g.init_cluster_cpp(Y0)
            for it in range(2):
                assert g.cluster_cpp(perms[it]) == 0
                g.moe_correct_ridge_cpp()
                g.check_convergence(1)
            res[name] = dict(Zo=Zo, Z=g.getZcorr().T.copy(), R=g.R.T.copy(),
                             Zt=g.get_tensor("Z_corr", torch.float64).cpu().numpy())
            dist.barrier()
        q.put((rank, res))
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, "ERR " + traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def test_two_gpu_device_shards_match_host_shards():
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_shard_run, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=600) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    for r in res.values():
        assert not isinstance(r, str), r
    for rank, r in res.items():
        h, dv = r["host"], r["device"]
        assert np.array_equal(h["Zo"], dv["Zo"])
        assert np.array_equal(dv["Zt"], dv["Z"])
        print(f"[2gpu device io] rank {rank}: relL2 Z {rel_l2(dv['Z'], h['Z']):.2e}, "
              f"max|dR| {np.abs(dv['R'] - h['R']).max():.2e}")
        assert rel_l2(dv["Z"], h["Z"]) < 2e-5
        assert np.abs(dv["R"] - h["R"]).max() < 1e-4
