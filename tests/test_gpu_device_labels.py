"""Batch labels in device memory, and the covariate-tuple index setup builds on the device (tuples.cuh).

The index is checked against a numpy restatement of its definition: keys are the mixed-radix numbers of a cell's
levels (covariate 0 most significant), tuple ids number the distinct keys in ascending order, and cells are stably
sorted by tuple id.  Host labels (hb_setup, and hb_setup_device with a host phi_i) and device labels must all give
exactly that index."""
import ctypes
import os
import sys
import warnings

import numpy as np
import pytest

from harmony_b200 import RunHarmony, prepare_inputs
from helpers import free_port, synthetic

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

D, K = 4, 4


def reference_index(phi, B_vec):
    """numpy restatement: (sort_perm, tuple_levels [J, C], tuple_start [J + 1], Pr_b as fp32)."""
    phi = np.asarray(phi, dtype=np.int64).reshape(len(phi), -1)
    B_vec = np.asarray(B_vec, dtype=np.int64)
    N, C = phi.shape
    base = np.concatenate([[0], np.cumsum(B_vec)[:-1]])
    radix = np.ones(C, dtype=np.uint64)
    for c in range(C - 2, -1, -1):
        radix[c] = radix[c + 1] * np.uint64(B_vec[c + 1])
    key = np.zeros(N, dtype=np.uint64)
    for c in range(C):
        key += (phi[:, c] - base[c]).astype(np.uint64) * radix[c]
    uniq, tuple_of = np.unique(key, return_inverse=True)
    tuple_of = tuple_of.reshape(-1)
    levels = np.empty((len(uniq), C), dtype=np.int64)
    rem = uniq.copy()
    for c in range(C):
        levels[:, c] = base[c] + (rem // radix[c]).astype(np.int64)
        rem = rem % radix[c]
    start = np.concatenate([[0], np.cumsum(np.bincount(tuple_of, minlength=len(uniq)))])
    counts = np.bincount(phi.reshape(-1), minlength=int(B_vec.sum()))
    Pr_b = (counts.astype(np.float32) / np.float32(N)).astype(np.float64)
    return np.argsort(tuple_of, kind="stable"), levels, start, Pr_b


def new_setup(phi, B_vec, Z, **kw):
    from harmony_b200.harmony import harmony
    B = int(np.sum(B_vec))
    g = harmony(device=0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")          # "Too few cells" below 40 cells
        g.setup(Z, phi, np.full(K, 0.1), np.ones(B), None, 0.2, 2, 1e-5, 1e-4, K, 0.05, np.asarray(B_vec), 1e-5, **kw)
    return g


def device_index(g):
    L, n, C = g._L, g._scalar("N_local"), g._scalar("C")
    J = L.hb_debug_tuple_index(g._h, None, None, None)
    assert J > 0
    perm = np.empty(n, np.int32)
    levels = np.empty((J, C), np.int32)
    start = np.empty(J + 1, np.int64)
    P = ctypes.c_void_p
    assert L.hb_debug_tuple_index(g._h, P(perm.ctypes.data), P(levels.ctypes.data), P(start.ctypes.data)) == J
    return perm, levels, start, g.Pr_b


def index_variants(phi, B_vec, seed=0):
    """The index from host labels with a host Z (hb_setup), host labels with a device Z and device labels."""
    N = len(phi)
    Z = np.random.default_rng(seed).standard_normal((N, D))
    Zd = torch.from_numpy(Z).to("cuda", torch.float32)
    phi_d = torch.from_numpy(np.ascontiguousarray(phi)).cuda()
    return {"host": device_index(new_setup(phi, B_vec, Z)),
            "host_phi_device_Z": device_index(new_setup(phi, B_vec, Zd)),
            "device": device_index(new_setup(phi_d, B_vec, Zd))}


def assert_index_equal(got, ref, what):
    for name, a, b in zip(("sort_perm", "tuple_levels", "tuple_start", "Pr_b"), got, ref):
        assert np.array_equal(np.asarray(a, np.float64), np.asarray(b, np.float64)), f"{what}: {name}"


def _random(N, B_vec, seed):
    rng = np.random.default_rng(seed)
    base = np.concatenate([[0], np.cumsum(B_vec)[:-1]])
    return np.stack([base[c] + rng.integers(0, B_vec[c], N) for c in range(len(B_vec))], axis=1)


def _nested(seed):
    rng = np.random.default_rng(seed)
    N = 50_000
    top = rng.integers(0, 5, N)
    sub = top * 3 + rng.integers(0, 3, N)          # each of the 15 sub-levels belongs to one of the 5 top levels
    return np.stack([top, 5 + sub], axis=1), [5, 15]


def _crossed_hash(seed):
    """C = 3, key space 6e6 > 2^22 (hash dictionary), ~5k tuples drawn from a pool."""
    rng = np.random.default_rng(seed)
    B_vec = [300, 200, 100]
    pool = _random(5200, B_vec, seed + 1)
    return pool[rng.integers(0, len(pool), 200_000)], B_vec


def _singletons(seed):
    """Every tuple holds one cell (J = N = 5000: two radix passes)."""
    keys = np.random.default_rng(seed).permutation(5000)
    return np.stack([keys // 50, 100 + keys % 50], axis=1), [100, 50]


def _reversed(seed):
    phi = np.sort(_random(30_000, [40, 7], seed), axis=0)[::-1]
    return np.ascontiguousarray(phi), [40, 7]


ROWS = {
    "c3_shape": lambda s: (_random(1_000_000, [20], s), [20]),
    "nested_C2": _nested,
    "crossed_C3_hash": _crossed_hash,
    "J1": lambda s: (np.zeros((10_000, 1), np.int64), [1]),
    "singletons": _singletons,
    "J300_two_passes": lambda s: (_random(100_000, [300], s), [300]),
    "J70k_three_passes": lambda s: (_random(500_000, [300, 250], s), [300, 250]),   # levels, not tuples, size the ridge
    "N_off_chunk": lambda s: (_random(3 * 2048 + 77, [3, 4], s), [3, 4]),
    "N6": lambda s: (np.array([[0], [1], [1], [0], [1], [0]]), [2]),
    "N39": lambda s: (_random(39, [2, 3], s), [2, 3]),
    "reverse_sorted_rows": _reversed,
}


@pytest.mark.parametrize("row", sorted(ROWS))
def test_index_matches_host_rule(row):
    phi, B_vec = ROWS[row](7)
    ref = reference_index(phi, B_vec)
    J = len(ref[1])
    if row == "J300_two_passes":
        assert 256 < J < 65536
    if row == "J70k_three_passes":
        assert J > 65536
    if row == "crossed_C3_hash":
        assert np.prod(B_vec) > 2 ** 22 and 4000 < J < 6000
    for name, got in index_variants(phi, B_vec).items():
        assert_index_equal(got, ref, f"{row} / {name}")


def test_bad_level_same_message():
    from harmony_b200.harmony import HarmonyError
    phi = _random(20_000, [4, 6], 3)
    phi[900, 0] = 9                  # a later bad level must not be the one reported
    phi[777, 1] = 3                  # level of covariate 0 given as covariate 1's
    phi[777 + 1, 0] = -5
    msgs = []
    Zh = np.zeros((len(phi), D))
    Zd = torch.zeros((len(phi), D), device="cuda")
    for Z, labels in ((Zh, phi), (Zd, phi), (Zd, torch.from_numpy(phi).cuda())):
        with pytest.raises(HarmonyError) as e:
            new_setup(labels, [4, 6], Z)
        msgs.append(str(e.value))
    assert msgs == ["phi row index 3 of cell 777 is not a level of covariate 1"] * 3, msgs


def _distinct(n, B_vec, seed):
    """n cells with distinct tuples (two covariates)."""
    keys = np.random.default_rng(seed).choice(B_vec[0] * B_vec[1], n, replace=False)
    return np.stack([keys // B_vec[1], B_vec[0] + keys % B_vec[1]], axis=1)


@pytest.mark.parametrize("B_vec,n", [([1001, 1001], 1_000_001),        # direct table
                                     ([2048, 2049], 1_000_001),        # hash table, one key over the limit
                                     ([4096, 4096], 3_000_000)])       # hash table past its capacity
def test_too_many_tuples(B_vec, n):
    from harmony_b200.harmony import HarmonyError
    phi = _distinct(n, B_vec, 5)
    Zd = torch.zeros((n, D), device="cuda")
    labels = [torch.from_numpy(phi).cuda()] + ([phi] if n < 2_000_000 else [])
    for lab in labels:
        with pytest.raises(HarmonyError, match="more than 1e6 distinct covariate tuples"):
            new_setup(lab, B_vec, Zd)
    # one tuple fewer is accepted on the same path
    if n == 1_000_001:
        g = new_setup(torch.from_numpy(phi[:-1]).cuda(), B_vec, Zd[:-1])
        assert g._L.hb_debug_tuple_index(g._h, None, None, None) == 1_000_000


def test_device_labels_rejected_by_hb_setup():
    from harmony_b200.harmony import harmony
    N = 1000
    phi = torch.from_numpy(_random(N, [3], 1)).to("cuda", torch.int32).contiguous()
    Z = np.zeros((N, D))
    B_vec, sigma, theta = np.array([3], np.int32), np.full(K, 0.1), np.ones(3)
    g = harmony(device=0)
    P = ctypes.c_void_p
    st = g._L.hb_setup(g._h, P(Z.ctypes.data), D, N, P(phi.data_ptr()), P(B_vec.ctypes.data), 1, P(sigma.ctypes.data),
                       P(theta.ctypes.data), None, 0.2, 2, 1e-5, 1e-4, K, 0.05, 1e-5, 0)
    assert st == 2 and "device memory" in g._L.hb_last_error(g._h).decode()
    assert g.kernel_launches == 0


def test_python_rejections():
    from harmony_b200.harmony import harmony
    Z, meta = synthetic(2000, 8, [3], seed=2)
    Zd = torch.from_numpy(Z).cuda()
    lab = torch.from_numpy(meta["cov0"]).cuda()
    with pytest.raises(ValueError):                     # device labels, host embedding
        prepare_inputs(Z, {"b": lab}, "b")
    with pytest.raises(TypeError):                      # floating-point labels
        prepare_inputs(Zd, {"b": lab.double()}, "b")
    with pytest.raises(TypeError):
        prepare_inputs(Zd, lab.float())
    g = harmony(device=0)
    with pytest.raises(ValueError):                     # device Phi, host Z
        g.setup(Z, lab, np.full(K, 0.1), np.ones(3), None, 0.2, 2, 1e-5, 1e-4, K, 0.05, [3], 1e-5)
    with pytest.raises(TypeError):
        g.setup(Zd, lab.float(), np.full(K, 0.1), np.ones(3), None, 0.2, 2, 1e-5, 1e-4, K, 0.05, [3], 1e-5)
    assert g.kernel_launches == 0
    # a bare CUDA vector is the batch variable, like a bare numpy one
    a, b = prepare_inputs(Zd, lab, nclust=10), prepare_inputs(Z, meta["cov0"], nclust=10)
    assert a["vars_use"] == b["vars_use"] == ["batch_variable"]
    assert torch.is_tensor(a["phi_i"]) and a["phi_i"].dtype == torch.int32 and a["phi_i"].is_cuda
    assert np.array_equal(a["phi_i"].cpu().numpy(), b["phi_i"]) and np.array_equal(a["theta"], b["theta"])
    if torch.cuda.device_count() < 2:
        return
    other = lab.to("cuda:1")
    with pytest.raises(ValueError):
        prepare_inputs(Zd, {"b": other}, "b")
    with pytest.raises(ValueError):
        g.setup(Zd, other, np.full(K, 0.1), np.ones(3), None, 0.2, 2, 1e-5, 1e-4, K, 0.05, [3], 1e-5)
    g2 = harmony(device=0)
    phi1 = other.to(torch.int32).reshape(-1, 1).contiguous()
    B_vec, sigma, theta = np.array([3], np.int32), np.full(K, 0.1), np.ones(3)
    P = ctypes.c_void_p
    st = g2._L.hb_setup_device(g2._h, P(Zd.data_ptr()), 1, 8, None, 8, 2000, P(phi1.data_ptr()), P(B_vec.ctypes.data),
                               1, P(sigma.ctypes.data), P(theta.ctypes.data), None, 0.2, 2, 1e-5, 1e-4, K, 0.05, 1e-5, 0)
    assert st == 2 and "device 1" in g2._L.hb_last_error(g2._h).decode()
    assert g2.kernel_launches == 0


def test_side_stream_ordering():
    """Labels written on a side stream behind a sleep, setup called on that stream without synchronisation."""
    phi, B_vec = _random(200_000, [30, 5], 11), [30, 5]
    ref = reference_index(phi, B_vec)
    src = torch.from_numpy(phi).cuda()
    Zd = torch.from_numpy(np.random.default_rng(1).standard_normal((len(phi), D))).cuda()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        lab = torch.full_like(src, -1)             # every level out of range until the copy lands
        torch.cuda._sleep(50_000_000)
        lab.copy_(src)
        g = new_setup(lab, B_vec, Zd)
    assert_index_equal(device_index(g), ref, "side stream")


def test_runharmony_with_device_labels():
    Z, meta = synthetic(20_000, 20, [6, 12], seed=4)
    flag = (np.arange(20_000) % 3 == 0)
    host_meta = {"b": meta["cov0"] + 100, "s": meta["cov1"].astype(np.int32), "f": flag}
    dev_meta = {"b": torch.from_numpy(host_meta["b"]).cuda(), "s": torch.from_numpy(host_meta["s"]).cuda(),
                "f": torch.from_numpy(flag).cuda()}
    Zd = torch.from_numpy(Z).to("cuda", torch.float32)
    vars_use = ["b", "s", "f"]
    kw = dict(nclust=30, max_iter=4, verbose=False, seed=17)
    a_h, a_d = prepare_inputs(Zd, host_meta, vars_use), prepare_inputs(Zd, dev_meta, vars_use)
    for x, y in zip(a_h["level_names"], a_d["level_names"]):
        assert isinstance(y, np.ndarray) and np.array_equal(x, y)
    assert np.array_equal(a_h["phi_i"], a_d["phi_i"].cpu().numpy())
    assert np.array_equal(a_h["theta"], a_d["theta"]) and np.array_equal(a_h["B_vec"], a_d["B_vec"])
    h1 = RunHarmony(Zd, host_meta, vars_use, **kw).cpu().numpy()
    h2 = RunHarmony(Zd, host_meta, vars_use, **kw).cpu().numpy()
    dv = RunHarmony(Zd, dev_meta, vars_use, **kw).cpu().numpy()
    mixed = RunHarmony(Zd, {"b": dev_meta["b"], "s": host_meta["s"], "f": flag}, vars_use, **kw).cpu().numpy()
    noise = float(np.abs(h1 - h2).max())
    print(f"[device labels] host/host max|dZ| {noise:.2e}; host/device {np.abs(h1 - dv).max():.2e}; "
          f"host/mixed {np.abs(h1 - mixed).max():.2e}")
    assert float(np.abs(h1 - dv).max()) <= 2 * noise + 1e-6
    assert float(np.abs(h1 - mixed).max()) <= 2 * noise + 1e-6


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
        Z, meta = synthetic(30011, 50, [20, 40], n_types=30, seed=11)
        # rank 0 holds no cell of level 0 of cov0: the union index has tuples without local cells
        meta["cov0"][: 15000][meta["cov0"][: 15000] == 0] = 1
        a = prepare_inputs(Z, meta, ["cov0", "cov1"], nclust=100, early_stop=False)
        N, T = Z.shape[0], a["max_iter_kmeans"]
        Y0 = make_Y0(Z, a["K"], 5)
        perms = make_perms(N, 2 * T, 6).reshape(2, T, N)
        lo, hi = shard_bounds(N, world, rank)
        res = {}
        for name in ("host", "device"):
            phi = a["phi_i"][lo:hi]
            if name == "device":
                phi = torch.from_numpy(phi).cuda(rank)
            comm = make_comm(N) if name == "host" else (rank, world, None, N, lo)
            g = harmony(device=rank, comm=comm)
            g.setup(torch.from_numpy(a["Z"][lo:hi]).cuda(rank), phi, a["sigma"], a["theta"], a["lambda_"], a["alpha"],
                    T, a["epsilon_kmeans"], a["epsilon_harmony"], a["K"], a["block_size"], a["B_vec"],
                    a["batch_proportion_cutoff"])
            L, n, C = g._L, g._scalar("N_local"), g._scalar("C")
            J = L.hb_debug_tuple_index(g._h, None, None, None)
            perm, levels, start = np.empty(n, np.int32), np.empty((J, C), np.int32), np.empty(J + 1, np.int64)
            P = ctypes.c_void_p
            L.hb_debug_tuple_index(g._h, P(perm.ctypes.data), P(levels.ctypes.data), P(start.ctypes.data))
            g.init_cluster_cpp(Y0)
            for it in range(2):
                assert g.cluster_cpp(perms[it]) == 0
                g.moe_correct_ridge_cpp()
                g.check_convergence(1)
            res[name] = dict(perm=perm, levels=levels, start=start, Pr_b=g.Pr_b, Z=g.getZcorr().T.copy(),
                             R=g.R.T.copy())
            dist.barrier()
        q.put((rank, res))
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, "ERR " + traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def test_two_gpu_device_label_shards_match_host_shards():
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
        for k in ("perm", "levels", "start", "Pr_b"):
            assert np.array_equal(h[k], dv[k]), (rank, k)
        assert np.array_equal(res[0]["device"]["levels"], res[1]["device"]["levels"])
        assert float(np.abs(dv["Z"] - h["Z"]).max()) < 1e-4
        assert float(np.abs(dv["R"] - h["R"]).max()) < 1e-4
