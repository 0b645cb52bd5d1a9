"""Shapes past the FFMA kernels' shared-memory limits: wide embeddings (d > 120 for the logits, d > 256 for the apply) and
large K (K x d beyond the FFMA assignment and k-means kernels).  They run on the d-chunked logits kernel with softmax
passes, the column-range ridge apply and the k-means initialisation from those logits (hb_debug_wide_paths).

The CPU tests restate today's fit tests of the FFMA kernels in Python and check, over every K in 2..1024 and d in
1..1024, that each stage keeps its kernel where that kernel fits and takes the new one everywhere else.  The GPU tests run
the four stages of stages.py on the rows of WIDE_ROWS, which straddle each new limit, against the fp64 numpy
restatement.
"""
import ctypes

import numpy as np
import pytest

from harmony_b200 import _lib
from helpers import compare, free_port, make_perms, num_sms, rel_l2, run_gpu
from stages import (A_FFMA, A_FUSED, A_LOGITS, A_WIDE, C_FUSED, C_LOGITS, C_NATURAL, C_WIDE, DEFAULT, HB_KS_WIDE,
                    M_FFMA, M_LOGITS, M_TC, M_WIDE, NB, P_COLS, P_FFMA, P_TC, SINGLE_PASS, T, TOL_R, TOL_R1, WIDE_ROWS,
                    _mix64, case_of, f32, fp32_errors, kernel_paths, make_Y0, native_order, numpy_model, planted_R,
                    planted_zy, setup_gpu, stage_s1, stage_s2, stage_s3, stage_s4, wide_paths)

SMEM = 227 * 1024


# ---- today's fit tests (harmony_b200/csrc), restated --------------------------------------------------------------------
def up(x, m):
    return (x + m - 1) // m * m


def assign_ffma_fits(K, d):      # k_assign: Ys, Zs, Ls, sig, part
    KP, DP4 = up(K, 64), up(d, 4)
    return 4 * (DP4 * KP + 64 * DP4 + 64 * (KP + 4) + 9 * KP) <= SMEM


def logits_tc_fits(d):           # k_logits_tc: A hi/lo, B hi/lo, U stage, 2/sigma, norms
    KD = up(d, 8)
    return d <= 128 and 4 * (2 * 128 * KD + 2 * 64 * KD + 128 * 68 + 64 + 4 * 128) + 256 <= SMEM - 256


def apply_ffma_fits(K, d):       # k_ridge_apply: d / 4 x 16 threads, V_q and the R tile
    DP, KP4 = up(d, 4), up(K, 4)
    return DP // 4 * 16 <= 1024 and 4 * (KP4 * DP + 64 * KP4) <= SMEM


def kmeans_ffma_fits(K, d):      # k_kmeans_race / k_kmeans_assign: all centroids
    return 4 * K * d <= 200 * 1024


def test_every_shape_has_a_kernel_and_keeps_the_one_that_fits():
    """K in 2..1024, d in 1..1024 (20 tuples, 1M cells, 132 SMs): the old kernel wherever it fits, the new one elsewhere."""
    L = _lib.lib()      # the hooks themselves, on reused buffers: kernel_paths / wide_paths double this loop's time
    old, new = (ctypes.c_int64 * 8)(), (ctypes.c_int64 * 4)()
    for K in range(2, 1025):
        for d in range(1, 1025):
            L.hb_debug_kernel_paths(K, d, 20, 1000000, NB, 132, 0, old)
            L.hb_debug_wide_paths(K, d, 20, 1000000, NB, 132, 0, new)
            lw = 0 if logits_tc_fits(d) else 1
            fused, logits, apply_tc, km_tc, plan = old[1] > 0, old[2], old[3], old[4], old[5]
            # natural-order assignment
            if fused:
                want = A_FUSED
            elif assign_ffma_fits(K, d):
                want = A_FFMA
            else:
                want = A_LOGITS + lw
            assert new[0] == want, (K, d, tuple(new))
            # plan-order cold start: today's where it exists, the new logits where k_assign does not fit and the call
            # runs single-pass; natural order otherwise
            if old[0] == SINGLE_PASS and not fused and not logits and not assign_ffma_fits(K, d):
                assert plan == 1 and new[1] == C_LOGITS + lw, (K, d, tuple(new))
            else:
                assert new[1] == (C_NATURAL if not plan else C_FUSED if fused else C_LOGITS), (K, d, tuple(new))
            # ridge apply
            assert apply_tc == (d <= 128)
            assert new[2] == (P_TC if apply_tc else P_FFMA if apply_ffma_fits(K, d) else P_COLS), (K, d, tuple(new))
            # k-means initialisation
            want = M_TC if km_tc else M_FFMA if kmeans_ffma_fits(K, d) else M_LOGITS + lw
            assert new[3] == want, (K, d, tuple(new))
            assert min(new[0], new[2], new[3]) > 0


def test_wide_hook_forces_the_new_kernels():
    """HB_KS_WIDE puts every stage on the new kernels, c3 included."""
    assert wide_paths(100, 50, 20, 1000000, 132, kernel_set=HB_KS_WIDE) == (A_WIDE, C_WIDE, P_COLS, M_WIDE)
    assert kernel_paths(100, 50, 20, 1000000, 132)[1:5] == (2, 0, 1, 1)   # unchanged without the bit


# ---- rows -------------------------------------------------------------------------------------------------------------
def _apply_launches(K, d, wide):
    """Launches of the ridge apply: cluster ranges (x column ranges for the column-range kernel)."""
    KS, DS = up(K, 4), up(d, 4)
    fixed = 4 * 2 * (128 if (wide or d > 64) else 64) * 112 + 32

    def passes(DC):
        npass = (K + 111) // 112
        while True:
            Kp = up((K + npass - 1) // npass, 8)
            RS = min(KS, Kp)
            st = 4 * 64 * (RS + DC)
            n = (SMEM - 256 - fixed) // st if fixed < SMEM - 256 else 0
            if (min(n, 4) & ~1) >= 2:
                return len(range(0, K, Kp))
            npass += 1
    if not wide:
        return passes(DS)
    return sum(passes(min(128, DS - c)) for c in range(0, DS, 128))


@pytest.mark.parametrize("name", list(WIDE_ROWS))
def test_wide_rows_reach_their_kernels(name):
    c = case_of(name, 132)
    K, d, _, want, update, ks = WIDE_ROWS[name]
    J = len(c["sizes"])
    assert wide_paths(K, d, J, c["N"], 132, kernel_set=ks) == want
    assert kernel_paths(K, d, J, c["N"], 132)[0] == update


# ---- GPU ----------------------------------------------------------------------------------------------------------------
def _assign_launches(K, wide_logits, plan, normalise):
    lg = 1 + (K + 127) // 128 if wide_logits else (K + 63) // 64
    return lg + 2 + (1 if normalise and not plan else 0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(WIDE_ROWS))
def test_wide_row_stages(name):
    sms = num_sms()
    c = case_of(name, sms)
    K, d, _, want, update, ks = WIDE_ROWS[name]
    N, J = c["N"], len(c["sizes"])
    paths = wide_paths(K, d, J, N, sms, kernel_set=ks)
    assert paths == want
    rng = np.random.default_rng(11)
    Zf = f32(c["Z"])
    Y0 = f32(make_Y0(c["Z"], K, rng))
    # the inputs of S2, S4 and S3, drawn here in the order the stages use them, then the fp32 oracle's R error per stage
    R2, _, _ = planted_R(c, rng)
    R4 = planted_R(c, rng, special=True)
    Zp, Yp = planted_zy(c, rng)
    e32 = fp32_errors(c, DEFAULT, Y0, R2, make_perms(N, T, 5), Zp, Yp, make_perms(N, T, 6))
    bar_R1, bar_R2, bar_R3 = max(TOL_R1, 2 * e32[0]), max(TOL_R, 2 * e32[1]), max(TOL_R, 2 * e32[2])
    print(f"[wide {name}] fp32 oracle max|dR| per stage {e32[0]:.2e} {e32[1]:.2e} {e32[2]:.2e} -> R bars "
          f"{bar_R1:.2e} {bar_R2:.2e} {bar_R3:.2e}")
    ratios = []
    g = setup_gpu(c, kernel_set=ks)
    npy = numpy_model(c, Zf)
    logits = paths[0] in (A_LOGITS, A_WIDE)
    stage_s1(name, g, npy, Y0, "wide", dict(R=bar_R1), ratios,
             assign_launches=_assign_launches(K, paths[0] == A_WIDE, False, False) if logits else None)
    assert stage_s2(name, g, npy, c, rng, tag="wide", bars=dict(R=bar_R2), ratios=ratios, R=R2) == T
    stage_s4(name, g, npy, c, rng, tag="wide", ratios=ratios, R=R4,
             apply_launches=_apply_launches(K, d, paths[2] == P_COLS) if paths[2] != P_FFMA else None)
    if paths[1] == C_WIDE:
        cold = _assign_launches(K, True, True, True)
    elif paths[1] == C_NATURAL and logits:
        cold = _assign_launches(K, paths[0] == A_WIDE, False, True)
    else:
        cold = None
    assert stage_s3(name, g, npy, c, rng, tag="wide", bars=dict(R=bar_R3), ratios=ratios, assign_launches=cold,
                    Zp=Zp, Yp=Yp) == T
    print(f"[wide {name}] largest ratio to a bar: {max(ratios):.2f}")


@pytest.mark.gpu
def test_parity_d300_K100():
    """A whole run at d = 300, K = 100 (50k cells, 3 iterations, injected centroids and orders) meets the parity bars of
    test_gpu_parity.py against the fp32 and fp64 oracles."""
    from harmony_b200 import prepare_inputs
    from helpers import make_Y0 as make_Y0_h, run_oracle, synthetic
    Z, meta = synthetic(50000, 300, [8], n_types=20, seed=41)
    a = prepare_inputs(Z, meta, "cov0", nclust=100, early_stop=False)
    N, T_ = Z.shape[0], a["max_iter_kmeans"]
    n_iter = 3
    Y0 = make_Y0_h(Z, a["K"], 17)
    perms = make_perms(N, n_iter * T_, 23).reshape(n_iter, T_, N)
    o32, _, _ = run_oracle(a, Y0, n_iter, perms=perms)
    o64, _, _ = run_oracle(a, Y0, n_iter, perms=perms, double=True)
    g, iters = run_gpu(a, Y0, n_iter, perms)
    assert iters == n_iter
    compare(g, o32, o64, "d300_K100")


# ---- RunHarmony on a CUDA tensor against the oracles, with the library's native update orders replayed ----------------
def test_native_order_replay_matches_the_library():
    """native_order restates hb_permute_inv exactly (checked through hb_debug_permute, host only)."""
    L = _lib.lib()
    for n, rc in [(50000, 0), (50000, 37), (1000003, 5)]:
        order = native_order(n, 123, rc)
        key = int(_mix64(np.array([123 ^ int(_mix64(np.array([rc + 0x1234567], dtype=np.uint64))[0])],
                                  dtype=np.uint64))[0])
        for p in list(range(50)) + list(range(n - 50, n)):
            assert L.hb_debug_permute(p, n, key, 1) == order[p]
        if n < 100000:
            assert np.array_equal(np.sort(order), np.arange(n))


@pytest.mark.gpu
def test_runharmony_cuda_tensor_d300(monkeypatch):
    """RunHarmony on a CUDA tensor (d = 300, K = 100, 50k cells, seeded native k-means initialisation and update orders,
    10 iterations) meets test_gpu_parity.py's bars against the fp32 and fp64 oracles: the oracles start from the
    centroids the library's initialisation produced and replay its native update orders."""
    import torch
    from harmony_b200 import harmony_options, prepare_inputs, ui
    from helpers import run_oracle, synthetic
    SEED, ITERS = 20261015, 10
    # one cell type per cluster: with 20 types for K = 100 many clusters end up as near-duplicates after 10 iterations,
    # and their exact ties (top-2 gaps <= 3e-6) flip the hard index of ~0.2 % of the cells in any fp32 evaluation (the fp32
    # oracle itself flips 264 of 50k cells there, this path 98; DESIGN.md §4), more than assert_argmax_bounded's 0.05 %
    Z, meta = synthetic(50000, 300, [8], n_types=100, seed=41)
    opts = harmony_options(epsilon_cluster=-np.inf)   # every call runs all its rounds: round i T + t is call i's round t
    seen = {}
    real = ui.harmonize

    def harmonize(obj, it, verbose):
        seen["Y0"] = np.asarray(obj.Y).T.copy()       # the normalised centroids of the native initialisation
        return real(obj, it, verbose)
    monkeypatch.setattr(ui, "harmonize", harmonize)
    Zt = torch.from_numpy(Z).cuda()
    g = ui.RunHarmony(Zt, meta, "cov0", nclust=100, max_iter=ITERS, early_stop=False, options=opts, seed=SEED,
                      return_object=True, verbose=False)
    zt = ui.RunHarmony(Zt, meta, "cov0", nclust=100, max_iter=ITERS, early_stop=False, options=opts, seed=SEED,
                       verbose=False)
    assert zt.is_cuda and zt.dtype == torch.float64 and zt.shape == Zt.shape
    a = prepare_inputs(Z, meta, "cov0", nclust=100, early_stop=False, options=opts)
    N, T_ = Z.shape[0], a["max_iter_kmeans"]
    perms = np.stack([native_order(N, SEED, r) for r in range(ITERS * T_)]).reshape(ITERS, T_, N)
    o32, _, _ = run_oracle(a, seen["Y0"], ITERS, perms=perms)
    o64, _, _ = run_oracle(a, seen["Y0"], ITERS, perms=perms, double=True)
    compare(g, o32, o64, "RunHarmony d300_K100 cuda")
    # the tensor result of the same seeded run is the object's Z_corr up to fp32 atomics
    assert rel_l2(zt.cpu().numpy(), g.getZcorr().T) < 1e-5


# ---- two GPUs: a wide row sharded over the cells ------------------------------------------------------------------------
def _run_sharded(rank, world, port, q):
    import os
    import sys
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
        Z, meta = synthetic(30011, 300, [8], n_types=20, seed=13)   # d = 300, K = 100: d-chunked logits, column ranges
        a = prepare_inputs(Z, meta, "cov0", nclust=100, early_stop=False)
        N, T_ = Z.shape[0], a["max_iter_kmeans"]
        Y0 = make_Y0(Z, a["K"], 5)
        perms = make_perms(N, 2 * T_, 6).reshape(2, T_, N)
        lo, hi = shard_bounds(N, world, rank)
        res = {}
        for name, comm, rows in (("sharded", make_comm(N), slice(lo, hi)), ("single", None, slice(0, N))):
            if name == "single" and rank != 0:
                break
            g = harmony(device=rank, comm=comm) if comm is not None else harmony(device=rank)
            g.setup(a["Z"][rows], a["phi_i"][rows], a["sigma"], a["theta"], a["lambda_"], a["alpha"], T_,
                    a["epsilon_kmeans"], a["epsilon_harmony"], a["K"], a["block_size"], a["B_vec"],
                    a["batch_proportion_cutoff"])
            g.init_cluster_cpp(Y0)
            r = dict(O0=g.O.copy(), E0=g.E.copy())
            for it in range(2):
                assert g.cluster_cpp(perms[it]) == 0
                g.moe_correct_ridge_cpp()
                g.check_convergence(1)
            r.update(lo=lo, hi=hi, Z=g.getZcorr().T.copy(), R=g.R.T.copy(), O=g.O.copy(), E=g.E.copy(), Y=g.Y.copy(),
                     obj=g.objective_kmeans.copy())
            res[name] = r
        dist.barrier()
        q.put((rank, res))
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, "ERR " + traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_two_gpu_wide_row_equals_one_gpu():
    """The wide kernels with sharded cells (the natural-order assignment's O / row-sum all-reduce, the plan-order cold
    start's removal-sum all-reduce, the column-range apply) give the single-GPU result up to fp32 reassociation."""
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    assert wide_paths(100, 300, 8, 15006, torch.cuda.get_device_properties(0).multi_processor_count)[:3] == \
        (A_WIDE, C_WIDE, P_COLS)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_run_sharded, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=600) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    for r in res.values():
        assert not isinstance(r, str), r
    single, s0, s1 = res[0]["single"], res[0]["sharded"], res[1]["sharded"]
    Zs, Rs = np.concatenate([s0["Z"], s1["Z"]]), np.concatenate([s0["R"], s1["R"]])
    relz = np.linalg.norm(Zs - single["Z"]) / np.linalg.norm(single["Z"])
    print(f"[2gpu wide d300_K100] relL2 Z = {relz:.2e}, max|dR| = {np.abs(Rs - single['R']).max():.2e}")
    assert relz < 2e-5
    assert np.abs(Rs - single["R"]).max() < 1e-4
    for f in ("O0", "E0", "O", "E", "Y"):
        np.testing.assert_allclose(s0[f], s1[f], rtol=0, atol=0)            # replicated state identical
        np.testing.assert_allclose(s0[f], single[f], rtol=2e-4, atol=2e-3)
    np.testing.assert_allclose(s0["obj"], single["obj"], rtol=1e-4)
