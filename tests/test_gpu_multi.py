"""2-GPU equivalence (gpu-marked; skipped with < 2 devices): the cell-sharded run with NCCL
all-reduces equals the single-GPU run on the same inputs up to fp32 reassociation."""
import os

import numpy as np
import pytest

from helpers import free_port

pytestmark = pytest.mark.gpu


def _run(rank, world, port, case, q):
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
        if case == "1cov":
            Z, meta = synthetic(30011, 50, [20], n_types=30, seed=11)
            a = prepare_inputs(Z, meta, "cov0", nclust=100, early_stop=False)
        else:
            Z, meta = synthetic(20007, 24, [4, 12, 3], seed=12)
            a = prepare_inputs(Z, meta, ["cov0", "cov1", "cov2"], nclust=40, early_stop=False)
        N, T = Z.shape[0], a["max_iter_kmeans"]
        Y0 = make_Y0(Z, a["K"], 5)
        perms = make_perms(N, 2 * T, 6).reshape(2, T, N)
        lo, hi = shard_bounds(N, world, rank)
        g = harmony(device=rank, comm=make_comm(N))
        g.setup(a["Z"][lo:hi], a["phi_i"][lo:hi], a["sigma"], a["theta"], a["lambda_"], a["alpha"], T,
                a["epsilon_kmeans"], a["epsilon_harmony"], a["K"], a["block_size"], a["B_vec"],
                a["batch_proportion_cutoff"])
        g.init_cluster_cpp(Y0)
        for it in range(2):
            assert g.cluster_cpp(perms[it]) == 0
            g.moe_correct_ridge_cpp()
            g.check_convergence(1)
        res = dict(lo=lo, hi=hi, Z=g.getZcorr().T.copy(), R=g.R.T.copy(), O=g.O.copy(), E=g.E.copy(), Y=g.Y.copy(),
                   obj=g.objective_kmeans.copy())
        if rank == 0:  # single-GPU run of the same problem on this device
            s = harmony(device=rank)
            s.setup(a["Z"], a["phi_i"], a["sigma"], a["theta"], a["lambda_"], a["alpha"], T, a["epsilon_kmeans"],
                    a["epsilon_harmony"], a["K"], a["block_size"], a["B_vec"], a["batch_proportion_cutoff"])
            s.init_cluster_cpp(Y0)
            for it in range(2):
                s.cluster_cpp(perms[it])
                s.moe_correct_ridge_cpp()
                s.check_convergence(1)
            res["single"] = dict(Z=s.getZcorr().T.copy(), R=s.R.T.copy(), O=s.O.copy(), E=s.E.copy(), Y=s.Y.copy(),
                                 obj=s.objective_kmeans.copy())
        dist.barrier()
        q.put((rank, res))
    except Exception as e:  # pragma: no cover
        import traceback
        q.put((rank, "ERR " + traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("case", ["1cov", "3cov"])
def test_two_gpu_equals_one_gpu(case):
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_run, args=(r, 2, port, case, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=600) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    for r in res.values():
        assert not isinstance(r, str), r
    single = res[0]["single"]
    Zs = np.concatenate([res[0]["Z"], res[1]["Z"]])
    Rs = np.concatenate([res[0]["R"], res[1]["R"]])
    relz = np.linalg.norm(Zs - single["Z"]) / np.linalg.norm(single["Z"])
    print(f"[2gpu {case}] relL2 Z = {relz:.2e}, max|dR| = {np.abs(Rs - single['R']).max():.2e}")
    assert relz < 2e-5
    assert np.abs(Rs - single["R"]).max() < 1e-4
    for f in ("O", "E", "Y"):
        np.testing.assert_allclose(res[0][f], res[1][f], rtol=0, atol=0)          # replicated state identical
        np.testing.assert_allclose(res[0][f], single[f], rtol=2e-4, atol=2e-3)
    np.testing.assert_allclose(res[0]["obj"], single["obj"], rtol=1e-4)
