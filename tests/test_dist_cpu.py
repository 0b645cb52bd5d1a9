"""world_size-2 gloo tests (CPU) of the multi-GPU host logic: shard geometry, communicator-id
broadcast, and that sharding the update order / the diversity statistics reproduces the unsharded
quantities (the identities the library relies on when it all-reduces O, E and the ridge statistics)."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from harmony_b200.dist import broadcast_bytes, make_comm, shard_bounds
from helpers import free_port


def test_shard_bounds():
    b = shard_bounds(10, 3)
    assert b.tolist() == [0, 4, 7, 10]
    assert shard_bounds(1_000_003, 8)[-1] == 1_000_003
    assert all(0 <= x - y <= 1 for x, y in zip(np.diff(shard_bounds(1_000_003, 8))[:-1],
                                              np.diff(shard_bounds(1_000_003, 8))[1:]))
    assert shard_bounds(12, 4, rank=2) == (6, 9)


def _worker(rank, world, port, N, K, B, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        # communicator id plumbing (a fake id source: there is no NCCL/GPU on this box)
        comm = make_comm(N, id_source=lambda: bytes(range(128)))
        assert comm[0] == rank and comm[1] == world and comm[2] == bytes(range(128)) and comm[3] == N
        lo, hi = shard_bounds(N, world, rank)
        assert comm[4] == lo
        # sharded block membership from ONE global update order == unsharded (harmony.cpp:279-300)
        rng = np.random.default_rng(0)
        order = rng.permutation(N)
        lev = rng.integers(0, B, N)
        R = rng.random((N, K)).astype(np.float32)
        nb, cpb = 20, int(np.float32(N) * np.float32(0.05))
        pos = np.empty(N, dtype=np.int64)
        pos[order] = np.arange(N)
        blk = np.minimum(pos // cpb, nb - 1)
        # per-rank partial O[b, k] of block 3, all-reduced
        sel = (blk[lo:hi] == 3)
        part = np.zeros((B, K), dtype=np.float64)
        np.add.at(part, lev[lo:hi][sel], R[lo:hi][sel].astype(np.float64))
        t = torch.from_numpy(part)
        dist.all_reduce(t)
        full = np.zeros((B, K), dtype=np.float64)
        gs = blk == 3
        np.add.at(full, lev[gs], R[gs].astype(np.float64))
        assert np.allclose(t.numpy(), full, rtol=1e-12)
        # level counts (N_b) summed over ranks
        cnt = torch.from_numpy(np.bincount(lev[lo:hi], minlength=B).astype(np.int64))
        dist.all_reduce(cnt)
        assert cnt.numpy().tolist() == np.bincount(lev, minlength=B).tolist()
        payload = broadcast_bytes(b"harmony" + b"\0" * 121, 128, 0)
        assert payload.startswith(b"harmony")
        out.put((rank, "ok"))
    except Exception as e:  # pragma: no cover
        out.put((rank, repr(e)))
    finally:
        dist.destroy_process_group()


def test_two_rank_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, 4001, 7, 3, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res
