#!/usr/bin/env python
"""bench_device_io.py — end-to-end cost of getting an embedding into Harmony and the corrected one back out.

    python bench_device_io.py [--config c3|c5] [--reps R] [--iters I]

Four ways in and out, alternated within one run on the same synthetic shard (bench.py's generator and settings):
  host      pinned host fp64 Z -> setup, getZcorr() -> host fp64 (bench.py's `e2e` leg)
  dev32     CUDA fp32 tensor   -> setup, get_tensor("Z_corr")           -> CUDA fp32 tensor
  dev64     CUDA fp64 tensor   -> setup, get_tensor("Z_corr", float64)  -> CUDA fp64 tensor
  dev32lab  dev32 with the batch labels (phi_i) in a CUDA int32 tensor as well
The other modes pass the labels as a host numpy array.
Every run is split into phases with a device synchronise around each: setup (object creation included), the native
k-means initialisation, I Harmony iterations and the getter.  The library's "upload" / "download" region times (CUDA
events around the row copies, host transfers included on the host path) are reported with the rate over the bytes the
copy kernels must move (source + destination rows + the row map), and so is the "tuple_index" region: setup's
covariate-tuple index, the upload of host labels included.  One more run of `host`, `dev32` and `dev32lab` with
HB_TRACE_HOST=1 prints the library's own phase laps to stderr.  Prints one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (synth_shard, setup_kwargs and the workloads)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20)
        return out.stdout.strip().splitlines()[0] if out.returncode == 0 else None
    except Exception:
        return None


def run(mode, Z, Zin, kw, K, iters, torch, phi=None):
    from harmony_b200.harmony import harmony
    sync = torch.cuda.synchronize
    ph = {}
    sync()
    t = time.perf_counter()
    g = harmony(device=0)
    g.enable_timing(True)          # only the setup and getter regions are timed: the loop runs without it
    g.setup(Zin, kw["phi"] if phi is None else phi, kw["sigma"], kw["theta"], None, kw["alpha"], bench.T, 1e-3, -np.inf, K, 0.05, kw["B_vec"],
            kw["cutoff"])
    g.enable_timing(False)
    g.set_seed(1234)
    sync()
    ph["setup"] = time.perf_counter() - t
    t = time.perf_counter()
    g.init_cluster_cpp()
    g.synchronize()
    ph["init"] = time.perf_counter() - t
    t = time.perf_counter()
    for _ in range(iters):
        assert g.cluster_cpp() == 0
        g.moe_correct_ridge_cpp()
        g.check_convergence(1)
    g.synchronize()
    ph["iterations"] = time.perf_counter() - t
    g.enable_timing(True)
    t = time.perf_counter()
    if mode == "host":
        out = g.getZcorr()
    else:
        out = g.get_tensor("Z_corr", torch.float32 if mode == "dev32" else torch.float64)
    sync()
    ph["getter"] = time.perf_counter() - t
    g.enable_timing(False)
    ph["total"] = sum(ph.values())
    reg = {r: g.region_time(r)[0] for r in ("upload", "download", "tuple_index")}
    assert out.shape[0] in (Z.shape[0], Z.shape[1])
    del g
    return {k: v * 1e3 for k, v in ph.items()}, reg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="c3", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_device_io.py needs a CUDA device")
    torch.cuda.set_device(0)
    bench.W.clear()
    bench.W.update(bench.WORKLOADS[args.config])
    n, d, K = bench.W["cells_per_gpu"], bench.W["d"], bench.W["K"]
    Z, b = bench.synth_shard(n, 0, 20260922 + int(args.config[1:]))
    kw = bench.setup_kwargs(b)
    inputs = {"host": torch.from_numpy(Z).pin_memory().numpy(),
              "dev32": torch.from_numpy(Z).to("cuda", torch.float32),
              "dev64": torch.from_numpy(Z).cuda()}
    inputs["dev32lab"] = inputs["dev32"]
    labels = {"dev32lab": torch.from_numpy(kw["phi"]).to("cuda", torch.int32)}
    el = {"host": 8, "dev32": 4, "dev64": 8, "dev32lab": 4}
    # bytes the copy kernels move: caller rows + the fp32 device rows + the 4-byte row map (host path: its staging rows)
    moved = {m: n * d * (el[m] + 4) + 4 * n for m in el}
    moved_dl = {"host": n * d * (4 + 4) + 4 * n, "dev32": n * d * 8 + 4 * n, "dev64": n * d * 12 + 4 * n,
                "dev32lab": n * d * 8 + 4 * n}
    # warm-up on a small shard: module loading and first-touch allocations stay out of the timed runs
    zs, bs = bench.synth_shard(20000, 0, 1)
    kws = bench.setup_kwargs(bs)
    for m in el:
        zin = zs if m == "host" else torch.from_numpy(zs).to("cuda", torch.float64 if m == "dev64" else torch.float32)
        run(m, zs, zin, kws, K, 1, torch, torch.from_numpy(kws["phi"]).cuda() if m in labels else None)
    res = {m: [] for m in el}
    for _ in range(args.reps):
        for m in el:
            res[m].append(run(m, Z, inputs[m], kw, K, args.iters, torch, labels.get(m)))
    summary = {}
    for m, rows in res.items():
        med = {k: float(np.median([r[0][k] for r in rows])) for k in rows[0][0]}
        up = float(np.median([r[1]["upload"] for r in rows]))
        dn = float(np.median([r[1]["download"] for r in rows]))
        ti = float(np.median([r[1]["tuple_index"] for r in rows]))
        summary[m] = {"ms_median": {k: round(v, 3) for k, v in med.items()},
                      "ms_all": {k: [round(r[0][k], 3) for r in rows] for k in rows[0][0]},
                      "upload_ms": round(up, 4), "upload_GBps": round(moved[m] / (up * 1e-3) / 1e9, 1) if up else None,
                      "download_ms": round(dn, 4), "tuple_index_ms": round(ti, 4),
                      "download_GBps": round(moved_dl[m] / (dn * 1e-3) / 1e9, 1) if dn else None,
                      "upload_kernel_bytes": moved[m], "download_kernel_bytes": moved_dl[m]}
    os.environ["HB_TRACE_HOST"] = "1"
    for m in ("host", "dev32", "dev32lab"):
        print(f"--- HB_TRACE_HOST laps, {m} ---", file=sys.stderr, flush=True)
        run(m, Z, inputs[m], kw, K, args.iters, torch, labels.get(m))
    del os.environ["HB_TRACE_HOST"]
    print(json.dumps({"config": args.config, "cells": n, "d": d, "K": K, "iterations": args.iters, "reps": args.reps,
                      "gpu": gpu_info(), "modes": summary}), flush=True)


if __name__ == "__main__":
    main()
