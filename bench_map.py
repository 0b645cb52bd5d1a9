#!/usr/bin/env python
"""bench_map.py — mapping new cells onto a finished integration, against rerunning Harmony on reference + query.

    python bench_map.py [--config c3|c5] [--reps R] [--no-rerun]

1. Integrates a reference shaped like bench.py's workload (c3: 1M cells x 50 PCs, K = 100, 20 batches; c5: 6.25M x 100,
   K = 200, 3 covariates) with 10 Harmony iterations and times hb_reference, the compression of that integration.
2. Maps queries of 1M and 100k cells, from the same generator with 4 query batches of planted shifts, from host fp64
   arrays and from CUDA fp32 tensors.  Per query: hb_map_setup, hb_map and the getter (wall-clock, synchronised), and
   hb_map's region split (CUDA events, in separate runs).  For each region, the fewest bytes per cell the unfused pass
   must move (from the shapes) and the achieved rate against the H100's 3.35 TB/s.
3. Times what users run today instead: RunHarmony on reference + 1M-cell query (10 iterations, host arrays).
Prints one JSON line with the card and its power limit.
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

import bench  # noqa: E402  (synth_shard, setup_kwargs, host_Y0 and the workloads)

HBM_TBPS = 3.35
ITERS = 10
QUERY_BATCHES = 4


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20)
        return out.stdout.strip().splitlines()[0] if out.returncode == 0 else None
    except Exception:
        return None


def min_bytes_per_cell(K, d):
    """fp32 bytes per query cell each region must move at least: the assignment reads z and writes R, the statistics
    read R and z, the apply reads R and z and writes z'."""
    r = {"assign": 4 * (d + K), "ridge_stats": 4 * (d + K), "ridge_apply": 4 * (2 * d + K)}
    r["total"] = sum(r.values())
    return r


def integrate(Z, kw, K):
    from harmony_b200.harmony import harmony
    g = harmony(device=0)
    g.setup(Z, kw["phi"], kw["sigma"], kw["theta"], None, kw["alpha"], bench.T, kw["epsilon_kmeans"], -np.inf, K,
            kw["block_size"], kw["B_vec"], kw["cutoff"])
    g.set_seed(1234)
    g.init_cluster_cpp(bench.host_Y0(Z, K, 7))
    for _ in range(ITERS):
        assert g.cluster_cpp() == 0
        g.moe_correct_ridge_cpp()
        g.check_convergence(1)
    g.synchronize()
    return g


def make_query(n, cell_offset, seed):
    """Cells of the reference's generator (other cells) with QUERY_BATCHES batches, each shifted by its own vector."""
    Z, _ = bench.synth_shard(n, cell_offset, seed)
    r = np.random.default_rng([seed, 77])
    lv = r.integers(0, QUERY_BATCHES, n).astype(np.int32)
    d = Z.shape[1]
    Z += (r.standard_normal((QUERY_BATCHES, d)) * 2.0 * (10.0 / np.sqrt(1.0 + np.arange(d))))[lv]
    return Z, lv


def map_once(Zin, lv, ref, torch, timing):
    from harmony_b200.harmony import harmony
    sync = torch.cuda.synchronize
    ph = {}
    sync()
    t = time.perf_counter()
    g = harmony(device=0)
    g.enable_timing(timing)
    g.map_setup(Zin, lv, [QUERY_BATCHES], 1.0, ref)
    sync()
    ph["setup"] = time.perf_counter() - t
    t = time.perf_counter()
    g.map()
    g.synchronize()
    ph["map"] = time.perf_counter() - t
    t = time.perf_counter()
    out = g.getZcorr() if isinstance(Zin, np.ndarray) else g.get_tensor("Z_corr")
    sync()
    ph["getter"] = time.perf_counter() - t
    ph = {k: v * 1e3 for k, v in ph.items()}
    ph["total"] = sum(ph.values())
    reg = {r: g.region_time(r)[0] for r in ("assign", "ridge_stats", "ridge_solve", "ridge_apply", "upload", "download")}
    del out, g
    return ph, reg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="c3", choices=["c3", "c5"])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-rerun", action="store_true", help="skip RunHarmony on reference + query")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_map.py needs a CUDA device")
    torch.cuda.set_device(0)
    bench.W.clear()
    bench.W.update(bench.WORKLOADS[args.config])
    n, d, K = bench.W["cells_per_gpu"], bench.W["d"], bench.W["K"]
    seed = 20261016 + int(args.config[1:])
    bench.log(f"[bench_map] {args.config}: reference {n} x {d}, K = {K}")
    Z, lv_ref = bench.synth_shard(n, 0, seed)
    kw = bench.setup_kwargs(lv_ref)
    t = time.perf_counter()
    g = integrate(Z, kw, K)
    integrate_s = time.perf_counter() - t
    g.enable_timing(True)
    ref = g.reference()   # warm-up
    ref_ms = []
    for _ in range(args.reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        ref = g.reference()
        ref_ms.append((time.perf_counter() - t) * 1e3)
    ref_region = g.region_time("reference")
    del g
    # warm-up of the mapping path on a small query
    zs, ls = make_query(20000, n + 10_000_000, seed)
    for timing in (False, True):
        map_once(zs, ls, ref, torch, timing)
        map_once(torch.from_numpy(zs).to("cuda", torch.float32), torch.from_numpy(ls).cuda(), ref, torch, timing)
    mb = min_bytes_per_cell(K, d)
    queries = {}
    for nq in (1_000_000, 100_000):
        Zq, lq = make_query(nq, n, seed)
        inputs = {"host": (torch.from_numpy(Zq).pin_memory().numpy(), lq),
                  "dev32": (torch.from_numpy(Zq).to("cuda", torch.float32), torch.from_numpy(lq).cuda())}
        for mode, (zin, lin) in inputs.items():
            walls, regs = [], []
            for _ in range(args.reps):     # wall-clock runs without events, region runs with them, alternated
                walls.append(map_once(zin, lin, ref, torch, False)[0])
                regs.append(map_once(zin, lin, ref, torch, True)[1])
            med = {k: round(float(np.median([w[k] for w in walls])), 3) for k in walls[0]}
            reg = {k: round(float(np.median([r[k] for r in regs])), 4) for k in regs[0]}
            rate = {k: round(mb[k] * nq / (reg[k] * 1e-3) / 1e12 / HBM_TBPS, 3) for k in ("assign", "ridge_stats", "ridge_apply") if reg[k]}
            map_regions = reg["assign"] + reg["ridge_stats"] + reg["ridge_solve"] + reg["ridge_apply"]
            queries[f"{nq}_{mode}"] = {"cells": nq, "wall_ms_median": med, "wall_map_ms_all": [round(w["map"], 3) for w in walls],
                                       "region_ms_median": reg, "map_regions_ms": round(map_regions, 4),
                                       "fraction_of_hbm_peak": rate,
                                       "map_regions_fraction_of_hbm_peak": round(mb["total"] * nq / (map_regions * 1e-3) / 1e12 / HBM_TBPS, 3)}
            bench.log(f"[bench_map] {nq} {mode}: {queries[f'{nq}_{mode}']}")
        del inputs
    rerun = None
    if not args.no_rerun:
        from harmony_b200 import RunHarmony
        Zq, lq = make_query(1_000_000, n, seed)
        Zall = np.concatenate([Z, Zq])
        batch = np.concatenate([lv_ref[:, 0], bench.W["B_vec"][0] + lq])   # the query batches are new levels
        meta = {"batch": batch}
        torch.cuda.synchronize()
        t = time.perf_counter()
        RunHarmony(Zall, meta, "batch", nclust=K, max_iter=ITERS, early_stop=False, verbose=False, seed=3)
        torch.cuda.synchronize()
        rerun = {"cells": int(Zall.shape[0]), "covariates": "first covariate + query batches", "ms": round((time.perf_counter() - t) * 1e3, 1)}
        bench.log(f"[bench_map] RunHarmony on reference + query: {rerun}")
    print(json.dumps({"config": args.config, "reference_cells": n, "d": d, "K": K, "iterations": ITERS, "reps": args.reps,
                      "gpu": gpu_info(), "hbm_TBps": HBM_TBPS, "integrate_s": round(integrate_s, 3),
                      "reference_ms": {"wall_median": round(float(np.median(ref_ms)), 3), "wall_all": [round(x, 3) for x in ref_ms],
                                       "region_total": round(ref_region[0], 3), "region_calls": args.reps + 1},
                      "min_bytes_per_cell": mb, "queries": queries, "rerun_harmony": rerun}), flush=True)


if __name__ == "__main__":
    main()
