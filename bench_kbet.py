"""kbet on embeddings of 100k and 1M cells (20 cell types at scale 6, 4 batch shifts at scale 2, unit noise, d = 50 and
100, fp32), k0 by scib's rule: CUDA-event time of the whole call over warmed repetitions, the split into the index and
preparation, the grouped sweep, the merge and k_kbet from one torch.profiler repetition, the sweep's issued TFLOP/s
(3 x 2 sum_l n_l^2 KD for 3xTF32) against the 495 TFLOP/s of dense TF32 on the data sheet, alternated with a yardstick:
per cell type chunked fp32 torch.cdist + topk(k0), then the statistic and scipy.stats.chi2.sf on the host.  Fails
without a GPU.  The card's name, power limit and max SM clock come first, then one JSON line per case.

    python bench_kbet.py [--reps 3] [--sizes 100000 1000000] [--dims 50 100]
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

TYPES, BATCHES = 20, 4
TF32_DENSE = 495.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def data(N, d, seed=0):
    rng = np.random.default_rng(seed)
    M = rng.standard_normal((TYPES, d)) * 6
    S = rng.standard_normal((BATCHES, d)) * 2
    t = rng.integers(0, TYPES, N)
    b = rng.integers(0, BATCHES, N)
    return (M[t] + S[b] + rng.standard_normal((N, d))).astype(np.float32), t.astype(np.int32), b.astype(np.int32)


def yardstick(x, t, b, alpha=0.05, chunk=2048):
    """Per cell type: exact fp32 neighbours by cdist + topk(k0) (the cell and k0 - 1 others) on the GPU, scib's k0
    rule, the package's statistic and scipy's tail on the host -> the scaled score."""
    import torch
    from scipy.stats import chi2
    rates = []
    for label in np.unique(t):
        rows = np.nonzero(t == label)[0]
        levels, counts = np.unique(b[rows], return_counts=True)
        k0 = int(min(70, max(10, np.floor(counts.mean() / 4))))
        xl = x[torch.as_tensor(rows, device=x.device)]
        nn = torch.cat([torch.cdist(xl[r0:r0 + chunk], xl).topk(k0, dim=1, largest=False).indices
                        for r0 in range(0, len(rows), chunk)]).cpu().numpy()
        code = np.searchsorted(levels, b[rows])[nn]
        obs = np.zeros((len(rows), len(levels)))
        np.add.at(obs, (np.repeat(np.arange(len(rows)), k0), code.reshape(-1)), 1.0)
        exp = counts / len(rows) * k0
        p = chi2.sf(((obs - exp) ** 2 / exp).sum(1), len(levels) - 1)
        rates.append(float((p < alpha).mean()))
    return 1 - float(np.mean(rates))


def kernel_split(g, x, bt, tt):
    """Device time (ms) of the index and preparation, the sweep, the merge and k_kbet in one profiled call."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.kbet(x, bt, tt)
        torch.cuda.synchronize()
    split = {"index_prepare_ms": 0.0, "sweep_ms": 0.0, "merge_ms": 0.0, "k_kbet_ms": 0.0}
    for e in prof.key_averages():
        ms = getattr(e, "device_time_total", None)
        ms = (e.cuda_time_total if ms is None else ms) / 1e3
        if "k_knn_tc" in e.key:
            split["sweep_ms"] += ms
        elif "k_knn_merge" in e.key:
            split["merge_ms"] += ms
        elif "k_kbet" in e.key:
            split["k_kbet_ms"] += ms
        elif e.key.startswith("_Z") or "hb::" in e.key or e.key.startswith("void hb"):
            split["index_prepare_ms"] += ms
    return {k: round(v, 3) for k, v in split.items()}


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--dims", type=int, nargs="+", default=[50, 100])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_kbet.py needs a CUDA device: there is no CPU path")
    from harmony_b200 import kbet
    from harmony_b200.harmony import harmony
    print(json.dumps({"card": card()}))
    for N in args.sizes:
        for d in args.dims:
            X, t, b = data(N, d)
            x = torch.as_tensor(X, device="cuda:0")
            meta = {"type": torch.as_tensor(t, device="cuda:0"), "batch": torch.as_tensor(b, device="cuda:0")}
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ours, theirs = [], []
            for rep in range(args.reps + 1):     # the first repetition warms both up
                ev[0].record()
                score = kbet(x, meta, "batch", "type")
                ev[1].record()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                ref = yardstick(x, t, b)
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                if rep:
                    ours.append(ev[0].elapsed_time(ev[1]))
                    theirs.append((t1 - t0) * 1e3)
            g = harmony(device=0)
            split = kernel_split(g, x, meta["batch"], meta["type"])
            KD = (d + 7) // 8 * 8
            flop = 3 * 2 * float((np.bincount(t).astype(np.float64) ** 2).sum()) * KD
            result = {"N": N, "d": d, "types": TYPES, "batches": BATCHES, "score": round(score, 5),
                      "kbet_ms": round(float(np.median(ours)), 2), "spread_ms": [round(min(ours), 2), round(max(ours), 2)],
                      **split, "sweep_tflops": round(flop / (split["sweep_ms"] * 1e-3) / 1e12, 1)
                      if split["sweep_ms"] else None, "tf32_dense_tflops": TF32_DENSE,
                      "yardstick_ms": round(float(np.median(theirs)), 1), "yardstick_score": round(ref, 5)}
            print(json.dumps(result), flush=True)
            del x, meta, g
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
