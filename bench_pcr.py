"""pcr on embeddings of 100k and 1M cells (4 or 1000 batch shifts at scale 2 on 20 cell types at scale 6, unit noise,
d = 50 and 128, fp32), 50 components: CUDA-event time of the whole call over warmed repetitions; the split into the
batch index, the batch sums (sums, mean, combine), the Grams and the rest (copies and the host eigensolve) from one
torch.profiler repetition; the host eigensolve alone (hb_debug_sym_eig on a d x d covariance); the covariance Gram's
bytes and issued DMMA FLOP over its kernel time against the data sheet's 3.35 TB/s of HBM3 and 67 TFLOP/s of FP64
tensor cores.  Alternated with the yardsticks: fp64 torch on the GPU (centring, Xc^T Xc, index_add_, eigh) and, at
100k cells and 4 batches, scib's pc_regression transcribed (sklearn + pandas) on the CPU.  Fails without a GPU.  The
card's name, power limit and max SM clock come first, then one JSON line per case.

    python bench_pcr.py [--reps 5] [--sizes 100000 1000000] [--dims 50 128] [--batches 4 1000]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

TYPES, N_COMPS = 20, 50
HBM_TBS, FP64_TC_TFLOPS = 3.35, 67.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def data(N, d, B, seed=0):
    rng = np.random.default_rng(seed)
    M = rng.standard_normal((TYPES, d)) * 6
    S = rng.standard_normal((B, d)) * 2
    t = rng.integers(0, TYPES, N)
    b = rng.integers(0, B, N)
    return (M[t] + S[b] + rng.standard_normal((N, d))).astype(np.float32), b.astype(np.int32)


def torch_fp64(x, bt, B, n_comps=N_COMPS):
    """The score by fp64 torch on the GPU: centring, the covariance, the batch sums by index_add_, eigh."""
    import torch
    X = x.double()
    Xc = X - X.mean(0)
    C = Xc.T @ Xc
    S = torch.zeros((B, X.shape[1]), dtype=torch.float64, device=X.device).index_add_(0, bt.long(), Xc)
    nb = torch.bincount(bt.long(), minlength=B).double()
    T = S[nb > 0] / nb[nb > 0].sqrt()[:, None]
    lam, V = torch.linalg.eigh(C)
    lam, V = lam.flip(0)[:n_comps], V.flip(1)[:, :n_comps]
    r2 = ((T @ V) ** 2).sum(0) / lam
    return float((r2.clamp(0, 1) * lam).sum() / lam.sum())


def gram_kernels(h, x, bt):
    """Device time (ms) by stage in one profiled call; the first k_pcr_gram is the covariance's."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        h.pcr(x, bt, N_COMPS)
        torch.cuda.synchronize()
    split = {"index_ms": 0.0, "sums_ms": 0.0, "gram_x_ms": 0.0, "gram_between_ms": 0.0, "reduce_ms": 0.0,
             "memcpy_ms": 0.0}
    grams = 0
    for e in sorted(prof.events(), key=lambda e: e.time_range.start):
        ms = getattr(e, "device_time_total", None)
        ms = (e.cuda_time_total if ms is None else ms) / 1e3
        if not ms:
            continue
        if "k_pcr_gram" in e.name:
            split["gram_x_ms" if grams == 0 else "gram_between_ms"] += ms
            grams += 1
        elif "k_pcr_reduce" in e.name:
            split["reduce_ms"] += ms
        elif "k_pcr_" in e.name:
            split["sums_ms"] += ms
        elif "emcpy" in e.name or "emset" in e.name:
            split["memcpy_ms"] += ms
        elif "hb::" in e.name or e.name.startswith("_Z") or e.name.startswith("void hb"):
            split["index_ms"] += ms
    return {k: round(v, 4) for k, v in split.items()}


def host_eig_ms(x, reps=5):
    """hb_debug_sym_eig on the d x d covariance of x, the eigensolve hb_pcr runs on the host."""
    from harmony_b200 import _lib
    X = x.double()
    C = np.ascontiguousarray(((X - X.mean(0)).T @ (X - X.mean(0))).cpu().numpy())
    d = C.shape[0]
    w, V = np.empty(d), np.empty((d, d))
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        assert _lib.lib().hb_debug_sym_eig(d, P(C), P(w), P(V)) == 0
        ts.append((time.perf_counter() - t0) * 1e3)
    return round(float(np.median(ts)), 3)


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--dims", type=int, nargs="+", default=[50, 128])
    ap.add_argument("--batches", type=int, nargs="+", default=[4, 1000])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_pcr.py needs a CUDA device: there is no CPU path")
    from harmony_b200.harmony import harmony
    print(json.dumps({"card": card()}))
    for N in args.sizes:
        for d in args.dims:
            for B in args.batches:
                X, b = data(N, d, B)
                x = torch.as_tensor(X, device="cuda:0")
                bt = torch.as_tensor(b, device="cuda:0")
                h = harmony(device=0)
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
                ours, theirs = [], []
                for rep in range(args.reps + 1):     # the first repetition warms both up
                    ev[0].record()
                    score = h.pcr(x, bt, N_COMPS)[3]
                    ev[1].record()
                    ev[2].record()
                    ref = torch_fp64(x, bt, B)
                    ev[3].record()
                    torch.cuda.synchronize()
                    if rep:
                        ours.append(ev[0].elapsed_time(ev[1]))
                        theirs.append(ev[2].elapsed_time(ev[3]))
                split = gram_kernels(h, x, bt)
                KD = (d + 15) // 16 * 16
                tiles = (KD // 16) ** 2 + KD // 16
                flop = 2.0 * N * tiles * 16 * 8          # issued: every 16 x 8 upper tile over every row
                gbytes = N * d * 4
                gms = split["gram_x_ms"]
                result = {"N": N, "d": d, "batches": B, "score": round(score, 10), "pcr_ms": round(float(np.median(ours)), 3),
                          "spread_ms": [round(min(ours), 3), round(max(ours), 3)], **split,
                          "host_eig_ms": host_eig_ms(x),
                          "gram_x_tbs": round(gbytes / (gms * 1e-3) / 1e12, 3) if gms else None,
                          "gram_x_tflops": round(flop / (gms * 1e-3) / 1e12, 2) if gms else None,
                          "gram_x_bound": "dmma" if flop / FP64_TC_TFLOPS / 1e12 > gbytes / HBM_TBS / 1e12 else "hbm",
                          "gram_x_share_of_bound": round(max(flop / FP64_TC_TFLOPS / 1e12, gbytes / HBM_TBS / 1e12)
                                                         / (gms * 1e-3), 3) if gms else None,
                          "torch_fp64_ms": round(float(np.median(theirs)), 3), "torch_fp64_score": round(ref, 10)}
                if N <= 100_000 and B <= 4:
                    import pcr_restatement as pr
                    t0 = time.perf_counter()
                    result["scib_score"] = round(float(pr.scib_pc_regression(X.astype(np.float64), b, N_COMPS)[0]), 10)
                    result["scib_cpu_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
                print(json.dumps(result), flush=True)
                del x, bt, h
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
