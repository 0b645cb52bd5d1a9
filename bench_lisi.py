"""hb_lisi on embeddings of 100k and 1M cells (the suite's seeded generator), d = 50 and 100, perplexity 30 (k = 89) and
two label sets (batch and type).  CUDA-event time of the whole call over warmed repetitions, the split into the
neighbour search (column sums, preparation, sweep, merge) and k_lisi from one torch.profiler repetition, the issued
sweep flop 3 * 2 * N^2 * KD and their share of the 495 TFLOP/s TF32 bound, next to a yardstick alternated with it:
chunked torch.cdist + topk(k + 1) in fp32 and a vectorised fp64 torch bisection.  On a sample of rows both must
return the same neighbours outside the band of DESIGN §9 and, where the neighbour sets match, LISI within 1e-4.
Fails without a GPU.  The card's name, power limit and max SM clock come first, then one JSON line per case; a part
not run is reported as "not measured".

    python bench_lisi.py [--reps 2] [--sizes 100000 1000000] [--yardstick-max 1000000]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

TF32_DENSE = 495e12   # H100 SXM data sheet, 700 W
P, K = 30, 89
SEARCH = ("k_knn_colsum", "k_knn_prepare", "k_knn_tc", "k_knn_merge")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def yardstick(x, codes, chunk=1024):
    """(lisi [N, sets], idx [N, k]): cdist + topk(k + 1) with the first column dropped, fp64 bisection and fold."""
    import torch
    idx, dist = [], []
    for r0 in range(0, x.shape[0], chunk):
        d, i = torch.cdist(x[r0:r0 + chunk], x).topk(K + 1, dim=1, largest=False)
        idx.append(i[:, 1:])
        dist.append(d[:, 1:])
    idx, D = torch.cat(idx), torch.cat(dist).double()
    D = D - D[:, :1]
    n = D.shape[0]
    beta = torch.ones(n, dtype=torch.float64, device=x.device)
    bmin, bmax = torch.full_like(beta, -math.inf), torch.full_like(beta, math.inf)
    H, Pm = torch.zeros_like(beta), torch.zeros_like(D)
    active = torch.ones(n, dtype=torch.bool, device=x.device)
    for _ in range(50):
        E = torch.exp(-beta[:, None] * D)
        s = E.sum(1)
        Hn = torch.log(s) + beta * (D * E).sum(1) / s
        H = torch.where(active, Hn, H)
        Pm = torch.where(active[:, None], E / s[:, None], Pm)
        diff = Hn - math.log(P)
        done = diff.abs() < 1e-5
        up, down = active & ~done & (diff > 0), active & ~done & ~(diff > 0)
        b_up = torch.where(torch.isinf(bmax), 2 * beta, (beta + bmax) / 2)
        b_down = torch.where(torch.isinf(bmin), beta / 2, (beta + bmin) / 2)
        bmin, bmax = torch.where(up, beta, bmin), torch.where(down, beta, bmax)
        beta = torch.where(up, b_up, torch.where(down, b_down, beta))
        active &= ~done
        if not bool(active.any()):
            break
    out = torch.empty((n, codes.shape[0]), dtype=torch.float64, device=x.device)
    for s in range(codes.shape[0]):
        for r0 in range(0, n, 16384):
            lab = codes[s][idx[r0:r0 + 16384]]
            p = Pm[r0:r0 + 16384]
            same = lab[:, :, None] == lab[:, None, :]
            out[r0:r0 + 16384, s] = 1.0 / (p * (same * p[:, None, :]).sum(2)).sum(1)
    out[H == 0] = -1.0
    return out, idx


def kernel_split(g, x, codes):
    """Device time (ms) of the search kernels and of k_lisi in one profiled call."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.lisi(x, codes, P)
        torch.cuda.synchronize()
    search = lisi = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if "k_lisi" in e.key:
            lisi += t / 1e3
        elif any(s in e.key for s in SEARCH):
            search += t / 1e3
    return search, lisi


def agree(x, idx_ours, lisi_ours, idx_ref, lisi_ref, rows):
    """The same neighbours outside the band on the sampled rows, and LISI within 1e-4 where the sets match."""
    from knn_restatement import band, centred_norms, distances
    xh = x.cpu().numpy()
    qh = xh[rows]
    D = distances(qh, xh, "euclidean")
    D[np.arange(len(rows)), rows] = np.inf
    qn, xn = centred_norms(qh, xh, "euclidean")
    Dk = np.partition(D, K - 1, axis=1)[:, K - 1]
    b = band(qn, xn, x.shape[1])
    outside = lambda ii: np.take_along_axis(D, ii, 1) < (Dk - b)[:, None]  # noqa: E731
    io, ir = idx_ours[rows].cpu().numpy().astype(np.int64), idx_ref[rows].cpu().numpy()
    same_band = bool((outside(io).sum(1) == outside(ir).sum(1)).all() and
                     (np.take_along_axis(D, io, 1) <= (Dk + b)[:, None]).all())
    same_set = (np.sort(io, 1) == np.sort(ir, 1)).all(1)
    lo, lr_ = lisi_ours[rows].cpu().numpy()[same_set], lisi_ref[rows].cpu().numpy()[same_set]
    rel = float((np.abs(lo - lr_) / np.abs(lr_)).max()) if len(lo) else float("nan")
    return same_band, float(same_set.mean()), rel


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--dims", type=int, nargs="+", default=[50, 100])
    ap.add_argument("--yardstick-max", type=int, default=1_000_000, help="largest N the yardstick runs at")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_lisi.py needs a CUDA device: there is no CPU path")
    from harmony_b200.harmony import harmony
    from helpers import synthetic
    print(json.dumps({"card": card()}))
    g = harmony(device=0)
    for N in args.sizes:
        for d in args.dims:
            Z, meta = synthetic(N, d, [20, 30], n_types=30, seed=7, nested=False)
            x = torch.as_tensor(Z, dtype=torch.float32, device="cuda:0")
            codes = torch.as_tensor(np.stack([meta["cov0"], meta["cov1"]]).astype(np.int32), device="cuda:0")
            del Z
            run_ref = N <= args.yardstick_max
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            ours, theirs = [], []
            for rep in range(args.reps + 1):     # the first repetition warms both up
                ev[0].record()
                lisi, idx, _ = g.lisi(x, codes, P, return_neighbors=True)
                ev[1].record()
                if run_ref:
                    ev[2].record()
                    ref, ref_idx = yardstick(x, codes)
                    ev[3].record()
                torch.cuda.synchronize()
                if rep:
                    ours.append(ev[0].elapsed_time(ev[1]))
                    if run_ref:
                        theirs.append(ev[2].elapsed_time(ev[3]))
            search_ms, lisi_ms = kernel_split(g, x, codes)
            KD = (d + 7) // 8 * 8
            issued = 3.0 * 2.0 * N * N * KD
            result = {"N": N, "d": d, "perplexity": P, "k": K, "label_sets": 2,
                      "hb_lisi_ms": round(float(np.median(ours)), 2),
                      "spread_ms": [round(min(ours), 2), round(max(ours), 2)],
                      "search_kernels_ms": round(search_ms, 2), "k_lisi_ms": round(lisi_ms, 2),
                      "issued_sweep_tflop": round(issued / 1e12, 1),
                      "issued_tflops_over_search": round(issued / search_ms / 1e9, 1),
                      "share_of_tf32_bound": round(issued / TF32_DENSE * 1e3 / search_ms, 3)}
            if run_ref:
                rows = np.random.default_rng(0).choice(N, 500, replace=False)
                same_band, same_sets, rel = agree(x, idx, lisi, ref_idx, ref, rows)
                result.update({"yardstick_ms": round(float(np.median(theirs)), 2),
                               "same_neighbours_outside_band": same_band, "sample_rows_same_set": same_sets,
                               "lisi_max_rel_diff_same_set": rel, "lisi_agrees": rel <= 1e-4})
            else:
                result.update({"yardstick_ms": "not measured", "same_neighbours_outside_band": "not measured"})
            print(json.dumps(result), flush=True)
            del x, codes, lisi, idx
            if run_ref:
                del ref, ref_idx
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
