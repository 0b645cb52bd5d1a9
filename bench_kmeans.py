"""kmeans on embeddings of 100k and 1M cells (K cell types at scale 6 with unit noise, d = 50 and 128, fp32), K = 20
and 200: CUDA-event time of the whole call at the defaults, of the seeding (region "kmeans_seed") and of an iteration
((a tol = 0, max_iter = 20 run - a max_iter = 0 run) / its iterations); the iteration's bytes and the sweep's issued
3xTF32 flop against the data sheet's 3.35 TB/s of HBM3 and 495 TFLOP/s of TF32.  Alternated with the yardsticks: an
fp32 torch Lloyd on the same card from the same seeds (cdist, argmin, index_add_, the same stopping rule) and, at 100k
x 50 with K = 20, sklearn's KMeans(algorithm="lloyd") on the CPU from the same seeds.  Fails without a GPU.  The
card's name, power limit and max SM clock come first, then one JSON line per case.

    python bench_kmeans.py [--reps 3] [--sizes 100000 1000000] [--dims 50 128] [--clusters 20 200]
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

HBM_TBS, TF32_TFLOPS = 3.35, 495.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def data(N, d, K, seed=0):
    rng = np.random.default_rng(seed)
    M = rng.standard_normal((K, d)) * 6
    t = rng.integers(0, K, N)
    return (M[t] + rng.standard_normal((N, d))).astype(np.float32), t


def timed(fn, reps):
    import torch
    best = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        best.append(e0.elapsed_time(e1))
    return out, min(best), max(best)


def torch_lloyd(X, C, max_iter, tol):
    """sklearn's Lloyd in fp32 torch: cdist + argmin, index_add_ means (empty clusters kept), the same stopping rule."""
    import torch
    N, d = X.shape
    K = C.shape[0]
    tol_abs = tol * float(X.var(dim=0, unbiased=False).mean())
    old = torch.full((N,), -1, dtype=torch.int64, device=X.device)
    strict, it = False, 0
    for i in range(max_iter):
        lab = torch.cdist(X, C).argmin(dim=1)
        S = torch.zeros_like(C).index_add_(0, lab, X)
        n = torch.bincount(lab, minlength=K).to(X.dtype)
        Cn = torch.where(n[:, None] > 0, S / n.clamp(min=1)[:, None], C)
        shift = float(((Cn - C) ** 2).sum())
        C, it = Cn, i + 1
        if torch.equal(lab, old):
            strict = True
            break
        if shift <= tol_abs:
            break
        old = lab
    if not strict:
        lab = torch.cdist(X, C).argmin(dim=1)
    return lab, C, it


def iteration_bytes(N, d, K):
    """An iteration's HBM traffic by the kernels' reads and writes: the sweep reads the prepared rows, the merge them
    again with the candidate lists, the labels kernel labels / old labels / finite flags / codes, the tuple index about
    eight passes of 4-byte codes and keys, and the segment sums the caller's rows gathered through sort_perm."""
    KD = (d + 7) // 8 * 8
    return N * (4 * KD * 2 + 4 + 4 * 4 + 1 + 8 * 8 + 4 * d + 4)


def sweep_flop(N, d, K):
    """3xTF32: three m64n64k8 products per k-step over the K centres padded to the 64-row tile."""
    KD = (d + 7) // 8 * 8
    return 3 * 2 * N * ((K + 63) // 64 * 64) * KD


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", type=int, nargs="+", default=[100000, 1000000])
    ap.add_argument("--dims", type=int, nargs="+", default=[50, 128])
    ap.add_argument("--clusters", type=int, nargs="+", default=[20, 200])
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_kmeans.py needs a CUDA device")
    from harmony_b200 import nmi_ari
    from harmony_b200.harmony import harmony
    print("card:", card(), flush=True)
    g = harmony(device=0)
    for N in args.sizes:
        for d in args.dims:
            for K in args.clusters:
                Xh, t = data(N, d, K)
                X = torch.as_tensor(Xh, device="cuda:0")
                g.kmeans(X, K, max_iter=2)  # warm every shape
                out, whole, whole_hi = timed(lambda: g.kmeans(X, K, return_seeds=True), args.reps)
                labels, C, inertia, n_iter, seeds = out
                g.enable_timing(True)
                s0 = g.region_time("kmeans_seed")[0]
                _, t0, _ = timed(lambda: g.kmeans(X, K, max_iter=0), 1)
                seed_ms = g.region_time("kmeans_seed")[0] - s0
                g.enable_timing(False)
                o20, t20, _ = timed(lambda: g.kmeans(X, K, max_iter=20, tol=0.0), args.reps)
                _, t0b, _ = timed(lambda: g.kmeans(X, K, max_iter=0), args.reps)
                it20 = int(o20[3][0])
                per_iter = (t20 - t0b) / max(it20, 1)
                # yardstick: torch fp32 Lloyd from the same seeds, alternated
                C0 = X[seeds[0].long()].clone()
                (tl, tC, tit), tt, _ = timed(lambda: torch_lloyd(X, C0, 300, 1e-4), args.reps)
                (_, _, tit20), tt20, _ = timed(lambda: torch_lloyd(X, C0, 20, 0.0), args.reps)
                (_, _, _), tt0, _ = timed(lambda: torch_lloyd(X, C0, 0, 0.0), args.reps)
                agree = nmi_ari(labels, tl.to(torch.int32))[0]
                rec = dict(N=N, d=d, K=K, whole_ms=round(whole, 2), whole_ms_max=round(whole_hi, 2), n_iter=int(n_iter[0]),
                           seed_ms=round(seed_ms, 2), iter_ms=round(per_iter, 3), iters_timed=it20,
                           iter_bytes=iteration_bytes(N, d, K), iter_hbm_share=round(
                               iteration_bytes(N, d, K) / (per_iter * 1e-3) / (HBM_TBS * 1e12), 4),
                           sweep_flop=sweep_flop(N, d, K), sweep_tf32_share=round(
                               sweep_flop(N, d, K) / (per_iter * 1e-3) / (TF32_TFLOPS * 1e12), 4),
                           torch_whole_ms=round(tt, 2), torch_n_iter=tit, torch_iter_ms=round((tt20 - tt0) / max(tit20, 1), 3),
                           nmi_vs_torch=round(agree, 6), nmi_vs_truth=round(nmi_ari(t, labels.cpu().numpy())[0], 6))
                if N == 100000 and d == 50 and K == 20:
                    from sklearn.cluster import KMeans
                    Xd = Xh.astype(np.float64)
                    t_0 = time.perf_counter()
                    km = KMeans(K, init=Xd[seeds[0].cpu().numpy()], n_init=1, algorithm="lloyd").fit(Xd)
                    rec["sklearn_s"] = round(time.perf_counter() - t_0, 3)
                    rec["sklearn_label_agreement"] = float((km.labels_ == labels.cpu().numpy()).mean())
                    rec["sklearn_n_iter"] = int(km.n_iter_)
                print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
