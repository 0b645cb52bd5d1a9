"""hb_knn on an embedding of c3's size (1M cells, the suite's seeded generator): (a) 100k query x 1M reference, k = 5 (label transfer) and (b) 1M x 1M self-search,
k = 15 (neighbour graph), both metrics, d = 50 and d = 100.  CUDA-event time of the whole call over warmed repetitions,
the flop and bytes it needs by count and the share of the bound that applies, next to chunked torch.cdist + topk in
fp32 on the same tensors (alternated), with a check that both return the same neighbours outside the band of DESIGN §9.
Fails without a GPU.  One JSON line per case; the card's name, power limit and max SM clock come first.

    python bench_knn.py [--reps 3] [--small]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

TF32_DENSE, HBM = 495e12, 3.35e12   # H100 SXM data sheet, 700 W


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def torch_topk(q, x, k, metric, exclude_self, chunk=2048):
    import torch
    if metric == "cosine":
        q, x = torch.nn.functional.normalize(q, dim=1), torch.nn.functional.normalize(x, dim=1)
    out = []
    for r0 in range(0, q.shape[0], chunk):
        D = torch.cdist(q[r0:r0 + chunk], x)
        if exclude_self:
            r = torch.arange(D.shape[0], device=D.device)
            D[r, r0 + r] = float("inf")
        out.append(D.topk(k, dim=1, largest=False).indices)
    return torch.cat(out)


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--small", action="store_true", help="a tenth of the cells (a check of the script, not a measurement)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_knn.py needs a CUDA device: there is no CPU path")
    from harmony_b200.harmony import harmony
    from knn_restatement import band, centred_norms, distances
    from helpers import synthetic
    print(json.dumps({"card": card()}))
    scale = 10 if args.small else 1
    g = harmony(device=0)
    for d in (50, 100):
        Z, _ = synthetic(1_000_000 // scale, d, [20], n_types=30, seed=7)
        x = torch.as_tensor(Z, dtype=torch.float32, device="cuda:0")
        del Z
        for name, nq, k, self_search in (("transfer_k5", 100_000 // scale, 5, False), ("graph_k15", 1_000_000 // scale, 15, True)):
            q = x if self_search else x[torch.randperm(x.shape[0], device=x.device)[:nq]] + 0.1
            for metric in ("euclidean", "cosine"):
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
                ours, theirs = [], []
                idx = None
                for rep in range(args.reps + 1):     # the first repetition warms both up
                    ev[0].record()
                    idx, _ = g.knn(q, None if self_search else x, k=k, metric=metric)
                    ev[1].record()
                    ev[2].record()
                    ref = torch_topk(q, x, k, metric, self_search)
                    ev[3].record()
                    torch.cuda.synchronize()
                    if rep:
                        ours.append(ev[0].elapsed_time(ev[1]))
                        theirs.append(ev[2].elapsed_time(ev[3]))
                # the same neighbours outside the band, on a sample of rows in fp64
                rows = np.random.default_rng(0).choice(nq, 500, replace=False)
                qh, xh = q[rows].cpu().numpy(), x.cpu().numpy()
                D = distances(qh, xh, metric)
                if self_search:
                    D[np.arange(len(rows)), rows] = np.inf
                qn, xn = centred_norms(qh, xh, metric)
                Dk = np.partition(D, k - 1, axis=1)[:, k - 1]
                b = band(qn, xn, d, metric)
                outside = lambda ii: np.take_along_axis(D, ii, 1) < (Dk - b)[:, None]  # noqa: E731
                io, it = idx[rows].cpu().numpy().astype(np.int64), ref[rows].cpu().numpy()
                same = bool((outside(io).sum(1) == outside(it).sum(1)).all() and
                            (np.take_along_axis(D, io, 1) <= (Dk + b)[:, None]).all())
                KD = (d + 7) // 8 * 8
                ms = float(np.median(ours))
                flop = 2.0 * nq * x.shape[0] * d
                issued = 3.0 * 2.0 * nq * x.shape[0] * KD
                ref_bytes = -(-nq // 128) * x.shape[0] * KD * 4.0      # the reference once per query tile, from L2 or HBM
                hbm_bytes = x.shape[0] * KD * 4.0 * max(1, -(-nq // 128) // 132)   # once per wave if the CTAs sweep together
                bound_ms = max(issued / TF32_DENSE, hbm_bytes / HBM) * 1e3
                print(json.dumps({"case": name, "Nq": nq, "Nx": int(x.shape[0]), "d": d, "metric": metric, "k": k, "hb_knn_ms": round(ms, 2),
                                  "spread_ms": [round(min(ours), 2), round(max(ours), 2)],
                                  "cdist_topk_ms": round(float(np.median(theirs)), 2),
                                  "useful_tflops": round(flop / ms / 1e9, 1), "issued_tflops": round(issued / ms / 1e9, 1),
                                  "reference_bytes_read_by_count": ref_bytes, "bound": "tf32 dense (3 products)",
                                  "bound_ms": round(bound_ms, 2), "share_of_bound": round(bound_ms / ms, 3),
                                  "same_neighbours_outside_band": same}))


if __name__ == "__main__":
    main()
