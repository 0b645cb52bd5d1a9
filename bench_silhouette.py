"""hb_silhouette on embeddings of 100k and 1M cells (seeded clusters), d = 50 and 100, in the two ways scib scores an
integration: cell-type ASW (one group, 20 labels) and batch ASW (20 cell types as groups, 4 batches as labels).
CUDA-event time of the whole call over warmed repetitions, the split into index / preparation and the sweep from one
torch.profiler repetition, the issued sweep flop 3 * 2 * sum_g n_g^2 * KD and their share of the 495 TFLOP/s TF32
bound, next to a yardstick alternated with it: chunked fp32 torch.cdist and index_add_ of the distances per label.
On a 2000-row fp64 sample both must agree with the fp64 restatement (tests/silhouette_restatement.py), the call within
its per-row bound.  Fails without a GPU.  The card's name, power limit and max SM clock come first, then one JSON line
per case; a part not run is reported as "not measured".

    python bench_silhouette.py [--reps 3] [--sizes 100000 1000000] [--yardstick-max 1000000]
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

TF32_DENSE = 495e12   # H100 SXM data sheet, 700 W
SWEEP = "k_silhouette_tc"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def data(N, d, seed=7):
    """20 cell types (cluster centres) x 4 batches (per-batch shifts), as an unintegrated embedding looks."""
    rng = np.random.default_rng(seed)
    t = rng.integers(0, 20, N)
    b = rng.integers(0, 4, N)
    X = (rng.standard_normal((20, d)) * 3.0)[t] + (rng.standard_normal((4, d)) * 1.0)[b]
    X += rng.standard_normal((N, d)).astype(np.float32)
    return X.astype(np.float32), t.astype(np.int32), b.astype(np.int32)


def yardstick(x, labels, groups, chunk=2048):
    """s [N]: chunked fp32 cdist against each group's rows, per-label sums by index_add_, the definition in fp64."""
    import torch
    N = x.shape[0]
    s = torch.full((N,), float("nan"), dtype=torch.float64, device=x.device)
    gs = torch.zeros(N, dtype=torch.int64, device=x.device) if groups is None else groups.long()
    for g in torch.unique(gs).tolist():
        rows = torch.nonzero(gs == g).flatten()
        lab = labels[rows].long()
        L = int(lab.max()) + 1
        n = torch.bincount(lab, minlength=L).double()
        xg = x[rows]
        sums = torch.empty((len(rows), L), dtype=torch.float64, device=x.device)
        for r0 in range(0, len(rows), chunk):
            D = torch.cdist(xg[r0:r0 + chunk], xg)
            part = torch.zeros((D.shape[0], L), dtype=torch.float32, device=x.device)
            part.index_add_(1, lab, D)
            sums[r0:r0 + chunk] = part.double()
        own = n[lab]
        i = torch.arange(len(rows), device=x.device)
        a = torch.where(own > 1, sums[i, lab] / (own - 1).clamp(min=1), torch.zeros_like(own))
        means = sums / n.clamp(min=1)
        means[:, n == 0] = float("inf")
        means[i, lab] = float("inf")
        b = means.min(1).values
        m = torch.maximum(a, b)
        sg = torch.where(m > 0, (b - a) / m, torch.zeros_like(m))
        sg[own == 1] = 0.0
        sg[torch.isinf(b)] = float("nan")
        s[rows] = sg
    return s


def kernel_split(g, x, labels, groups):
    """Device time (ms) of the sweep and of everything else (index, preparation, counts) in one profiled call."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.silhouette(x, labels, groups)
        torch.cuda.synchronize()
    sweep = other = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if e.key.startswith(("Memcpy", "Memset", "cudaMem")):
            other += t / 1e3
        elif SWEEP in e.key:
            sweep += t / 1e3
        else:
            other += t / 1e3
    return sweep, other


def check_sample(x, labels, groups, ours, theirs, n=2000):
    """Both against the fp64 restatement on a 2000-row sample re-scored on its own (fp64 rows)."""
    import torch
    import silhouette_restatement as sr
    from harmony_b200.harmony import harmony
    rows = torch.as_tensor(np.sort(np.random.default_rng(0).choice(x.shape[0], n, replace=False)), device=x.device)
    xs = x[rows].double()
    lab, grp = labels[rows], None if groups is None else groups[rows]
    got = harmony(device=0).silhouette(xs, lab, grp).cpu().numpy()
    ys = yardstick(xs.float(), lab, grp).cpu().numpy()
    want, bound = sr.silhouette(xs.cpu().numpy(), lab.cpu().numpy(), None if grp is None else grp.cpu().numpy(), bound=True)
    ok = ~np.isnan(want)
    ours_ok = bool((np.isnan(got) == np.isnan(want)).all() and (np.abs(got[ok] - want[ok]) <= bound[ok] + 1e-12).all())
    return {"sample_within_bound": ours_ok, "sample_max_err": float(np.abs(got[ok] - want[ok]).max()),
            "sample_yardstick_max_err": float(np.nanmax(np.abs(ys[ok] - want[ok]))),
            "full_max_diff_to_yardstick": float(np.nanmax(np.abs(ours.cpu().numpy() - theirs.cpu().numpy())))
            if theirs is not None else "not measured"}


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--dims", type=int, nargs="+", default=[50, 100])
    ap.add_argument("--yardstick-max", type=int, default=1_000_000, help="largest N the yardstick runs at")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_silhouette.py needs a CUDA device: there is no CPU path")
    from harmony_b200.harmony import harmony
    print(json.dumps({"card": card()}), flush=True)
    g = harmony(device=0)
    for N in args.sizes:
        for d in args.dims:
            X, t, b = data(N, d)
            x = torch.as_tensor(X, device="cuda:0")
            tt, bb = torch.as_tensor(t, device="cuda:0"), torch.as_tensor(b, device="cuda:0")
            for case, labels, groups in (("cell_type_asw", tt, None), ("batch_asw", bb, tt)):
                run_ref = N <= args.yardstick_max
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
                ours, theirs = [], []
                s = ref = None
                for rep in range(args.reps + 1):     # the first repetition warms both up
                    ev[0].record()
                    s = g.silhouette(x, labels, groups)
                    ev[1].record()
                    if run_ref:
                        ev[2].record()
                        ref = yardstick(x, labels, groups)
                        ev[3].record()
                    torch.cuda.synchronize()
                    if rep:
                        ours.append(ev[0].elapsed_time(ev[1]))
                        if run_ref:
                            theirs.append(ev[2].elapsed_time(ev[3]))
                sweep_ms, other_ms = kernel_split(g, x, labels, groups)
                KD = (d + 7) // 8 * 8
                sizes = np.bincount(t) if groups is not None else np.array([N])
                issued = 3.0 * 2.0 * float((sizes.astype(np.float64) ** 2).sum()) * KD
                result = {"N": N, "d": d, "case": case, "groups": len(sizes), "labels": int(labels.max()) + 1,
                          "hb_silhouette_ms": round(float(np.median(ours)), 2),
                          "spread_ms": [round(min(ours), 2), round(max(ours), 2)],
                          "sweep_ms": round(sweep_ms, 2), "index_prepare_ms": round(other_ms, 2),
                          "issued_sweep_tflop": round(issued / 1e12, 2),
                          "issued_tflops_over_sweep": round(issued / sweep_ms / 1e9, 1),
                          "share_of_tf32_bound": round(issued / TF32_DENSE * 1e3 / sweep_ms, 3),
                          "yardstick_ms": round(float(np.median(theirs)), 2) if run_ref else "not measured"}
                result.update(check_sample(x, labels, groups, s, ref))
                print(json.dumps(result), flush=True)
                del s, ref
                torch.cuda.empty_cache()
            del x, tt, bb


if __name__ == "__main__":
    main()
