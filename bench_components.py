"""graph_connectivity on embeddings of 100k and 1M cells (20 cell types at scale 6, 4 batch shifts at scale 2, unit
noise, d = 50, fp32), n_neighbors 15: CUDA-event time of the whole call over warmed repetitions and the split into the
neighbour search (column sums, preparation, sweep, merge) and the component kernels (k_cc_*) from one torch.profiler
repetition, alternated with a yardstick: chunked fp32 torch.cdist + topk(k + 1), then scib's scipy loop on the host
(symmetric connectivities, each cell type's subgraph, connected_components).  Then hb_graph_components alone on 1M-row
graphs (random at k = 14 and 64, a shuffled path, stars on the first and the last row) as edges (N k entries) per
second.  Fails without a GPU.  The card's name, power limit and max SM clock come first, then one JSON line per case.

    python bench_components.py [--reps 3] [--sizes 100000 1000000] [--yardstick-max 1000000]
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

NN, TYPES, BATCHES, D = 15, 20, 4, 50
SEARCH = ("k_knn_colsum", "k_knn_prepare", "k_knn_tc", "k_knn_merge")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def data(N, seed=0):
    rng = np.random.default_rng(seed)
    M = rng.standard_normal((TYPES, D)) * 6
    S = rng.standard_normal((BATCHES, D)) * 2
    t = rng.integers(0, TYPES, N)
    b = rng.integers(0, BATCHES, N)
    return (M[t] + S[b] + rng.standard_normal((N, D))).astype(np.float32), t


def yardstick(x, t, chunk=1024):
    """scib's route with an exact fp32 search: cdist + topk on the GPU, the per-type loop of scipy on the host."""
    import torch
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import connected_components
    idx = []
    for r0 in range(0, x.shape[0], chunk):
        idx.append(torch.cdist(x[r0:r0 + chunk], x).topk(NN, dim=1, largest=False).indices[:, 1:])
    idx = torch.cat(idx).cpu().numpy()
    N, k = idx.shape
    conn = csr_matrix((np.ones(N * k, np.float32), (np.repeat(np.arange(N), k), idx.reshape(-1))), shape=(N, N))
    conn = conn + conn.T
    res = []
    for label in np.unique(t):
        sub = np.nonzero(t == label)[0]
        _, lab = connected_components(conn[sub][:, sub], connection="strong")
        tab = np.bincount(lab)
        res.append(tab.max() / tab.sum())
    return float(np.mean(res))


def kernel_split(x, meta):
    """Device time (ms) of the search kernels and of the component kernels in one profiled call."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from harmony_b200 import graph_connectivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        graph_connectivity(x, meta, "type", NN)
        torch.cuda.synchronize()
    search = comp = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if "k_cc_" in e.key:
            comp += t / 1e3
        elif any(s in e.key for s in SEARCH):
            search += t / 1e3
    return search, comp


def graphs(N, rng):
    p = rng.permutation(N).astype(np.int32)
    path = np.full((N, 2), -1, np.int32)
    path[p[:-1], 0] = p[1:]
    path[p[1:], 1] = p[:-1]
    yield "random_k14", rng.integers(0, N, (N, 14)).astype(np.int32)
    yield "random_k64", rng.integers(0, N, (N, 64)).astype(np.int32)
    yield "shuffled_path", path
    yield "star_row_0", np.zeros((N, 1), np.int32)
    yield "star_last_row", np.full((N, 1), N - 1, np.int32)


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--yardstick-max", type=int, default=1_000_000, help="largest N the yardstick runs at")
    ap.add_argument("--graph-rows", type=int, default=1_000_000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_components.py needs a CUDA device: there is no CPU path")
    from harmony_b200 import graph_connectivity
    from harmony_b200.harmony import harmony
    print(json.dumps({"card": card()}))
    for N in args.sizes:
        X, t = data(N)
        x = torch.as_tensor(X, device="cuda:0")
        meta = {"type": torch.as_tensor(t, device="cuda:0")}
        del X
        run_ref = N <= args.yardstick_max
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ours, theirs = [], []
        for rep in range(args.reps + 1):     # the first repetition warms both up
            ev[0].record()
            score = graph_connectivity(x, meta, "type", NN)
            ev[1].record()
            torch.cuda.synchronize()
            if run_ref:
                t0 = time.perf_counter()
                ref = yardstick(x, t)
                torch.cuda.synchronize()
                t1 = time.perf_counter()
            if rep:
                ours.append(ev[0].elapsed_time(ev[1]))
                if run_ref:
                    theirs.append((t1 - t0) * 1e3)
        search_ms, comp_ms = kernel_split(x, meta)
        result = {"N": N, "d": D, "n_neighbors": NN, "types": TYPES, "batches": BATCHES, "score": round(score, 5),
                  "graph_connectivity_ms": round(float(np.median(ours)), 2),
                  "spread_ms": [round(min(ours), 2), round(max(ours), 2)],
                  "search_kernels_ms": round(search_ms, 2), "component_kernels_ms": round(comp_ms, 3)}
        if run_ref:
            result.update({"yardstick_ms": round(float(np.median(theirs)), 1), "yardstick_score": round(ref, 5)})
        else:
            result.update({"yardstick_ms": "not measured"})
        print(json.dumps(result), flush=True)
        del x, meta
        torch.cuda.empty_cache()
    g = harmony(device=0)
    rng = np.random.default_rng(1)
    N = args.graph_rows
    for name, idx in graphs(N, rng):
        it = torch.as_tensor(idx, device="cuda:0")
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        times = []
        for rep in range(args.reps + 1):
            ev[0].record()
            comp, largest = g.graph_components(it)
            ev[1].record()
            torch.cuda.synchronize()
            if rep:
                times.append(ev[0].elapsed_time(ev[1]))
        ms = float(np.median(times))
        print(json.dumps({"graph": name, "N": N, "k": idx.shape[1], "components": int(torch.unique(comp).numel()),
                          "largest": int(largest[0]), "hb_graph_components_ms": round(ms, 3),
                          "spread_ms": [round(min(times), 3), round(max(times), 3)],
                          "entries_per_s": float(f"{N * idx.shape[1] / ms * 1e3:.3g}")}), flush=True)
        del it, comp, largest


if __name__ == "__main__":
    main()
