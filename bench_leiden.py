"""UMAP connectivities and Leiden of embeddings of 100k and 1M cells (d = 50, 20 cell types at scale 6 shifted by 4
batches at scale 2, unit noise, fp32), n_neighbors = 15: CUDA-event medians of the exact neighbour search (hb_knn),
the connectivities (hb_umap_graph) and Leiden at resolution 1 (hb_leiden), the phase split of Leiden by its regions
(local moving, refinement, aggregation), its levels, sweeps, rounds and Q, and the 20-resolution
nmi_ari_cluster_labels_leiden call.  At 100k also networkx's Louvain on the host once, with its Q and time.  Fails
without a GPU.  The card's name, power limit and SM clocks come first, then one JSON line per size.

    python bench_leiden.py [--reps 3] [--sizes 100000 1000000] [--no-louvain]
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def data(N, d=50, types=20, batches=4, seed=0):
    rng = np.random.default_rng(seed)
    M = rng.standard_normal((types, d)) * 6
    S = rng.standard_normal((batches, d)) * 2
    t = rng.integers(0, types, N)
    b = rng.integers(0, batches, N)
    return (M[t] + S[b] + rng.standard_normal((N, d))).astype(np.float32), t


def timed(fn, reps):
    import torch
    ms, out = [], None
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return out, float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", type=int, nargs="+", default=[100000, 1000000])
    ap.add_argument("--no-louvain", action="store_true")
    args = ap.parse_args()
    import torch
    from harmony_b200 import nmi_ari_cluster_labels_leiden
    from harmony_b200._arrays import handle
    from harmony_b200.community import leiden_graph_on, umap_graph_on
    from harmony_b200.neighbors import knn_on
    print(card(), flush=True)
    g = handle(0)
    for N in args.sizes:
        X, t = data(N)
        x = torch.as_tensor(X, device="cuda:0")
        (idx, dist), knn_ms = timed(lambda: knn_on(g, x, None, 14), args.reps)
        G, umap_ms = timed(lambda: umap_graph_on(g, idx, dist, 15), args.reps)
        (labels, info), leiden_ms = timed(lambda: leiden_graph_on(g, G, 1.0, -1, True), args.reps)
        g.enable_timing(True)
        before = {r: g.region_time(r)[0] for r in ("leiden_move", "leiden_refine", "leiden_aggregate", "leiden")}
        leiden_graph_on(g, G, 1.0, -1)
        torch.cuda.synchronize()
        split = {r: round(g.region_time(r)[0] - before[r], 2) for r in before}
        g.enable_timing(False)
        t0 = time.perf_counter()
        scores = nmi_ari_cluster_labels_leiden(x, {"cell_type": torch.as_tensor(t, device="cuda:0")}, "cell_type")
        torch.cuda.synchronize()
        sweep_s = time.perf_counter() - t0
        out = dict(N=N, d=50, n_neighbors=15, nnz=int(G[1].numel()), knn_ms=round(knn_ms, 2),
                   umap_graph_ms=round(umap_ms, 2), leiden_ms=round(leiden_ms, 2),
                   graph_plus_leiden_over_search=round((umap_ms + leiden_ms) / knn_ms, 3), leiden_regions_ms=split,
                   **{k: info[k] for k in ("n_communities", "quality", "iterations", "levels", "sweeps", "rounds")},
                   nmi_ari_20_resolutions_s=round(sweep_s, 2), scores=scores)
        if N <= 100000 and not args.no_louvain:
            import networkx as nx
            import scipy.sparse as sp
            A = sp.csr_matrix((G[2].double().cpu().numpy(), G[1].cpu().numpy(), G[0].cpu().numpy()), shape=(N, N))
            H = nx.from_scipy_sparse_array(A, edge_attribute="weight")
            t0 = time.perf_counter()
            parts = nx.community.louvain_communities(H, weight="weight", seed=0)
            out["networkx_louvain_s"] = round(time.perf_counter() - t0, 2)
            out["networkx_louvain_Q"] = nx.community.modularity(H, parts, weight="weight")
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
