"""Timings of the shapes past the FFMA kernels' limits (d-chunked logits + softmax passes, column-range ridge apply, k-means
initialisation from logits) at N = 1M cells, 20 batches, on one GPU.  bench.py (config 3 and friends) stays the flagship
benchmark; this script only measures the wide shapes.

For each shape: CUDA-event region times per Harmony iteration (cluster_cpp + moe_correct_ridge_cpp) for the assignment
(the cold start of cluster_cpp), the ridge apply and the whole iteration, the native k-means initialisation, the bytes each
region must move and the achieved rate against the H100 SXM's 3.35 TB/s.  Then, at d = 200 / K = 100, the FFMA kernels
against the same shape under HB_KS_WIDE, alternated in one run.  Prints one JSON line.

    python bench_wide.py [--cells 1000000] [--steps 5] [--ab-rounds 3]
"""
import argparse
import json
import sys
import time

import numpy as np

HBM_TBS = 3.35
HB_KS_WIDE = 16
SHAPES = [(127, 200), (300, 100), (512, 200), (50, 1024)]   # (d, K)
T = 10


def up(x, m):
    return (x + m - 1) // m * m


def make_inputs(n, d, seed):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    types = torch.randn(30, d, device="cuda", generator=g)
    batch = torch.randn(20, d, device="cuda", generator=g)
    t = torch.randint(0, 30, (n,), device="cuda", generator=g)
    b = torch.randint(0, 20, (n,), device="cuda", generator=g)
    Z = types[t] + 0.5 * batch[b] + 0.6 * torch.randn(n, d, device="cuda", generator=g)
    Z *= (10.0 / torch.sqrt(1.0 + torch.arange(d, device="cuda")))[None, :]
    return Z.contiguous(), b.cpu().numpy().astype(np.int32)[:, None]


def new_model(Z, phi, K, kernel_set):
    from harmony_b200.harmony import harmony
    g = harmony()
    if kernel_set:
        g.kernel_set = kernel_set
    g.setup(Z, phi, np.full(K, 0.1), np.full(20, 2.0), None, 0.2, T, -np.inf, -np.inf, K, 0.05, [20], 1e-5)
    return g


def iteration_ms(g, steps):
    """Mean ms per Harmony iteration (no region timers), then the region times of `steps` more iterations."""
    import torch
    dev = torch.device("cuda", 0)
    g.cluster_cpp()
    g.moe_correct_ridge_cpp()
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        g.cluster_cpp()
        g.moe_correct_ridge_cpp()
    g.synchronize()
    e1.record()
    torch.cuda.synchronize(dev)
    whole = e0.elapsed_time(e1) / steps
    g.enable_timing(True)
    base = {r: g.region_time(r) for r in ("assign", "ridge_apply")}
    for _ in range(steps):
        g.cluster_cpp()
        g.moe_correct_ridge_cpp()
    g.synchronize()
    reg = {}
    for r in ("assign", "ridge_apply"):
        ms, n = g.region_time(r)
        reg[r] = ((ms - base[r][0]) / steps, (n - base[r][1]) // steps)
    g.enable_timing(False)
    return whole, reg


def bytes_per_cell(d, K, paths, apply_launches):
    """Bytes per cell each region must move on the kernels hb_debug_wide_paths reports (`paths`):
    logits: Z once per cluster range (128 clusters for the d-chunked kernel, 64 for k_logits_tc) + the U row;
    assignment (the cold start of cluster_cpp): plan order (single-pass shapes) = logits + one U read of the block-sum
    pass; natural order = logits + U read + R write of the softmax pass + k_normalise_rows (Z_corr read and written);
    ridge apply: R once per column range + minuend in and Z_corr out once per cluster range (FFMA and one-range wgmma: one
    column range); k-means initialisation from logits (None on the FFMA kernels): 11 logits passes with a U read each
    (the race, 10 picks), 10 one-hot R writes and 10 statistics passes (R + Z once per 128-cluster launch)."""
    KS, DS = up(K, 4), up(d, 4)
    wide = paths[0] == 4 or paths[1] == 3 or paths[3] == 4
    ranges = (K + 127) // 128 if wide else (K + 63) // 64
    logits = 4 * DS * ranges + 4 * KS
    if paths[1] in (2, 3):           # plan-order cold start
        assign = logits + 4 * KS
    elif paths[0] in (3, 4):         # natural order
        assign = logits + 8 * KS + 8 * DS
    else:
        assign = None
    ncr = (DS + 127) // 128 if paths[2] == 3 else 1
    nkr = max(1, apply_launches // ncr)
    apply = 4 * KS * ncr + 8 * DS * nkr
    kmeans = None
    if paths[3] in (3, 4):
        st = (K + 127) // 128
        kmeans = 11 * (logits + 4 * KS) + 10 * 4 * KS + 10 * st * (4 * KS // st + 4 * DS)
    return dict(assign=assign, ridge_apply=apply, kmeans_init=kmeans)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--cells", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--ab-rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    from harmony_b200 import _lib
    n = args.cells
    out = dict(cells=n, gpu=torch.cuda.get_device_name(0), shapes=[], ab=None)
    for d, K in SHAPES:
        Z, phi = make_inputs(n, d, 1000 + d + K)
        g = new_model(Z, phi, K, 0)
        paths = (__import__("ctypes").c_int64 * 4)()
        _lib.lib().hb_debug_wide_paths(K, d, 20, n, 20, torch.cuda.get_device_properties(0).multi_processor_count, 0, paths)
        g.set_seed(5)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        g.init_cluster_cpp()
        g.synchronize()
        km = (time.perf_counter() - t0) * 1e3
        whole, reg = iteration_ms(g, args.steps)
        b = bytes_per_cell(d, K, list(paths), reg["ridge_apply"][1])
        row = dict(d=d, K=K, wide_paths=list(paths), iteration_ms=round(whole, 3), kmeans_init_ms=round(km, 2))

        def rate(nbytes, ms):
            return None if nbytes is None else round(nbytes * n / (ms * 1e-3) / 1e12, 3)
        for r, (ms, launches) in reg.items():
            tbs = rate(b[r], ms)
            row[r] = dict(ms=round(ms, 4), launches=launches, bytes_per_cell=b[r], tbs=tbs,
                          of_peak=None if tbs is None else round(tbs / HBM_TBS, 3))
        row["kmeans_init"] = dict(bytes_per_cell=b["kmeans_init"], tbs=rate(b["kmeans_init"], km))
        print(f"[wide] {json.dumps(row)}", file=sys.stderr, flush=True)
        out["shapes"].append(row)
        del g, Z
        torch.cuda.empty_cache()
    # ---- A/B at d = 200, K = 100: today's FFMA kernels against HB_KS_WIDE, alternated
    d, K = 200, 100
    Z, phi = make_inputs(n, d, 77)
    Y0 = None
    runs = {0: [], HB_KS_WIDE: []}
    for _ in range(args.ab_rounds):
        for ks in (0, HB_KS_WIDE):
            g = new_model(Z, phi, K, ks)
            if Y0 is None:
                g.set_seed(5)
                g.init_cluster_cpp()
                Y0 = np.asarray(g.Y).T.copy()
            else:
                g.init_cluster_cpp(Y0)
            whole, reg = iteration_ms(g, args.steps)
            runs[ks].append(dict(iteration_ms=whole, assign_ms=reg["assign"][0], ridge_apply_ms=reg["ridge_apply"][0]))
            del g
    out["ab"] = {("ffma" if ks == 0 else "wide"): {k: [round(r[k], 4) for r in v] for k in v[0]} for ks, v in runs.items()}
    out["ab"]["shape"] = dict(d=d, K=K)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
