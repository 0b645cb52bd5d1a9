"""Shared helpers for the test-suite (test infrastructure; may use oracle/)."""
import os
import socket

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def load_cell_lines(small=True):
    f = np.load(os.path.join(GOLDEN, "cell_lines_small.npz" if small else "cell_lines.npz"))
    meta = {"dataset": f["dataset_levels"][f["dataset"]], "cell_type": f["cell_type_levels"][f["cell_type"]]}
    return f["scaled_pcs"], meta


def load_pbmc():
    f = np.load(os.path.join(GOLDEN, "pbmc_stim_pcs.npz"))
    return f["pcs"], {"stim": f["stim_levels"][f["stim"]]}


def synthetic(N, d, B_vec, n_types=8, seed=0, nested=True):
    """Small synthetic embedding following SURVEY.md §8d's generator (numpy, test sizes)."""
    rng = np.random.default_rng(seed)
    t = rng.integers(0, n_types, N)
    M = rng.standard_normal((n_types, d))
    sd = 10.0 / np.sqrt(1.0 + np.arange(d))
    Z = M[t] + 0.6 * rng.standard_normal((N, d))
    meta = {}
    prev = None
    for c, Bc in enumerate(B_vec):
        if c == 0 or not nested:
            lv = rng.integers(0, Bc, N)
        else:  # nested: each level of this covariate belongs to one level of the first
            parent = np.arange(Bc) % B_vec[0]
            lv = np.empty(N, dtype=np.int64)
            for p in range(B_vec[0]):
                cand = np.flatnonzero(parent == p)
                sel = prev == p
                lv[sel] = rng.choice(cand, sel.sum()) if len(cand) else 0
        if c == 0:
            prev = lv
        S = rng.standard_normal((Bc, d))
        Z = Z + 0.5 * S[lv]
        meta[f"cov{c}"] = lv
    return Z * sd[None, :], meta


def make_Y0(Z, K, seed=0):
    """K distinct random cells, cosine-normalised (stand-in for kmeans_centers, injected on both sides)."""
    rng = np.random.default_rng(seed)
    Zn = Z / np.maximum(np.linalg.norm(Z, axis=1, keepdims=True), 1e-30)
    idx = rng.choice(Z.shape[0], K, replace=False)
    Y = Zn[idx].copy()
    for _ in range(2):  # two Lloyd iterations on the cosine-normalised data
        a = np.argmax(Zn @ Y.T, axis=1)
        for k in range(K):
            if np.any(a == k):
                Y[k] = Zn[a == k].mean(axis=0)
    return Y


def make_perms(N, n, seed=0):
    rng = np.random.default_rng(seed)
    return np.stack([rng.permutation(N) for _ in range(n)]).astype(np.int64)


def setup_args(a):
    """prepare_inputs() dict -> positional args of OracleHarmony.setup / harmony.setup order differs; keep dict."""
    return dict(Z=a["Z"], phi_i=a["phi_i"], B_vec=a["B_vec"], sigma=a["sigma"], theta=a["theta"],
                lambda_=a["lambda_"], alpha=a["alpha"], max_iter_kmeans=a["max_iter_kmeans"],
                epsilon_kmeans=a["epsilon_kmeans"], epsilon_harmony=a["epsilon_harmony"], K=a["K"],
                block_size=a["block_size"], batch_proportion_cutoff=a["batch_proportion_cutoff"])


def run_oracle(a, Y0, n_iter, perm_seed=0, double=False, perms=None):
    """Drive the CPU oracle exactly like RunHarmony.default + harmonize (R/ui.R:269-283, R/utils.R:15-46)
    with injected centroids / update orders.  Returns the OracleHarmony object and the perms used."""
    from oracle.oracle import OracleHarmony
    o = OracleHarmony(double=double)
    o.setup(**setup_args(a))
    o.init_cluster_cpp(Y0)
    T = a["max_iter_kmeans"]
    N = a["Z"].shape[0]
    if perms is None:
        perms = make_perms(N, n_iter * T, perm_seed).reshape(n_iter, T, N)
    iters = 0
    for it in range(n_iter):
        o.cluster_cpp(perms[it])
        o.moe_correct_ridge_cpp()
        iters += 1
        if o.check_convergence(1):
            break
    return o, perms, iters


def rel_l2(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(np.asarray(b)), 1e-300))


def num_sms():
    """The SM count of GPU 0, which the geometry and kernel-path hooks take."""
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def gpu_harmony():
    """A fresh harmony object on GPU 0."""
    from harmony_b200.harmony import harmony
    return harmony(device=0)


def free_port():
    """A TCP port on 127.0.0.1 that was free a moment ago, for a test's process group."""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p
