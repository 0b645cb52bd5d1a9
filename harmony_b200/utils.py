"""Driver loop: mirror of /root/reference/R/utils.R:15-46 (``harmonize``) and :50-81."""
import sys

import numpy as np


def is_cuda_tensor(x):
    """True for a torch tensor on a CUDA device.  Never imports torch: a tensor exists only if torch is loaded."""
    torch = sys.modules.get("torch")
    return torch is not None and isinstance(x, torch.Tensor) and x.is_cuda


def harmonize(harmonyObj, iter_harmony, verbose=True):
    """R/utils.R:15-46: cluster_cpp -> moe_correct_ridge_cpp -> check_convergence(1)."""
    if iter_harmony < 1:
        return 0
    for it in range(1, iter_harmony + 1):
        if verbose:
            print(f"Harmony {it}/{iter_harmony}", file=sys.stderr)
        err_status = harmonyObj.cluster_cpp()
        if err_status == -1:
            raise KeyboardInterrupt("terminated by user")
        elif err_status != 0:
            raise RuntimeError(f"Harmony exited with non-zero exit status: {err_status}")
        harmonyObj.moe_correct_ridge_cpp()
        if harmonyObj.check_convergence(1):
            if verbose:
                print(f"Harmony converged after {it} iterations", file=sys.stderr)
            return 0
    return None


def HarmonyConvergencePlot(harmonyObj, round_start=1, round_end=float("inf")):
    """R/utils.R:50-81 without ggplot: returns the table the plot is drawn from
    (idx, kmeans_idx, harmony_idx, val) so callers can plot it with whatever they have."""
    rounds = np.asarray(harmonyObj.kmeans_rounds, dtype=np.int64)
    kmeans_idx = np.concatenate([np.arange(1, r + 1) for r in rounds]) if len(rounds) else np.zeros(0, np.int64)
    harmony_idx = np.repeat(np.arange(1, len(rounds) + 1), rounds)
    val = np.asarray(harmonyObj.objective_kmeans)[1:]
    sel = (harmony_idx >= round_start) & (harmony_idx <= round_end)
    return dict(idx=np.arange(1, sel.sum() + 1), kmeans_idx=kmeans_idx[sel], harmony_idx=harmony_idx[sel],
                val=val[sel])
