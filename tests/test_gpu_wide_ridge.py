"""The ridge step at embedding widths whose tensor-core statistics and apply kernels copy partial rows, and at a
shape where an odd number of apply stages would fit:
- d = 150: K3 runs two column ranges of [Z | 1], each copying part of every Z row (the apply runs on FFMA);
- d = 128, K = 112: the apply splits the clusters into two ranges so that two raw stages fit shared memory, each
  copying part of every R row;
- d = 100, K = 50: three raw stages of the apply would fit; the kernel uses two, since with an odd count a stage
  would pass between the two warpgroups.
The GPU's own R, O, E after cluster_cpp() are handed to the fp64 numpy restatement, both run the ridge step, and
Z_corr and Y must agree as in test_gpu_parity.test_ridge_step_against_plain_formulas."""
import numpy as np
import pytest

from harmony_b200 import prepare_inputs
from helpers import gpu_setup, make_perms, make_Y0, rel_l2, synthetic

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("d,K", [(150, 20), (128, 112), (100, 50)])
def test_ridge_step_wide_embeddings(d, K):
    from numpy_restatement import NumpyHarmony
    Z, meta = synthetic(6000, d, [5], n_types=12, seed=40 + d)
    a = prepare_inputs(Z, meta, "cov0", nclust=K, early_stop=False)
    N, T = Z.shape[0], a["max_iter_kmeans"]
    Y0 = make_Y0(Z, a["K"], 17)
    perms = make_perms(N, T, 31)
    g = gpu_setup(a)
    g.init_cluster_cpp(Y0)
    assert g.cluster_cpp(perms) == 0
    npy = NumpyHarmony(a["Z"], a["phi_i"], a["B_vec"], a["sigma"], a["theta"], a["lambda_"], a["alpha"], T, a["K"],
                       a["block_size"], a["batch_proportion_cutoff"])
    npy.Y = g.Y.T.astype(np.float64)
    npy.R, npy.O, npy.E = g.R.T.astype(np.float64), g.O.astype(np.float64), g.E.astype(np.float64)
    g.moe_correct_ridge_cpp()
    npy.moe_correct_ridge()
    e = rel_l2(g.getZcorr().T, npy.Z_corr)
    dY = float(np.abs(g.Y.T - npy.Y).max())
    print(f"[ridge vs plain formulas, d={d} K={K}] relL2(Z)={e:.2e} max|dY|={dY:.2e}")
    assert e <= 2e-5
    assert dY <= 5e-5
