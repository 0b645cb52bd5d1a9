"""Native update orders when a call needs more rounds than the plan buffers hold.

The native update order of every round is keyed by (seed, round counter).  A cluster_cpp call on a persistent update
path prebuilds the next call's plan, which draws the next T rounds of the counter.  When the next call does not use
it (here: max_iter_kmeans was raised), the prebuilt plan is discarded and its rounds are drawn again, whether or not
the plan buffers have to grow for the longer call.  Two handles with the same seed run the same calls:
- A is set up for 6 rounds, so its second call (6 rounds) fits the buffers and only discards the 4-round prebuild;
- B is set up for 4 rounds, so its second call also grows the buffers.
Their results may differ only by the run-to-run noise of the kernels' float atomics, which two runs of A measure.
Measured on an H100 80GB HBM3 (700 W): run-to-run max|dR| 9e-7, relative |dO| 6e-7, relative objective 1e-7; A
against B 1e-6 / 7e-7 / 2e-7.  With B's orders shifted by the 4 prebuilt rounds (no rollback when the buffers
grow) A and B differed by 2.6e-2 / 6.7e-4 / 2.6e-5."""
import numpy as np
import pytest

from harmony_b200 import prepare_inputs
from helpers import synthetic

pytestmark = pytest.mark.gpu

SEED = 11


def run(a, T_setup):
    from harmony_b200.harmony import harmony
    g = harmony()
    # epsilon_kmeans = -inf: no call stops early, so every round of the plan runs
    g.setup(a["Z"], a["phi_i"], a["sigma"], a["theta"], a["lambda_"], a["alpha"], T_setup, float("-inf"),
            a["epsilon_harmony"], a["K"], a["block_size"], a["B_vec"], a["batch_proportion_cutoff"], False)
    g.set_seed(SEED)
    g.max_iter_kmeans = 4
    g.init_cluster_cpp()
    assert g.cluster_cpp() == 0
    g.max_iter_kmeans = 6
    assert g.cluster_cpp() == 0
    assert list(g.kmeans_rounds) == [4, 6]
    return g.R.T.copy(), g.O.T.copy(), np.asarray(g.objective_kmeans)


def deviation(x, y):
    (Rx, Ox, ox), (Ry, Oy, oy) = x, y
    assert len(ox) == len(oy)
    return (float(np.abs(Rx - Ry).max()), float(np.abs(Ox - Oy).max() / np.abs(Oy).max()),
            float(np.abs(ox - oy).max() / np.abs(oy).max()))


def test_grown_plan_keeps_native_orders():
    Z, meta = synthetic(5000, 16, [4], seed=5)
    a = prepare_inputs(Z, meta, "cov0", nclust=20, early_stop=False)
    A1, A2, B = run(a, 6), run(a, 6), run(a, 4)
    noise, dev = deviation(A1, A2), deviation(A1, B)
    print(f"[plan growth] run-to-run (A, A): max|dR| {noise[0]:.2e}, rel|dO| {noise[1]:.2e}, rel|dobj| {noise[2]:.2e}; "
          f"(A, B): max|dR| {dev[0]:.2e}, rel|dO| {dev[1]:.2e}, rel|dobj| {dev[2]:.2e}")
    for d in (noise, dev):
        assert d[0] <= 1e-4 and d[1] <= 1e-5 and d[2] <= 2e-6, d
