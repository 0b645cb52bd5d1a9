"""End-to-end tests through RunHarmony() with the native (seeded) k-means initialisation and update
orders — the reference's own testthat files, test for test
(/root/reference/tests/testthat/test_integration.R, test_two_variable.R), plus determinism and
size-independent properties at BASELINE.json's 1M-cell configuration."""
import numpy as np
import pytest

from harmony_b200 import RunHarmony, harmony_options
from helpers import load_cell_lines, load_pbmc, synthetic

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def obj_small():
    Z, meta = load_cell_lines(True)
    # test_integration.R:5-7
    return RunHarmony(Z, meta, "dataset", theta=1, nclust=50, max_iter=5, return_object=True, verbose=False,
                      options=harmony_options(max_iter_cluster=10), seed=1)


def test_dimensions_match(obj_small):
    obj = obj_small  # test_integration.R:9-14
    assert obj.Y.shape == (obj.d, obj.K)
    assert obj.getZcorr().shape == (obj.d, obj.N)
    assert obj.getZorig().shape == (obj.d, obj.N)
    assert obj.R.shape == (obj.K, obj.N)


def test_R_is_a_probability_distribution(obj_small):
    R = obj_small.R  # test_integration.R:16-20
    assert R.min() >= 0 and R.max() <= 1
    np.testing.assert_allclose(R.sum(axis=0), 1.0, atol=1e-5)


def test_no_null_values(obj_small):
    Z = obj_small.getZcorr()  # test_integration.R:22-26
    assert np.all(np.isfinite(Z))


def _chi2(o):
    return float((((o.O - o.E) ** 2) / o.E).sum())


def test_theta_decreases_chi2():
    Z, meta = load_cell_lines(True)  # test_integration.R:29-41
    o0 = RunHarmony(Z, meta, "dataset", theta=0, nclust=20, max_iter=2, return_object=True, verbose=False, seed=2)
    o1 = RunHarmony(Z, meta, "dataset", theta=1, nclust=5, max_iter=2, return_object=True, verbose=False, seed=2)
    assert _chi2(o0) > _chi2(o1)


def test_error_messages():
    Z, meta = load_cell_lines(True)  # test_integration.R:43-55
    with pytest.raises(ValueError):
        RunHarmony(Z, meta, "fake_variable", verbose=False)
    with pytest.raises(ValueError):
        RunHarmony(Z, meta, "dataset", lambda_=[1, 2], verbose=False)
    with pytest.raises(ValueError):
        RunHarmony(Z, {k: v[:-1] for k, v in meta.items()}, "dataset", verbose=False)
    with pytest.raises(TypeError):
        RunHarmony(Z, meta, "dataset", tau=1, verbose=False)   # legacy argument


def test_two_variable_run():
    Z, meta = load_cell_lines(False)  # test_two_variable.R:5-55
    obj = RunHarmony(Z, meta, ["cell_type", "dataset"], theta=[1, 1], nclust=50, max_iter=10, return_object=True,
                     verbose=False, options=harmony_options(max_iter_cluster=10), seed=3)
    assert obj.Y.shape == (obj.d, obj.K) and obj.R.shape == (obj.K, obj.N)
    assert obj.O.shape[1] == 5 and obj.E.shape[1] == 5
    R = obj.R
    assert R.min() >= 0 and R.max() <= 1
    np.testing.assert_allclose(R.sum(axis=0), 1.0, atol=1e-5)
    assert np.all(np.isfinite(obj.getZcorr()))
    lo = RunHarmony(Z, meta, ["cell_type", "dataset"], theta=[0, 0], nclust=20, max_iter=2, return_object=True,
                    verbose=False, seed=4)
    hi = RunHarmony(Z, meta, ["cell_type", "dataset"], theta=[2, 2], nclust=20, max_iter=2, return_object=True,
                    verbose=False, seed=4)
    assert _chi2(lo) > _chi2(hi)


def test_returns_embedding_and_mixes_batches():
    """Default call returns cells x PCs; on pbmc_stim (config 2) the stim/ctrl batches mix: the mean
    per-cluster batch imbalance drops markedly."""
    Z, meta = load_pbmc()
    out = RunHarmony(Z, meta, "stim", nclust=50, verbose=False, seed=5)
    assert out.shape == Z.shape and np.all(np.isfinite(out))
    obj = RunHarmony(Z, meta, "stim", nclust=50, verbose=False, seed=5, return_object=True)
    first = RunHarmony(Z, meta, "stim", nclust=50, verbose=False, seed=5, return_object=True, max_iter=0)
    assert _chi2(obj) < _chi2(first)
    assert len(obj.objective_harmony) == len(obj.kmeans_rounds) + 1


def test_seed_reproducible_and_seed_dependent():
    Z, meta = synthetic(5000, 20, [4], seed=9)
    a = RunHarmony(Z, meta, "cov0", nclust=20, max_iter=3, verbose=False, seed=11)
    b = RunHarmony(Z, meta, "cov0", nclust=20, max_iter=3, verbose=False, seed=11)
    c = RunHarmony(Z, meta, "cov0", nclust=20, max_iter=3, verbose=False, seed=12)
    assert np.linalg.norm(a - b) / np.linalg.norm(a) < 1e-5      # same seed: same orders (atomics reorder sums)
    assert np.linalg.norm(a - c) / np.linalg.norm(a) > 1e-6      # another seed: another run


def test_properties_at_full_size():
    """BASELINE.json config 3 (1M cells x 50 PCs, 20 batches, K=100): size-independent invariants."""
    import sys
    import os
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from bench import synth_shard
    from harmony_b200.harmony import harmony
    N = 1_000_000
    Z, b = synth_shard(N, 0, 123)
    g = harmony()
    g.setup(Z, b.reshape(-1, 1), np.full(100, 0.1), np.full(20, 2.0), None, 0.2, 4, 1e-3, -np.inf, 100, 0.05,
            np.array([20], dtype=np.int32), 1e-5)
    g.set_seed(7)
    g.init_cluster_cpp()
    N_b = np.bincount(b[:, 0], minlength=20)
    for it in range(2):
        assert g.cluster_cpp() == 0
        O, E = g.O, g.E
        # O column sums = batch sizes, E column sums = batch sizes, rows of O and E agree (sum_b O_kb = sum_i R_ik)
        np.testing.assert_allclose(O.sum(axis=0), N_b, rtol=2e-4)
        np.testing.assert_allclose(E.sum(axis=0), N_b, rtol=2e-4)
        np.testing.assert_allclose(O.sum(axis=1), E.sum(axis=1), rtol=2e-4)
        g.moe_correct_ridge_cpp()
        g.check_convergence(1)
    R = g.R
    np.testing.assert_allclose(R.sum(axis=0), 1.0, atol=2e-5)
    assert R.min() >= 0
    np.testing.assert_allclose(R.sum(axis=1), g.O.sum(axis=1), rtol=2e-4)   # O is consistent with the stored R
    Zc = g.getZcorr()
    assert np.all(np.isfinite(Zc))
    np.testing.assert_allclose(np.linalg.norm(g.Y, axis=0), 1.0, atol=1e-5)  # centroids are unit vectors
    ok = g.objective_kmeans
    assert len(ok) == 1 + 2 * 4 and np.all(np.isfinite(ok))
    # idempotence of the read path and un-sorting: getZorig returns the input (fp32-rounded), in input order
    np.testing.assert_array_equal(g.getZorig().T[:1000], Z[:1000].astype(np.float32))


def test_library_reproduces_the_tables_printed_by_the_reference_vignette():
    """Same golden values as tests/test_oracle.py (doc/detailedWalkthrough.html:656-708 of the reference), through
    the C ABI: init_cluster_cpp with the matching centroids must leave round(O), round(E) equal to the 30 integers
    the reference printed (the closest value to a rounding boundary, 398.52, is 0.02 away — 20x the fp32 error)."""
    import os
    from harmony_b200 import prepare_inputs
    from helpers import GOLDEN, gpu_setup
    g = np.load(os.path.join(GOLDEN, "vignette_walkthrough.npz"))
    Z, meta = load_cell_lines(small=False)
    a = prepare_inputs(Z, meta, "dataset", nclust=5, theta=1.0)
    h = gpu_setup(a, device=0)
    h.init_cluster_cpp(g["Y"])
    assert np.array_equal(np.round(np.asarray(h.O)), g["O_init"])
    assert np.array_equal(np.round(np.asarray(h.E)), g["E_init"])
    R = np.asarray(h.R)                      # K x N like harmonyObj$R
    ct = np.stack([(meta["cell_type"] == lv) for lv in ("jurkat", "t293")], axis=1).astype(np.float64)
    assert np.abs(np.round(R @ ct) - g["celltype_init"]).max() <= 1


# update orders 0-3 under the default kernels (fused wgmma at this shape; ids "0" .. "3"), the FFMA contractions
# (HB_KS_FFMA_CONTRACTIONS = 1) and the wide kernels (HB_KS_WIDE = 16)
@pytest.mark.parametrize("seed,kernel_set", [pytest.param(s, ks, id=str(s) if ks == 0 else f"{s}-ks{ks}")
                                             for ks in (0, 1, 16) for s in (0, 1, 2, 3)])
def test_library_reproduces_the_vignette_tables_after_cluster_cpp(seed, kernel_set):
    """The tables the reference's vignette prints after `max_iter_kmeans <- 10; cluster_cpp()`
    (doc/detailedWalkthrough.html:733-786) through the C ABI, with the centroid step of harmony.cpp:235-238
    switched on as in the package version that rendered them: 25 integers, exactly, for any update order, after
    exactly 5 rounds (see tests/test_oracle.py for the same check on the restatements), whichever kernel the step's
    assignment runs on."""
    import os
    from harmony_b200 import prepare_inputs
    from helpers import GOLDEN, gpu_setup, make_perms
    g = np.load(os.path.join(GOLDEN, "vignette_walkthrough.npz"))
    Z, meta = load_cell_lines(small=False)
    a = prepare_inputs(Z, meta, "dataset", nclust=5, theta=1.0)
    h = gpu_setup(a, T=10, kernel_set=kernel_set, device=0)
    h.legacy_centroid_step = 1
    assert h.legacy_centroid_step == 1
    h.init_cluster_cpp(g["Y"])
    assert h.cluster_cpp(make_perms(Z.shape[0], 10, seed)) == 0
    assert int(h.kmeans_rounds[-1]) == 5
    assert np.array_equal(np.round(np.asarray(h.O)), g["O_clustered"])
    ct = np.stack([(meta["cell_type"] == lv) for lv in ("jurkat", "t293")], axis=1).astype(np.float64)
    counts = np.asarray(h.R) @ ct
    assert np.array_equal(np.round(counts), g["celltype_clustered"])
    err = (counts / counts.sum(axis=1, keepdims=True)).min(axis=1) * 100.0
    assert np.abs(err - g["error_rate_clustered"]).max() < 2e-3


def test_abort_callback_stops_cluster_cpp():
    """hb_set_abort_callback = Progress::check_abort (harmony.cpp:233): cluster_cpp returns -1 once the callback
    says so, harmonize() reports "terminated by user" like R/utils.R:27-29, and the object stays usable."""
    from harmony_b200 import prepare_inputs
    from harmony_b200.utils import harmonize
    from helpers import gpu_setup, make_Y0
    Z, meta = load_cell_lines(True)
    a = prepare_inputs(Z, meta, "dataset", nclust=5, early_stop=False)
    g = gpu_setup(a, device=0)
    g.init_cluster_cpp(make_Y0(Z, a["K"], 0))
    calls, state = [], {"abort": False}
    g.set_abort_callback(lambda: calls.append(1) or state["abort"])
    assert g.cluster_cpp() == 0            # polled, not yet aborting
    g.moe_correct_ridge_cpp()
    assert len(calls) >= 1
    state["abort"] = True
    with pytest.raises(KeyboardInterrupt):
        harmonize(g, 5, verbose=False)
    g.set_abort_callback(None)
    assert g.cluster_cpp() == 0            # the handle survives an abort
