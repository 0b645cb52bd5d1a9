"""Mapping a query onto a reference, without a GPU: the maths of the fp64 restatement, the reference's file format and
MapQuery's argument checks."""
import numpy as np
import pytest

from harmony_b200 import HarmonyReference, MapQuery, prepare_inputs
from helpers import synthetic
from map_restatement import (correct, lambda_levels, map_query, reference_stats, weights_dense, weights_folded)


def _query(rng, N, d, K, B_vec, absent=(), zero_nr=None):
    """Random query labels over B_vec (levels in `absent` never used), Z, a row-stochastic R and a reference."""
    phi = []
    off = 0
    for Bc in B_vec:
        lv = np.array([b for b in range(Bc) if off + b not in absent])
        phi.append(off + rng.choice(lv, N))
        off += Bc
    phi = np.stack(phi, axis=1)
    Z = rng.standard_normal((N, d)) * 3.0
    A = np.exp(rng.standard_normal((N, K)) * 2.0)
    R = A / A.sum(axis=1, keepdims=True)
    Nr = rng.uniform(10.0, 100.0, K)
    Cref = rng.standard_normal((K, d)) * Nr[:, None]
    if zero_nr is not None:
        Nr[zero_nr] = 0.0
        Cref[zero_nr] = 0.0
    return phi, Z, R, Nr, Cref


@pytest.mark.parametrize("B_vec,absent,zero_nr", [
    ([3], (), None),
    ([1], (), None),                 # a single query level
    ([4, 3], (), None),
    ([2, 3, 2], (), None),
    ([4], (1, 3), None),             # declared levels absent from the query
    ([3, 4], (4,), 2),               # ... and a cluster without reference mass
    ([2], (), 0),
])
def test_folded_solve_matches_dense(B_vec, absent, zero_nr):
    rng = np.random.default_rng(len(B_vec) * 10 + len(absent))
    phi, Z, R, Nr, Cref = _query(rng, 300, 7, 5, B_vec, absent, zero_nr)
    B = sum(B_vec)
    lam = rng.uniform(0.1, 2.0, B)
    Wd = weights_dense(R, Z, phi, B, lam, Nr, Cref)
    Wf = weights_folded(R, Z, phi, B, lam, Nr, Cref)
    assert np.abs(Wf - Wd).max() <= 1e-10 * max(1.0, np.abs(Wd).max())
    out = correct(Z, R, phi, Wf)
    assert np.isfinite(out).all()
    if len(B_vec) == 1 and B_vec[0] == 1:
        assert np.abs(out - Z).max() > 1e-3   # one query batch is corrected, not left alone


def test_empty_cluster_contributes_nothing():
    rng = np.random.default_rng(3)
    phi, Z, R, Nr, Cref = _query(rng, 100, 5, 4, [2], zero_nr=1)
    R[:, 1] = 0.0                              # no query mass either: G_k[0, 0] == 0
    W = weights_folded(R, Z, phi, 2, np.ones(2), Nr, Cref)
    assert np.all(W[1] == 0) and np.isfinite(W).all()


def test_planted_reference_cells_map_back():
    """Query = the reference's own cells shifted by a constant, with their own R and lambda -> 0: the mapping returns
    the reference's Z_corr exactly (the reference anchors each intercept, the one query level absorbs the shift)."""
    rng = np.random.default_rng(7)
    N, d, K = 2000, 10, 12
    Zc = rng.standard_normal((N, d)) * 4.0
    A = np.exp(rng.standard_normal((N, K)) * 2.0)
    R = A / A.sum(axis=1, keepdims=True)
    Nr, Cref, Y = reference_stats(Zc, R)
    shift = rng.standard_normal(d) * 5.0
    phi = np.zeros((N, 1), dtype=np.int64)
    out, _ = map_query(Zc + shift, phi, [1], [1e-8], Y, Nr, Cref, np.full(K, 0.1), R=R)
    assert np.abs(out - Zc).max() <= 1e-6


def test_lambda_broadcast():
    np.testing.assert_array_equal(lambda_levels(0.5, [2, 3]), np.full(5, 0.5))
    np.testing.assert_array_equal(lambda_levels([1.0, 2.0], [2, 3]), [1, 1, 2, 2, 2])


def _reference(K=6, d=4, seed=0):
    rng = np.random.default_rng(seed)
    C = rng.standard_normal((K, d))
    return HarmonyReference(C / np.linalg.norm(C, axis=1, keepdims=True), rng.uniform(1, 9, K), C * 3,
                            np.full(K, 0.1))


@pytest.mark.parametrize("suffix", [".npz", ""])
def test_reference_save_load_round_trip(tmp_path, suffix):
    ref = _reference()
    path = str(tmp_path / f"ref{suffix}")
    ref.save(path)
    back = HarmonyReference.load(path)
    for f in HarmonyReference.FIELDS:
        np.testing.assert_array_equal(getattr(back, f), getattr(ref, f))
    assert (back.K, back.d) == (6, 4)


def test_reference_rejects_inconsistent_arrays():
    with pytest.raises(ValueError):
        HarmonyReference(np.zeros((3, 4)), np.ones(3), np.zeros((3, 5)), np.ones(3))
    with pytest.raises(ValueError):
        HarmonyReference(np.zeros((3, 4)), np.ones(3), np.zeros((3, 4)), np.ones(2))


def test_map_query_checks_arguments_before_the_device():
    """Each of these is refused by the argument checks, before a harmony object (and so a GPU) is needed."""
    ref = _reference(d=4)
    Z = np.random.default_rng(0).standard_normal((50, 4))
    meta = {"batch": np.repeat([0, 1], 25), "other": np.zeros(50)}
    with pytest.raises(ValueError, match="dimensions"):
        MapQuery(Z[:, :3], meta, "batch", ref, verbose=False)
    for bad in (0.0, -1.0, [1.0, 0.0], np.nan):
        with pytest.raises(ValueError, match="positive"):
            MapQuery(Z, meta, ["batch", "other"], ref, lambda_=bad, verbose=False)
    with pytest.raises(ValueError, match="per covariate"):
        MapQuery(Z, meta, "batch", ref, lambda_=[1.0, 2.0], verbose=False)
    with pytest.raises(ValueError, match="variables names"):
        MapQuery(Z, meta, "nope", ref, verbose=False)
    with pytest.raises(ValueError, match="variables names"):
        MapQuery(Z, meta, None, ref, verbose=False)
    with pytest.raises(TypeError):
        MapQuery(Z, meta, "batch", {"centroids": ref.centroids}, verbose=False)


def test_prepare_inputs_unchanged_by_the_label_helper():
    """prepare_inputs still factorises the labels into the same phi_i / B_vec / theta it did."""
    Z, meta = synthetic(300, 6, [3, 4], seed=2)
    a = prepare_inputs(Z, meta, ["cov0", "cov1"], nclust=5, lambda_=[1.0, 2.0])
    lv0, lv1 = np.unique(meta["cov0"]), np.unique(meta["cov1"])
    np.testing.assert_array_equal(a["B_vec"], [len(lv0), len(lv1)])
    np.testing.assert_array_equal(a["phi_i"][:, 0], np.searchsorted(lv0, meta["cov0"]))
    np.testing.assert_array_equal(a["phi_i"][:, 1], len(lv0) + np.searchsorted(lv1, meta["cov1"]))
    np.testing.assert_array_equal(a["lambda_"], np.r_[0.0, np.repeat([1.0, 2.0], a["B_vec"])])
