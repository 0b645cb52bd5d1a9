"""hb_lisi without a GPU: the fp64 restatement against a literal loop over a cKDTree search, its invariants, the
refusals of compute_lisi and the geometry of the search."""
import ctypes
import math

import numpy as np
import pytest
from scipy.spatial import cKDTree

import knn_restatement as kr
import lisi_restatement as lr
from harmony_b200 import compute_lisi


def literal(X, label_sets, p):
    """The package's rules as plain loops: 3 p neighbours with the cell itself by cKDTree, the first column dropped,
    the bisection on unshifted distances (a zero sum of weights gives H = 0), 1 / Simpson per label set."""
    dd, ii = cKDTree(X).query(X, k=int(3 * p))
    D, I = dd[:, 1:], ii[:, 1:]
    out, underflow = np.empty((len(X), len(label_sets))), False
    for i in range(len(X)):
        beta, bmin, bmax = 1.0, -math.inf, math.inf
        for _ in range(50):
            P = np.exp(-D[i] * beta)
            total = P.sum()
            if total == 0:
                H, P, underflow = 0.0, np.zeros_like(P), True
            else:
                H = math.log(total) + beta * float((D[i] * P).sum()) / total
                P = P / total
            diff = H - math.log(p)
            if abs(diff) < 1e-5:
                break
            if diff > 0:
                bmin = beta
                beta = 2 * beta if math.isinf(bmax) else (beta + bmax) / 2
            else:
                bmax = beta
                beta = beta / 2 if math.isinf(bmin) else (beta + bmin) / 2
        for s, codes in enumerate(label_sets):
            if H == 0:
                out[i, s] = -1.0
                continue
            mass = {}
            for j, pj in zip(I[i], P):
                mass[codes[j]] = mass.get(codes[j], 0.0) + pj
            out[i, s] = 1.0 / sum(m * m for m in mass.values())
    return out, underflow


def _data(seed, n=400, d=6, types=5, scale=1.0):
    rng = np.random.default_rng(seed)
    M = rng.standard_normal((types, d)) * 3.0
    t = rng.integers(0, types, n)
    X = (M[t] + rng.standard_normal((n, d))) * scale
    batch = rng.integers(0, 3, n)
    return X, np.stack([batch, t, rng.integers(0, 40, n)])


@pytest.mark.parametrize("p,scale", [(5, 1.0), (10, 0.3), (30, 1.0), (30, 0.05)])
def test_restatement_matches_a_literal_loop(p, scale):
    X, labels = _data(p, scale=scale)
    got, flag = lr.lisi(X, labels, p)
    want, underflow = literal(X, labels, p)
    assert not underflow, "choose data where the unshifted weights do not underflow"
    keep = ~flag
    assert keep.mean() > 0.95
    np.testing.assert_allclose(got[keep], want[keep], rtol=1e-9)
    idx, dist = lr.neighbours(X, p)
    dd, ii = cKDTree(X).query(X, k=int(3 * p))
    np.testing.assert_array_equal(idx, ii[:, 1:])
    np.testing.assert_allclose(dist, dd[:, 1:], rtol=1e-9)


def test_shifted_entropy_is_the_unshifted_one():
    rng = np.random.default_rng(3)
    dist = np.sort(rng.uniform(0.5, 3.0, (200, 29)), axis=1)
    P, H, _, beta = lr.calibrate(dist, 10)
    E = np.exp(-beta[:, None] * dist)
    H0 = np.log(E.sum(1)) + beta * (dist * E).sum(1) / E.sum(1)
    np.testing.assert_allclose(H, H0, rtol=1e-12)
    np.testing.assert_allclose(P, E / E.sum(1, keepdims=True), rtol=1e-12)


def test_invariants():
    p = 30
    X, labels = _data(7, n=600, d=8)
    out, flag = lr.lisi(X, labels, p)
    # one label: 1
    one, _ = lr.lisi(X, np.zeros((1, len(X)), int), p)
    np.testing.assert_allclose(one, 1.0, rtol=1e-12)
    # exp(H) within the tolerance of p
    idx, dist = lr.neighbours(X, p)
    _, H, _, _ = lr.calibrate(dist, p)
    assert (np.abs(H - math.log(p)) < 1e-5).all()
    # relabelling the codes (a bijection onto negative and large values) changes nothing
    perm = np.array([-2 ** 31, 7, 2 ** 31 - 1, -5, 123456789] + list(range(1000, 1035)))
    again, _ = lr.lisi(X, perm[labels], p)
    np.testing.assert_array_equal(again, out)
    # 1 <= LISI <= the number of distinct labels among the neighbours
    for s in range(len(labels)):
        distinct = np.array([len(np.unique(labels[s][r])) for r in idx])
        assert (out[:, s] >= 1 - 1e-12).all() and (out[:, s] <= distinct + 1e-9).all()
    assert flag.mean() < 0.01


@pytest.mark.parametrize("k", [2, 29, 89])
def test_equal_distances(k):
    """Every neighbour at one distance: P = 1 / k, and LISI = 1 / sum_b (n_b / k)^2 for n_b neighbours with label b
    (H = ln k stays off ln p, so all 50 evaluations run; beta ends near 2^50)."""
    p = (k + 1) / 3
    assert lr.neighbours_for(p) == k
    idx = np.array([np.delete(np.arange(k + 1), i) for i in range(k + 1)])
    dist = np.full(idx.shape, 3.0 * math.sqrt(2.0))
    codes = np.arange(k + 1) % 3
    out, _ = lr.lisi(None, codes[None], p, idx, dist)
    for i in range(k + 1):
        n_b = np.bincount(np.delete(codes, i), minlength=3)
        assert out[i, 0] == pytest.approx(1.0 / ((n_b / k) ** 2).sum(), rel=1e-12)


def test_special_rows():
    X, labels = _data(9, n=200)
    X[[3, 50]] = np.nan
    X[7, 2] = np.inf
    out, _ = lr.lisi(X, labels, 10)
    assert np.isnan(out[[3, 7, 50]]).all() and not np.isnan(np.delete(out, [3, 7, 50], 0)).any()
    # one neighbour left: all weight on it, H = 0
    Y = np.array([[0.0], [1.0], [np.nan], [np.nan]])
    out, _ = lr.lisi(Y, np.zeros((1, 4), int), 1)
    assert (out[:2] == -1).all() and np.isnan(out[2:]).all()


def test_compute_lisi_refusals_need_no_device(monkeypatch):
    from harmony_b200 import _lib
    monkeypatch.setattr(_lib, "lib", lambda: pytest.fail("the library was loaded"))
    X, labels = _data(5, n=100)
    meta = {"batch": labels[0], "type": labels[1]}
    missing = "column 'batch' holds missing labels"
    bad = [(dict(perplexity=0.5), "perplexity must be finite and at least 1, not 0.5"),
           (dict(perplexity=float("nan")), "perplexity must be finite and at least 1, not nan"),
           (dict(perplexity=float("inf")), "perplexity must be finite and at least 1, not inf"),
           (dict(perplexity=43.34), "perplexity 43.34 needs k = floor(3 p) - 1 = 129 neighbours; at most 128 "
                                    "(perplexity < 43 1/3)"),
           (dict(perplexity=34), "perplexity 34 needs k = 101 neighbours, 100 rows have 99"),
           (dict(perplexity=True), "perplexity must be a number, not True"),
           (dict(perplexity="30"), "perplexity must be a number, not '30'"),
           (dict(X=X[:, 0]), "X must be an [N, d] matrix"),
           (dict(X=np.zeros((100, 129))), "d = 129 is not supported (1 <= d <= 128)"),
           (dict(X=np.zeros((100, 0))), "d = 0 is not supported (1 <= d <= 128)"),
           (dict(label_colnames=[]), "label_colnames names no column"),
           (dict(label_colnames="nope"), "meta_data has no column 'nope'"),
           (dict(meta_data=labels[0]), "meta_data must be a DataFrame or a dict of columns"),
           (dict(meta_data={"batch": labels[0][:99]}), "column 'batch' must hold one label per row of X (100)"),
           (dict(meta_data={"batch": np.where(labels[0] == 1, np.nan, labels[0])}), missing),
           (dict(meta_data={"batch": np.array(["a", None] * 50, dtype=object)}), missing),
           (dict(meta_data={"batch": np.array(["a", float("nan")] * 50, dtype=object)}), missing)]
    for change, msg in bad:
        kw = dict(X=X, meta_data=meta, label_colnames="batch", perplexity=10)
        kw.update(change)
        with pytest.raises(ValueError) as e:
            compute_lisi(kw.pop("X"), **kw)
        assert e.type is ValueError and str(e.value) == msg, change


def _geometry(d, p, N, sms):
    from harmony_b200 import _lib
    out = (ctypes.c_int64 * 8)(*([-7] * 8))
    return _lib.lib().hb_debug_lisi_geometry(d, p, N, sms, out), list(out)


def _knn_geometry(d, k, N, sms):
    from harmony_b200 import _lib
    out = (ctypes.c_int64 * 8)(*([-7] * 8))
    return _lib.lib().hb_debug_knn_geometry(d, k, N, N, sms, out), list(out)


def test_geometry_hook_matches_the_rule():
    seen = set()
    for p in (1, 21, 21.67, 22, 30, 36, 43):         # k = 2, 62, 64, 65, 89, 107, 128
        k = lr.neighbours_for(p)
        for d in range(1, 129):
            for N in (k + 1, 1000, 20_000, 1_000_000):
                st, g = _geometry(d, p, N, 132)
                assert st == 0 and g == lr.geometry(d, p, N, 132), (d, p, N, g)
                tq, tn, stages, splits, smem, per, KD, threads = g
                seen.add((tq, stages))
                assert smem <= 227 * 1024 and (splits - 1) * per * tn < N <= splits * per * tn and splits * k <= 1024
                if k <= 64:   # the same search as hb_knn's
                    assert _knn_geometry(d, k, N, 132) == (0, g)
                else:
                    assert _knn_geometry(d, k, N, 132)[0] == 2
    assert seen == {(128, 2), (128, 1), (64, 2), (64, 1)}
    # (64, 1) is reached by k > 64 only: d = 128 from k = 107 and d = 120 at k = 128
    assert _geometry(128, 36, 5000, 132)[1][:3] == [64, 64, 1]
    assert _geometry(120, 43, 5000, 132)[1][:3] == [64, 64, 1]
    assert _geometry(128, 35, 5000, 132)[1][:3] == [64, 64, 2]      # k = 104
    assert _geometry(112, 43, 5000, 132)[1][:3] == [64, 64, 2]
    for k in range(1, 65):
        for d in range(1, 129):
            assert tuple(kr.geometry(d, k, 1000, 1000, 132)[:3:2]) != (64, 1)
    assert [lr.neighbours_for(p) for p in (1, 21, 21.67, 22, 30, 36, 43, 43.33)] == [2, 62, 64, 65, 89, 107, 128, 128]


def test_geometry_hook_refusals():
    for d, p, N in ((0, 30, 1000), (129, 30, 1000), (50, 0.999, 1000), (50, float("nan"), 1000),
                    (50, float("inf"), 1000), (50, 130 / 3, 1000), (50, 30, 89), (50, 30, 2 ** 31)):
        assert _geometry(d, p, N, 132) == (2, [-7] * 8), (d, p, N)
    assert _geometry(50, 30, 90, 132)[0] == 0 and _geometry(50, 43, 129, 132)[0] == 0 and _geometry(1, 1, 3, 132)[0] == 0
