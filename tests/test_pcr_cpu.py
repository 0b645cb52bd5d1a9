"""hb_pcr without a GPU: the restatement against a transcription of scib's pc_regression, the trace identity, the
comparison fold against scib's, the library's eigensolver against numpy.linalg.eigh, the Python refusals and the
restatement's scores of the fixtures."""
import ctypes
import warnings

import numpy as np
import pytest

import pcr_restatement as pr
from harmony_b200 import pcr, pcr_comparison
from harmony_b200.pcr import pcr_fold, pcr_on
from helpers import load_cell_lines, load_pbmc

pytest.importorskip("pandas")
pytest.importorskip("sklearn")


def _data(rng, N, d, B, shift=1.0):
    b = rng.integers(0, B, N)
    X = rng.standard_normal((N, d)) * np.linspace(3.0, 0.5, d) + rng.standard_normal((B, d))[b] * shift
    return X, b


CASES = [
    # name, N, d, B, n_comps, options
    ("n_comps_below_d", 500, 20, 4, 5, {}),
    ("n_comps_at_d", 500, 20, 4, 20, {}),
    ("n_comps_above_d", 500, 20, 4, 50, {}),
    ("N_below_d", 12, 30, 3, 50, {}),
    ("one_batch", 300, 10, 1, 10, {}),
    ("singletons_and_unused_codes", 200, 8, 4, 8, dict(singletons=True)),
    ("non_finite_rows", 400, 12, 3, 12, dict(nan=True)),
    ("offset_1e4", 600, 16, 5, 16, dict(offset=1e4)),
    ("offset_1e4_few_comps", 600, 16, 5, 3, dict(offset=1e4)),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_restatement_is_scibs(case):
    name, N, d, B, n_comps, o = case
    rng = np.random.default_rng(sum(map(ord, name)))
    X, b = _data(rng, N, d, B)
    if o.get("singletons"):   # codes 0, 3, 7, 9 of 10, two batches of one row
        b = np.array([0, 3, 7, 9])[b]
        b[:2] = [11, 12]
    if o.get("offset"):
        X += o["offset"]
    if o.get("nan"):
        X[[3, 50, 399]] = np.nan
        X[10, 4] = np.inf
        X[77, 0] = -np.inf
    r = pr.pcr(X, b, n_comps)
    keep = pr.finite(X)
    want, var, r2 = pr.scib_pc_regression(X[keep], b[keep], n_comps)
    m = len(var)
    assert r.score == pytest.approx(want, abs=1e-12)
    lam1 = r.lam[0]
    np.testing.assert_allclose(r.var[:m], var, rtol=0, atol=1e-12 * lam1 / (r.n - 1))
    gap = np.abs(np.diff(r.lam)) / lam1
    iso = np.ones(m, bool)     # a component whose eigenvalue is separated from its neighbours'
    iso[:-1] &= gap[:m - 1] >= 1e-3
    iso[1:] &= gap[:m - 1] >= 1e-3
    iso &= r.var[:m] > 1e-10 * lam1
    np.testing.assert_allclose(r.r2[:m][iso], r2[iso], rtol=0, atol=1e-10)
    if m >= min(r.n - 1, d):   # full rank: the trace identity
        assert r.score == pytest.approx(pr.trace_score(X, b), abs=1e-12)
    if B == 1:
        assert r.score == 0 and (r.r2 == 0).all()


def test_degenerate_spectrum_trace_identity():
    """Repeated eigenvalues at full rank: the per-PC R^2 are not unique, their weighted sum is tr(M) / tr(C)."""
    rng = np.random.default_rng(3)
    Q = np.linalg.qr(rng.standard_normal((10, 10)))[0]
    X = rng.standard_normal((2000, 10)) @ np.diag([2, 2, 2, 1, 1, 1, 1, 0.5, 0.5, 0.5]) @ Q
    b = rng.integers(0, 3, 2000)
    X += rng.standard_normal((3, 10))[b] * 0.3
    r = pr.pcr(X, b, 10)
    assert r.score == pytest.approx(pr.trace_score(X, b), abs=1e-13)
    assert r.score == pytest.approx(pr.scib_pc_regression(X, b, 10)[0], abs=1e-12)


def test_fold_is_scibs():
    for before, after in [(0.4, 0.1), (0.2, 0.2), (0.1, 0.3), (0.5, 0.0)]:
        for scale in (True, False):
            with warnings.catch_warnings(record=True) as w:
                warnings.simplefilter("always")
                got = pcr_fold(before, after, scale)
            assert got == pytest.approx(pr.comparison(before, after, scale), abs=1e-15)
            assert bool(w) == (scale and after > before)


def _eig(L, A):
    n = A.shape[0]
    A = np.ascontiguousarray(A, np.float64)
    w, V = np.empty(n), np.empty((n, n))
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    assert L.hb_debug_sym_eig(n, P(A), P(w), P(V)) == 0
    return w, V


def _matrices(n, rng):
    G = rng.standard_normal((n, n))
    Q = np.linalg.qr(rng.standard_normal((n, n)))[0]
    yield "random", (G + G.T) / 2
    yield "diagonal", np.diag(rng.standard_normal(n))
    rep = np.repeat(rng.standard_normal((n + 3) // 4), 4)[:n]
    yield "repeated", Q @ np.diag(rep) @ Q.T
    k = max(1, n // 3)
    F = rng.standard_normal((n, k))
    yield "rank_deficient", F @ F.T
    yield "graded", Q @ np.diag(10.0 ** -np.linspace(0, 12, n)) @ Q.T
    Y = rng.standard_normal((3 * n, n)) + 1e2
    yield "covariance", (Y - Y.mean(0)).T @ (Y - Y.mean(0))


@pytest.mark.parametrize("n", list(range(1, 17)) + [20, 31, 32, 33, 50, 64, 100, 127, 128])
def test_sym_eig_hook_is_eigh(n):
    from harmony_b200 import _lib
    L = _lib.lib()
    rng = np.random.default_rng(n)
    for name, A in _matrices(n, rng):
        A = (A + A.T) / 2
        w, V = _eig(L, A)
        norm = np.linalg.norm(A, 2)
        want = np.linalg.eigvalsh(A)[::-1]
        assert (np.diff(w) <= 0).all(), name
        np.testing.assert_allclose(w, want, rtol=0, atol=1e-13 * max(norm, 1e-300) * max(1, n / 16), err_msg=name)
        assert np.linalg.norm(A @ V - V * w, 2) <= 1e-13 * norm, name
        assert np.abs(V.T @ V - np.eye(n)).max() <= 1e-13, name
        np.testing.assert_array_equal(V, pr.sign_rule(V), err_msg=name)
    w0, V0 = np.full(4, -7.0), np.full(16, -7.0)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    for bad in (0, 129, -1):
        assert L.hb_debug_sym_eig(bad, P(np.eye(4)), P(w0), P(V0)) == 2
    assert (w0 == -7).all() and (V0 == -7).all()


def test_sym_eig_isolated_vectors_are_eighs():
    """Away from degenerate eigenspaces the vectors are eigh's, under the sign rule."""
    from harmony_b200 import _lib
    L = _lib.lib()
    rng = np.random.default_rng(5)
    for n in (7, 50, 128):
        Q = np.linalg.qr(rng.standard_normal((n, n)))[0]
        A = Q @ np.diag(np.linspace(10, 1, n)) @ Q.T
        w, V = _eig(L, (A + A.T) / 2)
        lam, U = np.linalg.eigh((A + A.T) / 2)
        np.testing.assert_allclose(V, pr.sign_rule(U[:, ::-1]), rtol=0, atol=1e-11)


def test_refusals_need_no_device(monkeypatch):
    from harmony_b200 import _lib
    monkeypatch.setattr(_lib, "lib", lambda: pytest.fail("the library was loaded"))
    rng = np.random.default_rng(8)
    X = rng.standard_normal((50, 4))
    meta = {"batch": rng.integers(0, 3, 50)}
    calls = [(dict(X=X[:, 0]), ValueError, "X must be an [N, d] matrix"),
             (dict(X=np.zeros((50, 129))), ValueError, "d = 129 is not supported (1 <= d <= 128)"),
             (dict(X=np.zeros((50, 0))), ValueError, "d = 0 is not supported (1 <= d <= 128)"),
             (dict(X=X[:1], meta_data={"batch": [0]}), ValueError, "X has 1 rows, at least 2 are needed"),
             (dict(n_comps=0), ValueError, "n_comps = 0, at least one component is needed"),
             (dict(n_comps=2.5), ValueError, "n_comps must be an integer, not 2.5"),
             (dict(n_comps=True), ValueError, "n_comps must be an integer, not True"),
             (dict(meta_data={"batch": meta["batch"][:49]}), ValueError,
              "column 'batch' must hold one label per row of X (50)"),
             (dict(batch_key="nope"), ValueError, "meta_data has no column 'nope'"),
             (dict(meta_data={"batch": np.where(meta["batch"] == 1, np.nan, meta["batch"])}), ValueError,
              "column 'batch' holds missing labels"),
             (dict(meta_data=meta["batch"]), ValueError, "meta_data must be a DataFrame or a dict of columns")]
    for change, exc, msg in calls:
        args = dict(dict(X=X, meta_data=meta, batch_key="batch"), **change)
        with pytest.raises(exc) as e:
            pcr(**args)
        assert str(e.value) == msg, change
    with pytest.raises(ValueError) as e:
        pcr_comparison(X, X[:40], meta, "batch")
    assert str(e.value) == "X_before has 50 rows and X_after 40: they must hold the same cells"
    with pytest.raises(ValueError) as e:
        pcr_comparison(X, X, meta, "batch", n_comps=-1)
    assert str(e.value) == "n_comps = -1, at least one component is needed"
    with pytest.raises(ValueError) as e:
        pcr_comparison(X, X, {"batch": meta["batch"][1:]}, "batch")
    assert str(e.value) == "column 'batch' must hold one label per row of X (50)"
    obj = object()   # pcr_on refuses by shape before it touches the object
    with pytest.raises(ValueError, match=r"batches must be \[50\]"):
        pcr_on(obj, X, meta["batch"][:40])
    with pytest.raises(ValueError, match="n_comps = 0"):
        pcr_on(obj, X, meta["batch"], 0)
    with pytest.raises(TypeError, match="batches must be integers"):
        pcr_on(obj, X, meta["batch"].astype(float))


def test_restatement_scores_fixtures():
    Z, meta = load_cell_lines(True)
    assert pr.pcr(Z, meta["dataset"]).score == pytest.approx(0.4830351865, abs=1e-10)
    Z, meta = load_cell_lines(False)
    assert pr.pcr(Z, meta["dataset"], 50).score == pytest.approx(0.4685829545, abs=1e-10)
    assert pr.pcr(Z, meta["dataset"], 5).score == pytest.approx(0.5594197236, abs=1e-10)
    assert pr.trace_score(Z, meta["dataset"]) == pytest.approx(0.4685829545, abs=1e-10)
    Z, meta = load_pbmc()
    assert pr.pcr(Z, meta["stim"]).score == pytest.approx(0.0178766554, abs=1e-10)
