"""hb_silhouette without a GPU: the fp64 restatement against sklearn's silhouette_samples, with groups and non-finite
rows, the scib folds against literal loops of scib's code, the Python refusals and the geometry of the sweep."""
import ctypes

import numpy as np
import pytest

import silhouette_restatement as sr
from harmony_b200 import silhouette_batch, silhouette_label, silhouette_samples
from harmony_b200.silhouette import batch_fold

sklearn_metrics = pytest.importorskip("sklearn.metrics")


def _data(seed, n=300, d=5, types=4):
    rng = np.random.default_rng(seed)
    M = rng.standard_normal((types, d)) * 2.0
    t = rng.integers(0, types, n)
    return M[t] + rng.standard_normal((n, d)), t


@pytest.mark.parametrize("case", ["plain", "two_labels", "singletons", "duplicates", "all_equal", "unused_codes"])
def test_restatement_is_sklearn(case):
    X, t = _data(len(case))
    if case == "two_labels":
        t = t % 2
    if case == "singletons":      # labels with one row: s = 0
        t = t.copy()
        t[[0, 5, 9]] = [10, 11, 12]
    if case == "duplicates":      # exact duplicates inside and across labels
        X[100:150] = X[:50]
        X = np.round(X * 4) / 4
    if case == "all_equal":       # a = b = 0 for every row: 0 / 0 -> 0
        X = np.ones((40, 3))
        t = np.arange(40) % 3
    if case == "unused_codes":    # codes 0, 7, 20: levels that no row has play no part
        t = np.array([0, 7, 20, 7])[t]
    want = sklearn_metrics.silhouette_samples(X, t)
    got = sr.silhouette(X, t)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)
    if case == "singletons":
        assert (got[[0, 5, 9]] == 0).all()
    if case == "all_equal":
        assert (got == 0).all()


def test_groups_are_sklearn_per_group():
    X, t = _data(3, n=500)
    rng = np.random.default_rng(3)
    g = rng.integers(0, 4, len(X))
    g[:7] = 9              # a group of one label: NaN
    t[:7] = 2
    got = sr.silhouette(X, t, g)
    for grp in (0, 1, 2, 3):
        rows = g == grp
        np.testing.assert_allclose(got[rows], sklearn_metrics.silhouette_samples(X[rows], t[rows]), rtol=0, atol=1e-12)
    assert np.isnan(got[:7]).all()
    one = sr.silhouette(X[:1], t[:1], g[:1])   # a group of one row
    assert np.isnan(one).all()


def test_non_finite_rows():
    X, t = _data(5)
    bad = [3, 40, 41, 200]
    X[3] = np.nan
    X[40, 1] = np.inf
    X[41, 0] = -np.inf
    X[200, 2] = 1e20           # |x - c|^2 overflows fp32 (the centre moves by 1e20 / N only)
    got = sr.silhouette(X, t)
    assert np.isnan(got[bad]).all()
    keep = np.setdiff1d(np.arange(len(X)), bad)
    np.testing.assert_allclose(got[keep], sklearn_metrics.silhouette_samples(X[keep], t[keep]), rtol=0, atol=1e-12)
    fin, _, _ = sr.finite_rows(X)
    assert (np.nonzero(~fin)[0] == bad).all()


def scib_silhouette_batch(X, batch, label, scale=True):
    """scib.metrics.silhouette_batch, its loops as published, on arrays"""
    sil_per_label = []
    for group in list(dict.fromkeys(label)):          # adata.obs[label_key].unique()
        rows = label == group
        n_batches = len(set(batch[rows]))
        if (n_batches == 1) or (n_batches == rows.sum()):
            continue
        sil = sklearn_metrics.silhouette_samples(X[rows], batch[rows])
        sil = [abs(i) for i in sil]
        if scale:
            sil = [1 - i for i in sil]
        sil_per_label.extend([(group, score) for score in sil])
    if len(sil_per_label) == 0:
        return np.nan, {}
    means = {}
    for group, score in sil_per_label:
        means.setdefault(group, []).append(score)
    means = {k: float(np.mean(v)) for k, v in means.items()}
    return float(np.mean(list(means.values()))), means


@pytest.mark.parametrize("scale", [True, False])
def test_batch_fold_is_scib(scale):
    X, t = _data(11, n=400)
    rng = np.random.default_rng(11)
    batch = rng.integers(0, 3, len(X))
    t[:5] = 7                      # a cell type in one batch: skipped
    batch[:5] = 0
    t[5:8] = 8                     # as many batches as cells: skipped
    batch[5:8] = [0, 1, 2]
    s = sr.silhouette(X, batch, t)
    asw, means = batch_fold(s, batch, t, scale)
    want, want_means = scib_silhouette_batch(X, batch, t, scale)
    assert set(means) == set(want_means) and 7 not in means and 8 not in means
    for k in means:
        assert means[k] == pytest.approx(want_means[k], abs=1e-12)
    assert asw == pytest.approx(want, abs=1e-12)
    only = batch_fold(s[:8], batch[:8], t[:8], scale)    # every cell type skipped
    assert np.isnan(only[0]) and only[1] == {}


def test_label_fold_is_scib():
    X, t = _data(12)
    s = sr.silhouette(X, t)
    want = (sklearn_metrics.silhouette_score(X, t) + 1) / 2
    assert (s.mean() + 1) / 2 == pytest.approx(want, abs=1e-12)


def test_refusals_need_no_device(monkeypatch):
    from harmony_b200 import _lib
    monkeypatch.setattr(_lib, "lib", lambda: pytest.fail("the library was loaded"))
    X, t = _data(6, n=50)
    meta = {"batch": t % 2, "type": t}
    n_labels = "Number of labels is {}. Valid values are 2 to n_samples - 1 (inclusive)"
    no_column, type_rows = "meta_data has no column 'nope'", "column 'type' must hold one label per row of X (50)"
    calls = [(silhouette_samples, dict(X=X[:, 0], labels=t), "X must be an [N, d] matrix"),
             (silhouette_samples, dict(X=np.zeros((50, 129)), labels=t), "d = 129 is not supported (1 <= d <= 128)"),
             (silhouette_samples, dict(X=np.zeros((50, 0)), labels=t), "d = 0 is not supported (1 <= d <= 128)"),
             (silhouette_samples, dict(X=X[:1], labels=t[:1]), "X has 1 rows, at least 2 are needed"),
             (silhouette_samples, dict(X=X, labels=t[:49]), "labels must hold one label per row of X (50)"),
             (silhouette_samples, dict(X=X, labels=np.zeros(50)), n_labels.format(1)),
             (silhouette_samples, dict(X=X, labels=np.arange(50)), n_labels.format(50)),
             (silhouette_samples, dict(X=X, labels=np.where(t == 1, np.nan, t)), "labels holds missing labels"),
             (silhouette_samples, dict(X=X, labels=np.array(["a", None] * 25, dtype=object)),
              "labels holds missing labels"),
             (silhouette_samples, dict(X=X, labels=t, groups=t[:10]), "groups must hold one label per row of X (50)")]
    for kw, msg in ((dict(meta_data=t), "meta_data must be a DataFrame or a dict of columns"),
                    (dict(meta_data={"type": t[:49]}), type_rows), (dict(label_key="nope"), no_column),
                    (dict(meta_data={"type": np.zeros(50)}), n_labels.format(1))):
        calls.append((silhouette_label, dict(dict(X=X, meta_data=meta, label_key="type"), **kw), msg))
    for kw, msg in ((dict(batch_key="nope"), no_column), (dict(label_key="nope"), no_column),
                    (dict(meta_data={"batch": t, "type": t[:3]}), type_rows)):
        calls.append((silhouette_batch, dict(dict(X=X, meta_data=meta, batch_key="batch", label_key="type"), **kw), msg))
    for f, kw, msg in calls:
        with pytest.raises(ValueError) as e:
            f(**kw)
        assert e.type is ValueError and str(e.value) == msg, (f.__name__, kw)


def _geometry(d, N, sms):
    from harmony_b200 import _lib
    out = (ctypes.c_int64 * 8)(*([-7] * 8))
    return _lib.lib().hb_debug_silhouette_geometry(d, N, sms, out), list(out)


def test_geometry_hook_matches_the_rule():
    for d in range(1, 129):
        for N in (2, 129, 20_000, 1_000_000, 2 ** 31 - 1):
            st, g = _geometry(d, N, 132)
            assert st == 0 and g == sr.geometry(d, N, 132), (d, N, g)
            assert g[:3] == [128, 64, 2] and g[3] <= 227 * 1024 - 256   # (128, 2) fits every d <= 128
    assert _geometry(50, 1000, 0)[0] == 2
    for d, N in ((0, 100), (129, 100), (50, 1), (50, 0), (50, 2 ** 31)):
        assert _geometry(d, N, 132) == (2, [-7] * 8), (d, N)
