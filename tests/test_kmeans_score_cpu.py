"""k-means and the NMI / ARI scores without a GPU (DESIGN §15): the restatement's Lloyd against sklearn's, the fold
against sklearn.metrics, the restatement's scores of the fixtures, and every Python refusal before the library loads."""
import numpy as np
import pytest

import kmeans_score_restatement as kr
from harmony_b200 import kmeans, nmi_ari, nmi_ari_cluster_labels_kmeans
from helpers import load_cell_lines


@pytest.mark.parametrize("tol", [1e-4, 0.0])
def test_restatement_lloyd_is_sklearns(tol):
    from sklearn.cluster import KMeans
    rng = np.random.default_rng(0)
    checked = 0
    for rep in range(12):
        N, d, K = int(rng.integers(200, 2000)), int(rng.integers(2, 12)), int(rng.integers(2, 9))
        X = rng.standard_normal((N, d)) + rng.standard_normal((K, d))[rng.integers(0, K, N)] * 2
        fin, P, _ = kr.prepare(X)
        seeds = kr.seeding(P, fin, K, rep)
        labels, C, inertia, n_iter = kr.lloyd(X, X[seeds], 300, tol)
        if len(np.unique(labels)) < K:
            continue  # sklearn relocates an empty cluster; the library keeps it
        km = KMeans(K, init=X[seeds], n_init=1, algorithm="lloyd", tol=tol, max_iter=300).fit(X)
        np.testing.assert_array_equal(labels, km.labels_)
        assert n_iter == km.n_iter_
        assert abs(inertia - km.inertia_) <= 1e-10 * inertia
        assert np.abs(C - km.cluster_centers_).max() <= 1e-10 * (np.abs(C).max() + 1)
        checked += 1
    assert checked >= 8


def test_seeding_draws_by_d2():
    """The seeds are distinct finite rows, and with three tight, far-apart clusters the D^2 draws put one seed in each,
    under every seed."""
    rng = np.random.default_rng(1)
    X = np.concatenate([rng.standard_normal((300, 3)) * 0.01 + c for c in ([0, 0, 0], [10, 0, 0], [0, 10, 0])])
    X[5] = np.nan
    fin, P, _ = kr.prepare(X)
    spread = 0
    for init in range(20):
        s = kr.seeding(P, fin, 3, init)
        assert fin[s].all() and len(set(s.tolist())) == 3
        spread += len(set((s // 300).tolist())) == 3
    assert spread == 20


def _sk(t, p):
    from sklearn.metrics import adjusted_rand_score, normalized_mutual_info_score
    return normalized_mutual_info_score(t, p), adjusted_rand_score(t, p)


def test_nmi_ari_is_sklearns():
    rng = np.random.default_rng(2)
    cases = []
    for _ in range(20):
        n = int(rng.integers(3, 3000))
        cases.append((rng.integers(0, rng.integers(1, 12), n), rng.integers(0, rng.integers(1, 12), n)))
    t = rng.integers(0, 5, 500)
    cases += [(t, t), (t, (t + 1) % 5), (t * 7 + 100, t), (t, rng.integers(0, 5, 500) * 3)]   # unused codes
    cases += [(np.array(["b", "a", "c", "a"] * 50), rng.integers(0, 3, 200))]                # string labels
    cases += [(np.zeros(10), np.zeros(10)), (np.zeros(10), np.arange(10)), (np.arange(10), np.arange(10)),
              (np.arange(10), np.zeros(10)), (np.array([1]), np.array([2])), (np.array([1, 2]), np.array([3, 3])),
              (np.array([1, 2]), np.array([3, 4])), (np.array([], int), np.array([], int))]    # special cases
    for t, p in cases:
        want = _sk(t, p)
        got = nmi_ari(t, p)
        assert got == pytest.approx(want, abs=1e-12), (t[:5], p[:5])
        assert kr.nmi_ari(t, p) == pytest.approx(want, abs=1e-12)


def test_nmi_ari_leaves_out_unassigned_rows():
    rng = np.random.default_rng(3)
    t, p = rng.integers(0, 4, 400), rng.integers(0, 4, 400)
    p[::7] = -1
    keep = p != -1
    assert nmi_ari(t, p) == pytest.approx(_sk(t[keep], p[keep]), abs=1e-12)


def test_restatement_scores_fixtures():
    """K = 2 by cell type on scaled_pcs: sklearn's KMeans gives NMI 0.9909829259 / ARI 0.9966258397 on cell_lines and
    1.0 / 1.0 on cell_lines_small, for every random seed; the restatement reaches them from its own seeds."""
    Z, meta = load_cell_lines(False)
    t = meta["cell_type"]
    K = len(np.unique(t))
    for seed in range(3):
        labels = kr.kmeans(Z, K, seed)[1]
        assert nmi_ari(t, labels) == pytest.approx((0.9909829259, 0.9966258397), abs=1e-9)
    Z, meta = load_cell_lines(True)
    labels = kr.kmeans(Z, len(np.unique(meta["cell_type"])), 0)[1]
    assert nmi_ari(meta["cell_type"], labels) == (1.0, 1.0)


def test_refusals_need_no_device(monkeypatch):
    from harmony_b200 import _lib
    monkeypatch.setattr(_lib, "lib", lambda: pytest.fail("the library was loaded"))
    X = np.random.default_rng(4).standard_normal((50, 4))
    calls = [(dict(X=X[:, 0]), "X must be an [N, d] matrix"),
             (dict(X=np.zeros((50, 129))), "d = 129 is not supported (1 <= d <= 128)"),
             (dict(X=np.zeros((0, 3))), "X has no rows"),
             (dict(n_clusters=0), "n_clusters = 0, at least 1 is needed"),
             (dict(n_clusters=51), "n_clusters = 51 is not supported (1 <= n_clusters <= min(N, 1024) = 50)"),
             (dict(n_clusters=2.0), "n_clusters must be an integer, not 2.0"),
             (dict(seed=-1), "seed = -1, at least 0 is needed"),
             (dict(seed=2 ** 64), f"seed = {2 ** 64} does not fit 64 bits"),
             (dict(n_init=0), "n_init = 0, at least 1 is needed"),
             (dict(max_iter=-1), "max_iter = -1, at least 0 is needed"),
             (dict(max_iter=2 ** 32 + 5), f"max_iter = {2 ** 32 + 5} does not fit 32 bits"),
             (dict(n_init=2 ** 31), f"n_init = {2 ** 31} does not fit 32 bits"),
             (dict(tol=-1.0), "tol must be a finite number >= 0, not -1.0"),
             (dict(tol=float("nan")), "tol must be a finite number >= 0, not nan"),
             (dict(tol=True), "tol must be a finite number >= 0, not True")]
    for change, msg in calls:
        args = dict(dict(X=X, n_clusters=3), **change)
        with pytest.raises(ValueError) as e:
            kmeans(**args)
        assert str(e.value) == msg
    meta = {"ct": np.arange(50) % 3}
    for change, msg in [(dict(label_key="nope"), "meta_data has no column 'nope'"),
                        (dict(meta_data={"ct": meta["ct"][:49]}), "column 'ct' must hold one label per row of X (50)"),
                        (dict(meta_data=meta["ct"]), "meta_data must be a DataFrame or a dict of columns"),
                        (dict(n_init=0), "n_init = 0, at least 1 is needed")]:
        args = dict(dict(X=X, meta_data=meta, label_key="ct"), **change)
        with pytest.raises(ValueError) as e:
            nmi_ari_cluster_labels_kmeans(**args)
        assert str(e.value) == msg
    with pytest.raises(ValueError, match="must label the same rows"):
        nmi_ari([0, 1], [0])
