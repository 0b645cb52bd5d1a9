"""hb_knn without a GPU: the fp64 restatement against cKDTree, the vote rule, the Python refusals and the geometry."""
import ctypes

import numpy as np
import pytest
from scipy.spatial import cKDTree

import knn_restatement as kr
from harmony_b200 import TransferLabels, knn
from harmony_b200 import neighbors


def _sets(seed, nq=200, nx=700, d=7):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((nx, d)) + 3.0
    Q = rng.standard_normal((nq, d)) + 3.0
    X[50:60] = X[40:50]           # exact duplicates
    return Q, X


@pytest.mark.parametrize("k", [1, 5, 15])
def test_restatement_matches_ckdtree(k):
    Q, X = _sets(k)
    idx, dist = kr.brute_force(Q, X, k, block=64)
    dd, ii = cKDTree(X).query(Q, k=k)
    np.testing.assert_allclose(dist, dd.reshape(dist.shape), rtol=1e-9, atol=1e-6)
    assert (np.sort(X[idx].sum(-1), axis=1) == pytest.approx(np.sort(X[ii.reshape(idx.shape)].sum(-1), axis=1)))
    # cosine: 1 - cos = |q^ - x^|^2 / 2 on normalised rows
    idx, dist = kr.brute_force(Q, X, k, "cosine")
    dd, _ = cKDTree(kr.unit_rows(X)).query(kr.unit_rows(Q), k=k)
    np.testing.assert_allclose(dist, dd.reshape(dist.shape) ** 2 / 2, atol=1e-12)


def test_restatement_excludes_self_and_zero_rows():
    _, X = _sets(3)
    X[5] = 0.0
    idx, dist = kr.brute_force(X, X, 4, exclude_self=True)
    assert not (idx == np.arange(len(X))[:, None]).any()
    dd, ii = cKDTree(X).query(X, k=5)
    np.testing.assert_allclose(dist, dd[:, 1:], atol=1e-6)  # duplicates: sqrt of the expansion's 1e-15
    _, dist = kr.brute_force(X[5:6], X[:5], 3, "cosine")
    np.testing.assert_allclose(dist, 1.0)


def test_vote_rule():
    codes = np.array([0, 0, 1, 1, 2, 2])
    idx = np.array([[0, 2, 3], [0, 2, 4], [4, 2, 0], [5, -1, -1], [-1, -1, -1], [2, 0, 3]])
    dist = np.array([[.1, .2, .3], [.3, .2, .1], [.1, .1, .1], [.5, np.inf, np.inf], [np.inf] * 3, [.1, .1, .2]])
    want_code, want_share = [1, 2, 0, 2, -1, 1], [2 / 3, 1 / 3, 1 / 3, 1.0, 0.0, 2 / 3]
    for f in (kr.vote, neighbors.vote):
        code, share = f(idx, dist, codes, 3)
        assert list(code) == want_code, f
        np.testing.assert_allclose(share, want_share)
    rng = np.random.default_rng(0)
    idx = rng.integers(-1, 40, (300, 7))
    dist = np.sort(rng.integers(0, 4, (300, 7)) / 4.0, axis=1)
    codes = rng.integers(0, 5, 40)
    a, b = kr.vote(idx, dist, codes, 5), neighbors.vote(idx, dist, codes, 5)
    np.testing.assert_array_equal(a[0], b[0])
    np.testing.assert_allclose(a[1], b[1])


class _Categorical:
    """What TransferLabels needs of a pandas Categorical."""

    def __init__(self, codes, categories):
        self.codes, self.categories = np.asarray(codes), np.asarray(categories)

    @classmethod
    def from_codes(cls, codes, categories):
        return cls(codes, categories)


@pytest.mark.parametrize("kind", ["str", "int", "categorical"])
def test_transfer_labels_kinds(kind, monkeypatch):
    Q, X = _sets(11, nq=60, nx=300)
    types = np.random.default_rng(1).integers(0, 4, len(X))
    labels = {"str": np.array(["b", "a", "d", "c"])[types], "int": 10 * types + 3,
              "categorical": _Categorical(types, ["t3", "t1", "t2", "t0"])}[kind]
    monkeypatch.setattr(neighbors, "knn", lambda q, r, k, metric, device: tuple(
        a.astype(t) for a, t in zip(kr.brute_force(q, r, k, metric), (np.int32, np.float32))))
    pred, share = TransferLabels(Q, X, labels, k=5, return_prob=True)
    idx, dist = kr.brute_force(Q, X, 5)
    if kind == "categorical":
        code, want_share = kr.vote(idx, dist.astype(np.float32), types, 4)
        assert isinstance(pred, _Categorical) and list(pred.categories) == ["t3", "t1", "t2", "t0"]
        np.testing.assert_array_equal(pred.codes, code)
    else:
        cats, codes = np.unique(labels, return_inverse=True)
        code, want_share = kr.vote(idx, dist.astype(np.float32), codes, len(cats))
        assert pred.dtype == labels.dtype
        np.testing.assert_array_equal(pred, cats[code])
    np.testing.assert_allclose(share, want_share)


def test_python_refusals_need_no_device(monkeypatch):
    from harmony_b200 import _lib
    monkeypatch.setattr(_lib, "lib", lambda: pytest.fail("the library was loaded"))
    Q, X = _sets(5, nq=10, nx=30)
    ref_k = "is not supported here (1 <= k <= 30: at most 64, and the rows of ref)"
    matrices = "query and ref must be [rows, d] matrices"
    bad = [(dict(query=Q, ref=X, k=0), f"k = 0 {ref_k}"), (dict(query=Q, ref=X, k=65), f"k = 65 {ref_k}"),
           (dict(query=Q, ref=X, k=31), f"k = 31 {ref_k}"),
           (dict(query=Q, k=10), "k = 10 is not supported here (1 <= k <= 9: at most 64, and the other rows)"),
           (dict(query=Q, ref=X, k=2.5), "k must be an integer, not 2.5"),
           (dict(query=Q, ref=X[:, :5]), "query has 7 dimensions, ref 5"), (dict(query=Q[0], ref=X), matrices),
           (dict(query=Q, ref=X[0]), matrices),
           (dict(query=Q, ref=X, metric="manhattan"), "metric must be one of ['cosine', 'euclidean'], not 'manhattan'"),
           (dict(query=np.zeros((4, 129)), ref=np.zeros((9, 129)), k=2), "d = 129 is not supported (1 <= d <= 128)"),
           (dict(query=np.zeros((0, 3)), ref=X[:, :3], k=1), "query and ref need at least one row")]
    for kw, msg in bad:
        with pytest.raises(ValueError) as e:
            knn(**kw)
        assert e.type is ValueError and str(e.value) == msg, kw
    for kw, msg in ((dict(ref_labels=np.zeros(29)), "ref has 30 rows, ref_labels 29 labels"),
                    (dict(ref_labels=np.zeros((30, 2))), "ref_labels must hold one label per row of ref"),
                    (dict(ref_labels=np.zeros(30), k=0), f"k = 0 {ref_k}"),
                    (dict(ref_labels=_Categorical([-1] * 30, ["a"])), "ref_labels holds missing values"),
                    (dict(ref=None, ref_labels=np.zeros(10)), "TransferLabels needs a reference embedding")):
        kw = dict(dict(query=Q, ref=X), **kw)
        with pytest.raises(ValueError) as e:
            TransferLabels(**kw)
        assert e.type is ValueError and str(e.value) == msg, kw


def _geometry(d, k, Nq, Nx, sms):
    from harmony_b200 import _lib
    out = (ctypes.c_int64 * 8)(*([-7] * 8))
    return _lib.lib().hb_debug_knn_geometry(d, k, Nq, Nx, sms, out), list(out)


def test_geometry_hook_matches_the_rule():
    shapes = [(1000, 1_000_000), (100_000, 1_000_000), (1_000_000, 1_000_000), (1, 64), (20_000, 50_000), (129, 127)]
    for d in range(1, 129):
        for k in (1, 5, 15, 64):
            for Nq, Nx in shapes:
                st, g = _geometry(d, k, Nq, Nx, 132)
                assert st == 0 and g == kr.geometry(d, k, Nq, Nx, 132), (d, k, Nq, Nx, g)
                tq, tn, stages, splits, smem, per, KD, threads = g
                assert smem <= 227 * 1024 and KD >= d and KD % 8 == 0 and stages in (1, 2)
                assert (splits - 1) * per * tn < Nx <= splits * per * tn          # every split has rows, none is left out
                assert splits * k <= 1024
                if -(-Nq // tq) >= 132:
                    assert splits == 1
    assert _geometry(50, 5, 1000, 1_000_000, 132)[1][3] > 1
    assert _geometry(50, 15, 1_000_000, 1_000_000, 132)[1][:4] == [128, 64, 2, 1]
    assert _geometry(128, 64, 5000, 5000, 132)[1][0] == 64
    for d, k in ((129, 5), (0, 5), (50, 65), (50, 0)):
        st, g = _geometry(d, k, 1000, 1000, 132)
        assert st == 2 and g == [-7] * 8


def test_row_layout_reads_only_unit_stride_rows_in_place():
    """The layout rule of every caller array the scores read (_arrays.row_layout), on CPU tensors: row-strided [N, d]
    views are read in place with their stride; a transposed view, and a single row whose column stride is not 1, are
    made contiguous first."""
    import torch
    from harmony_b200._arrays import row_layout
    A = torch.arange(20.).reshape(4, 5)
    one = A.T[:1]                                   # [1, 4], strides (1, 5): elements 0, 5, 10, 15
    t, ld = row_layout(one, 4)
    assert t.stride(1) == 1 and ld == 4 and t.flatten().tolist() == [0.0, 5.0, 10.0, 15.0]
    t, ld = row_layout(A[:1], 5)                    # one dense row: in place
    assert t.data_ptr() == A.data_ptr() and ld == 5
    t, ld = row_layout(A[:, :3], 3)                 # [4, 3] of row stride 5: in place
    assert t.data_ptr() == A.data_ptr() and ld == 5
    t, ld = row_layout(A.T, 4)                      # [5, 4] transposed: contiguous
    assert t.is_contiguous() and ld == 4 and torch.equal(t, A.T)
