"""hb_kbet without a GPU: the statistic's forms against the kBET package's chi_batch_test, the k0 rule and skips of the
restatement against a transcription of scib's loop, the Python fold against scib's, the p-value function against
scipy, the Python refusals, and the restatement's score of the cell_lines fixture."""
import ctypes

import numpy as np
import pytest
from scipy.stats import chi2

import kbet_restatement as kr
from harmony_b200 import kbet
from harmony_b200.kbet import kbet_fold, kbet_on
from helpers import load_cell_lines

pd = pytest.importorskip("pandas")


def kernel_stat(env, levels, counts, k0):
    """k_kbet's form: over the batches present in the neighbourhood, (o - e)^2 / e, plus the absent batches' e summed
    as k0 (n - their rows) / n."""
    out = []
    n = counts.sum()
    for row in env:
        b, o = np.unique(row, return_counts=True)
        c = counts[np.searchsorted(levels, b)]
        e = k0 * c / n
        out.append(((o - e) ** 2 / e).sum() + k0 * (n - c.sum()) / n)
    return np.array(out)


def closed_stat(env, levels, counts, k0):
    """The closed form of DESIGN §13: sum over the batches present of o^2 / (k0 p) - k0."""
    n = counts.sum()
    out = []
    for row in env:
        b, o = np.unique(row, return_counts=True)
        p = counts[np.searchsorted(levels, b)] / n
        out.append((o * o / (k0 * p)).sum() - k0)
    return np.array(out)


@pytest.mark.parametrize("B,k0", [(2, 10), (3, 70), (12, 25), (300, 70), (5, 129)])
def test_statistic_forms_are_chi_batch_test(B, k0):
    rng = np.random.default_rng(B * 1000 + k0)
    counts = rng.integers(1, 400, B)
    levels = np.sort(rng.choice(10 * B, B, replace=False))
    p = counts / counts.sum()
    skew = rng.dirichlet(np.ones(B) * 0.3)         # mixed, skewed and one-batch neighbourhoods
    env = np.concatenate([rng.choice(levels, (200, k0), p=p), rng.choice(levels, (200, k0), p=skew),
                          np.repeat(levels[rng.integers(0, B, 5)], k0).reshape(5, k0)])
    want = kr.chi_batch_test(env, levels, counts, k0)
    assert (want >= 0).all()
    np.testing.assert_allclose(kernel_stat(env, levels, counts, k0), want, rtol=1e-13, atol=0)
    np.testing.assert_allclose(closed_stat(env, levels, counts, k0), want, rtol=1e-12, atol=1e-12 * k0)


def scib_k0(obs, batch_key, label_key):
    """scib's loop over cell types, transcribed: skip (NaN) a type with fewer than 10 cells or one batch category in
    the subset (categories are those the subset has), else k0 from the mean of value_counts and the 2^31 guard."""
    size_max = np.iinfo(np.int32).max
    out = {}
    for clus in obs[label_key].unique():
        sub = obs[obs[label_key] == clus].copy()
        sub[batch_key] = sub[batch_key].cat.remove_unused_categories()
        if sub.shape[0] < 10 or len(sub[batch_key].cat.categories) == 1:
            out[clus] = 0
            continue
        quarter_mean = np.floor(np.mean(sub[batch_key].value_counts()) / 4).astype("int")
        k0 = np.min([70, np.max([10, quarter_mean])])
        if k0 * sub.shape[0] >= size_max:
            k0 = np.floor(size_max / sub.shape[0]).astype("int")
        out[clus] = int(k0)
    return out


def test_k0_rule_and_skips_are_scibs():
    rng = np.random.default_rng(1)
    sizes = {0: [500, 300, 20], 1: [9], 2: [4, 5], 3: [40, 0, 0, 2], 4: [3000, 3000, 3000, 3000], 5: [60, 60],
             6: [100], 7: [11, 1], 8: [37, 38, 39, 40, 41]}
    lab, bat = [], []
    for l, per in sizes.items():
        for b, n in enumerate(per):
            lab += [l] * n
            bat += [b] * n
    bat = np.array(bat)
    bat[bat == 4] = 9      # batch code 4 becomes 9: codes 4..8 are used by no row
    perm = rng.permutation(len(bat))
    lab, bat = np.array(lab)[perm], bat[perm]
    obs = pd.DataFrame({"batch": pd.Categorical(bat, categories=range(10)), "type": lab})
    want = scib_k0(obs, "batch", "type")
    for l in sizes:
        rows = lab == l
        assert kr.k0_rule(int(rows.sum()), len(np.unique(bat[rows]))) == want[l], l
    assert want[0] == 68 and want[4] == 70 and want[1] == want[2] == want[6] == 0 and want[3] == 10 and want[5] == 15
    # the guard: k0 n reaching 2^31 - 1
    assert kr.k0_rule(40_000_000, 2) == 53 and kr.k0_rule(2 ** 31 - 2, 4) == 1
    # a fixed k0: a label smaller than k0 is skipped
    assert kr.k0_rule(12, 2, fixed=13) == 0 and kr.k0_rule(13, 2, fixed=13) == 13 and kr.k0_rule(9, 2, fixed=2) == 0


def test_fold_is_scibs():
    rng = np.random.default_rng(2)
    N = 3000
    codes = rng.integers(0, 6, N)
    pval = rng.random(N) ** 3
    k0 = np.array([10, 0, 25, 70, 0, 12])
    pval[np.isin(codes, [1, 4])] = np.nan
    pval[rng.integers(0, N, 30)] = np.nan               # non-finite rows of tested labels
    rates = kbet_fold(pval, codes, k0, 0.05)
    scib = []
    for l in range(6):     # scib: per cell type the package's mean rejection rate, NaN for a skipped one
        p = pval[(codes == l) & ~np.isnan(pval)]
        scib.append(np.nan if k0[l] == 0 else np.mean(p < 0.05))
    np.testing.assert_array_equal(rates, np.array(scib))
    np.testing.assert_array_equal(rates, kr.rates(pval, codes, k0))
    assert 1 - np.nanmean(scib) == pytest.approx(1 - rates[~np.isnan(rates)].mean(), abs=0)


DOFS = [1, 2, 3, 4, 19, 20, 99, 299, 1000, 10000]


@pytest.mark.parametrize("dof", DOFS)
def test_chi2_sf_hook_is_scipy(dof):
    from harmony_b200 import _lib
    L = _lib.lib()
    out = ctypes.c_double()
    xs = np.concatenate([[0.0, 1e-300, 1e-12, 1e-3], np.linspace(0, 50 * dof, 4001)[1:],
                         dof * (1 + np.array([-1e-9, 1e-9, -1e-3, 1e-3, -0.1, 0.1])), [dof - 2, dof + 2, dof + 1, dof - 1]])
    xs = xs[xs >= 0]
    for x in xs:
        assert L.hb_debug_chi2_sf(float(x), dof, ctypes.byref(out)) == 0
        want, got = chi2.sf(x, dof), out.value
        if want >= 1e-300:
            assert abs(got - want) <= 1e-13 * (1 + dof) * want, (x, dof, got, want)
        else:
            assert 0 <= got <= 1e-290, (x, dof, got, want)
    assert L.hb_debug_chi2_sf(0.0, dof, ctypes.byref(out)) == 0 and out.value == 1.0
    assert L.hb_debug_chi2_sf(float("inf"), dof, ctypes.byref(out)) == 0 and out.value == 0.0
    out.value = -5.0
    assert L.hb_debug_chi2_sf(1.0, 0, ctypes.byref(out)) == 2 and out.value == -5.0


def test_refusals_need_no_device(monkeypatch):
    from harmony_b200 import _lib
    monkeypatch.setattr(_lib, "lib", lambda: pytest.fail("the library was loaded"))
    rng = np.random.default_rng(8)
    X = rng.standard_normal((50, 4))
    meta = {"batch": rng.integers(0, 3, 50), "type": rng.integers(0, 2, 50)}
    k0_msg = "k0 = {} is not supported (None or 0 for scib's rule, or 2 <= k0 <= 129)"
    calls = [(dict(X=X[:, 0]), ValueError, "X must be an [N, d] matrix"),
             (dict(X=np.zeros((50, 129))), ValueError, "d = 129 is not supported (1 <= d <= 128)"),
             (dict(X=X[:1], meta_data={"batch": [0], "type": [0]}), ValueError, "X has 1 rows, at least 2 are needed"),
             (dict(k0=1), ValueError, k0_msg.format(1)),
             (dict(k0=130), ValueError, k0_msg.format(130)),
             (dict(k0=-3), ValueError, k0_msg.format(-3)),
             (dict(k0=2.5), ValueError, "k0 must be None or an integer, not 2.5"),
             (dict(k0=True), ValueError, "k0 must be None or an integer, not True"),
             (dict(alpha=0), ValueError, "alpha must be a number in (0, 1), not 0"),
             (dict(alpha=1.0), ValueError, "alpha must be a number in (0, 1), not 1.0"),
             (dict(alpha=float("nan")), ValueError, "alpha must be a number in (0, 1), not nan"),
             (dict(alpha="0.05"), ValueError, "alpha must be a number in (0, 1), not '0.05'"),
             (dict(meta_data={"batch": meta["batch"][:49], "type": meta["type"]}), ValueError,
              "column 'batch' must hold one label per row of X (50)"),
             (dict(meta_data={"batch": meta["batch"], "type": meta["type"][1:]}), ValueError,
              "column 'type' must hold one label per row of X (50)"),
             (dict(batch_key="nope"), ValueError, "meta_data has no column 'nope'"),
             (dict(meta_data={"batch": np.where(meta["batch"] == 1, np.nan, meta["batch"]), "type": meta["type"]}),
              ValueError, "column 'batch' holds missing labels")]
    for change, exc, msg in calls:
        args = dict(dict(X=X, meta_data=meta, batch_key="batch", label_key="type"), **change)
        with pytest.raises(exc) as e:
            kbet(**args)
        assert str(e.value) == msg, change
    obj = object()   # kbet_on refuses by shape before it touches the object
    with pytest.raises(ValueError, match="k0 = 1 is not supported"):
        kbet_on(obj, X, meta["batch"], k0=1)
    with pytest.raises(ValueError, match=r"batches must be \[50\]"):
        kbet_on(obj, X, meta["batch"][:40])
    with pytest.raises(ValueError, match="X has 1 rows"):
        kbet_on(obj, X[:1], meta["batch"][:1])


def test_restatement_scores_cell_lines():
    """The raw PCs of the full cell_lines fixture: k0 = 70 for both cell types and a scaled kBET of 0.0972."""
    Z, meta = load_cell_lines(False)
    b = np.unique(meta["dataset"], return_inverse=True)[1]
    types, t = np.unique(meta["cell_type"], return_inverse=True)
    r = kr.kbet(Z, b, t)
    np.testing.assert_array_equal(r.k0, [70, 70])
    rates = kr.rates(r.pval, t, r.k0)
    np.testing.assert_allclose(rates, [0.9913, 0.8143], atol=5e-5)
    assert 1 - rates.mean() == pytest.approx(0.0972, abs=5e-5)
