"""hb_silhouette on the GPU against the fp64 restatement (silhouette_restatement.py): a table of shapes, each row naming
the limit it straddles and compared within its per-row bound (DESIGN §11), the inputs Python takes, repeatability, the
handle's state left untouched, the refusals, and the two scib scores of an integration end to end."""
import ctypes

import numpy as np
import pytest

import silhouette_restatement as sr
from harmony_b200 import RunHarmony, silhouette_batch, silhouette_label, silhouette_samples
from harmony_b200._arrays import ptr
from helpers import gpu_harmony, load_cell_lines
from score_helpers import Frame, generic, handle_state_untouched, non_finite_rows, refusals_launch_nothing, strided

pytestmark = pytest.mark.gpu


ROWS = [
    # name, N, d, dtype, options
    ("N2_both_alone", 2, 8, np.float32, {}),
    ("N3_one_pair_one_alone", 3, 8, np.float32, {}),
    ("d1", 3000, 1, np.float32, {}),
    ("d8_one_k_step", 3000, 8, np.float32, {}),
    ("d50_KD56", 3000, 50, np.float32, {}),
    ("d64", 3000, 64, np.float32, {}),
    ("d100", 3000, 100, np.float32, {}),
    ("d127", 3000, 127, np.float32, {}),
    ("d128_widest", 3000, 128, np.float32, {}),
    ("N65_one_past_a_reference_tile", 65, 20, np.float32, {}),
    ("N129_one_past_a_query_tile", 129, 20, np.float32, {}),
    ("N5121_one_past_40_query_tiles", 5121, 30, np.float32, {}),
    ("label_runs_straddle_tiles", 337, 16, np.float32, dict(runs=[100, 37, 200])),
    ("3000_labels_of_3_many_runs_per_tile", 9000, 30, np.float32, dict(labels=3000)),
    ("20_groups_singletons_one_label_group", 4000, 30, np.float32, dict(groups=20)),
    ("f64_strided", 3000, 50, np.float64, dict(strided=True)),
    ("f32_strided_groups", 3000, 40, np.float32, dict(strided=True, groups=4)),
    ("offset_1e3", 3000, 50, np.float32, dict(offset=1e3)),
    ("offset_1e3_f64", 3000, 50, np.float64, dict(offset=1e3)),
    ("duplicates", 3000, 50, np.float32, dict(duplicates=True)),
    ("nan_inf_rows", 3000, 20, np.float32, dict(nan=True)),
]


def _case(name, N, d, o):
    rng = np.random.default_rng(sum(map(ord, name)))
    X, t = generic(rng, N, d)
    g = None
    if N == 2:
        t = np.array([0, 1])
    if N == 3:
        t = np.array([0, 1, 0])
    if "runs" in o:
        t = np.repeat(np.arange(len(o["runs"])), o["runs"])
    if "labels" in o:
        t = np.arange(N) % o["labels"]
    if "groups" in o:
        g = rng.integers(0, o["groups"], N)
        if o["groups"] == 20:
            g = rng.integers(0, 17, N)
            g[:3] = [17, 18, 19]          # groups 17-19: one row each
            t[g == 16] = 5                # group 16: one label
    if o.get("offset"):
        X += o["offset"]
    if o.get("duplicates"):
        X[N // 2:N // 2 + 1000] = X[:1000]
    if o.get("nan"):
        non_finite_rows(X)
    return X, t.astype(np.int32), None if g is None else g.astype(np.int32)


@pytest.mark.parametrize("row", ROWS, ids=[r[0] for r in ROWS])
def test_silhouette_table(row):
    import torch
    name, N, d, dtype, o = row
    X, t, g = _case(name, N, d, o)
    xt = strided(X.astype(dtype)) if o.get("strided") else torch.as_tensor(X.astype(dtype), device="cuda:0")
    h = gpu_harmony()
    lab = torch.as_tensor(t, device="cuda:0")
    grp = None if g is None else torch.as_tensor(g, device="cuda:0")
    got = h.silhouette(xt, lab, grp)
    assert got.is_cuda and got.dtype == torch.float64 and got.shape == (N,)
    got = got.cpu().numpy()
    want, bound = sr.silhouette(X.astype(dtype), t, g, bound=True)
    assert (np.isnan(got) == np.isnan(want)).all(), "NaN rows differ"
    ok = ~np.isnan(want)
    err = np.abs(got[ok] - want[ok])
    bar = np.minimum(bound[ok], 2.0) + 1e-12
    ratio = err / bar
    worst = int(np.argmax(ratio)) if ratio.size else 0
    assert (err <= bar).all(), f"s off by {err[worst]:.3e}, bound {bar[worst]:.3e}"
    if o.get("nan"):
        assert np.isnan(got[[3, 11, 700, 1200, 2000, 2500]]).all()
    if "groups" in o and o["groups"] == 20:
        assert np.isnan(got[:3]).all() and np.isnan(got[g == 16]).all()
    if N == 2:   # both rows alone in their label: 0 by rule
        np.testing.assert_array_equal(got, 0.0)
    finite_bound = bound[ok][np.isfinite(bound[ok])]
    print(f"[silhouette {name}] worst error {err.max() if err.size else 0:.2e} "
          f"(ratio to bound {ratio.max() if ratio.size else 0:.3f}), median bound {np.median(finite_bound) if finite_bound.size else 0:.2e}")


def test_inputs_agree_and_repeat():
    """Host arrays, CUDA tensors, a DataFrame and CUDA integer labels give one result; two calls are bit-identical."""
    import torch
    rng = np.random.default_rng(4)
    X, t = generic(rng, 6000, 30)
    batch = np.array(["b1", "b0", "b2"])[rng.integers(0, 3, len(X))]
    host = silhouette_samples(X, batch, groups=t)
    assert isinstance(host, np.ndarray) and host.dtype == np.float64 and host.shape == (len(X),)
    Xd = torch.as_tensor(X, device="cuda:0")
    bcodes = np.unique(batch, return_inverse=True)[1]
    dev = silhouette_samples(Xd, torch.as_tensor(bcodes * 1000 - 7, device="cuda:0"),
                             groups=torch.as_tensor(t, device="cuda:0"))
    assert dev.is_cuda and dev.dtype == torch.float64
    np.testing.assert_array_equal(host, dev.cpu().numpy())
    np.testing.assert_array_equal(host, silhouette_samples(X, batch, groups=t))
    want, bound = sr.silhouette(X, bcodes, t, bound=True)
    assert (np.abs(host - want) <= bound + 1e-12).all()
    meta = Frame({"batch": batch, "type": t})
    b_host, per = silhouette_batch(X, meta, "batch", "type", return_all=True)
    b_dev = silhouette_batch(Xd, {"batch": batch, "type": torch.as_tensor(t, device="cuda:0")}, "batch", "type")
    assert b_host == b_dev and set(per) == set(range(12))
    l_host = silhouette_label(X, meta, "type")
    assert l_host == silhouette_label(Xd, {"type": torch.as_tensor(t, device="cuda:0")}, "type")
    s = silhouette_samples(X, t)
    assert l_host == (s.mean() + 1) / 2
    with pytest.raises(ValueError):
        silhouette_samples(X, torch.as_tensor(t, device="cuda:0"))   # device labels, host X


def test_handle_state_untouched():
    """hb_silhouette between cluster_cpp and moe_correct_ridge_cpp and on a mapping handle: Z_corr, R, Y and the
    covariate-tuple index read bit for bit the same before and after the call."""
    import torch
    from harmony_b200 import _lib
    L = _lib.lib()

    def index(h, n):
        perm, start = np.zeros(n, np.int32), np.zeros(64, np.int64)
        J = L.hb_debug_tuple_index(h._h, perm.ctypes.data_as(ctypes.c_void_p), None, start.ctypes.data_as(ctypes.c_void_p))
        return J, perm, start[:J + 1].copy()

    def call(h, phase, data):
        if phase == "setup":
            h.silhouette(data.probe, data.codes)
            return
        n = 20000 if phase == "run" else 6000
        ib = index(h, n)
        if phase == "run":
            assert not torch.isnan(h.silhouette(data.probe, data.codes)).any()
        else:
            h.silhouette(h.get_tensor("Z_corr"), data.mapped_codes)
        ia = index(h, n)
        assert ib[0] == ia[0]
        np.testing.assert_array_equal(ib[1], ia[1])
        if phase == "run":
            assert ia[0] == 4
            np.testing.assert_array_equal(ib[2], ia[2])

    handle_state_untouched(call)


def test_refusals_launch_nothing():
    import torch
    from harmony_b200 import _lib
    L = _lib.lib()
    g = gpu_harmony()
    dev = torch.device("cuda", 0)
    N, d = 200, 8
    X = torch.zeros((N, d), device=dev)
    lab = torch.zeros(N, dtype=torch.int32, device=dev)
    grp = torch.zeros(N, dtype=torch.int32, device=dev)
    out = torch.zeros(N, dtype=torch.float64, device=dev)
    host = np.zeros(N, np.float64)
    H = host.ctypes.data_as(ctypes.c_void_p)
    good = dict(X=ptr(X), xt=0, xld=d, N=N, d=d, lab=ptr(lab), nl=2, grp=ptr(grp), ng=1, out=ptr(out))
    bad = [dict(N=1), dict(N=0), dict(N=2 ** 31), dict(d=0), dict(d=129, xld=129), dict(nl=0), dict(ng=0),
           dict(nl=N + 1), dict(ng=N + 1), dict(xt=2), dict(xt=-1), dict(xld=d - 1), dict(X=None), dict(lab=None),
           dict(out=None), dict(X=H), dict(lab=H), dict(grp=H), dict(out=H)]
    call = lambda a: L.hb_silhouette(g._h, a["X"], a["xt"], a["xld"], a["N"], a["d"], a["lab"], a["nl"], a["grp"],  # noqa: E731
                                     a["ng"], a["out"], None)
    refusals_launch_nothing(g, call, good, bad)
    # codes out of range: found by the index pass, status 2 naming the cell
    lab[17] = 2
    assert call(good) == 2 and b"labels of cell 17" in L.hb_last_error(g._h)
    lab[17] = 0
    grp[5] = -1
    assert call(good) == 2 and b"groups of cell 5" in L.hb_last_error(g._h)
    grp[5] = 0
    lab[::2] = 1
    assert call(good) == 0 and call(dict(good, grp=None, ng=0)) == 0
    assert g.kernel_launches > 0
    np.testing.assert_array_equal(out.cpu().numpy(), 0.0)   # all rows equal: a = b = 0


def test_integration_scores_end_to_end():
    """On the PCs of cell_lines, sklearn 1.9.0 gives batch ASW (`dataset` within `cell_type`) 0.829918 and scaled
    cell-type ASW 0.740870.  The CPU oracle's integration (default parameters, make_Y0 centroids, seeds 1 and 2)
    scores 0.971 / 0.971 and 0.757 / 0.758; the bars below it allow for the native k-means initialisation."""
    import torch
    Z, meta = load_cell_lines(False)
    b0 = silhouette_batch(Z, meta, "dataset", "cell_type")
    l0 = silhouette_label(Z, meta, "cell_type")
    assert b0 == pytest.approx(0.8299178087618779, abs=1e-5)
    assert l0 == pytest.approx(0.7408698953900408, abs=1e-5)
    Zc = RunHarmony(torch.as_tensor(Z, device="cuda:0"), meta, "dataset", verbose=False, seed=1)
    b1, per = silhouette_batch(Zc, meta, "dataset", "cell_type", return_all=True)
    l1 = silhouette_label(Zc, meta, "cell_type")
    print(f"[silhouette cell_lines] batch ASW {b0:.4f} -> {b1:.4f} {per}, cell-type ASW {l0:.4f} -> {l1:.4f}")
    assert b1 > 0.93
    assert l1 > 0.72
