"""hb_kbet on the GPU against the fp64 restatement (kbet_restatement.py): a table of cases, each row's neighbours held
to DESIGN §9's band within its own label and its statistic and p-value to the restatement's, the inputs Python takes,
repeatability, the handle's state left untouched, the refusals, stream order, the launch count and the score of an
integration end to end."""
import ctypes

import numpy as np
import pytest
from scipy.stats import chi2

import kbet_restatement as kr
import knn_restatement as knr
from harmony_b200 import RunHarmony, kbet
from harmony_b200._arrays import ptr
from helpers import gpu_harmony, load_cell_lines
from score_helpers import (Frame, after_late_write, check_band, generic, handle_state_untouched, non_finite_rows,
                           refusals_launch_nothing, strided, unwritten)
from silhouette_restatement import finite_rows

pytestmark = pytest.mark.gpu

STAT_REL, STAT_ABS = 1e-12, 1e-15   # the absolute floor covers a statistic that is 0 up to the rounding of k0 p_b
P_REL = 1e-13                       # times 1 + dof


ROWS = [
    # name, N, d, dtype, options
    ("N10_one_label_all_neighbours", 10, 8, np.float32, dict(batches=2, labels=0)),
    ("d1", 3000, 1, np.float32, dict(batches=3, labels=4)),
    ("d4_N200k_40_labels", 200000, 4, np.float32, dict(batches=4, labels=40)),
    ("d50_f64_strided_offset_1e3", 20000, 50, np.float64, dict(batches=3, labels=5, strided=True, offset=1e3)),
    ("d50_f32_offset_1e3", 20000, 50, np.float32, dict(batches=3, labels=5, offset=1e3)),
    ("d100_f32_strided", 8000, 100, np.float32, dict(batches=5, labels=3, strided=True)),
    ("d128_one_label_code", 8000, 128, np.float32, dict(batches=2, labels=1)),
    ("labels_straddle_64_128", 0, 20, np.float32, dict(batches=2, sizes=[63, 65, 129, 64, 128, 127, 200, 9, 10])),
    ("3000_tiny_labels_all_skipped", 9000, 16, np.float32, dict(batches=2, labels=3000)),
    ("no_labels", 5000, 30, np.float32, dict(batches=3, labels=None)),
    ("300_batches_dof_299", 30000, 20, np.float32, dict(batches=300, labels=2)),
    ("unused_codes", 6000, 30, np.float32, dict(batches=3, labels=3, unused=True)),
    ("nan_inf_rows", 3000, 20, np.float32, dict(batches=3, labels=2, nan=True)),
    ("k0_2", 5000, 30, np.float32, dict(batches=3, labels=3, k0=2)),
    ("k0_10", 5000, 30, np.float32, dict(batches=3, labels=3, k0=10)),
    ("k0_129_one_label_too_small", 5000, 30, np.float32, dict(batches=3, labels=3, k0=129, small=100)),
    ("duplicates", 4000, 30, np.float32, dict(batches=3, labels=2, duplicates=True)),
]


def _case(name, N, d, o):
    rng = np.random.default_rng(sum(map(ord, name)))
    if "sizes" in o:
        N = sum(o["sizes"])
    X, t = generic(rng, N, d)
    b = rng.integers(0, o["batches"], N)
    X += rng.standard_normal((o["batches"], d))[b] * 0.7           # batch shifts
    n_labels = o.get("labels", 1) or 0
    lab = None
    if "sizes" in o:
        lab = np.repeat(np.arange(len(o["sizes"])), o["sizes"])
        n_labels = len(o["sizes"])
    elif n_labels == 3000:
        lab = np.arange(N) % 3000
    elif n_labels:
        lab = t % n_labels if n_labels <= 12 else rng.integers(0, n_labels, N)
    n_batches = o["batches"]
    if o.get("unused"):              # batch codes 0, 4, 7 of 8 and label codes 0, 2, 5 of 6
        b, lab = np.array([0, 4, 7])[b], np.array([0, 2, 5])[lab]
        n_batches, n_labels = 8, 6
    if o.get("small"):
        lab[:o["small"]] = n_labels - 1
        lab[o["small"]:][lab[o["small"]:] == n_labels - 1] = 0
    if o.get("offset"):
        X += o["offset"]
    if o.get("duplicates"):
        X[N // 2:N // 2 + 1000] = X[:1000]
    if o.get("nan"):
        non_finite_rows(X)
    lab = None if lab is None else lab.astype(np.int32)
    return X, b.astype(np.int32), lab, max(n_labels, 1), n_batches


def check_lists(X, lab, idx, k0, nn, block=2000):
    """Each tested row's list: k0_l - 1 distinct finite rows of its label other than itself, then -1; every other row
    all -1; the set differs from fp64's only inside DESIGN §9's band of the (k0_l - 1)-th same-label distance.
    Returns the rows whose set equals fp64's."""
    N = len(X)
    lab = np.zeros(N, np.int64) if lab is None else lab
    fin, c, norm = finite_rows(X)
    same = np.zeros(N, bool)
    assert idx.shape[1] == max(int(k0.max()) - 1, 0)
    for l in range(len(k0)):
        rows = np.flatnonzero(lab == l)
        if k0[l] == 0:
            assert (idx[rows] == -1).all()
            continue
        m = k0[l] - 1
        assert (idx[rows[~fin[rows]]] == -1).all()
        rows = rows[fin[rows]]
        got = idx[rows]
        assert (got[:, m:] == -1).all() and (got[:, :m] >= 0).all()
        back = np.full(N, -1)
        back[rows] = np.arange(len(rows))
        pos = back[got[:, :m]]
        assert (pos >= 0).all(), "a listed row is not a finite row of the label"
        assert (np.sort(pos, 1)[:, 1:] != np.sort(pos, 1)[:, :-1]).all(), "a row is listed twice"
        assert (pos != np.arange(len(rows))[:, None]).all(), "a row lists itself"
        F = X[rows] - c
        xn = norm[rows].max()
        for r0 in range(0, len(rows), block):
            r1 = min(len(rows), r0 + block)
            D = np.maximum((F[r0:r1] ** 2).sum(1)[:, None] - 2.0 * F[r0:r1] @ F.T + (F ** 2).sum(1)[None, :], 0.0)
            D[np.arange(r1 - r0), np.arange(r0, r1)] = np.inf
            check_band(D, np.take_along_axis(D, pos[r0:r1], 1), m, knr.band(norm[rows[r0:r1]], xn, X.shape[1]))
        same[rows] = (np.sort(got[:, :m], 1) == np.sort(nn[rows, :m], 1)).all(1)
    return same


def check_values(got, want, dof, rows):
    """stat within STAT_REL of want's, pval within P_REL (1 + dof) of scipy's tail of the call's own stat."""
    s, p = got
    err = np.abs(s[rows] - want[rows])
    assert (err <= STAT_REL * np.abs(want[rows]) + STAT_ABS).all(), f"stat off by {err.max():.3e}"
    ref = chi2.sf(s[rows], dof[rows])
    big = ref >= 1e-300
    perr = np.abs(p[rows] - ref)
    assert (perr[big] <= P_REL * (1 + dof[rows][big]) * ref[big]).all(), "pval off scipy's tail"
    assert ((p[rows][~big] >= 0) & (p[rows][~big] <= 1e-290)).all()


@pytest.mark.parametrize("row", ROWS, ids=[r[0] for r in ROWS])
def test_kbet_table(row):
    import torch
    name, N, d, dtype, o = row
    X, b, lab, n_labels, n_batches = _case(name, N, d, o)
    X = X.astype(dtype)
    N = len(X)
    xt = strided(X) if o.get("strided") else torch.as_tensor(X, device="cuda:0")
    h = gpu_harmony()
    bt = torch.as_tensor(b, device="cuda:0")
    lt = None if lab is None else torch.as_tensor(lab, device="cuda:0")
    if o.get("unused"):    # the codes' counts come from the call's arguments: through the C ABI
        from harmony_b200 import _lib
        L = _lib.lib()
        stat, pval = (torch.empty(N, dtype=torch.float64, device="cuda:0") for _ in range(2))
        k0_out = torch.empty(n_labels, dtype=torch.int32, device="cuda:0")
        idx = torch.empty((N, 69), dtype=torch.int32, device="cuda:0")
        assert L.hb_kbet(h._h, ptr(xt), 0, d, N, d, ptr(bt), n_batches, ptr(lt), n_labels, 0, ptr(stat), ptr(pval),
                         ptr(k0_out), ptr(idx), 69, None) == 0
        idx = idx[:, :int(k0_out.max()) - 1]
    else:
        stat, pval, k0_out, idx = h.kbet(xt, bt, lt, o.get("k0", 0), return_neighbors=True)
    assert stat.is_cuda and stat.dtype == torch.float64 and pval.dtype == torch.float64 and idx.dtype == torch.int32
    stat, pval, k0_out, idx = (v.cpu().numpy() for v in (stat, pval, k0_out, idx))
    want = kr.kbet(X, b, lab, o.get("k0", 0), n_labels)
    np.testing.assert_array_equal(k0_out, want.k0)
    tested = ~np.isnan(want.stat)
    assert (np.isnan(stat) == ~tested).all() and (np.isnan(pval) == ~tested).all()
    same = check_lists(X.astype(np.float64), lab, idx, want.k0, want.nn)
    from_idx = kr.kbet(X, b, lab, o.get("k0", 0), n_labels, idx=np.where(idx < 0, 0, idx))
    check_values((stat, pval), from_idx.stat, want.dof, tested)
    np.testing.assert_array_equal(from_idx.stat[same], want.stat[same])
    check_values((stat, pval), want.stat, want.dof, same)
    if o.get("nan"):
        assert np.isnan(stat[[3, 11, 700, 1200, 2000, 2500]]).all()
    if name.startswith("3000"):
        assert not tested.any() and (k0_out == 0).all()
    if "small" in o:
        assert k0_out[-1] == 0 and (k0_out[:-1] == 129).all()
    print(f"[kbet {name}] tested {tested.sum()}, sets equal to fp64's {same[tested].mean() if tested.any() else 1:.5f}, "
          f"k0 {sorted(set(k0_out.tolist()))}")


def test_inputs_agree_and_repeat():
    """Host arrays, CUDA tensors, a DataFrame and CUDA integer labels give one score; two calls are bit-identical."""
    import torch
    rng = np.random.default_rng(4)
    X, t = generic(rng, 20000, 30)
    bcode = rng.integers(0, 3, len(X))
    X += rng.standard_normal((3, 30))[bcode]
    batch = np.array(["b1", "b0", "b2"])[bcode]
    meta = Frame({"batch": batch, "type": t})
    s_host, rates, (stat, pval) = kbet(X, meta, "batch", "type", return_all=True)
    assert isinstance(stat, np.ndarray) and set(rates) == set(range(12))
    Xd = torch.as_tensor(X, device="cuda:0")
    s_dev, _, (sd, pd) = kbet(Xd, {"batch": batch, "type": torch.as_tensor(t, device="cuda:0")}, "batch", "type",
                              return_all=True)
    assert sd.is_cuda and s_dev == s_host
    np.testing.assert_array_equal(sd.cpu().numpy(), stat)
    np.testing.assert_array_equal(pd.cpu().numpy(), pval)
    assert kbet(X, meta, "batch", "type", scaled=False) == pytest.approx(1 - s_host, abs=1e-15)
    h = gpu_harmony()
    bt, lt = torch.as_tensor(bcode.astype(np.int32), device="cuda:0"), torch.as_tensor(t.astype(np.int32), device="cuda:0")
    first = [v.cpu().numpy() for v in h.kbet(Xd, bt, lt, 0, return_neighbors=True)]
    second = [v.cpu().numpy() for v in h.kbet(Xd, bt, lt, 0, return_neighbors=True)]
    for u, v in zip(first, second):
        np.testing.assert_array_equal(u, v)
    assert np.isnan(kbet(X[:9], {"batch": batch[:9]}, "batch"))      # no label tested: NaN
    with pytest.raises(ValueError):
        kbet(X, {"batch": torch.as_tensor(bcode, device="cuda:0")}, "batch")   # device labels, host X


def test_handle_state_untouched():
    """hb_kbet between cluster_cpp and moe_correct_ridge_cpp and on a mapping handle: Z_corr, R and Y read bit for bit
    the same before and after the call."""
    import torch

    def call(h, phase, data):
        if phase == "mapped":
            stat = h.kbet(h.get_tensor("Z_corr"), data.mapped_codes)[0]
        else:
            stat = h.kbet(data.probe, data.codes)[0]
        assert not torch.isnan(torch.as_tensor(stat)).all()

    handle_state_untouched(call)


def _call(L, g, a):
    return L.hb_kbet(g._h, a["X"], a["xt"], a["xld"], a["N"], a["d"], a["bat"], a["nb"], a["lab"], a["nl"], a["k0"],
                     a["stat"], a["pval"], a["k0o"], a["idx"], a["ld"], a.get("stream"))


def _buffers(N, d, k):
    import torch
    dev = torch.device("cuda", 0)
    X = torch.as_tensor(np.random.default_rng(0).standard_normal((N, d)).astype(np.float32), device=dev)
    bat = torch.as_tensor(np.arange(N, dtype=np.int32) % 2, device=dev)
    lab = torch.zeros(N, dtype=torch.int32, device=dev)
    stat, pval = torch.full((N,), -9.0, dtype=torch.float64, device=dev), torch.full((N,), -9.0, dtype=torch.float64, device=dev)
    k0o = torch.full((1,), -9, dtype=torch.int32, device=dev)
    idx = torch.full((N, k), -9, dtype=torch.int32, device=dev)
    return X, bat, lab, stat, pval, k0o, idx


def test_refusals_launch_nothing():
    from harmony_b200 import _lib
    L = _lib.lib()
    g = gpu_harmony()
    N, d = 200, 8
    X, bat, lab, stat, pval, k0o, idx = _buffers(N, d, 69)
    host = np.zeros(N, np.float64)
    H = host.ctypes.data_as(ctypes.c_void_p)
    good = dict(X=ptr(X), xt=0, xld=d, N=N, d=d, bat=ptr(bat), nb=2, lab=ptr(lab), nl=1, k0=0, stat=ptr(stat),
                pval=ptr(pval), k0o=ptr(k0o), idx=ptr(idx), ld=69)
    bad = [dict(N=1), dict(N=0), dict(N=2 ** 31), dict(d=0), dict(d=129, xld=129), dict(nb=0), dict(nl=0),
           dict(nb=N + 1), dict(nl=N + 1), dict(k0=1), dict(k0=-1), dict(k0=130), dict(xt=2), dict(xt=-1),
           dict(xld=d - 1), dict(X=None), dict(bat=None), dict(stat=None), dict(pval=None), dict(X=H), dict(bat=H),
           dict(lab=H), dict(stat=H), dict(pval=H), dict(k0o=H), dict(idx=H)]
    refusals_launch_nothing(g, lambda a: _call(L, g, a), good, bad)
    assert _call(L, g, dict(good, lab=None, nl=0, k0o=None, idx=None)) == 0     # n_labels is ignored without labels
    assert g.kernel_launches > 0


@pytest.mark.parametrize("case", ["batch_past_n_batches", "label_negative", "short_idx_ld", "short_idx_ld_fixed_k0"])
def test_late_refusals_write_nothing(case):
    """A code out of range or an idx_ld below the largest k0 - 1: status 2 after the index pass, outputs unwritten."""
    from harmony_b200 import _lib
    L = _lib.lib()
    g = gpu_harmony()
    N, d = 2000, 8
    X, bat, lab, stat, pval, k0o, idx = _buffers(N, d, 69)
    a = dict(X=ptr(X), xt=0, xld=d, N=N, d=d, bat=ptr(bat), nb=2, lab=ptr(lab), nl=1, k0=0, stat=ptr(stat),
             pval=ptr(pval), k0o=ptr(k0o), idx=ptr(idx), ld=69)
    if case == "batch_past_n_batches":
        bat[17] = 2
        msg = "hb_kbet: batches of cell 17 is not a code in 0..1"
    elif case == "label_negative":
        lab[5] = -1
        msg = "hb_kbet: labels of cell 5 is not a code in 0..0"
    elif case == "short_idx_ld":          # 1000 rows per batch: k0 = 70 by the rule
        a["ld"] = 68
        msg = "hb_kbet: idx_ld = 68 is smaller than the 69 neighbours of the largest k0"
    else:
        a.update(k0=30, ld=28)
        msg = "hb_kbet: idx_ld = 28 is smaller than the 29 neighbours of the largest k0"
    assert _call(L, g, a) == 2 and L.hb_last_error(g._h).decode() == msg
    unwritten(-9, stat, pval, k0o, idx)


def test_launch_count_and_stream_order():
    """The index pass's launches (as hb_silhouette's on the same codes) plus colsum, prepare, count, sweep, merge and
    k_kbet; with no label tested no sweep or merge.  The call reads X after the work queued on the caller's stream."""
    import torch
    rng = np.random.default_rng(9)
    X, t = generic(rng, 30000, 20)
    b = rng.integers(0, 3, len(X)).astype(np.int32)
    t = (t % 4).astype(np.int32)
    xt, bt, lt = (torch.as_tensor(v, device="cuda:0") for v in (X.astype(np.float32), b, t))
    g = gpu_harmony()
    g.silhouette(xt, bt, lt)
    sil = g.kernel_launches
    g = gpu_harmony()
    want = [v.cpu().numpy() for v in g.kbet(xt, bt, lt)]
    assert g.kernel_launches == g.region_time("kbet")[1] == sil + 2
    small = torch.as_tensor(np.arange(40, dtype=np.int32) % 5, device="cuda:0")   # 8 rows per label: none tested
    g = gpu_harmony()
    g.silhouette(xt[:40], bt[:40], small)
    sil = g.kernel_launches
    g = gpu_harmony()
    g.kbet(xt[:40], bt[:40], small)
    assert g.kernel_launches == sil
    g = gpu_harmony()
    got = after_late_write(xt, float("nan"), 200_000_000, lambda dst: [v.cpu().numpy() for v in g.kbet(dst, bt, lt)])
    for u, v in zip(want, got):
        np.testing.assert_array_equal(u, v)


def test_integration_scores_end_to_end():
    """The raw PCs of cell_lines: the restatement gives rejection rates 0.9913 / 0.8143 and a scaled kBET of 0.0972.
    The CPU oracle's fp64 integration (make_Y0 centroids, seeds 0 and 1) scores 0.7604 and 0.7635 there."""
    import torch
    Z, meta = load_cell_lines(False)
    s0, rates0, _ = kbet(Z, meta, "dataset", "cell_type", return_all=True)
    assert s0 == pytest.approx(0.0972, abs=0.005)
    Zc = RunHarmony(torch.as_tensor(Z, device="cuda:0"), meta, "dataset", verbose=False, seed=1)
    s1, rates1, _ = kbet(Zc, meta, "dataset", "cell_type", return_all=True)
    print(f"[kbet cell_lines] {s0:.4f} {rates0} -> {s1:.4f} {rates1}")
    assert s1 >= 0.6
