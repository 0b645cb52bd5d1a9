"""Mapping a query onto a reference on the GPU, against the fp64 restatement (map_restatement.py), stage by stage with
the bars of stages.py: the compression of an integration, the query's assignment and its correction, on every
assignment and apply kernel, then device I/O, the end-to-end MapQuery and the refusals."""
import ctypes

import numpy as np
import pytest

from harmony_b200 import HarmonyReference, MapQuery, RunHarmony, prepare_inputs
from helpers import gpu_harmony, gpu_setup, make_perms, make_Y0, num_sms, rel_l2, synthetic
from map_restatement import assign, correct, lambda_levels, map_query, reference_stats, type_offset, weights_folded
from stages import HB_KS_FFMA_CONTRACTIONS, HB_KS_WIDE, TOL_OE, TOL_R1, TOL_Y, TOL_Z, f32, wide_paths

pytestmark = pytest.mark.gpu


# ---- compression ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,K,N", [(50, 100, 20000), (300, 100, 20000), (64, 1024, 40000)])
def test_reference_compression(d, K, N):
    """hb_reference after two injected iterations against fp64 sums of the same object's getZcorr() / getR(); at
    d = 50 also after a further cluster_cpp, whose Z_corr the library normalises on the first read."""
    Z, meta = synthetic(N, d, [4], n_types=12, seed=d + K)
    a = prepare_inputs(Z, meta, "cov0", nclust=K, early_stop=False)
    g = gpu_setup(a, T=5, device=0)
    g.init_cluster_cpp(make_Y0(Z, K, 1))
    perms = make_perms(N, 15, 2).reshape(3, 5, N)
    for it in range(2):
        assert g.cluster_cpp(perms[it]) == 0
        g.moe_correct_ridge_cpp()
    states = ["after ridge"]
    if d == 50:
        states.append("after cluster_cpp")
    for state in states:
        if state == "after cluster_cpp":
            assert g.cluster_cpp(perms[2]) == 0
        ref = g.reference()
        Nr, Cref, Y = reference_stats(g.getZcorr().T, g.getR().T)
        errs = dict(Nr=float(np.abs(ref.Nr - Nr).max() / max(1.0, np.abs(Nr).max())),
                    Cref=float(np.abs(ref.Cref - Cref).max() / max(1.0, np.abs(Cref).max())),
                    Y=float(np.abs(ref.centroids - Y).max()))
        print(f"[map compression d={d} K={K} {state}] {errs}")
        assert errs["Nr"] <= TOL_OE and errs["Cref"] <= TOL_OE and errs["Y"] <= TOL_Y, errs
        np.testing.assert_array_equal(ref.sigma, g.sigma)
        assert g.region_time("reference")[1] > 0


# ---- assignment and correction, row by row --------------------------------------------------------------------------
def planted_reference(rng, K, d, M, sigma, zero=None):
    """A reference around the type centres M: unit centroids, masses, Cref along the centroids.  zero: a cluster with
    Nr = 0, Cref = 0, small sigma and a centroid opposite the query's cells (its assignment underflows to 0)."""
    Y = M[np.arange(K) % len(M)] + 0.3 * rng.standard_normal((K, d)) * np.abs(M).mean()
    Nr = rng.uniform(20.0, 3000.0, K)
    Cref = Nr[:, None] * (Y + 0.1 * rng.standard_normal((K, d)) * np.abs(M).mean())
    Y = Y / np.linalg.norm(Y, axis=1, keepdims=True)
    sigma = np.broadcast_to(np.asarray(sigma, dtype=np.float64), (K,)).copy()
    if zero is not None:
        u = M.mean(axis=0)
        Y[zero] = -u / np.linalg.norm(u)
        Nr[zero], Cref[zero], sigma[zero] = 0.0, 0.0, 0.005
    return HarmonyReference(Y, Nr, Cref, sigma)


def planted_query(rng, N, d, B_vec, absent=(), special=False):
    """Query cells around shared type centres (with a common offset, so a planted opposite centroid is far from all),
    a shift per level; labels over B_vec with the levels in `absent` unused.  special: rows at 0, 1e-25 and 1e20."""
    n_types = 8
    M = rng.standard_normal((n_types, d)) * 2.0 + 3.0
    phi = []
    off = 0
    for Bc in B_vec:
        lv = np.array([b for b in range(Bc) if off + b not in absent])
        phi.append(off + rng.choice(lv, N))
        off += Bc
    phi = np.stack(phi, axis=1)
    Z = M[rng.integers(0, n_types, N)] + 0.7 * rng.standard_normal((N, d))
    Z += 1.5 * rng.standard_normal((off, d))[phi].sum(axis=1)
    scale = 10.0 / np.sqrt(1.0 + np.arange(d))
    Z *= scale
    if special and N >= 9:
        s = rng.choice(N, 9, replace=False)
        Z[s[:3]] = 0.0
        Z[s[3:6]] *= 1e-25 / np.abs(Z[s[3:6]]).max(axis=1, keepdims=True)
        Z[s[6:]] *= 1e20 / np.abs(Z[s[6:]]).max(axis=1, keepdims=True)
    return Z, phi, M * scale


ROWS = [
    # name, K, d, B_vec, kernel_set, (assign, apply) kernels, Nq, options
    ("fused_c1", 100, 50, [3], 0, (1, 1), 50000, dict(special=True, zero=5)),
    ("ffma_c2_sigma_lam_cov", 100, 50, [3, 2], HB_KS_FFMA_CONTRACTIONS, (2, 2), 5000,
     dict(sigma="per_cluster", lam=[0.5, 2.0], special=True)),
    ("logits_c3", 300, 100, [2, 2, 2], 0, (3, 1), 129, dict(lam=0.3)),
    ("dchunk_cols_b1", 100, 50, [1], HB_KS_WIDE, (4, 3), 5, dict()),
    ("ffma_cols_absent_zero", 64, 300, [4], 0, (2, 3), 2000, dict(absent=(1, 3), zero=7, sigma="per_cluster")),
    ("fused_nq1", 100, 50, [2], 0, (1, 1), 1, dict()),
    ("wide_c2_absent", 200, 64, [3, 3], HB_KS_WIDE, (4, 3), 3000, dict(absent=(4,), lam=[1.0, 0.2])),
]


def _map_row(K, d, B_vec, kernel_set, Nq, opts, seed):
    rng = np.random.default_rng(seed)
    Z, phi, M = planted_query(rng, Nq, d, B_vec, opts.get("absent", ()), opts.get("special", False))
    sigma = rng.uniform(0.05, 0.2, K) if opts.get("sigma") == "per_cluster" else 0.1
    ref = planted_reference(rng, K, d, M, sigma, opts.get("zero"))
    lam = lambda_levels(opts.get("lam", 1.0), B_vec)
    g = gpu_harmony()
    if kernel_set:
        g.kernel_set = kernel_set
    g.map_setup(Z, phi, B_vec, lam, ref)
    g.map()
    return g, Z, phi, ref, lam


@pytest.mark.parametrize("row", ROWS, ids=[r[0] for r in ROWS])
def test_map_stages(row):
    name, K, d, B_vec, kernel_set, paths, Nq, opts = row
    g, Z, phi, ref, lam = _map_row(K, d, B_vec, kernel_set, Nq, opts, seed=sum(map(ord, name)))
    J = len(np.unique(phi, axis=0))
    got = wide_paths(K, d, J, Nq, num_sms(), nb=1, kernel_set=kernel_set)
    assert (got[0], got[2]) == paths          # natural-order assignment, ridge apply
    Rg = g.getR().T
    Zg = g.getZcorr().T
    np.testing.assert_array_equal(g.getZorig().T, f32(Z))
    np.testing.assert_array_equal(g.Y.T, f32(ref.centroids))
    np.testing.assert_array_equal(g.sigma, f32(ref.sigma))
    assert np.isfinite(Rg).all() and np.isfinite(Zg).all()
    # assignment: the fp64 softmax of the same fp32 query and reference
    Rn = assign(f32(Z), f32(ref.centroids), f32(ref.sigma))
    # correction: the fp64 steps 3-4 driven by the library's own assignment
    Zn, _ = map_query(f32(Z), phi, B_vec, f32(lam), None, f32(ref.Nr), f32(ref.Cref), None, R=Rg)
    errs = dict(R=float(np.abs(Rg - Rn).max()), Z=rel_l2(Zg, Zn))
    print(f"[map {name}] {errs}")
    assert errs["R"] <= TOL_R1 and errs["Z"] <= TOL_Z, errs
    if sum(B_vec) == 1:
        assert np.abs(Zg - f32(Z)).max() > 1e-3 * np.abs(Z).max()   # one query batch is corrected
    if opts.get("zero") is not None:
        k = opts["zero"]
        assert np.all(Rg[:, k] == 0)
        B = sum(B_vec)
        W = weights_folded(Rg, f32(Z), phi, B, f32(lam), f32(ref.Nr), f32(ref.Cref))
        assert np.all(W[k] == 0)
        Rk = Rg.copy()
        Rk[:, k] = 0.0
        assert rel_l2(Zg, correct(f32(Z), Rk, phi, W)) <= TOL_Z   # the cluster contributes nothing
    for region in ("assign", "ridge_stats", "ridge_solve", "ridge_apply"):
        assert g.region_time(region)[1] > 0, region


def test_map_is_repeatable():
    g, Z, phi, ref, lam = _map_row(100, 50, [3], 0, 2000, {}, seed=11)
    Z1, R1 = g.getZcorr(), g.getR()
    g.map()
    assert rel_l2(g.getZcorr(), Z1) <= TOL_Z and np.abs(g.getR() - R1).max() <= TOL_R1


# ---- device I/O -----------------------------------------------------------------------------------------------------
def test_map_device_io():
    import torch
    K, d, B_vec, Nq = 100, 50, [3, 2], 3000
    g, Z, phi, ref, lam = _map_row(K, d, B_vec, 0, Nq, dict(sigma="per_cluster"), seed=21)
    Zh, Rh = g.getZcorr().T, g.getR().T
    dev = torch.device("cuda", 0)
    wide = torch.zeros((Nq, d + 7), dtype=torch.float32, device=dev)
    wide[:, :d] = torch.from_numpy(Z).to(dev, torch.float32)
    inputs = {
        "fp32 rows": torch.from_numpy(Z).to(dev, torch.float32),
        "fp64 columns": torch.from_numpy(np.ascontiguousarray(Z.T)).to(dev),
        "fp32 strided rows": wide[:, :d],
    }
    phis = {"host labels": phi, "device labels": torch.from_numpy(phi).to(dev)}
    for zname, Zt in inputs.items():
        for pname, ph in phis.items():
            h = gpu_harmony()
            h.map_setup(Zt, ph, B_vec, lam, ref)
            h.map()
            for dtype in (torch.float32, torch.float64):
                Zd = h.get_tensor("Z_corr", dtype=dtype).cpu().numpy()
                Rd = h.get_tensor("R", dtype=dtype).cpu().numpy()
                errs = dict(Z=rel_l2(Zd, Zh), R=float(np.abs(Rd - Rh).max()))
                print(f"[map device io {zname}, {pname}, {dtype}] {errs}")
                assert errs["Z"] <= TOL_Z and errs["R"] <= TOL_R1, (zname, pname, dtype, errs)
    # MapQuery on a CUDA tensor with device labels returns a tensor of the input's dtype
    Zt = torch.from_numpy(Z).to(dev)
    out = MapQuery(Zt, {"a": torch.from_numpy(phi[:, 0]).to(dev), "b": torch.from_numpy(phi[:, 1] - 3).to(dev)},
                   ["a", "b"], ref, lambda_=lam[[0, 3]], verbose=False)
    assert out.dtype == torch.float64 and out.device == Zt.device
    assert rel_l2(out.cpu().numpy(), Zh) <= TOL_Z


# ---- end to end -----------------------------------------------------------------------------------------------------
# MapQuery against the fp64 restatement on the same reference arrays: rel-L2 bar of the mapped embedding (measured
# 8.1e-7 at lambda = 1 and 8.6e-7 at lambda = 0.1 on an H100 80GB HBM3 at 700 W), and the margin on the reduction of
# the per-type offset to the reference (measured: x3.82 and x3.87, equal to the fp64 restatement's to two decimals)
TOL_E2E = 1e-5
OFFSET_MARGIN = 0.05


@pytest.mark.parametrize("lam", [1.0, 0.1])
def test_map_query_end_to_end(tmp_path, lam):
    N, d, K, n_types = 20000, 20, 30, 8
    Z, meta = synthetic(N, d, [2], n_types=n_types, seed=3)
    t = np.random.default_rng(3).integers(0, n_types, N)   # synthetic's first draw: the cell types
    rng = np.random.default_rng(0)
    is_ref = rng.random(N) < 0.7
    obj = RunHarmony(Z[is_ref], {"cov0": meta["cov0"][is_ref]}, "cov0", nclust=K, return_object=True, verbose=False,
                     seed=4)
    Zr = obj.getZcorr().T
    path = str(tmp_path / "ref.npz")
    obj.reference().save(path)
    ref = HarmonyReference.load(path)
    Zq0 = Z[~is_ref]
    lv = rng.integers(0, 2, len(Zq0))
    delta = rng.standard_normal((2, d)) * 2.0 * (10.0 / np.sqrt(1 + np.arange(d)))
    Zq = Zq0 + delta[lv]
    out = MapQuery(Zq, {"sample": lv}, "sample", ref, lambda_=lam, verbose=False)
    expect, _ = map_query(Zq, lv.reshape(-1, 1), [2], np.full(2, lam), ref.centroids, ref.Nr, ref.Cref, ref.sigma)
    tq, tr = t[~is_ref], t[is_ref]
    before = type_offset(Zq, tq, Zr, tr)
    gain_gpu = before / type_offset(out, tq, Zr, tr)
    gain_np = before / type_offset(expect, tq, Zr, tr)
    err = rel_l2(out, expect)
    print(f"[map end to end lambda={lam}] rel-L2 {err:.2e} (bar {TOL_E2E:.0e}); offset {before:.2f} -> "
          f"{before / gain_gpu:.2f} (x{gain_gpu:.2f}; fp64 x{gain_np:.2f})")
    assert err <= TOL_E2E
    assert gain_gpu >= gain_np * (1 - OFFSET_MARGIN)
    assert gain_np > 2.0


# ---- refusals -------------------------------------------------------------------------------------------------------
def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


HB_FLOAT64 = 1


def _raw_map_setup(g, Z, phi, B_vec, lam, ref, K=None, d=None, N=None, C=None, phi_ptr=None, z_dev=None,
                   dtype=HB_FLOAT64, ld=None):
    """Status of hb_map_setup called directly (the Python layer checks shapes first), or of hb_map_setup_device on the
    device pointer z_dev.  K, d, N, C, phi_ptr and ld replace what the arrays give."""
    Z = np.ascontiguousarray(Z, dtype=np.float64)
    phi = np.ascontiguousarray(phi, dtype=np.int32).reshape(len(Z), -1)
    B_vec = np.ascontiguousarray(B_vec, dtype=np.int32)
    lam = np.ascontiguousarray(lam, dtype=np.float64)
    arrs = [np.ascontiguousarray(a, dtype=np.float64) for a in (ref.centroids, ref.Nr, ref.Cref, ref.sigma)]
    d = Z.shape[1] if d is None else d
    labels = _ptr(phi) if phi_ptr is None else ctypes.c_void_p(phi_ptr)
    rest = (d, len(Z) if N is None else N, labels, _ptr(B_vec), len(B_vec) if C is None else C, _ptr(lam),
            ref.K if K is None else K, *(_ptr(a) for a in arrs))
    if z_dev is None:
        return g._L.hb_map_setup(g._h, _ptr(Z), *rest)
    return g._L.hb_map_setup_device(g._h, ctypes.c_void_p(z_dev), dtype, d if ld is None else ld, None, *rest)


def test_map_refusals():
    from harmony_b200.harmony import HarmonyError
    rng = np.random.default_rng(5)
    Z, phi, M = planted_query(rng, 200, 16, [2])
    ref = planted_reference(rng, 10, 16, M, 0.1)
    lam = np.ones(2)
    # status 2: lambda, sigma, labels outside their levels, K beyond the library's range
    for bad_lam in ([0.0, 1.0], [1.0, -2.0], [np.nan, 1.0], [np.inf, 1.0]):
        assert _raw_map_setup(gpu_harmony(), Z, phi, [2], bad_lam, ref) == 2
    for bad_sigma in (0.0, -0.1, np.inf, np.nan):
        r = HarmonyReference(ref.centroids, ref.Nr, ref.Cref, np.r_[ref.sigma[:-1], bad_sigma])
        assert _raw_map_setup(gpu_harmony(), Z, phi, [2], lam, r) == 2
    assert _raw_map_setup(gpu_harmony(), Z, np.where(phi == 1, 2, phi), [2], lam, ref) == 2
    assert _raw_map_setup(gpu_harmony(), Z, phi, [2], lam, ref, K=0) == 2
    # status 2 from the setup steps hb_setup shares, through the host and the device entry point: dimensions, K past
    # the library's range, device labels given to the host entry point, and the device entry point's Z checks
    import torch
    Zt = torch.from_numpy(Z).cuda()
    for z_dev in (None, Zt.data_ptr()):
        for bad in (dict(d=0), dict(N=0), dict(C=0), dict(K=0), dict(K=1025)):
            assert _raw_map_setup(gpu_harmony(), Z, phi, [2], lam, ref, z_dev=z_dev, **bad) == 2, (z_dev, bad)
    phi_t = torch.from_numpy(np.ascontiguousarray(phi, dtype=np.int32)).cuda()
    h = gpu_harmony()
    assert _raw_map_setup(h, Z, phi, [2], lam, ref, phi_ptr=phi_t.data_ptr()) == 2
    assert "hb_map_setup_device" in h._L.hb_last_error(h._h).decode()
    Zh = np.ascontiguousarray(Z)
    for z_dev, dtype, ld in ((Zt.data_ptr(), 7, None), (Zt.data_ptr(), HB_FLOAT64, 15), (Zh.ctypes.data, HB_FLOAT64, None)):
        assert _raw_map_setup(gpu_harmony(), Z, phi, [2], lam, ref, z_dev=z_dev, dtype=dtype, ld=ld) == 2, (dtype, ld)
    # d or K not matching the reference arrays: the Python layer refuses before the library
    with pytest.raises(ValueError):
        gpu_harmony().map_setup(Z[:, :15], phi, [2], lam, ref)
    with pytest.raises(ValueError):
        HarmonyReference(ref.centroids, ref.Nr[:-1], ref.Cref, ref.sigma)
    # status 3: a second setup, a sharded handle
    g = gpu_harmony()
    assert _raw_map_setup(g, Z, phi, [2], lam, ref) == 0
    assert _raw_map_setup(g, Z, phi, [2], lam, ref) == 3
    assert _raw_map_setup(g, Z, phi, [2], lam, ref, z_dev=Zt.data_ptr()) == 3
    with pytest.raises(HarmonyError):
        g.setup(Z, phi, 0.1, np.full(2, 2.0), None, 0.2, 5, 1e-5, 1e-4, 10, 0.05, [2], 1e-5)
    s = gpu_harmony()
    assert s._L.hb_set_shard(s._h, 400, 0) == 0
    assert _raw_map_setup(s, Z, phi, [2], lam, ref) == 3
    # status 3: the Harmony steps on a mapping handle, hb_map on an ordinary one, hb_reference before init
    L = g._L
    g.map()
    assert L.hb_init_cluster(g._h, None) == 3
    assert L.hb_cluster(g._h, None) == 3
    assert L.hb_moe_correct_ridge(g._h) == 3
    assert L.hb_compute_objective(g._h) == 3
    assert L.hb_check_convergence(g._h, 0) == -3
    assert L.hb_reference(g._h, None, None, None, None) == 3
    out = np.empty(64)
    assert L.hb_get_field(g._h, 6, _ptr(out)) == 3            # HB_W
    assert L.hb_set_field(g._h, 9, _ptr(np.full(10, 0.1))) == 3  # HB_SIGMA
    h = gpu_harmony()
    assert L.hb_reference(h._h, None, None, None, None) == 3   # before setup
    h.setup(Z, phi, 0.1, np.full(2, 2.0), None, 0.2, 5, 1e-5, 1e-4, 10, 0.05, [2], 1e-5)
    assert L.hb_reference(h._h, None, None, None, None) == 3   # before init_cluster_cpp
    assert L.hb_map(h._h) == 3
    # a query of one cell maps (no "fewer than 6 cells" refusal)
    one = gpu_harmony()
    one.map_setup(Z[:1], phi[:1], [2], lam, ref)
    one.map()
    assert np.isfinite(one.getZcorr()).all()
    assert L.hb_version() == 400
