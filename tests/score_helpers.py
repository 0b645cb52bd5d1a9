"""What the GPU tests of the score calls share: data, non-finite rows, input stand-ins, the band check of the neighbour
search, the handle-state, refusal, unwritten-output and stream-order scenarios."""
import ctypes
from types import SimpleNamespace

import numpy as np

from helpers import gpu_harmony, num_sms, synthetic


def generic(rng, n, d, types=12):
    """n rows around `types` centres in d dimensions -> (rows, each row's centre)."""
    M = rng.standard_normal((types, d)) * 3.0
    t = rng.integers(0, types, n)
    return M[t] + rng.standard_normal((n, d)), t


def non_finite_rows(X):
    """The non-finite values of the table cases, written into the rows X in place: NaN rows 3, 700 and 2000, +inf in
    column 5 of rows 11 and 2500, -inf in column 0 of row 1200."""
    X[[3, 700, 2000]] = np.nan
    X[[11, 2500], 5] = np.inf
    X[1200, 0] = -np.inf


class Frame:
    """What the scores need of a pandas DataFrame."""

    def __init__(self, cols):
        self._cols, self.columns = cols, list(cols)

    def __getitem__(self, name):
        return self._cols[name]


def strided(X):
    """The numpy rows X on cuda:0 as a view of row stride d + 3 that ends exactly where its allocation does."""
    import torch
    N, d = X.shape
    ld = d + 3
    buf = torch.zeros(N * ld - 3, dtype=getattr(torch, X.dtype.name), device="cuda:0")
    view = torch.as_strided(buf, (N, d), (ld, 1))
    view.copy_(torch.as_tensor(X, device="cuda:0"))
    return view


def geometry(hook, *args):
    """The eight values of the geometry test hook `hook` for these arguments on this device's SMs."""
    from harmony_b200 import _lib
    out = (ctypes.c_int64 * 8)()
    assert getattr(_lib.lib(), hook)(*args, num_sms(), out) == 0
    return list(out)


def check_band(D, got, k, b):
    """The bar of DESIGN §9 on a block of query rows: D the fp64 distances to every candidate (inf where excluded), got
    those of the rows returned, b each query row's band.  Every row closer than the k-th distance minus the band is
    returned and none beyond it plus the band, so a set that differs from fp64's differs inside the band only."""
    Dk = np.partition(D, k - 1, axis=1)[:, k - 1]
    must = (D < (Dk - b)[:, None]).sum(axis=1)
    have = (got < (Dk - b)[:, None]).sum(axis=1)
    assert (have == must).all(), f"rows {np.nonzero(have != must)[0][:5]} of the block miss a neighbour inside the band"
    assert (got <= (Dk + b)[:, None]).all(), "a row outside the band was returned"


def handle_state_untouched(call, baseline=False):
    """A score call between cluster_cpp and moe_correct_ridge_cpp in two rounds (``call(h, "run", data)``), and on a
    mapping handle before hb_map (``"setup"``) and after it (``"mapped"``): Z_corr, R and Y read bit for bit the same
    before and after the "run" and "mapped" calls.  ``data.probe`` holds 5000 CUDA rows and ``data.codes`` their int32
    CUDA labels, ``data.mapped_codes`` the host labels of the 6000 mapped cells.  With ``baseline`` the same run and
    mapping without the call come first, and both end where those end (to the run-to-run noise of the atomics' order);
    the two mappings use the reference of the run with the call."""
    import torch
    from harmony_b200 import prepare_inputs
    from helpers import gpu_setup, make_perms, make_Y0, rel_l2
    Z, meta = synthetic(20000, 50, [4], n_types=10, seed=3)
    a = prepare_inputs(Z, meta, "cov0", nclust=50, early_stop=False)
    Y0, perms = make_Y0(Z, 50, 1), make_perms(20000, 2 * a["max_iter_kmeans"], 2).reshape(2, a["max_iter_kmeans"], -1)
    data = SimpleNamespace(probe=torch.as_tensor(Z[:5000], device="cuda:0"),
                           codes=torch.as_tensor(meta["cov0"][:5000].astype(np.int32), device="cuda:0"),
                           mapped_codes=np.asarray(meta["cov0"][:6000], np.int32))
    state = lambda h: (h.getZcorr(), h.getR(), h.Y)  # noqa: E731

    def untouched(h, phase):
        before = state(h)
        call(h, phase, data)
        for u, v in zip(before, state(h)):
            np.testing.assert_array_equal(u, v)

    runs = (False, True) if baseline else (True,)
    outs = []
    for with_call in runs:
        g = gpu_setup(a, K=50, device=0)
        g.init_cluster_cpp(Y0)
        for it in range(2):
            assert g.cluster_cpp(perms[it]) == 0
            if with_call:
                untouched(g, "run")
            g.moe_correct_ridge_cpp()
        outs.append(state(g))
        ref = g.reference()
    maps = []
    for with_call in runs:
        m = gpu_harmony()
        m.map_setup(Z[:6000], a["phi_i"][:6000], a["B_vec"], 1.0, ref)
        if with_call:
            call(m, "setup", data)
        m.map()
        if with_call:
            untouched(m, "mapped")
        maps.append(state(m))
    if baseline:
        for u, v in zip(*outs):
            assert rel_l2(u, v) < 1e-4
        for u, v in zip(*maps):
            assert rel_l2(u, v) < 1e-4


def refusals_launch_nothing(g, call, good, bad):
    """``call(args)`` with each change of ``bad`` applied to the arguments ``good``: status 2 with a message on the
    handle ``g``, and not one kernel launched."""
    from harmony_b200 import _lib
    L = _lib.lib()
    for change in bad:
        assert call(dict(good, **change)) == 2 and L.hb_last_error(g._h), change
        assert g.kernel_launches == 0, change


def unwritten(fill, *outs):
    """Every output tensor of a refused call still holds the value ``fill`` it was filled with."""
    for t in outs:
        assert (t.cpu().numpy() == fill).all()


def after_late_write(src, fill, sleep, call):
    """What ``call(dst)`` returns on a new stream right after torch fills ``dst`` with ``fill`` (None: uninitialised),
    spins for ``sleep`` cycles and copies ``src`` into it there: a call ordered on that stream reads the copy."""
    import torch
    with torch.cuda.stream(torch.cuda.Stream()):
        dst = torch.empty_like(src) if fill is None else torch.full_like(src, fill)
        torch.cuda._sleep(sleep)
        dst.copy_(src)
        return call(dst)
