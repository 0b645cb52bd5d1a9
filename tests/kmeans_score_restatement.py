"""An fp64 restatement of hb_kmeans (DESIGN §15) and of the NMI / ARI fold, written from the definitions: greedy
k-means++ on the prepared rows (float32 after centring on the column mean of the finite rows) with the library's
keyed-hash races, sklearn's Lloyd iteration, and the scores from a contingency table."""
import math

import numpy as np

from kmeans_restatement import CELL_TAG, U24
from stages import _mix64

SEED_TAG = 0x6b6d2b2b73636f72     # kmeans_score_key: hb_mix64(seed ^ SEED_TAG ^ hb_mix64(init))
MAX_T = 8                          # the uniform of (round, trial) sits at kmeans_uniform's index round * MAX_T + trial
KEY_REL = 4.0 * U24                # fp32 rounding of a race key, and the log's last bits


def trials(K):
    return 2 + int(math.floor(math.log(K)))


def score_key(seed, init):
    s = np.array([int(seed)], dtype=np.uint64)
    return _mix64(s ^ np.uint64(SEED_TAG) ^ _mix64(np.array([int(init)], dtype=np.uint64)))[0]


def uniform(key, rnd, t, rows):
    """kmeans_uniform(key, rnd * MAX_T + t, rows) as float32."""
    i = np.uint64(rnd * MAX_T + t)
    g = np.asarray(rows, dtype=np.uint64)
    h = _mix64(np.uint64(key) ^ _mix64((i << np.uint64(40)) ^ g ^ np.uint64(CELL_TAG)))
    u = ((h >> np.uint64(40)).astype(np.float32) + np.float32(0.5)) * np.float32(U24)
    return np.minimum(u, np.float32(1.0 - U24))


def prepare(X):
    """-> (finite mask, the prepared rows fp32(x - m) as float64, m): m the fp64 column mean of the finite rows."""
    X = np.asarray(X, dtype=np.float64)
    fin = np.isfinite(X).all(axis=1)
    m = X[fin].mean(axis=0)
    P = np.zeros_like(X)
    P[fin] = (X[fin] - m).astype(np.float32)
    return fin, P, m


def sqdist(P, c):
    """|p - c|^2 in fp64 for every row of P."""
    e = P - P[c]
    return np.einsum("ij,ij->i", e, e)


def race_keys(key, rnd, w, fin):
    """The fp32 race keys -ln(u) / w of every row for each trial of round `rnd` ([T, N], +inf where a row takes no
    part: non-finite or w = 0)."""
    N = len(w)
    out = []
    for t in range(MAX_T):
        e = -np.log(uniform(key, rnd, t, np.arange(N)).astype(np.float64))
        with np.errstate(divide="ignore"):
            k = (e / w).astype(np.float32).astype(np.float64)
        out.append(np.where(fin & (w > 0), k, np.inf))
    return np.array(out)


def race_weights(D2, fin):
    """The weights of a round after the first: D^2, or 1 for every finite row when no finite row has D^2 > 0."""
    return D2 if (D2[fin] > 0).any() else np.where(fin, 1.0, 0.0)


def seeding(P, fin, K, seed, init=0):
    """Greedy k-means++ by the library's rule -> the K seed rows."""
    key = score_key(seed, init)
    T = trials(K)
    ones = np.where(fin, 1.0, 0.0)
    s0 = int(np.argmin(race_keys(key, 0, ones, fin)[0]))   # argmin: the lowest row on a tie, as the packed key
    seeds, D2 = [s0], sqdist(P, s0)
    for r in range(1, K):
        keys = race_keys(key, r, race_weights(D2, fin), fin)[:T]
        cand = keys.argmin(axis=1)
        pots = [np.minimum(D2, sqdist(P, c))[fin].sum() for c in cand]
        c = int(cand[int(np.argmin(pots))])
        seeds.append(c)
        D2 = np.minimum(D2, sqdist(P, c))
    return np.array(seeds)


def admissible(keys, rel=KEY_REL):
    """The rows whose race key may be the smallest once each is known to a relative rel: lo <= min hi."""
    lo, hi = keys * (1 - rel), keys * (1 + rel)
    return np.nonzero(lo <= hi.min())[0]


def replay_seeds(P, fin, K, seed, init, got, pot_rel=1e-12):
    """Replays the seeding from the GPU's seeds `got`, round by round: each must be an admissible race winner of one
    of the round's trials, and the potential argmin among the candidates where every trial's winner is unambiguous.
    -> the rounds in which every draw was unambiguous."""
    key = score_key(seed, init)
    T = trials(K)
    ones = np.where(fin, 1.0, 0.0)
    assert int(got[0]) in admissible(race_keys(key, 0, ones, fin)[0]), "round 0"
    exact = 1 if len(admissible(race_keys(key, 0, ones, fin)[0])) == 1 else 0
    D2 = sqdist(P, int(got[0]))
    for r in range(1, K):
        keys = race_keys(key, r, race_weights(D2, fin), fin)[:T]
        sets = [admissible(k) for k in keys]
        g = int(got[r])
        assert any(g in s for s in sets), f"round {r}: seed {g} wins no race"
        if all(len(s) == 1 for s in sets):
            cand = [int(s[0]) for s in sets]
            pots = np.array([np.minimum(D2, sqdist(P, c))[fin].sum() for c in cand])
            ok = {cand[t] for t in range(T) if pots[t] <= pots.min() * (1 + pot_rel)}
            assert g in ok, f"round {r}: seed {g} is not the potential argmin {cand[int(np.argmin(pots))]}"
            exact += len(ok) == 1
        D2 = np.minimum(D2, sqdist(P, g))
    return exact


def assign(X, C):
    """The nearest centre of every row (fp64, the lower index on a tie) and the distances to all."""
    D = ((X[:, None, :] - C[None, :, :]) ** 2).sum(axis=2) if len(X) * len(C) * X.shape[1] < 4e7 else \
        (X ** 2).sum(1)[:, None] - 2 * X @ C.T + (C ** 2).sum(1)[None, :]
    return D.argmin(axis=1), D


def lloyd(X, centres, max_iter=300, tol=1e-4):
    """sklearn's algorithm="lloyd" on the finite rows of X from `centres`, with empty clusters kept -> (labels, -1 for
    non-finite rows, centres, inertia, n_iter)."""
    X = np.asarray(X, dtype=np.float64)
    fin = np.isfinite(X).all(axis=1)
    Xf = X[fin]
    C = np.array(centres, dtype=np.float64)
    K = len(C)
    tol_abs = tol * Xf.var(axis=0).mean()
    old = np.full(len(Xf), -1)
    strict, it = False, 0
    for i in range(max_iter):
        lab = assign(Xf, C)[0]
        Cn = C.copy()
        for k in range(K):
            m = lab == k
            if m.any():
                Cn[k] = Xf[m].mean(axis=0)
        shift = ((Cn - C) ** 2).sum()
        C, it = Cn, i + 1
        if (lab == old).all():
            strict = True
            break
        if shift <= tol_abs:
            break
        old = lab
    if not strict:
        lab = assign(Xf, C)[0]
    labels = np.full(len(X), -1)
    labels[fin] = lab
    inertia = ((Xf - C[lab]) ** 2).sum()
    return labels, C, inertia, it


def kmeans(X, K, seed=0, max_iter=300, tol=1e-4):
    """One init of the whole call: the seeds, then Lloyd from their rows."""
    X = np.asarray(X, dtype=np.float64)
    fin, P, _ = prepare(X)
    seeds = seeding(P, fin, K, seed)
    return (seeds,) + lloyd(X, X[seeds], max_iter, tol)


def nmi_ari(t, p):
    """NMI (arithmetic mean of the entropies) and ARI of two labelings, rows with p == -1 left out, from the
    definitions; sklearn's special cases: NMI 1 when both have one class (or no row), 0 when the mutual information is
    0; ARI 1 when the pair counts agree."""
    t, p = np.asarray(t), np.asarray(p)
    keep = p != -1 if p.dtype.kind in "iuf" else np.ones(len(p), bool)
    t, p = np.unique(t[keep], return_inverse=True)[1], np.unique(p[keep], return_inverse=True)[1]
    n = len(t)
    C = np.zeros((t.max() + 1 if n else 0, p.max() + 1 if n else 0))
    np.add.at(C, (t, p), 1)
    a, b = C.sum(1), C.sum(0)
    H = lambda v: -sum(x / n * math.log(x / n) for x in v if x > 0)  # noqa: E731
    if n == 0 or (len(a) == 1 and len(b) == 1):
        nmi = 1.0
    else:
        mi = sum(C[i, j] / n * math.log(n * C[i, j] / (a[i] * b[j])) for i, j in zip(*np.nonzero(C)))
        nmi = 0.0 if mi <= 1e-15 else mi / ((H(a) + H(b)) / 2)
    comb = lambda v: sum(int(x) * (int(x) - 1) // 2 for x in v)  # noqa: E731
    sij, sa, sb, tot = comb(C.ravel()), comb(a), comb(b), n * (n - 1) // 2
    if sa == sb == sij:  # the two labelings pair up the same rows
        return nmi, 1.0
    expected = sa * sb / tot
    return nmi, (sij - expected) / ((sa + sb) / 2 - expected)
