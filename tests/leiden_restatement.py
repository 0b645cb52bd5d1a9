"""fp64 numpy restatement of DESIGN §16: umap's connectivities of neighbour lists, and deterministic Leiden (local
moving with the up/down rule, greedy refinement with cancelled proposals, aggregation, iterations until no label
changes).  ``leiden`` also reports whether any decision lay within 1e-12 of a tie."""
import math

import numpy as np
import scipy.sparse as sp

TIE = 1e-12


def umap_graph(idx, dist, n_neighbors):
    """The symmetric CSR (scipy, fp64) of umap's fuzzy union of neighbour lists [N][k] (-1 / inf fill)."""
    idx, dist = np.asarray(idx), np.asarray(dist, np.float64)
    N, k = idx.shape
    ok = (idx >= 0) & np.isfinite(dist)
    target = math.log2(n_neighbors)
    mean_all = dist[ok].sum() / (ok.sum() + N)
    W = np.zeros((N, k))
    for i in range(N):
        d = dist[i][ok[i]]
        pos = d[d > 0]
        rho = pos.min() if pos.size else 0.0
        lo, hi, mid = 0.0, np.inf, 1.0
        for _ in range(64):
            x = d - rho
            ps = float(np.where(x > 0, np.exp(-(np.maximum(x, 0) / mid)), 1.0).sum())
            if abs(ps - target) < 1e-5:
                break
            if ps > target:
                hi = mid
                mid = (lo + hi) / 2
            else:
                lo = mid
                mid = mid * 2 if hi == np.inf else (lo + hi) / 2
        s = mid
        fl = 1e-3 * (d.sum() / (d.size + 1) if rho > 0 else mean_all)
        s = max(s, fl)
        for m in range(k):
            j = idx[i, m]
            if not ok[i, m] or j == i:
                continue
            t = dist[i, m] - rho
            W[i, m] = 1.0 if (t <= 0 or s == 0) else math.exp(-(t / s))
    rows = np.repeat(np.arange(N), k)
    Wm = sp.csr_matrix((W.ravel(), (rows, np.where(idx.ravel() >= 0, idx.ravel(), 0))), shape=(N, N))
    Wm.eliminate_zeros()
    P = Wm + Wm.T - Wm.multiply(Wm.T)
    P = sp.csr_matrix(P)
    P.setdiag(0)
    P.eliminate_zeros()
    P.sort_indices()
    return P


def _rows(ip):
    return np.repeat(np.arange(len(ip) - 1), np.diff(ip))


class _Ties:
    near = False

    def check(self, a, b):
        if np.any((np.abs(a - b) <= TIE * np.maximum(1.0, np.maximum(np.abs(a), np.abs(b)))) & (a != b)):
            self.near = True


def _move(n, row, col, w, k, inv2m, g, comm, ties, stats):
    quiet, moved_any, s = 0, False, 0
    off = row != col
    r, c0, ww = row[off], col[off], w[off]
    while s < 128:
        tot = np.bincount(comm, k, n)
        key = r * n + comm[c0]
        u, inv = np.unique(key, return_inverse=True)
        S = np.bincount(inv, ww)
        ur, uc = u // n, u % n
        own = comm[ur] == uc
        f = g * k * inv2m
        stay = -f * (tot[comm] - k)
        stay[ur[own]] += S[own]
        gain = S - f[ur] * tot[uc]
        o = ~own
        best_g = np.full(n, -np.inf)
        best_c = np.full(n, -1)
        if o.any():
            orr, ouc, og = ur[o], uc[o], gain[o]
            order = np.lexsort((ouc, -og, orr))
            first = np.ones(len(order), bool)
            first[1:] = orr[order][1:] != orr[order][:-1]
            sel = order[first]
            best_g[orr[sel]] = og[sel]
            best_c[orr[sel]] = ouc[sel]
            second = order[~first]
            # near ties among the top two and against staying
            if len(order) > 1:
                nxt = np.flatnonzero(first) + 1
                nxt = nxt[nxt < len(order)]
                nxt = nxt[~first[nxt]]
                ties.check(og[order][nxt - 1], og[order][nxt])
            del second
        has = best_c >= 0
        ties.check(best_g[has], stay[has])
        allowed = (best_c < comm) if s % 2 == 0 else (best_c > comm)
        go = has & (best_g > stay) & allowed
        nxt_comm = np.where(go, best_c, comm)
        m = int(go.sum())
        comm = nxt_comm
        stats["sweeps"] += 1
        s += 1
        if m:
            moved_any = True
        quiet = 0 if m else quiet + 1
        if quiet == 2:
            break
    return comm, moved_any


def _refine(n, row, col, w, k, inv2m, g, comm, ties, stats):
    off = row != col
    r, c0, ww = row[off], col[off], w[off]
    same = comm[r] == comm[c0]
    tot = np.bincount(comm, k, n)
    win = np.bincount(r[same], ww[same], n)
    sub = np.arange(n)
    moved_any = False
    for _ in range(1024):
        size = np.bincount(sub, minlength=n)
        stot = np.bincount(sub, k, n)
        ext_e = same & (sub[r] != sub[c0])
        sext = np.bincount(sub[r[ext_e]], ww[ext_e], n)
        T = tot[comm]
        single = (sub == np.arange(n)) & (size[np.arange(n)] == 1)
        wc_v = single & (win >= g * k * (T - k) * inv2m)
        ties.check(win[single], (g * k * (T - k) * inv2m)[single])
        e = same & wc_v[r]
        key = r[e] * n + sub[c0[e]]
        u, inv = np.unique(key, return_inverse=True)
        S = np.bincount(inv, ww[e]) if len(u) else np.zeros(0)
        ur, us = u // n, u % n
        Tc = tot[comm[ur]]
        wc_s = sext[us] >= g * stot[us] * (Tc - stot[us]) * inv2m
        ties.check(sext[us], g * stot[us] * (Tc - stot[us]) * inv2m)
        val = S - g * k[ur] * stot[us] * inv2m
        ok = wc_s & (val > 0)
        ties.check(val, np.zeros_like(val))
        target = np.full(n, -1)
        if ok.any():
            orr, os_, ov = ur[ok], us[ok], val[ok]
            order = np.lexsort((os_, -ov, orr))
            first = np.ones(len(order), bool)
            first[1:] = orr[order][1:] != orr[order][:-1]
            nxt = np.flatnonzero(first) + 1
            nxt = nxt[nxt < len(order)]
            nxt = nxt[~first[nxt]]
            ties.check(ov[order][nxt - 1], ov[order][nxt])
            sel = order[first]
            target[orr[sel]] = os_[sel]
        proposed = np.zeros(n, bool)
        proposed[target[target >= 0]] = True
        join = (target >= 0) & ~proposed
        stats["rounds"] += 1
        if not join.any():
            break
        sub = np.where(join, target, sub)
        moved_any = True
    return sub, moved_any


def _iteration(N, ip, col, w, inv2m, g, start, ties, stats):
    n, row, k = N, _rows(ip), np.bincount(_rows(ip), w, N)
    comm = start.copy()
    omap = np.arange(N)
    while True:
        comm, moved = _move(n, row, col, w, k, inv2m, g, comm, ties, stats)
        stats["levels"] += 1
        sub, refined = _refine(n, row, col, w, k, inv2m, g, comm, ties, stats)
        if not refined:
            break
        used = np.zeros(n, bool)
        used[sub] = True
        newid = np.cumsum(used) - 1
        vmap = newid[sub]
        n2 = int(used.sum())
        cmin = np.full(n, np.iinfo(np.int64).max)
        np.minimum.at(cmin, comm, vmap)
        nc = np.empty(n2, np.int64)
        nc[vmap] = cmin[comm]
        omap = vmap[omap]
        A = sp.csr_matrix((w, (vmap[row], vmap[col])), shape=(n2, n2))
        A.sum_duplicates()
        A.sort_indices()
        ip, col, w = A.indptr, A.indices.astype(np.int64), A.data
        row = _rows(ip)
        k = np.bincount(row, w, n2)
        n, comm = n2, nc
    return comm[omap]


def number(labels):
    """Labels numbered by decreasing size, ties by the smallest member."""
    labels = np.asarray(labels)
    u, first, inv, size = np.unique(labels, return_index=True, return_inverse=True, return_counts=True)
    order = np.lexsort((first, -size))
    rank = np.empty(len(u), np.int64)
    rank[order] = np.arange(len(u))
    return rank[inv.reshape(-1)].astype(np.int32)


def modularity(A, labels, gamma):
    A = sp.csr_matrix(A)
    k = np.asarray(A.sum(axis=1)).ravel()
    two_m = k.sum()
    if two_m == 0:
        return 0.0
    r = _rows(A.indptr)
    inside = A.data[labels[r] == labels[A.indices]].sum()
    tot = np.bincount(labels, k)
    inv2m = 1.0 / two_m  # the library's form: exact for integer weights, so Q replays bit for bit
    return float((inside - gamma * (tot ** 2).sum() * inv2m) * inv2m)


def leiden(A, gamma=1.0, n_iterations=-1):
    """-> (labels, n_communities, Q, iterations, near_tie, stats) of the §16 definition on the symmetric CSR A."""
    A = sp.csr_matrix(A, dtype=np.float64)
    A.sort_indices()
    N = A.shape[0]
    ip, col, w = A.indptr.astype(np.int64), A.indices.astype(np.int64), A.data.astype(np.float64)
    two_m = w.sum()
    ties = _Ties()
    stats = {"levels": 0, "sweeps": 0, "rounds": 0}
    labels = np.arange(N)
    iters = 0
    if two_m > 0:
        inv2m = 1.0 / two_m
        prev = None
        cap = 64 if n_iterations < 0 else n_iterations
        for it in range(cap):
            labels = number(_iteration(N, ip, col, w, inv2m, gamma, labels if it else np.arange(N), ties, stats))
            iters += 1
            if n_iterations >= 0:
                continue
            if prev is not None and np.array_equal(prev, labels):
                break
            prev = labels
    labels = number(labels)
    return labels, int(labels.max()) + 1, modularity(A, labels, gamma), iters, ties.near, stats


def connected_communities(A, labels):
    """Whether every community induces one connected piece: the graph without its edges between communities has as
    many components as there are communities."""
    from scipy.sparse.csgraph import connected_components
    A = sp.csr_matrix(A)
    r = _rows(A.indptr)
    keep = labels[r] == labels[A.indices]
    B = sp.csr_matrix((A.data[keep], (r[keep], A.indices[keep])), shape=A.shape)
    return connected_components(B, directed=False)[0] == len(np.unique(labels))


def improving_move(A, labels, gamma, tol=1e-12):
    """The largest gain in Q of moving one vertex to a neighbouring community (<= tol * |Q| when converged)."""
    A = sp.csr_matrix(A, dtype=np.float64)
    k = np.asarray(A.sum(axis=1)).ravel()
    two_m = k.sum()
    tot = np.bincount(labels, k, labels.max() + 1)
    r = _rows(A.indptr)
    key = r * (labels.max() + 1) + labels[A.indices]
    u, inv = np.unique(key, return_inverse=True)
    S = np.bincount(inv, A.data)
    ur, uc = u // (labels.max() + 1), u % (labels.max() + 1)
    own = labels[ur] == uc
    w_own = np.zeros(len(k))
    w_own[ur[own]] = S[own]
    stay = w_own - gamma * k * (tot[labels] - k) / two_m
    gain = S - gamma * k[ur] * tot[uc] / two_m
    d = (gain - stay[ur])[~own]
    return float(d.max() / two_m) if d.size else 0.0
