"""fp64 restatement of hb_kbet (DESIGN.md §13): per label a k-d tree on the label's finite rows, the neighbourhood of
the cell and its k0 - 1 nearest others, the chi-square statistic of its batch counts as the kBET package's
chi_batch_test forms it (the full table of the label's batches, zeros included) and scipy's upper tail."""
from types import SimpleNamespace

import numpy as np
from scipy.spatial import cKDTree
from scipy.stats import chi2

from silhouette_restatement import finite_rows

TOP = 2 ** 31 - 1


def k0_rule(n, present, fixed=0):
    """A label's k0 from its n finite rows in `present` batches: 0 (not tested) for n < 10 or one batch; a fixed k0,
    0 when n < k0; else scib's min(70, max(10, floor(mean / 4))) with its 2^31 guard."""
    if n < 10 or present < 2:
        return 0
    if fixed:
        return fixed if fixed <= n else 0
    k0 = int(min(70, max(10, np.floor(n / present / 4))))
    if k0 * n >= TOP:
        k0 = TOP // n
    return k0


def chi_batch_test(env_batches, levels, counts, k0):
    """The package's statistic for neighbourhoods env_batches [rows, k0] of batch values: observed counts over the
    label's batch levels (zeros included) against k0 times their frequencies, sum of (o - e)^2 / e."""
    code = np.searchsorted(levels, env_batches)
    obs = np.stack([np.bincount(c, minlength=len(levels)) for c in code]).astype(np.float64)
    exp = counts / counts.sum() * k0
    return ((obs - exp) ** 2 / exp).sum(axis=1)


def kbet(X, batches, labels=None, k0=0, n_labels=None, idx=None):
    """hb_kbet's outputs by definition -> namespace of stat, pval [N] (NaN for rows not tested), k0 [n_labels], dof [N]
    (-1 for rows not tested) and nn [N][max k0 - 1] (each tested row's other rows by ascending fp64 distance, -1 after).
    With idx (hb_kbet's own lists) the neighbourhoods are taken from it instead of the tree."""
    X = np.asarray(X, dtype=np.float64)
    N = len(X)
    batches = np.asarray(batches)
    labels = np.zeros(N, np.int64) if labels is None else np.asarray(labels)
    n_labels = int(labels.max()) + 1 if n_labels is None else n_labels
    fin = finite_rows(X)[0]
    stat, pval, dof = np.full(N, np.nan), np.full(N, np.nan), np.full(N, -1)
    k0_out = np.zeros(n_labels, np.int64)
    lists = {}
    for l in range(n_labels):
        rows = np.flatnonzero((labels == l) & fin)
        levels, counts = np.unique(batches[rows], return_counts=True)
        k = k0_rule(len(rows), len(levels), k0)
        k0_out[l] = k
        if k == 0:
            continue
        if idx is None:
            _, nn = cKDTree(X[rows]).query(X[rows], k)
            nn = np.asarray(nn).reshape(len(rows), k)
            others = np.empty((len(rows), k - 1), np.int64)
            for r in range(len(rows)):   # the row itself, wherever exact duplicates put it, or the farthest
                keep = nn[r][nn[r] != r]
                others[r] = keep[:k - 1]
            others = rows[others]
        else:
            others = np.asarray(idx)[rows, :k - 1].astype(np.int64)
        env = np.concatenate([others, rows[:, None]], axis=1)
        s = chi_batch_test(batches[env], levels, counts, k)
        stat[rows], pval[rows], dof[rows] = s, chi2.sf(s, len(levels) - 1), len(levels) - 1
        for r, o in zip(rows, others):
            lists[r] = o
    width = max(int(k0_out.max()) - 1, 0)
    nn = np.full((N, width), -1, np.int64)
    for r, o in lists.items():
        nn[r, :len(o)] = o
    return SimpleNamespace(stat=stat, pval=pval, k0=k0_out, dof=dof, nn=nn)


def rates(pval, labels, k0, alpha=0.05):
    """Each label's rejection rate, NaN where k0 = 0."""
    return np.array([np.nan if k0[l] == 0 else float((pval[(labels == l) & ~np.isnan(pval)] < alpha).mean())
                     for l in range(len(k0))])
