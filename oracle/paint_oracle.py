"""TEST INFRASTRUCTURE — distPaint.py's per-window assignment in numpy / scipy, and two pure-Python restatements of the
orders the result depends on bit for bit.

    paint_window   : the worker loop of distPaint.py:67-83 on a dense window, with which_lowest_test /
                     which_lowest_delta (26-44) calling scipy.stats.ranksums and np.nanmean themselves
    pairwise_sum   : numpy's summation order for np.sum / np.nansum of a 1-d float64 array
    cpython_sort   : CPython's list.sort of fewer than 64 floats (nan included), as sorted() gives it

The engine's kernel (k2_paint_epi) follows the two orders; the CPU tests check them against np.nansum and sorted()."""
import warnings

import numpy as np
from scipy.stats import ranksums


def pairwise_sum(a):
    """np.add.reduce order of numpy's pairwise_sum (numpy/_core/src/umath/loops_utils.h.src): fewer than 8 values are
    added one by one from 0.0; up to 128 go to eight strided accumulators combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)),
    then the tail one by one; above 128 the list is split at n/2 rounded down to a multiple of 8."""
    n = len(a)
    if n < 8:
        res = 0.0
        for v in a:
            res += float(v)
        return res
    if n <= 128:
        r = [float(v) for v in a[:8]]
        i = 8
        while i < n - n % 8:
            for k in range(8):
                r[k] += float(a[i + k])
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for v in a[i:]:
            res += float(v)
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return pairwise_sum(a[:n2]) + pairwise_sum(a[n2:])


def nanmean(a):
    """np.nanmean through pairwise_sum: nans count as 0 in the sum, which is divided by the non-nan count"""
    vals = [0.0 if v != v else float(v) for v in a]
    cnt = sum(1 for v in a if v == v)
    return pairwise_sum(vals) / cnt if cnt else float("nan")


def cpython_sort(vals):
    """list.sort of fewer than 64 items (Objects/listobject.c, CPython 3.12): one count_run over the whole list (a strictly
    descending run is reversed), then binarysort of the rest into it; every comparison is <."""
    s = list(vals)
    n = len(s)
    assert n < 64
    run = 1
    if n > 1:
        run = 2
        if s[1] < s[0]:
            while run < n and s[run] < s[run - 1]:
                run += 1
            s[:run] = s[:run][::-1]
        else:
            while run < n and not (s[run] < s[run - 1]):
                run += 1
    for st in range(run, n):
        pivot = s[st]
        lo, hi = 0, st
        while lo < hi:
            m = lo + ((hi - lo) >> 1)
            if pivot < s[m]:
                hi = m
            else:
                lo = m + 1
        s[lo + 1:st + 1] = s[lo:st]
        s[lo] = pivot
    return s


def pair_counts(win):
    """diff_ij, n_ij of every haplotype-column pair of a window (Alignment.pairDist's numerator and nanMask count); win int8
    [S, H], negative = missing"""
    valid = (win >= 0).astype(np.int64)
    n = valid.T @ valid
    same = sum(((win == b).astype(np.int64).T @ (win == b).astype(np.int64)) for b in range(4))
    return n - same, n


def member_distances(diff, n, i, members, min_sites):
    """Alignment.pairDist(i, j) = np.mean of the mismatches at the jointly called sites (diff / n, one division), nan when
    fewer than minSites (distPaint.py:73-76); one float64 array in member order, which np.nanmean and ranksums read as
    they read the reference's list of np.float64"""
    m = np.asarray(members, dtype=np.int64)
    nij = n[i, m]
    with np.errstate(all="ignore"):
        d = diff[i, m].astype(np.float64) / nij.astype(np.float64)
    d[nij < min_sites] = np.nan
    return d


def paint_window(win, query_hap, pops, min_sites, delta=None, p_threshold=0.05, noresult=-1):
    """-> assign [n_query], means [n_query, P], pvals [n_query, P] (ranksums' p-value of the chosen population against
    each other one: nan for the chosen one itself and under the delta rule).  pops: member column lists."""
    nq, P = len(query_hap), len(pops)
    assign = np.empty(nq, dtype=np.int64)
    means = np.full((nq, P), np.nan)
    pvals = np.full((nq, P), np.nan)
    diff, n = pair_counts(win)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for k, i in enumerate(query_hap):
            lists = [member_distances(diff, n, i, m, min_sites) for m in pops]
            means[k] = [np.nanmean(a) for a in lists]
            best = int(np.argmin(means[k]))
            if delta is not None:
                s = sorted(list(means[k]))
                assign[k] = noresult if s[1] - s[0] < delta else best
                continue
            assign[k] = best
            for j in range(P):
                if j != best:
                    pvals[k, j] = ranksums(lists[best], lists[j], alternative="less").pvalue
                    if pvals[k, j] > p_threshold:
                        assign[k] = noresult
    return assign, means, pvals
