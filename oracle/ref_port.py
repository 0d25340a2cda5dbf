"""TEST INFRASTRUCTURE — loop-faithful CPU port of the reference's per-window numerics.

Same role and import rules as ``dense_oracle.py`` (checker / CPU baseline only; never on
the product path).  Where ``dense_oracle.py`` is vectorised so that tests finish in
seconds, THIS file keeps the reference's *cost structure* — the interpreter-level O(N²)
pair loops and per-site loops — because it is what ``bench.py`` times as the CPU
baseline (``cpu_baseline.kind = "port"``) and as the ``--impl reference`` arm on the GPU
box, where /root/reference does not exist.  It is validated against the reference itself
through tests/golden (tests/test_oracle_golden.py) and its throughput against the
survey's measurements of the unmodified scripts (BASELINE.md §2).

Citations are genomics_general/<file>:<line>.
"""
from __future__ import annotations

import itertools

import numpy as np

NAN = float("nan")


class PortAlignment:
    """numArray int64 [N haplotypes, L sites] + nanMask, as Alignment.__init__ builds them
    (genomics.py:813-869); rows are haplotypes here exactly like the reference."""

    def __init__(self, g_sites_by_haps, groups):
        # genoToAlignment/seqArrayToNumArray produce int64 rows per haplotype (74-77, 1101-1127)
        self.numArray = np.ascontiguousarray(np.asarray(g_sites_by_haps).T.astype(np.int64))
        self.numArray[self.numArray < 0] = -999
        self.nanMask = self.numArray >= 0                                      # 834
        self.N, self.l = self.numArray.shape
        self.groups = np.asarray(groups)
        self._distMat_ = None
        self._pairNonNan_ = None

    # genomics.py:903-905 + 1219-1221
    def pairDist(self, i, j):
        nanMask = self.nanMask[i, :] & self.nanMask[j, :]
        a = self.numArray[i, :][nanMask]
        b = self.numArray[j, :][nanMask]
        dif = a - b
        with np.errstate(invalid="ignore"):
            import warnings
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                return np.mean(dif != 0)

    # genomics.py:907-916
    def distMatrix(self):
        distMat = np.zeros((self.N, self.N))
        for i in range(self.N - 1):
            for j in range(i + 1, self.N):
                distMat[i, j] = distMat[j, i] = self.pairDist(i, j)
        self._distMat_ = distMat
        return distMat

    # genomics.py:1042-1047
    def pairNonNan(self):
        self._pairNonNan_ = np.zeros((self.N, self.N))
        for i in range(self.N - 1):
            for j in range(i + 1, self.N):
                self._pairNonNan_[i, j] = self._pairNonNan_[j, i] = np.sum(self.nanMask[i, :] & self.nanMask[j, :])
        return self._pairNonNan_

    # genomics.py:956-995
    def groupDistStats(self, pops, doPairs=True, minSites=None, minData=0.01):
        from .dense_oracle import nanmean_min
        distMat = self.distMatrix()
        if minSites:
            distMat[self.pairNonNan() < minSites] = np.nan
        np.fill_diagonal(distMat, np.nan)
        popIndices = [list(np.where(self.groups == p)[0]) for p in pops]
        out = {}
        for x, p in enumerate(pops):
            out["pi_%s" % p] = nanmean_min(distMat[np.ix_(popIndices[x], popIndices[x])], minData)
        if len(pops) == 1 or not doPairs:
            return out
        for x in range(len(pops) - 1):
            for y in range(x + 1, len(pops)):
                px, py = pops[x], pops[y]
                out["dxy_%s_%s" % (px, py)] = nanmean_min(distMat[np.ix_(popIndices[x], popIndices[y])], minData)
                n_x, n_y = len(popIndices[x]), len(popIndices[y])
                w = 1.0 * n_x / (n_x + n_y)
                pi_s = w * out["pi_%s" % px] + (1 - w) * out["pi_%s" % py]
                both = popIndices[x] + popIndices[y]
                pi_t = nanmean_min(distMat[np.ix_(both, both)], minData)
                with np.errstate(divide="ignore", invalid="ignore"):
                    out["Fst_%s_%s" % (px, py)] = 1 - np.float64(pi_s) / np.float64(pi_t)
        return out

    # genomics.py:1049-1052 (+592-599)
    def siteFreqs(self, rows, sites=None, asCounts=False):
        if sites is None:
            sites = range(self.l)
        out = []
        for x in sites:
            col = self.numArray[rows, x][self.nanMask[rows, x]]
            n = len(col)
            if n == 0:
                out.append(np.zeros(4, dtype=int) if asCounts else np.array([np.nan] * 4))
            else:
                c = np.bincount(col, minlength=4)
                out.append(c if asCounts else 1.0 * c / n)
        return np.array(out).reshape(-1, 4)


def abbababa_port(aln: PortAlignment, P1, P2, P3, P4, minData):
    """genomics.py:1647-1695 with its per-site np.unique / siteFreqs loops."""
    rows = {p: np.where(aln.groups == p)[0] for p in (P1, P2, P3, P4)}
    allrows = np.unique(np.concatenate([rows[p] for p in (P1, P2, P3, P4)]))
    biallelic = np.array([len(np.unique(aln.numArray[allrows, x][aln.nanMask[allrows, x]])) == 2
                          for x in range(aln.l)], dtype=bool)
    enough = np.ones(aln.l, dtype=bool)
    for p in (P1, P2, P3, P4):
        enough &= (np.sum(aln.nanMask[rows[p], :], axis=0) * 1.0 / len(rows[p]) >= minData)
    good = np.where(biallelic & enough)[0]
    if len(good) < 1:
        return dict(D=NAN, fd=NAN, fdM=NAN, ABBA=NAN, BABA=NAN, sitesUsed=NAN)
    allf = aln.siteFreqs(allrows, good)
    f = {p: aln.siteFreqs(rows[p], good) for p in (P1, P2, P3, P4)}
    with np.errstate(invalid="ignore", divide="ignore"):
        ai = np.where((allf > 0) & (f[P4] == 0))
        p1, p2, p3, p4 = (f[p][ai[0], ai[1]] for p in (P1, P2, P3, P4))
        f4 = lambda a, b, c, d: (1 - a) * b * c * (1 - d) - a * (1 - b) * c * (1 - d)
        abba = (1 - p1) * p2 * p3 * (1 - p4)
        baba = p1 * (1 - p2) * p3 * (1 - p4)
        D = f4(p1, p2, p3, p4).sum() * 1.0 / (abba + baba).sum()
        pd = p2 * (p2 > p3) + p3 * (p3 >= p2)
        fd = f4(p1, p2, p3, p4).sum() * 1.0 / f4(p1, pd, pd, p4).sum()
        a = p3 > p1
        b = p3 > p2
        x = p1 > p2
        y = ~x
        pdm1 = p3 * (x & a) + p1 * (~(x & a))
        pdm2 = p3 * (y & b) + p2 * (~(y & b))
        pdm3 = -p3 * (x & a) + p3 * (y & b) - p1 * (x & ~a) + p2 * (y & ~b)
        fdm = f4(p1, p2, p3, p4).sum() * 1.0 / f4(pdm1, pdm2, pdm3, p4).sum()
    return dict(D=float(D), fd=float(fd), fdM=float(fdm), ABBA=float(abba.sum()), BABA=float(baba.sum()),
                sitesUsed=len(ai[0]))


def ind_pair_dists_port(aln: PortAlignment, hap_ind, n_ind, includeSameWithSame=False):
    """genomics.py:934-954: O(N²) distMatrix + n² np.nanmean calls."""
    import warnings
    distMat = aln.distMatrix()
    if not includeSameWithSame:
        np.fill_diagonal(distMat, np.nan)
    idx = [np.where(np.asarray(hap_ind) == a)[0] for a in range(n_ind)]
    out = np.zeros((n_ind, n_ind))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for i, j in itertools.product(range(n_ind), repeat=2):
            out[i, j] = np.nanmean(distMat[np.ix_(idx[i], idx[j])])
    return out


def popgen_window_port(g, hap_pop, n_pops, min_sites, min_data):
    """One popgenWindows worker iteration on an already-parsed window
    (popgenWindows.py:41-66 minus text handling): returns pi, dxy, fst arrays."""
    L = np.asarray(g).shape[0]
    pairs = list(itertools.combinations(range(n_pops), 2))
    if L < min_sites:
        return np.full(n_pops, np.nan), np.full(len(pairs), np.nan), np.full(len(pairs), np.nan)
    aln = PortAlignment(g, hap_pop)
    d = aln.groupDistStats(list(range(n_pops)), True, min_sites, min_data)
    pi = np.array([d["pi_%d" % x] for x in range(n_pops)])
    dxy = np.array([d["dxy_%d_%d" % p] for p in pairs])
    fst = np.array([d["Fst_%d_%d" % p] for p in pairs])
    return pi, dxy, fst
