"""``genomics``-compatible host API backed by libpgwin.so (the H100 engine).

This mirrors the slice of genomics_general/genomics.py that the four hot scripts use (SURVEY.md §8b):
``SampleData`` (1264-1290), ``GenoWindow`` (1721-1797), the window generators (1971-2171),
``parseGenoFile`` (1949-1967), ``genoToAlignment`` (1101-1127), ``Alignment`` with
``distMatrix / pairNonNan / groupDistStats / indPairDists / siteFreqs / siteNonNan / seqNonNan / subset``
(808-1098) and ``ABBABABA`` (1647-1695) — same names, argument meaning and return shapes, so code written
against the reference module runs unchanged.  Every number is computed on the GPU through the C-ABI;
there is no CPU fallback (creating the engine without a CUDA device raises).

Differences, on purpose: windows are views into one dense int8 matrix instead of lists of strings; the
haplotype order of an ``Alignment`` is file order (``ind_A, ind_B`` adjacent) instead of sorted by name —
no statistic depends on it; letters other than ACGTN are missing (the reference reads uninitialised
memory for them, genomics.py:75).
"""
from __future__ import annotations

import itertools
import string

import numpy as np

from . import geno_io, windows as _win
from .engine import Engine

_BASES = np.array(list("ACGTN"))
_DIPLO_OF = {"AA": "A", "CC": "C", "GG": "G", "TT": "T", "GT": "K", "TG": "K", "AC": "M", "CA": "M", "CG": "S",
             "GC": "S", "AG": "R", "GA": "R", "AT": "W", "TA": "W", "CT": "Y", "TC": "Y"}

_engine = None


def default_engine(device: int = 0) -> Engine:
    """Process-wide engine used by the Alignment methods (one pg_ctx on `device`)."""
    global _engine
    if _engine is None:
        _engine = Engine(device)
    return _engine


# ------------------------------------------------------------------------------------------------
class SampleData:
    """Populations -> samples, sample -> ploidy (behaviour of genomics.py:1264-1290).

    popInds[k] lists the individuals of population popNames[k]; an individual missing from indNames is
    appended to it; populations are addressable by name and by number; ploidy defaults to 2."""

    def __init__(self, indNames=None, popNames=None, popInds=None, popNumbers=None, ploidyDict=None):
        members = [list(m) for m in (popInds or [])]
        numbers = list(popNumbers) if popNumbers is not None else list(range(len(members)))
        labels = list(popNames) if popNames is not None else [str(k) for k in numbers]
        if not (len(labels) == len(members) == len(numbers)):
            raise AssertionError("Names, inds and numbers should be same length.")
        roster = indNames if indNames is not None else []
        known = set(roster)
        self.popInds = {}
        for label, number, inds in zip(labels, numbers, members):
            for ind in inds:
                if ind not in known:
                    roster.append(ind)
                    known.add(ind)
            self.popInds[label] = inds
            self.popInds[number] = inds
        self.popNames, self.popNumbers, self.indNames = labels, numbers, roster
        self.ploidy = {ind: (ploidyDict[ind] if ploidyDict else 2) for ind in roster}

    def getPop(self, indName):
        """population of an individual: None, a name, or a tuple of names when it sits in several"""
        hits = tuple(p for p in self.popNames if indName in self.popInds[p])
        return None if not hits else (hits[0] if len(hits) == 1 else hits)

    def getPopNumber(self, popName):
        return self.popNumbers[self.popNames.index(popName)] if popName in self.popNames else None


# ------------------------------------------------------------------------------------------------
class GenoWindow:
    """genomics.py:1721-1797.  Dense-backed: ``geno`` is an int8 [sites, haplotypes] view of the file matrix
    (``sites`` — the reference's list of per-sample genotype strings — is produced on demand)."""

    def __init__(self, scaffold=None, limits=None, sites=None, names=None, positions=None, ID=None, geno=None,
                 ploidy=None, genoFormat="phased"):
        self.scaffold = scaffold
        self.limits = [-np.inf, np.inf] if limits is None else limits
        self.names = list(names) if names is not None else []
        self.n = len(self.names)
        self.positions = list(positions) if positions is not None else []
        self.ID = ID
        self.genoFormat = genoFormat
        self.ploidy = np.asarray(ploidy if ploidy is not None else [2] * self.n, dtype=np.int64)
        self._sites = sites
        self.geno = geno
        if geno is None and sites is not None:
            self.geno = _encode_sites(sites, self.ploidy, genoFormat)

    @property
    def sites(self):
        if self._sites is None:
            self._sites = _decode_sites(self.geno, self.ploidy, self.genoFormat) if self.geno is not None else []
        return self._sites

    def _cut(self, sl):
        """keep the sites of a Python slice (positions, dense rows and the token cache stay aligned)"""
        self.positions = self.positions[sl]
        if self.geno is not None:
            self.geno = self.geno[sl]
        if self._sites is not None:
            self._sites = self._sites[sl]

    def addBlock(self, sites, positions):
        """genomics.py:1745-1751"""
        assert len(set([len(site) for site in sites])) == 1, "Number of genotypes per site must be equal."
        assert len(sites[0]) == self.n, "Number of genotypes per site must match number of names."
        assert len(positions) == len(sites), "Positions must match number of sites"
        assert all(self.limits[0] <= p <= self.limits[1] for p in positions), "Position outside of window limit"
        rows = _encode_sites(sites, self.ploidy, self.genoFormat)
        self.geno = rows if self.geno is None or len(self.positions) == 0 else np.concatenate([self.geno, rows], axis=0)
        if self._sites is not None:
            self._sites = list(self._sites) + list(sites)
        self.positions = list(self.positions) + list(positions)

    def addSite(self, GTs, position=np.nan, ignorePosition=False):
        """genomics.py:1753-1759"""
        assert len(GTs) == self.n, "Number of genotypes per site must match number of names."
        if not ignorePosition:
            assert self.limits[0] <= position <= self.limits[1], "Position: " + str(position) + " outside of window limits: " + \
                "-".join([str(l) for l in self.limits])
        else:
            position = np.nan
        row = _encode_sites([GTs], self.ploidy, self.genoFormat)
        self.geno = row if self.geno is None or len(self.positions) == 0 else np.concatenate([self.geno, row], axis=0)
        if self._sites is not None:
            self._sites = list(self._sites) + [GTs]
        self.positions = list(self.positions) + [position]

    def slide(self, step=None, newLimits=None):
        """genomics.py:1767-1777: move the limits, drop the sites that now lie before the window"""
        assert step is not None or newLimits is not None
        if step:
            self.limits = [l + step for l in self.limits]
        else:
            self.limits = newLimits
        i, end = 0, len(self.positions)
        while i < end and self.positions[i] < self.limits[0]:
            i += 1
        self._cut(slice(i, None))

    def trim(self, right=False, remove=None, leave=None):
        """genomics.py:1779-1788 (with its slices: `right=True, remove=0` empties the window, [:-0])"""
        assert remove is not None or leave is not None
        if not remove:
            remove = self.seqLen() - leave
        self._cut(slice(remove, None) if not right else slice(None, -remove))

    def seqLen(self):
        return len(self.positions)

    def firstPos(self):
        return min(self.positions)

    def lastPos(self):
        return max(self.positions)

    def midPos(self):
        try:
            return int(round(sum(self.positions) / len(self.positions)))
        except Exception:
            return np.nan

    def seqDict(self, names=None):
        if names is None:
            names = self.names
        idx = [self.names.index(n) for n in names]
        s = self.sites
        return dict(zip(names, [[site[i] for site in s] for i in idx]))

    def copy(self):
        return GenoWindow(scaffold=self.scaffold, limits=self.limits[:], names=self.names[:],
                          positions=self.positions[:], ID=self.ID, geno=self.geno, ploidy=self.ploidy,
                          genoFormat=self.genoFormat)


def _decode_sites(geno, ploidy, fmt):
    ch = _BASES[np.where(geno < 0, 4, geno)]
    out = []
    offs = np.concatenate([[0], np.cumsum(ploidy)])
    for s in range(geno.shape[0]):
        row = []
        for k in range(len(ploidy)):
            al = ch[s, offs[k]:offs[k + 1]]
            if fmt == "phased":
                row.append("/".join(al))
            elif fmt == "diplo":
                row.append(_DIPLO_OF.get("".join(al), "N"))
            else:
                row.append("".join(al))
        out.append(row)
    return out


def _encode_tokens(tokens, ploidy, fmt):
    """list of genotype strings of ONE individual -> int8 [L, ploidy]"""
    lut = {"A": 0, "C": 1, "G": 2, "T": 3}
    dip = {"A": "AA", "C": "CC", "G": "GG", "K": "GT", "M": "AC", "N": "NN", "S": "CG", "R": "AG", "T": "TT", "W": "AT",
           "Y": "CT"}
    out = np.full((len(tokens), ploidy), -1, dtype=np.int8)
    for s, t in enumerate(tokens):
        if fmt == "phased":
            al = t[::2]
        elif fmt == "diplo":
            al = dip[t]
            if ploidy == 1:
                al = al[0] if al[0] == al[1] else "N"           # forceHomo (genomics.py:407)
        else:
            al = t
        assert len(al) == ploidy, "Sample ploidy (%d) doesn't match number of sequences (%d)" % (ploidy, len(al))
        for a in range(ploidy):
            out[s, a] = lut.get(al[a], -1)
    return out


def _encode_sites(sites, ploidy, fmt):
    L = len(sites)
    n = len(ploidy)
    cols = [_encode_tokens([sites[s][k] for s in range(L)], int(ploidy[k]), fmt) for k in range(n)]
    return np.concatenate(cols, axis=1) if cols else np.zeros((L, 0), dtype=np.int8)


# ------------------------------------------------------------------------------------------------
class Alignment:
    """genomics.py:808-1098, GPU-backed.  ``numArray`` is int64 [N, l] with -999 for missing, like the
    reference; the device copy is the int8 site-major matrix."""

    def __init__(self, geno, names=None, groups=None, sampleNames=None, positions=None, engine=None):
        self._geno = np.ascontiguousarray(geno, dtype=np.int8)            # [l, N]
        self.l, self.N = self._geno.shape
        self.names = np.array(names if names is not None else np.arange(self.N))
        self.sampleNames = np.array(sampleNames if sampleNames is not None else self.names)
        self.groups = np.array(groups if groups is not None else [None] * self.N, dtype=object)
        self.positions = positions if positions is not None else range(1, self.l + 1)
        self._eng = engine
        self._uploaded = False
        self._distMat_ = None
        self._pairNonNan_ = None
        # what the reference's analyses did IN PLACE to its cached distance matrix (genomics.py:959-963, 940)
        self._masked_min_sites = 0
        self._diag_nan = False
        self.groupIndDict = {}
        for n, g in zip(self.names, self.groups):
            for gg in (g if isinstance(g, (tuple, list)) else [g]):
                if gg is not None:
                    self.groupIndDict.setdefault(gg, []).append(n)

    # -- reference attributes
    @property
    def numArray(self):
        a = self._geno.T.astype(np.int64)
        a[a < 0] = -999
        return a

    @property
    def nanMask(self):
        return self._geno.T >= 0

    @property
    def array(self):
        return _BASES[np.where(self._geno < 0, 4, self._geno)].T

    def _engine(self):
        eng = self._eng or default_engine()
        if not self._uploaded or getattr(eng, "_owner", None) is not self:
            pos = np.asarray(list(self.positions), dtype=np.int64)
            pos = np.where(np.isfinite(pos.astype(np.float64)), pos, 0).astype(np.int32) if len(pos) else None
            eng.upload(self._geno, pos)
            eng.set_windows([0], [self.l])
            eng._owner = self
            self._uploaded = True
        return eng

    def subset(self, indices=None, names=None, groups=None):
        idx = list(indices) if indices is not None else []
        names = list(names) if names is not None else []
        for g in (groups or []):
            names += self.groupIndDict.get(g, [])
        idx += [int(np.where(self.names == n)[0][0]) for n in names]
        idx = np.unique(idx).astype(np.int64)
        return Alignment(self._geno[:, idx], names=self.names[idx], groups=self.groups[idx],
                         sampleNames=self.sampleNames[idx], positions=self.positions, engine=self._eng)

    def _pair_counts(self):
        diff, n = self._engine().pair_counts(0)
        return diff.astype(np.int64), n.astype(np.int64)

    def distMatrix(self, minSites=None):
        """genomics.py:907-916."""
        diff, n = self._pair_counts()
        with np.errstate(divide="ignore", invalid="ignore"):
            d = diff / n.astype(np.float64)
        d[n == 0] = np.nan
        np.fill_diagonal(d, 0.0)
        self._distMat_ = d
        # a fresh matrix replaces the cached one: earlier in-place masks are gone (genomics.py:908-912)
        self._masked_min_sites, self._diag_nan = 0, False
        if minSites:
            d[self.pairNonNan() < minSites] = np.nan
            self._masked_min_sites = int(minSites)
        return d

    def pairNonNan(self):
        """genomics.py:1042-1047 (diagonal left at 0)."""
        _, n = self._pair_counts()
        n = n.astype(np.float64)
        np.fill_diagonal(n, 0.0)
        self._pairNonNan_ = n
        return n

    def pairDist(self, i, j):
        return self.distMatrix()[i, j]

    def siteNonNan(self, sites=None, prop=False):
        m = self._geno >= 0
        if sites is not None:
            m = m[np.atleast_1d(sites)]
        return m.mean(axis=1) if prop else m.sum(axis=1)

    def seqNonNan(self, prop=False):
        m = self._geno >= 0
        return m.mean(axis=0) if prop else m.sum(axis=0)

    def siteFreqs(self, sites=None, asCounts=False):
        """genomics.py:1049-1052: [n_sites, 4] counts (int) or frequencies (nan x4 where no data)."""
        eng = self._engine()
        eng.set_pops(np.zeros(self.N, dtype=np.int32), 1)
        c = eng.site_counts()[:, 0, :].astype(np.int64)
        if sites is not None:
            c = c[np.atleast_1d(sites)]
        if asCounts:
            return c
        with np.errstate(divide="ignore", invalid="ignore"):
            return c / c.sum(axis=1, keepdims=True).astype(np.float64)

    def _pop_index(self):
        pops = sorted({g for g in self.groups if g is not None and not isinstance(g, tuple)})
        hp = np.array([pops.index(g) if (g is not None and not isinstance(g, tuple)) else -1 for g in self.groups],
                      dtype=np.int32)
        return pops, hp

    def groupDistStats(self, doPairs=True, minSites=None, minData=0.01):
        """genomics.py:956-995 -> dict pi_X, dxy_X_Y (both orders), Fst_X_Y (both orders)."""
        pops, hp = self._pop_index()
        eng = self._engine()
        eng.set_pops(hp, len(pops))
        r = eng.popgen(minSites if minSites else 0, minData)
        self._masked_min_sites = max(self._masked_min_sites, int(minSites or 0))
        self._diag_nan = True
        out = {}
        for x, p in enumerate(pops):
            out["pi_" + str(p)] = float(r["pi"][0, x])
        if len(pops) == 1 or not doPairs:
            return out
        for k, (x, y) in enumerate(itertools.combinations(range(len(pops)), 2)):
            a, b = str(pops[x]), str(pops[y])
            out["dxy_%s_%s" % (a, b)] = out["dxy_%s_%s" % (b, a)] = float(r["dxy"][0, k])
            out["Fst_%s_%s" % (a, b)] = out["Fst_%s_%s" % (b, a)] = float(r["fst"][0, k])
        return out

    def groupFreqStats(self):
        """genomics.py:1002-1028 -> dict l_X, S_X, thetaPi_X, thetaW_X, TajD_X per group (the popFreq columns): only sites
        without missing data in ANY sequence count (1010); l is an int, S an int or nan (no such site), like the
        reference's Python values."""
        pops, hp = self._pop_index()
        if np.any(hp < 0):
            raise NotImplementedError("groupFreqStats with sequences outside every group is not supported (the reference "
                                      "itself fails on mixed None / str groups, genomics.py:1007)")
        eng = self._engine()
        eng.set_pops(hp, len(pops))
        eng.set_freqstats(True)
        try:
            eng.popgen(0, 0.01)
            f = eng.popgen_freqstats()
        finally:
            eng.set_freqstats(False)
        out = {}
        for x, p in enumerate(pops):
            S = f["S"][0, x]
            out["l_" + str(p)] = int(f["l"][0])
            out["S_" + str(p)] = np.nan if np.isnan(S) else int(S)
            for k in ("thetaPi", "thetaW", "TajD"):
                out["%s_%s" % (k, p)] = float(f[k][0, x])
        return out

    def indPairDists(self, asDict=True, includeSameWithSame=False, minSites=None):
        """genomics.py:934-954 (order of first appearance of sample names)."""
        samples = list(dict.fromkeys(self.sampleNames.tolist()))
        hap_ind = np.array([samples.index(s) for s in self.sampleNames], dtype=np.int32)
        eng = self._engine()
        self._masked_min_sites = max(self._masked_min_sites, int(minSites or 0))
        m = eng.pairdist(hap_ind, len(samples), includeSameWithSame or False, min_sites=self._masked_min_sites)["dist"][0]
        if not includeSameWithSame:
            self._diag_nan = True
        if not asDict:
            return m
        return {a: {b: m[i, j] for j, b in enumerate(samples)} for i, a in enumerate(samples)}

    def sampleHet(self, sampleNames=None, asList=False, minSites=None):
        """genomics.py:918-929, operator-precedence quirk included: `len(x)==2 & n >= minSites` is the chained comparison
        len(x) == (2 & n) >= minSites, so a two-haplotype sample has a value iff bit 1 of n_ij is set AND minSites <= 2."""
        samples = list(dict.fromkeys(self.sampleNames.tolist()))
        hap_ind = np.array([samples.index(s) for s in self.sampleNames], dtype=np.int32)
        het = self._engine().ind_het(hap_ind, len(samples), min_sites=self._masked_min_sites)[0]
        if minSites is not None and minSites > 2:
            het = np.full(len(samples), np.nan)
        if sampleNames is not None:
            het = np.array([het[samples.index(s)] for s in sampleNames])
            samples = list(sampleNames)
        return dict(zip(samples, het.tolist())) if not asList else het.tolist()

    def H12stats(self, maxDist=0):
        """genomics.py:1079-1098 -> dict H1_X, H12_X, H2_X."""
        pops, hp = self._pop_index()
        eng = self._engine()
        eng.set_pops(hp, len(pops))
        r = eng.hapstats(maxDist, min_sites=self._masked_min_sites, diag_nan=self._diag_nan)[0]
        out = {}
        for x, p in enumerate(pops):
            out["H1_" + str(p)], out["H12_" + str(p)], out["H2_" + str(p)] = (float(v) for v in r[x])
        return out


def genoToAlignment(seqDict, sampleData=None, genoFormat="diplo", positions=None):
    """genomics.py:1101-1127: dict individual -> list of genotype strings  ->  Alignment."""
    if sampleData is None:
        sampleData = SampleData()
    cols, names, sampleNames, groups = [], [], [], []
    for ind, toks in seqDict.items():
        pl = sampleData.ploidy.get(ind)
        if pl is None:
            pl = 1 if genoFormat == "haplo" else (len(toks[0][::2]) if genoFormat == "phased" and toks else 2)
        cols.append(_encode_tokens(toks, int(pl), genoFormat))
        if pl != 1:
            names += [ind + "_" + string.ascii_uppercase[a] for a in range(pl)]
        else:
            names.append(ind)
        sampleNames += [ind] * pl
        groups += [sampleData.getPop(ind)] * pl
    geno = np.concatenate(cols, axis=1) if cols else np.zeros((0, 0), dtype=np.int8)
    order = np.argsort(names)                       # genomics.py:1121: haplotypes sorted by sequence name
    return Alignment(geno[:, order], names=[names[i] for i in order], groups=[groups[i] for i in order],
                     sampleNames=[sampleNames[i] for i in order], positions=positions)


def ABBABABA(aln, P1, P2, P3, P4, minData, polarize=True, fixed=False):
    """genomics.py:1647-1695.  polarize=True (default): the derived allele is the one absent from P4 (1672);
    polarize=False, fixed=True: additionally fixed in P1..P3 (1673-1676); both False: the less common of the two
    alleles (1677) — the latter two share fourPop's allele selection (the K1 FOURPOP site pass)."""
    pops = [P1, P2, P3, P4]
    hp = np.full(aln.N, -1, dtype=np.int32)
    for k, p in enumerate(pops):
        for i, g in enumerate(aln.groups):
            if g == p or (isinstance(g, tuple) and p in g):
                hp[i] = k
    eng = aln._engine()
    eng.set_pops(hp, 4)
    if polarize:
        r = eng.abbababa(0, 1, 2, 3, minData)
        used = r["sitesUsed"][0]
        return {"D": float(r["D"][0]), "fd": float(r["fd"][0]), "fdM": float(r["fdM"][0]), "ABBA": float(r["ABBA"][0]),
                "BABA": float(r["BABA"][0]), "sitesUsed": (np.nan if np.isnan(used) else int(used))}
    r = eng.fourpop(0, 1, 2, 3, minData, polarize=False, fixed=fixed)
    # no site passed the filters: every value nan, sitesUsed included (1694-1695).  With sites but no selected allele the
    # sums run over empty arrays: ABBA = 0.0, sitesUsed = 0.
    no_good = int(r["sitesUsed"][0]) == 0 and bool(np.isnan(r["ABBA"][0]))
    return {"D": float(r["D"][0]), "fd": float(r["fd"][0]), "fdM": float(r["fdm"][0]), "ABBA": float(r["ABBA"][0]),
            "BABA": float(r["BABA"][0]), "sitesUsed": (np.nan if no_good else int(r["sitesUsed"][0]))}


def fourPop(aln, P1, P2, P3, P4, minData, polarize=False, fixed=False):
    """genomics.py:1585-1643 -> dict of the 14 statistics + sitesUsed."""
    pops = [P1, P2, P3, P4]
    hp = np.full(aln.N, -1, dtype=np.int32)
    for k, p in enumerate(pops):
        for i, g in enumerate(aln.groups):
            if g == p or (isinstance(g, tuple) and p in g):
                hp[i] = k
    eng = aln._engine()
    eng.set_pops(hp, 4)
    r = eng.fourpop(0, 1, 2, 3, minData, polarize=polarize, fixed=fixed)
    out = {k: float(r[k][0]) for k in eng.FOURPOP_KEYS}
    out["sitesUsed"] = int(r["sitesUsed"][0])
    return out


# ------------------------------------------------------------------------------------------------
# window generators over a parsed file
# ------------------------------------------------------------------------------------------------
# ------------------------------------------------------------------------------------------------
# line-by-line readers (genomics.py:1884-1945): host Python, kept for scripts that walk a genotype file site by site —
# the command lines of this package tokenise whole files on the device instead (geno_io.ingest_geno)
# ------------------------------------------------------------------------------------------------
def makeHaploidNames(names, ploidy=2):
    """genomics.py:448-453: `ind_A`, `ind_B`, ... per individual (the plain names when every ploidy is 1)"""
    pl = list(ploidy) if isinstance(ploidy, (list, tuple, np.ndarray)) else [ploidy]
    if len(pl) == 1:
        pl = pl * len(names)
    if all(int(x) == 1 for x in pl):
        return names
    per = dict(zip(names, pl))              # (a repeated name keeps its LAST ploidy, as the reference's dict does)
    return [n + "_" + string.ascii_uppercase[k] for n in names for k in range(int(per[n]))]


def parseGenoLine(line, names, scafCol=0, posCol=1, firstSampleCol=2, type=str, splitPhased=False, asDict=True,
                  precompDict=None, addToPrecomp=True):
    """One line of a .geno / counts table -> {"scaffold", "position", "GTs"} (genomics.py:1884-1904).  GTs: the genotype
    fields as `type`, as a name -> value dict (asDict) or a list; splitPhased turns "A|T" into its alleles.  precompDict
    caches the parsed fields by their text (identical lines are common), counting insertions in "__counter__"."""
    if not line:
        return {"scaffold": None, "position": None, "GTs": None}
    fields = line.split(None, firstSampleCol)
    text = fields[-1]
    if precompDict and text in precompDict:
        gts = precompDict[text]
    else:
        gts = text.split()
        if splitPhased:
            gts = [a for tok in gts for a in tok[::2]]
        if type is float:
            gts = [float(t) for t in gts]
        elif type is not str:
            gts = [int(t) for t in gts]
        if asDict:
            gts = dict(zip(names, gts))
        if precompDict is not None and addToPrecomp:
            precompDict[text] = gts
            precompDict["__counter__"] += 1
    return {"scaffold": fields[scafCol] if scafCol >= 0 else None,
            "position": int(fields[posCol]) if posCol >= 0 else None, "GTs": gts}


class GenoFileReader:
    """genomics.py:1913-1945: iterates the data lines of an open genotype file ('#' lines skipped); `names` come from the
    header line (read from the file unless given)."""

    def __init__(self, genoFile, headerLine=None, scafCol=0, posCol=1, firstSampleCol=2, type=str, splitPhased=False,
                 ploidy=None, precomp=True, precompMaxSize=10000):
        self.genoFile = genoFile
        if not headerLine:
            headerLine = next(genoFile)
        self.names = headerLine.split()[firstSampleCol:]
        self.scafCol, self.posCol, self.firstSampleCol = scafCol, posCol, firstSampleCol
        self.type, self.splitPhased = type, splitPhased
        if splitPhased:
            assert ploidy is not None, "Ploidy must be defined for splitting phased sequences"
            if self.names:
                self.names = makeHaploidNames(self.names, ploidy)
        self.precompDict = {"__maxSize__": precompMaxSize, "__counter__": 0}

    def _parse(self, line, asDict):
        d = self.precompDict
        return parseGenoLine(line, self.names, self.scafCol, self.posCol, self.firstSampleCol, self.type, self.splitPhased,
                             asDict, d, addToPrecomp=d["__counter__"] < d["__maxSize__"])

    def siteBySite(self, asDict=True):
        for line in self.genoFile:
            if line[0] != "#":
                yield self._parse(line, asDict)

    def nextSite(self, asDict=True):
        while True:
            line = next(self.genoFile, None)
            if not (line and line[0] == "#"):
                return self._parse(line, asDict)


def _windows_from(gd: geno_io.GenoData, ws: _win.WindowSet, genoFormat):
    for k in range(len(ws)):
        lo, hi = ws.lo[k], ws.hi[k]
        limits = [ws.start[k], ws.end[k]] if ws.start[k] is not None else [-np.inf, np.inf]
        yield GenoWindow(scaffold=ws.scaffold[k], limits=limits, names=gd.names, positions=gd.pos[lo:hi].tolist(),
                         ID=ws.ID[k], geno=gd.geno[lo:hi], ploidy=gd.ploidy, genoFormat=genoFormat)


def _parse(genoFile, headerLine, names, genoFormat, ploidy):
    return geno_io.parse_geno(genoFile, geno_format=genoFormat, samples=names, ploidy=ploidy, header=headerLine)


def slidingCoordWindows(genoFile, windSize, stepSize, headerLine=None, names=None, include=None, exclude=None,
                        genoFormat="phased", ploidy=None, **_):
    gd = _parse(genoFile, headerLine, names, genoFormat, ploidy)
    ws = _win.sliding_coord_windows(gd.scaf_ids, gd.scaf_names, gd.pos, windSize, stepSize, include, exclude)
    return _windows_from(gd, ws, genoFormat)


def slidingSitesWindows(genoFile, windSites, overlap, maxDist=np.inf, minSites=None, headerLine=None, names=None,
                        include=None, exclude=None, genoFormat="phased", ploidy=None, **_):
    gd = _parse(genoFile, headerLine, names, genoFormat, ploidy)
    ws = _win.sliding_sites_windows(gd.scaf_ids, gd.scaf_names, gd.pos, windSites, overlap,
                                    None if maxDist is None or np.isinf(maxDist) else maxDist, minSites, include, exclude)
    return _windows_from(gd, ws, genoFormat)


def predefinedCoordWindows(genoFile, windCoords, headerLine=None, names=None, genoFormat="phased", ploidy=None, **_):
    gd = _parse(genoFile, headerLine, names, genoFormat, ploidy)
    ws = _win.predefined_coord_windows(gd.scaf_ids, gd.scaf_names, gd.pos, windCoords)
    return _windows_from(gd, ws, genoFormat)


def parseGenoFile(genoFile, headerLine=None, names=None, includePositions=False, genoFormat="phased", ploidy=None, **_):
    """genomics.py:1949-1967: the whole file as one window (positions are nan unless includePositions)."""
    gd = _parse(genoFile, headerLine, names, genoFormat, ploidy)
    positions = gd.pos.tolist() if includePositions else [np.nan] * gd.n_sites
    return GenoWindow(names=gd.names, positions=positions, geno=gd.geno, ploidy=gd.ploidy, genoFormat=genoFormat)


# ------------------------------------------------------------------------------------------------
def _rounded(distArray, roundTo):
    return np.asarray(distArray, dtype=np.float64).round(roundTo)


def makeDistMatString(distArray, roundTo=10):
    """genomics.py:2288-2289: rows joined with spaces, no trailing newline.  Numbers are printed by the native formatter
    (pg_format_matrix_rows) exactly as numpy's round(roundTo).astype(str) prints them."""
    return geno_io.format_matrix_rows(_rounded(distArray, roundTo))[:-1]


def makeDistMatPhylipString(distArray, names, roundTo=10):
    m = _rounded(distArray, roundTo)
    return "%d\n" % m.shape[0] + geno_io.format_matrix_rows(m, prefixes=["%s  " % nm for nm in names])


def makeDistMatNexusString(distArray, names, roundTo=10):
    m = _rounded(distArray, roundTo)
    taxa = "".join("[%d] '%s'\n" % (i + 1, nm) for i, nm in enumerate(names))
    body = geno_io.format_matrix_rows(m, prefixes=["[%d] '%s'    " % (i + 1, nm) for i, nm in enumerate(names)])
    return ("\nBEGIN Taxa;\nDIMENSIONS ntax=%d;\nTAXLABELS\n%s;\nEND; [Taxa]\n"
            "\nBEGIN Distances;\nDIMENSIONS ntax=%d;\nFORMAT labels=left diagonal triangle=both;\nMATRIX\n%s;\nEND; [Distances]\n"
            % (len(names), taxa, len(names), body))
