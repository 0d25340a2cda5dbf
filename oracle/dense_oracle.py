"""TEST INFRASTRUCTURE — CPU oracle (vectorised numpy restatement).

This file is the *checker* for the CUDA path.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl
reference`` legs may import it; the product (``genomics_general_b200``) never
does and fails loudly when its CUDA library is missing.

It restates, over dense int8 arrays, the algorithms of the reference's per-window
numerics (all citations are genomics_general/<file>:<line>):

  pair counts / p-distance .... genomics.py:903-916, 1042-1047, 1219-1221
  nanmean_min ................. genomics.py:88-90
  groupDistStats .............. genomics.py:956-995
  indPairDists ................ genomics.py:934-954  (+ distMat.py:42-45)
  siteFreqs / siteNonNan ...... genomics.py:1032-1036, 1049-1052, 592-599
  ABBABABA (+ f4,D,fd,fdM) .... genomics.py:1647-1695, 1409-1475, 1565-1569
  sampleHet / H12stats ........ genomics.py:918-929, 1079-1098, 1239-1261 (in the cache states of popgenWindows.py:50-64)
  groupFreqStats .............. genomics.py:1002-1028, 609-632
  fourPop ..................... genomics.py:1585-1643, 1409-1583
  freq.py --target ............ freq.py:62-98; genomics.py:636-668
  sfs.py ...................... sfs.py:68-92, 94-125, 430-474
  window generators ........... genomics.py:1971-2027, 2032-2108, 2112-2171
  row prefix (start,end,mid) .. popgenWindows.py:37-39, genomics.py:1795-1797

PINNING: the reference has no tests or golden vectors (SURVEY.md §4), so this
oracle is pinned against outputs of the *reference itself* executed in the
build container: ``oracle/make_golden.py`` imports genomics_general/genomics.py,
runs it on small seeded inputs and commits inputs + outputs under
``tests/golden/`` (``oracle/make_golden2.py`` adds the second batch); ``tests/test_oracle_golden.py`` and
``tests/test_oracle_golden2.py`` check every function here against those fixtures.

Data model: ``g`` is int8 ``[L sites, H haplotypes]`` with A0 C1 G2 T3 and any
negative value = missing (the reference's ``numArray`` transposed,
genomics.py:74-77,834).  ``hap_pop[h]`` is the population index of haplotype h
(-1 = in the alignment but in no population).
"""
from __future__ import annotations

import itertools
import math

import numpy as np

NAN = float("nan")


# ----------------------------------------------------------------------------------------
# pairwise counts  (genomics.py:903-916 distMatrix/pairDist, 1042-1047 pairNonNan)
# ----------------------------------------------------------------------------------------
def pair_counts(g: np.ndarray):
    """diff[i,j] = #sites both non-missing and different; n[i,j] = #sites both non-missing.

    Integer-exact: one-hot indicator products in float64 (exact below 2**53).
    Diagonal entries: diff=0, n=#non-missing (the reference leaves n_ii = 0 in
    pairNonNan, genomics.py:1043-1047; callers below never read n_ii)."""
    g = np.asarray(g)
    L, H = g.shape
    valid = (g >= 0)
    V = valid.astype(np.float64)
    n = V.T @ V
    same = np.zeros((H, H), dtype=np.float64)
    for a in range(4):
        X = (g == a).astype(np.float64)
        same += X.T @ X
    diff = n - same
    return np.rint(diff).astype(np.int64), np.rint(n).astype(np.int64)


def dist_matrix(diff, n):
    """d_ij = diff/n, nan where n == 0 (np.mean of an empty array, genomics.py:1221);
    diagonal 0.0 as in distMatrix (genomics.py:908)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        d = diff.astype(np.float64) / n.astype(np.float64)
    d[n == 0] = np.nan
    np.fill_diagonal(d, 0.0)
    return d


def nanmean_min(a, min=0.0):
    """genomics.py:88-90."""
    a = np.asarray(a, dtype=np.float64)
    if a.size == 0:
        return NAN
    if 1 - (1.0 * np.isnan(a).sum() / a.size) < min:
        return NAN
    good = a[~np.isnan(a)]
    if good.size == 0:
        return NAN
    return float(good.sum() / good.size)


# ----------------------------------------------------------------------------------------
# groupDistStats  (genomics.py:956-995)
# ----------------------------------------------------------------------------------------
def group_dist_stats(g, hap_pop, n_pops, min_sites=None, min_data=0.01, do_pairs=True):
    """Returns (pi[P], dxy[npairs], fst[npairs]); pairs in itertools.combinations order
    of the population indices.  Statistics are symmetric in the pair, so this equals the
    reference's name-keyed dict regardless of its np.unique name ordering (965)."""
    hap_pop = np.asarray(hap_pop)
    diff, n = pair_counts(g)
    d = dist_matrix(diff, n)
    if min_sites:
        nn = n.copy()
        np.fill_diagonal(nn, 0)                     # pairNonNan leaves the diagonal 0 (1043)
        d[nn < min_sites] = np.nan                  # 959-961
    np.fill_diagonal(d, np.nan)                     # 963
    idx = [np.where(hap_pop == x)[0] for x in range(n_pops)]
    pi = np.array([nanmean_min(d[np.ix_(idx[x], idx[x])], min_data) for x in range(n_pops)])
    pairs = list(itertools.combinations(range(n_pops), 2))
    dxy = np.full(len(pairs), np.nan)
    fst = np.full(len(pairs), np.nan)
    if do_pairs:
        for k, (x, y) in enumerate(pairs):
            dxy[k] = nanmean_min(d[np.ix_(idx[x], idx[y])], min_data)          # 984
            n_x, n_y = len(idx[x]), len(idx[y])
            w = 1.0 * n_x / (n_x + n_y)                                        # 988-990
            pi_s = w * pi[x] + (1 - w) * pi[y]                                 # 991
            both = np.concatenate([idx[x], idx[y]])
            pi_t = nanmean_min(d[np.ix_(both, both)], min_data)                # 992
            with np.errstate(divide="ignore", invalid="ignore"):
                fst[k] = 1 - np.float64(pi_s) / np.float64(pi_t)               # 993
    return pi, dxy, fst


def group_dist_stats_closed_form(g, hap_pop, n_pops, min_sites=None, min_data=0.01):
    """The allele-count closed form the K1 kernel uses (SURVEY.md §0 routing rule).

    Valid iff every site of the window is non-missing in ALL haplotypes that belong to a
    population, or missing in all of them.  Returns (ok, pi, dxy, fst); ``ok`` False means
    the window is "ragged" and the pairwise path must be used."""
    g = np.asarray(g)
    hap_pop = np.asarray(hap_pop)
    used = hap_pop >= 0
    gu = g[:, used]
    pops = hap_pop[used]
    nvalid = (gu >= 0).sum(axis=1)
    Hu = gu.shape[1]
    ragged = (nvalid > 0) & (nvalid < Hu)
    if ragged.any():
        return False, None, None, None
    present = nvalid == Hu
    Lp = int(present.sum())
    gp = gu[present]
    N = np.array([(pops == x).sum() for x in range(n_pops)], dtype=np.int64)
    counts = np.zeros((Lp, n_pops, 4), dtype=np.int64)
    for x in range(n_pops):
        sub = gp[:, pops == x]
        for a in range(4):
            counts[:, x, a] = (sub == a).sum(axis=1)
    pairs = list(itertools.combinations(range(n_pops), 2))
    pi = np.full(n_pops, np.nan)
    dxy = np.full(len(pairs), np.nan)
    fst = np.full(len(pairs), np.nan)
    all_nan = (Lp == 0) or (bool(min_sites) and Lp < min_sites)
    sq = (counts * counts).sum(axis=(0, 2))                                    # [P] sum_a c^2

    def frac_ok(nonnan, size):
        return not (1 - (1.0 * (size - nonnan) / size) < min_data)

    def pi_of(sumsq, n):
        # mean over the n(n-1) off-diagonal ordered pairs of diff/L'
        if all_nan or n < 2 or not frac_ok(n * n - n, n * n):
            return NAN
        return ((n * n * Lp - sumsq) / 2.0) / ((n * (n - 1) / 2.0) * Lp)

    for x in range(n_pops):
        pi[x] = pi_of(int(sq[x]), int(N[x]))
    for k, (x, y) in enumerate(pairs):
        cross = int((counts[:, x, :] * counts[:, y, :]).sum())
        if not all_nan and frac_ok(N[x] * N[y], N[x] * N[y]):
            dxy[k] = (N[x] * N[y] * Lp - cross) / float(N[x] * N[y] * Lp)
        nt = int(N[x] + N[y])
        sq_t = int(sq[x] + sq[y] + 2 * cross)
        pi_t = pi_of(sq_t, nt)
        w = 1.0 * N[x] / (N[x] + N[y])
        pi_s = w * pi[x] + (1 - w) * pi[y]
        with np.errstate(divide="ignore", invalid="ignore"):
            fst[k] = 1 - np.float64(pi_s) / np.float64(pi_t)
    return True, pi, dxy, fst


# ----------------------------------------------------------------------------------------
# groupFreqStats  (genomics.py:1002-1028, baseCountPi 609-616, TajimaD 619-632)
# ----------------------------------------------------------------------------------------
def group_freq_stats(g, hap_pop, n_pops):
    """dict of arrays l, S, thetaPi, thetaW, TajD (length P).  Only sites with no missing data in ANY
    haplotype of the alignment are used (1010)."""
    g = np.asarray(g)
    hap_pop = np.asarray(hap_pop)
    keep = np.all(g >= 0, axis=1)
    gp = g[keep]
    l = int(keep.sum())
    out = dict(l=np.full(n_pops, float(l)), S=np.full(n_pops, np.nan), thetaPi=np.full(n_pops, np.nan),
               thetaW=np.full(n_pops, np.nan), TajD=np.full(n_pops, np.nan))
    if l < 1:
        return out
    counts = site_counts(gp, hap_pop, n_pops).astype(np.float64)          # [l,P,4]
    for x in range(n_pops):
        N = int((hap_pop == x).sum())
        c = counts[:, x, :]
        pairs = (c[:, 0] * c[:, 1] + c[:, 0] * c[:, 2] + c[:, 0] * c[:, 3] + c[:, 1] * c[:, 2] + c[:, 1] * c[:, 3]
                 + c[:, 2] * c[:, 3])
        with np.errstate(divide="ignore", invalid="ignore"):
            site_pi = pairs / (.5 * N * (N - 1))
            S = float((site_pi != 0.).sum())
            theta_pi = float(site_pi.sum())
            a = sum(1. / i for i in range(1, N))
            a2 = sum(1. / (i ** 2) for i in range(1, N))
            theta_w = np.float64(S) / np.float64(a)
            b1 = (N + 1.) / (3 * (N - 1)) if N > 1 else np.nan
            b2 = (2. * (N ** 2 + N + 3)) / (9 * N * (N - 1)) if N > 1 else np.nan
            c1 = b1 - np.float64(1.) / np.float64(a)
            c2 = b2 - np.float64(N + 2) / np.float64(a * N) + np.float64(a2) / np.float64(a ** 2)
            e1 = c1 / np.float64(a)
            e2 = c2 / np.float64(a ** 2 + a2)
            D = (theta_pi - theta_w) / np.sqrt(e1 * S + e2 * S * (S - 1))
        out["S"][x], out["thetaPi"][x], out["thetaW"][x], out["TajD"][x] = S, theta_pi, float(theta_w), float(D)
    return out


# ----------------------------------------------------------------------------------------
# indPairDists  (genomics.py:934-954) in distMat.py's individual order (distMat.py:42-45)
# ----------------------------------------------------------------------------------------
def ind_pair_dists(g, hap_ind, n_ind, include_same_with_same=False, min_sites=None):
    """[n_ind, n_ind] matrix: entry (a,b) = nanmean of the haplotype-distance block of
    individuals a and b.  Haplotypes with hap_ind < 0 are ignored."""
    hap_ind = np.asarray(hap_ind)
    diff, n = pair_counts(g)
    d = dist_matrix(diff, n)
    if min_sites:
        nn = n.copy()
        np.fill_diagonal(nn, 0)
        d[nn < min_sites] = np.nan
    if not include_same_with_same:
        np.fill_diagonal(d, np.nan)                                            # 940
    idx = [np.where(hap_ind == a)[0] for a in range(n_ind)]
    out = np.full((n_ind, n_ind), np.nan)
    for a in range(n_ind):
        for b in range(n_ind):
            blk = d[np.ix_(idx[a], idx[b])]
            good = blk[~np.isnan(blk)]
            out[a, b] = good.sum() / good.size if good.size else np.nan        # np.nanmean, 947
    return out


# ----------------------------------------------------------------------------------------
# sampleHet  (genomics.py:918-929) as called by popgenWindows.py:59-61 (no arguments)
# ----------------------------------------------------------------------------------------
def _masked_dist(g, masked_min_sites=None, diag_nan=False):
    """The state of Alignment._distMat_ inside one popgenWindows worker call: distMatrix()
    (zero diagonal, 907-916); an earlier groupDistStats in the same window has set entries with
    n_ij < minSites to nan IN PLACE (959-961) and the diagonal to nan (963); an earlier
    indPairDists has set the diagonal to nan (940)."""
    diff, n = pair_counts(g)
    d = dist_matrix(diff, n)
    if masked_min_sites:
        nn = n.copy()
        np.fill_diagonal(nn, 0)
        d[nn < masked_min_sites] = np.nan
    if diag_nan:
        np.fill_diagonal(d, np.nan)
    return d, n


def sample_het(g, hap_ind, n_ind, masked_min_sites=None):
    """het[a] for each individual.  The reference's condition (924, 927)

        len(x)==2 & np.sum(mask_i & mask_j) >= _minSites        (_minSites = 1)

    parses as the chained comparison  len(x) == (2 & n_ij) >= 1 : the value is d_ij iff the
    individual has exactly two haplotypes AND bit 1 of n_ij is set, else nan.  Kept as is."""
    hap_ind = np.asarray(hap_ind)
    d, n = _masked_dist(g, masked_min_sites)
    out = np.full(n_ind, np.nan)
    for a in range(n_ind):
        x = np.where(hap_ind == a)[0]
        if len(x) == 2 and (2 & int(n[x[0], x[1]])) == 2:
            out[a] = d[x[0], x[1]]
    return out


# ----------------------------------------------------------------------------------------
# H12stats  (genomics.py:1079-1098) + distMat_to_cluster_sizes (1239-1261)
# ----------------------------------------------------------------------------------------
def cluster_sizes(match):
    """Greedy clustering, restated step by step (1239-1261): take the row with the most matches
    (first one on ties, np.argmax); if it has more than one match its matches form a cluster and
    are removed (the row itself stays when the diagonal does not match, i.e. was nan); otherwise
    every remaining entry is a cluster of one."""
    match = np.asarray(match, dtype=bool)
    alive = np.ones(match.shape[0], dtype=bool)
    sizes = []
    while alive.any():
        idx = np.where(alive)[0]
        sub = match[np.ix_(idx, idx)]
        cnt = sub.sum(axis=1)
        k = int(cnt.argmax())
        m = int(cnt[k])
        if m > 1:
            sizes.append(m)
            alive[idx[sub[k]]] = False
        else:
            sizes += [1] * len(idx)
            break
    return sizes


def h12_stats(g, hap_pop, n_pops, max_dist=0.0, masked_min_sites=None, diag_nan=False):
    """[P,3] = H1, H12, H2 per population.  ``masked_min_sites`` / ``diag_nan`` describe what
    earlier analyses of the same window did to the cached matrix (see _masked_dist)."""
    hap_pop = np.asarray(hap_pop)
    d, _ = _masked_dist(g, masked_min_sites, diag_nan)
    out = np.full((n_pops, 3), np.nan)
    for x in range(n_pops):
        idx = np.where(hap_pop == x)[0]
        with np.errstate(invalid="ignore"):
            match = d[np.ix_(idx, idx)] <= max_dist                            # nan <= x is False (1244)
        cs = np.array(cluster_sizes(match))
        f = cs / cs.sum()
        H1 = float((f ** 2).sum())
        if len(f) > 1:
            H12 = H1 + 2 * f[0] * f[1]
            H2 = float((f[1:] ** 2).sum())
        else:
            H12, H2 = H1, 0.0
        out[x] = (H1, H12, H2)
    return out


# ----------------------------------------------------------------------------------------
# freq.py --target derived | minor  (freq.py:62-92; genomics.py:636-668)
# ----------------------------------------------------------------------------------------
def target_freqs(g, hap_pop, n_pops, target, min_data=0.0, as_counts=False, threshold=None):
    """float64 [L,P] (nan = no value; counts mode: 0).  ``target``: "derived" (last population is
    the outgroup: the in-group allele that is not the outgroup's, when the in-group has exactly two
    alleles and the outgroup exactly one of them, 654-655) or "minor" (the rarer of exactly two
    alleles over all haplotypes that belong to a population; the reference picks at random on a
    tie (667) — here ties give -1 in the second return value so that callers can skip them).
    Returns (values, tie[L] bool).  Values are NOT rounded (freq.py:91 rounds to 4 dp)."""
    c = site_counts(g, hap_pop, n_pops)                                        # [L,P,4]
    L = c.shape[0]
    tgt = np.full(L, -1, dtype=np.int64)
    tie = np.zeros(L, dtype=bool)
    if target == "derived":
        cin = c[:, :-1, :].sum(axis=1)
        cout = c[:, -1, :]
        for s in range(L):
            ia = np.where(cin[s] > 0)[0]
            oa = np.where(cout[s] > 0)[0]
            if len(oa) == 1 and len(ia) == 2 and oa[0] in ia:
                tgt[s] = ia[ia != oa[0]][0]
    elif target == "minor":
        tot = c.sum(axis=1)
        for s in range(L):
            al = np.where(tot[s] > 0)[0]
            if len(al) == 2:
                if tot[s, al[0]] == tot[s, al[1]]:
                    tie[s] = True
                else:
                    tgt[s] = al[np.argmin(tot[s, al])]
    else:
        raise ValueError(target)
    nk = c.sum(axis=2)                                                         # [L,P]
    out = np.zeros((L, n_pops)) if as_counts else np.full((L, n_pops), np.nan)
    for s in range(L):
        if tgt[s] < 0:
            continue
        for x in range(n_pops):
            if not (nk[s, x] >= min_data):                                     # siteNonNan() >= minData: a COUNT (freq.py:79)
                continue
            if as_counts:
                out[s, x] = c[s, x, tgt[s]]
            else:
                out[s, x] = c[s, x, tgt[s]] / nk[s, x] if nk[s, x] > 0 else np.nan
    if threshold and not as_counts:                                            # 96-98
        r = np.around(out, 4)                                                  # the comparison sees the rounded value (91)
        hi = r >= threshold
        lo = r < threshold
        out[hi] = 1
        out[lo] = 0
    return out, tie


# ----------------------------------------------------------------------------------------
# per-site counts  (genomics.py:1049-1052 siteFreqs, 592-599 binBaseFreqs, 1032-1036)
# ----------------------------------------------------------------------------------------
def site_counts(g, hap_pop, n_pops):
    """int64 [L, P, 4]: A,C,G,T counts over each population's non-missing haplotypes."""
    g = np.asarray(g)
    hap_pop = np.asarray(hap_pop)
    L = g.shape[0]
    out = np.zeros((L, n_pops, 4), dtype=np.int64)
    for x in range(n_pops):
        sub = g[:, hap_pop == x]
        for a in range(4):
            out[:, x, a] = (sub == a).sum(axis=1)
    return out


# ----------------------------------------------------------------------------------------
# ABBA-BABA  (genomics.py:1647-1695)
# ----------------------------------------------------------------------------------------
def _f4(p1, p2, p3, p4):                                                       # 1409-1411
    return (1 - p1) * p2 * p3 * (1 - p4) - p1 * (1 - p2) * p3 * (1 - p4)


def abbababa_sites(g, hap_pop, P1, P2, P3, O, min_data):
    """Site classification + derived-allele frequencies (1649-1682, polarize=True).
    Returns (site_index[], p1[], p2[], p3[], p4[]) for every (site, derived allele) hit."""
    c = site_counts(g, hap_pop, max(P1, P2, P3, O) + 1)[:, [P1, P2, P3, O], :]   # [L,4,4]
    hap_pop = np.asarray(hap_pop)
    N = np.array([(hap_pop == x).sum() for x in (P1, P2, P3, O)], dtype=np.float64)
    nk = c.sum(axis=2)                                                         # [L,4] non-missing per pop
    tot = c.sum(axis=1)                                                        # [L,4] allele counts over all 4
    biallelic = (tot > 0).sum(axis=1) == 2                                     # 1655
    with np.errstate(divide="ignore", invalid="ignore"):
        enough = np.all(nk * 1.0 / N[None, :] >= min_data, axis=1)             # 1657-1660
    good = np.where(biallelic & enough)[0]
    cg = c[good].astype(np.float64)
    nkg = nk[good].astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        freqs = cg / nkg[:, :, None]                                           # nan where a pop has no data (597)
        allf = tot[good] / tot[good].sum(axis=1, keepdims=True)
    hit_s, hit_a = np.where((allf > 0) & (freqs[:, 3, :] == 0))               # 1672
    return good[hit_s], freqs[hit_s, 0, hit_a], freqs[hit_s, 1, hit_a], freqs[hit_s, 2, hit_a], freqs[hit_s, 3, hit_a]


def abbababa(g, hap_pop, P1, P2, P3, O, min_data):
    """dict D, fd, fdM, ABBA, BABA, sitesUsed  (1684-1695).  With no usable sites the
    reference zips 6 keys with 7 values, so sitesUsed is nan too (1694-1695)."""
    L = np.asarray(g).shape[0]
    # the reference takes the good-site branch iff len(goodSites) >= 1 (1671)
    hap_pop_a = np.asarray(hap_pop)
    c = site_counts(g, hap_pop_a, max(P1, P2, P3, O) + 1)[:, [P1, P2, P3, O], :]
    N = np.array([(hap_pop_a == x).sum() for x in (P1, P2, P3, O)], dtype=np.float64)
    nk = c.sum(axis=2)
    tot = c.sum(axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        n_good = int((((tot > 0).sum(axis=1) == 2) & np.all(nk * 1.0 / N[None, :] >= min_data, axis=1)).sum())
    if n_good < 1:
        return dict(D=NAN, fd=NAN, fdM=NAN, ABBA=NAN, BABA=NAN, sitesUsed=NAN)
    _, p1, p2, p3, p4 = abbababa_sites(g, hap_pop, P1, P2, P3, O, min_data)
    with np.errstate(divide="ignore", invalid="ignore"):
        abba = ((1 - p1) * p2 * p3 * (1 - p4))
        baba = (p1 * (1 - p2) * p3 * (1 - p4))
        D = _f4(p1, p2, p3, p4).sum() * 1.0 / (abba + baba).sum()              # 1430-1431
        pd = p2 * (p2 > p3) + p3 * (p3 >= p2)                                  # 1446
        fd = _f4(p1, p2, p3, p4).sum() * 1.0 / _f4(p1, pd, pd, p4).sum()
        a = p3 > p1                                                            # 1460-1468
        b = p3 > p2
        x = p1 > p2
        y = ~x
        pdm1 = p3 * (x & a) + p1 * (~(x & a))
        pdm2 = p3 * (y & b) + p2 * (~(y & b))
        pdm3 = -p3 * (x & a) + p3 * (y & b) - p1 * (x & ~a) + p2 * (y & ~b)
        fdm = _f4(p1, p2, p3, p4).sum() * 1.0 / _f4(pdm1, pdm2, pdm3, p4).sum()  # 1470-1475
    return dict(D=float(D), fd=float(fd), fdM=float(fdm), ABBA=float(abba.sum()),
                BABA=float(baba.sum()), sitesUsed=int(len(p1)))


# ----------------------------------------------------------------------------------------
# fourPop  (genomics.py:1585-1643; statistics 1409-1583)
# ----------------------------------------------------------------------------------------
FOURPOP_KEYS = ('fhom', "fhom'", 'D', 'fd', "fd'", 'fdm', "fdm'", 'fdh', 'fdh2', 'fh', "ABBA", "BABA", "ABAA", "BAAA",
                "sitesUsed")


def _f4c(p1, p2, p3, p4):                                                      # 1413-1418
    return _f4(p1, p2, p3, p4) + _f4(1 - p1, 1 - p2, 1 - p3, 1 - p4)


def four_pop_sites(g, hap_pop, P1, P2, P3, P4, min_data, polarize=False, fixed=False):
    """(p1,p2,p3,p4) of every (site, allele) the reference selects (1595-1621), n_good_sites."""
    hap_pop = np.asarray(hap_pop)
    c = site_counts(g, hap_pop, max(P1, P2, P3, P4) + 1)[:, [P1, P2, P3, P4], :]
    N = np.array([(hap_pop == x).sum() for x in (P1, P2, P3, P4)], dtype=np.float64)
    nk = c.sum(axis=2)
    tot = c.sum(axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        good = np.where(((tot > 0).sum(axis=1) == 2) & np.all(nk * 1.0 / N[None, :] >= min_data, axis=1))[0]
        freqs = c[good].astype(np.float64) / nk[good].astype(np.float64)[:, :, None]
        allf = tot[good] / tot[good].sum(axis=1, keepdims=True)
    if polarize:
        hs, ha = np.where((allf > 0) & (freqs[:, 3, :] == 0))
    elif fixed:
        fx = lambda f: (f == 0) | (f == 1)   # noqa: E731
        hs, ha = np.where((allf > 0) & (freqs[:, 3, :] == 0) & fx(freqs[:, 0, :]) & fx(freqs[:, 1, :]) & fx(freqs[:, 2, :]))
    else:
        hs = np.arange(len(good))
        ha = np.argsort(allf, axis=1, kind="stable")[:, 2] if len(good) else np.zeros(0, dtype=np.int64)   # 1615
    return freqs[hs, 0, ha], freqs[hs, 1, ha], freqs[hs, 2, ha], freqs[hs, 3, ha], len(good)


def four_pop(g, hap_pop, P1, P2, P3, P4, min_data, polarize=False, fixed=False):
    p1, p2, p3, p4, n_good = four_pop_sites(g, hap_pop, P1, P2, P3, P4, min_data, polarize, fixed)
    if n_good < 1:
        return dict(zip(FOURPOP_KEYS, [NAN] * 14 + [0]))                      # 1641-1643
    with np.errstate(divide="ignore", invalid="ignore"):
        abba = (1 - p1) * p2 * p3 * (1 - p4)
        baba = p1 * (1 - p2) * p3 * (1 - p4)
        f4 = _f4(p1, p2, p3, p4)
        f4c = _f4c(p1, p2, p3, p4)
        pd = p2 * (p2 > p3) + p3 * (p3 >= p2)
        a = p3 > p1
        b = p3 > p2
        x = p1 > p2
        y = ~x
        pdm1 = p3 * (x & a) + p1 * (~(x & a))
        pdm2 = p3 * (y & b) + p2 * (~(y & b))
        pdm3 = -p3 * (x & a) + p3 * (y & b) - p1 * (x & ~a) + p2 * (y & ~b)
        t11 = _f4c(p1, p3, p3, p4)
        t12 = _f4c(p4, p2, p3, p4)
        t21 = _f4c(p3, p2, p3, p4)
        t22 = _f4c(p1, p4, p3, p4)
        t31 = _f4c(p1, p2, p2, p4)
        t32 = _f4c(p1, p2, p3, p1)
        t41 = _f4c(p1, p2, p1, p4)
        t42 = _f4c(p1, p2, p3, p2)
        u1 = np.abs(p1 - p2)
        u2 = np.abs(p3 - p4)
        vals = [
            f4.sum() * 1. / _f4(p1, p3, p3, p4).sum(),                                              # fhom_old 1420
            f4c.sum() * 1. / t11.sum(),                                                             # fhom_new 1423
            f4.sum() * 1. / (abba + baba).sum(),                                                    # D 1430
            f4.sum() * 1. / _f4(p1, pd, pd, p4).sum(),                                              # fd 1445
            f4c.sum() * 1. / _f4c(p1, pd, pd, p4).sum(),                                            # fd_new 1450
            f4.sum() * 1. / _f4(pdm1, pdm2, pdm3, p4).sum(),                                        # fdm 1470
            f4c.sum() * 1. / _f4c(pdm1, pdm2, pdm3, p4).sum(),                                      # fdm_new 1476
            f4c.sum() * 1. / np.amax([t11, t12, t21, t22], axis=0).sum() if len(p1) else NAN,       # fdh 1488
            f4c.sum() * 1. / np.amax([t11, t12, t21, t22, t31, t32, t41, t42], axis=0).sum() if len(p1) else NAN,
            f4c.sum() * 1. / ((u1 * (u1 > u2) + u2 * (u2 >= u1)) ** 2).sum(),                       # fh 1527
            abba.sum(), baba.sum(),
            ((1 - p1) * p2 * (1 - p3) * (1 - p4)).sum(),                                            # ABAA 1558
            (p1 * (1 - p2) * (1 - p3) * (1 - p4)).sum(),                                            # BAAA 1561
            len(p1)]
    return dict(zip(FOURPOP_KEYS, [float(v) for v in vals]))


# ----------------------------------------------------------------------------------------
# sfs.py, --inputType genotypes without subsampling  (sfs.py:430-470, 68-92, 94-125)
# ----------------------------------------------------------------------------------------
def sfs_target_counts_from_counts(c, n_in, outgroup=-1, N=None):
    """Per-site target-allele counts from base counts c int [L, P, 4]: (counts int64 [L, n_in], used bool [L]).
    N (haplotypes per population) switches on the completeness test of genotype input (sfs.py:449); base-count input
    (sfs.py:456-470) has none.  getTargetCounts: sfs.py:68-92."""
    c = np.asarray(c, dtype=np.int64)
    L = c.shape[0]
    out = np.zeros((L, n_in), dtype=np.int64)
    used = np.zeros(L, dtype=bool)
    for s in range(L):
        cin = c[s, :n_in]
        if N is not None and not np.all(cin.sum(axis=1) == np.asarray(N)[:n_in]):
            continue
        tot = cin.sum(axis=0)
        alleles = tot > 0
        if outgroup >= 0:
            oa = c[s, outgroup] > 0
            alla = alleles | oa
            if not 1 <= alla.sum() <= 2:
                continue
            n_out = int(oa.sum())
            if n_out == 0 or (True & n_out) != 1:           # `outgroupMono & nOutAlleles != 1` (84): precedence kept
                continue
            cand = np.where(~oa & alleles)[0]
            target = cand[0] if len(cand) else np.where(~alleles)[0][0]
        else:
            if not 1 <= alleles.sum() <= 2:
                continue
            target = np.argsort(tot, kind="stable")[-2]     # (90); the reference's unstable sort is free on exact ties
        out[s] = cin[:, target]
        used[s] = True
    return out, used


def sfs_target_counts(g, hap_pop, n_in, outgroup=-1):
    """The same from genotypes: a site is used iff every in-group haplotype is called (449) and getTargetCounts returns
    a value."""
    hap_pop = np.asarray(hap_pop)
    P = int(hap_pop.max()) + 1
    c = site_counts(g, hap_pop, P)
    N = np.array([(hap_pop == x).sum() for x in range(P)])
    return sfs_target_counts_from_counts(c, n_in, outgroup, N)


def sfs_chains(tc, used, groups):
    """insertion-ordered (key tuple, count) lists, one per group, from per-site target counts (SparseFS.add / asChains)"""
    out = []
    for grp in groups:
        nested = {}
        for s in np.where(used)[0]:
            d = nested
            for x in grp[:-1]:
                d = d.setdefault(int(tc[s, x]), {})
            k = int(tc[s, grp[-1]])
            d[k] = d.get(k, 0) + 1
        chains = []

        def walk(d, prefix):
            for k, v in d.items():
                if isinstance(v, dict):
                    walk(v, prefix + (k,))
                else:
                    chains.append((prefix + (k,), v))
        walk(nested, ())
        out.append(chains)
    return out


def sfs(g, hap_pop, n_in, groups, outgroup=-1, site_mask=None):
    """For each group of populations: the spectrum as an insertion-ordered list of (key tuple, count) in the order the
    reference's nested SparseFS dicts are written (asChains, 117-125): first appearance at each nesting level."""
    tc, used = sfs_target_counts(g, hap_pop, n_in, outgroup)
    if site_mask is not None:
        used = used & np.asarray(site_mask, dtype=bool)
    return sfs_chains(tc, used, groups), int(used.sum())


# ----------------------------------------------------------------------------------------
# window generators restated over (scaffold id, position) arrays -> half-open site ranges
# ----------------------------------------------------------------------------------------
def _scaffold_runs(scaf):
    """Maximal runs of equal scaffold id: list of (id, lo, hi)."""
    scaf = np.asarray(scaf)
    runs = []
    S = len(scaf)
    lo = 0
    while lo < S:
        hi = lo
        while hi < S and scaf[hi] == scaf[lo]:
            hi += 1
        runs.append((scaf[lo], lo, hi))
        lo = hi
    return runs


def sliding_coord_windows(scaf, pos, wind_size, step_size=None, include=None, exclude=None):
    """genomics.py:1971-2027.  Returns list of dict(scaffold,start,end,lo,hi).

    Literal restatement of the generator's state machine driven by an index into the
    site arrays (the 'site in hand')."""
    if not step_size:
        step_size = wind_size
    scaf = list(scaf)
    pos = list(pos)
    S = len(pos)
    out = []

    def wanted(sc):
        return (not include and not exclude) or (include and sc in include) or (exclude and sc not in exclude)

    i = 0                                           # index of the site in hand; S == end of file
    w_scaf = None
    limits = [-math.inf, math.inf]
    w_lo = 0                                        # index of the first site currently held by the window
    held = []                                       # indices of the sites in the window
    while i < S:
        while i < S and scaf[i] == w_scaf and pos[i] <= limits[1]:
            if pos[i] >= limits[0]:
                held.append(i)
            i += 1
        if w_scaf is not None:
            out.append(dict(scaffold=w_scaf, start=limits[0], end=limits[1], sites=list(held)))
        cur_scaf = scaf[i] if i < S else None
        if cur_scaf == w_scaf:
            limits = [l + step_size for l in limits]
            held = [k for k in held if pos[k] >= limits[0]]      # GenoWindow.slide 1767-1777
        else:
            if wanted(cur_scaf):
                w_scaf = cur_scaf
                limits = [1, wind_size]
                held = []
            else:
                bad = cur_scaf
                while i < S and (scaf[i] == bad or (include and scaf[i] not in include)
                                 or (exclude and scaf[i] in exclude)):
                    i += 1
        if i >= S:
            break
    return out


def sliding_sites_windows(scaf, pos, wind_sites, overlap=0, max_dist=math.inf, min_sites=None,
                          include=None, exclude=None):
    """genomics.py:2032-2108.  Returns list of dict(scaffold,sites=[indices])."""
    if not min_sites:
        min_sites = wind_sites
    scaf = list(scaf)
    pos = list(pos)
    S = len(pos)
    out = []

    def wanted(sc):
        return (not include and not exclude) or (include and sc in include) or (exclude and sc not in exclude)

    def skip_bad(i, bad):
        while i < S and (scaf[i] == bad or (include and scaf[i] not in include)
                         or (exclude and scaf[i] in exclude)):
            i += 1
        return i

    i = 0
    w_scaf = None
    held = []
    guard = 0
    while True:
        guard += 1
        assert guard < 10 * S + 100, "window state machine did not terminate"
        while (i < S and scaf[i] == w_scaf and len(held) < wind_sites
               and (len(held) == 0 or pos[i] - min(pos[k] for k in held[:1]) <= max_dist)):
            held.append(i)
            i += 1
        cur_scaf = scaf[i] if i < S else None
        if len(held) >= min_sites:
            out.append(dict(scaffold=w_scaf, sites=list(held)))
            if cur_scaf == w_scaf:
                held = held[len(held) - overlap:] if overlap else []           # trim(leave=overlap) 1779-1788
            else:
                if wanted(cur_scaf):
                    w_scaf, held = cur_scaf, []
                else:
                    i = skip_bad(i, cur_scaf)
        else:
            if cur_scaf == w_scaf:
                held = held[1:]                                                # trim(remove=1)
            else:
                if wanted(cur_scaf):
                    w_scaf, held = cur_scaf, []
                else:
                    i = skip_bad(i, cur_scaf)
        if i >= S:
            break
    return out


def predefined_coord_windows(scaf, pos, wind_coords):
    """genomics.py:2112-2171.  wind_coords: list of (scaffold, start, end[, ID])."""
    scaf = list(scaf)
    pos = list(pos)
    S = len(pos)
    all_scafs = [w[0] for w in wind_coords]
    scafs = sorted(set(all_scafs), key=lambda x: all_scafs.index(x))
    out = []
    i = 0
    w_scaf = None
    held = []
    for w in wind_coords:
        limits = [w[1], w[2]]
        if w_scaf is not None and w_scaf == w[0]:
            held = [k for k in held if pos[k] >= limits[0]]                    # slide(newLimits=)
        else:
            w_scaf, held = w[0], []
        wsi = scafs.index(w_scaf)
        while i < S and (scaf[i] not in scafs or scafs.index(scaf[i]) < wsi):
            bad = scaf[i]
            while i < S and scaf[i] == bad:
                i += 1
        while i < S and scaf[i] == w_scaf and pos[i] < limits[0]:
            i += 1
        while i < S and scaf[i] == w_scaf and limits[0] <= pos[i] <= limits[1]:
            held.append(i)
            i += 1
        out.append(dict(scaffold=w_scaf, start=limits[0], end=limits[1], sites=list(held),
                        ID=(w[3] if len(w) > 3 else "NA")))
        if i >= S:
            break
    return out


def mid_pos(positions):
    """GenoWindow.midPos, genomics.py:1795-1797 (Python-3 banker's rounding; nan if empty)."""
    try:
        return int(round(sum(int(p) for p in positions) / len(positions)))
    except ZeroDivisionError:
        return NAN


# ----------------------------------------------------------------------------------------
# row formatting  (popgenWindows.py:37-39,66-74; ABBABABAwindows.py:31-51)
# ----------------------------------------------------------------------------------------
def popgen_row(scaffold, start, end, mid, sites, values, round_to=4, window_id=None):
    vals = [round(np.float64(v), round_to) for v in values]
    res = ([] if window_id is None else [window_id]) + [scaffold, start, end, mid, sites] + vals
    return ",".join(str(x) for x in res)
