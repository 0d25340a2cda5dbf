"""distPaint's epilogue (k2_paint_epi) at its edges, every query against oracle/paint_oracle.paint_window
(np.nanmean, np.argmin, sorted() and scipy's ranksums): assignments equal, means equal bit for bit, p-values within 1e-12
with the same nan pattern.

Windows are short (3 to 40 sites), so distances are ratios of small integers and the means of different populations tie
or differ in the last bit, where argmin, the delta test and the rank-sum threshold decide.  The groups:
  - summation lengths at numpy's pairwise boundaries (8 accumulators up to 128, a split above), nans inside the lists;
  - rank counts past one warp (n1 > 32) under heavy ties, and complete separation (512 vs 512, p ~ 1e-169);
  - 1 to 32 populations, identical member lists, members called nowhere, means in every count_run order, delta edges;
  - the pair path's layouts: tile edges, queries that are members, missing calls shared by a sample's two haplotypes;
  - window batches, the call without statistics (the command line's), noresult, and min_sites at the window length;
and the command line against reference fixtures with populations of 9, 130 and 300 samples."""
import numpy as np
import pytest

from oracle import paint_oracle as po
from test_gpu_paint import _same_bits
from test_paint_cpu import CASES8, DIR8, expected, run_cli

pytestmark = pytest.mark.gpu

NR = -1


def _geno(rng, S, H, miss=0.0, shared=False):
    """haplotypes from four source populations whose allele frequencies differ per site -> (g int8 [S, H], source [H]).
    shared: a missing call hits both haplotypes (2k, 2k + 1) of a sample"""
    src = rng.integers(0, 4, H)
    freq = rng.choice([0.05, 0.3, 0.7, 0.95], size=(S, 4))
    alt = rng.random((S, H)) < freq[:, src]
    bases = rng.permuted(np.tile(np.arange(4, dtype=np.int8), (S, 1)), axis=1)[:, :2]
    g = np.where(alt, bases[:, 1:2], bases[:, 0:1]).astype(np.int8)
    if shared:
        g[np.repeat(rng.random((S, (H + 1) // 2)) < miss, 2, axis=1)[:, :H]] = -1
    elif miss:
        g[rng.random((S, H)) < miss] = -1
    return g, src


def _csr(pops):
    return (np.cumsum([0] + [len(m) for m in pops]).astype(np.int32),
            np.array([j for m in pops for j in m], dtype=np.int32))


def _paint(g, wins, query, pops, min_sites, delta=False, thr=0.05, noresult=NR, with_stats=True):
    from genomics_general_b200.engine import Engine
    ref_off, ref_hap = _csr(pops)
    with Engine(0) as eng:
        eng.upload(g, np.arange(len(g), dtype=np.int32) * 10 + 1)
        eng.set_windows(np.array([w[0] for w in wins], np.int64), np.array([w[1] for w in wins], np.int64))
        return eng.distpaint(np.asarray(query, np.int32), ref_off, ref_hap, min_sites, delta=delta, threshold=thr,
                             noresult=noresult, with_stats=with_stats)


def _oracle(g, wins, query, pops, min_sites, delta=False, thr=0.05, noresult=NR):
    """per window (assign, means, pvals) of every query, None for an empty window"""
    return [po.paint_window(g[lo:hi], list(query), pops, min_sites, thr if delta else None, thr, noresult) if hi > lo
            else None for lo, hi in wins]


def _check(r, want, noresult=NR, what=""):
    for w, o in enumerate(want):
        if o is None:
            assert (r["assign"][w] == noresult).all(), (what, w)
            assert np.isnan(r["means"][w]).all() and np.isnan(r["pvals"][w]).all(), (what, w)
            continue
        a, m, p = o
        bad = np.flatnonzero(r["assign"][w] != a)
        assert bad.size == 0, (what, w, bad[:8], r["assign"][w][bad[:8]], a[bad[:8]])
        _same_bits(r["means"][w], m, (what, w))
        got = r["pvals"][w]
        assert np.array_equal(np.isnan(got), np.isnan(p)), (what, w)
        ok = ~np.isnan(p)
        np.testing.assert_allclose(got[ok], p[ok], rtol=1e-12, atol=0, err_msg=str((what, w)))


def _case(g, wins, query, pops, min_sites, delta=False, thr=0.05, noresult=NR, what=""):
    """the engine against the oracle -> the oracle's windows, for the callers' coverage checks"""
    want = _oracle(g, wins, query, pops, min_sites, delta, thr, noresult)
    _check(_paint(g, wins, query, pops, min_sites, delta, thr, noresult), want, noresult, what)
    return want


def _best_sizes(want, pops):
    """sizes of the chosen population over every (window, query) whose tests all ran (every p-value but the chosen
    population's is a number)"""
    out = set()
    for o in want:
        if o is None:
            continue
        a, m, p = o
        for k in range(len(m)):
            best = int(np.argmin(m[k]))
            if not np.isnan(m[k, best]) and np.isnan(p[k]).sum() == 1:
                out.add(len(pops[best]))
    return out


# ---- summation lengths ----------------------------------------------------------------------------------------------
# numpy's pairwise sum: one by one below 8, 8 strided accumulators up to 128, a split at n/2 rounded down to a
# multiple of 8 above; each call's member entries stay within the epilogue's 1024
SUM_GROUPS = [
    [7, 8, 9, 15, 16, 17, 63, 64, 65, 127, 128, 129, 135, 136],
    [137, 255, 256, 257],
    [263, 264, 257, 129, 8, 9, 65],
    [511, 513],
]


@pytest.mark.parametrize("sizes", SUM_GROUPS, ids=lambda s: "M%d" % sum(s))
def test_summation_lengths(sizes):
    rng = np.random.default_rng(sum(sizes))
    S, H, dead = 160, 96, 0
    g, _ = _geno(rng, S, H, 0.05)
    g[:, dead] = -1                                           # called nowhere: nan against every query
    pops = []
    for n in sizes:
        m = [int(x) for x in rng.integers(1, H, n)]
        for k in (0, 7, 8, 15, 16, 63, 64, 127, 128, n // 2, n - 1):   # nans on accumulator-block starts and ends
            if k < n and rng.random() < 0.5:
                m[k] = dead
        pops.append(m)
    rest = 1024 - sum(sizes)
    if rest >= 2:                                             # all nan but one value, somewhere inside the list
        pops.append([dead] * (rest // 3) + [int(rng.integers(1, H))] + [dead] * (rest - rest // 3 - 1))
    query = [int(x) for x in rng.permutation(H)[:40]] + [dead]
    # min_sites just under the window length: nans wherever a pair misses a site or two
    wins = [(0, 18), (18, 37), (40, 60), (61, 80), (80, 99)]
    nan = po.pair_counts(g[0:18])[1][np.ix_(query, [j for m in pops for j in m])] < 17
    assert 0.3 < nan.mean() < 0.8
    _case(g, wins, query, pops, 17, what="nans")
    _case(g, wins, query, pops, 17, delta=True, thr=1e-3, what="nans delta")
    wins = [(0, 3), (3, 8), (10, 27), (30, 70), (70, 110), (120, 160)]
    _case(g, wins, query, pops, 1, what="few nans")


# ---- rank counts past one warp --------------------------------------------------------------------------------------
def test_rank_counts_past_a_warp_with_heavy_ties():
    """windows of 3 to 5 sites leave a handful of distinct distances; the chosen population has 31 to 500 members"""
    rng = np.random.default_rng(31)
    S, H = 60, 120
    g, src = _geno(rng, S, H)
    sizes = [31, 32, 33, 64, 65, 500]
    pops = [[int(x) for x in rng.choice(np.flatnonzero(src == p % 4), n)] for p, n in enumerate(sizes)]
    query = list(range(H))
    wins = [(0, 3), (3, 7), (7, 12), (12, 15), (20, 25), (30, 34)]
    want = _case(g, wins, query, pops, 1, thr=0.05)
    assert {33, 64, 65, 500} <= _best_sizes(want, pops)


def test_complete_separation():
    """512 distances of 0 against 512 of 1: z = -27.7, p = 3.6e-169, deep in normcdf's tail.  CUDA's normcdf meets the
    1e-12 tolerance there: measured on an H100 80GB HBM3, it differs from scipy's ndtr by 8.4e-15 relative at 512 vs 512
    and by at most 8.6e-14 from 8 vs 8 (p = 3.9e-4) to 512 vs 512."""
    rng = np.random.default_rng(5)
    S, H = 40, 64
    base, _ = _geno(rng, S, 1)
    g = np.concatenate([np.repeat(base, 32, axis=1), np.repeat((base + 1) % 4, 32, axis=1)], axis=1).astype(np.int8)
    pops = [[k % 32 for k in range(512)], [32 + k % 32 for k in range(512)]]
    want = _case(g, [(0, 10), (10, 40), (5, 6)], [0, 7, 40, 63], pops, 1)
    p = want[0][2]
    assert np.nanmax(p) < 1e-160
    assert (want[0][0] == [0, 0, 1, 1]).all()


# ---- populations and ordering ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("P, delta", [(1, False), (2, False), (2, True), (3, False), (3, True), (31, False), (31, True),
                                      (32, False), (32, True)])
def test_population_counts(P, delta):
    rng = np.random.default_rng(100 + P)
    S, H = 120, 80
    g, src = _geno(rng, S, H, 0.03)
    pops = [[int(x) for x in rng.choice(np.flatnonzero(src == p % 4), int(rng.integers(1, 14)))] for p in range(P)]
    query = [int(x) for x in rng.permutation(H)[:48]]
    wins = [(0, 5), (5, 25), (25, 65), (70, 74), (80, 120)]
    _case(g, wins, query, pops, 2, delta, 0.01 if delta else 0.05)


@pytest.mark.parametrize("delta", [False, True])
def test_identical_lists_take_the_first(delta):
    """two populations with the same member list have the same mean bit for bit; argmin takes the first, and under the
    delta rule a difference of 0 is not below a threshold of 0"""
    rng = np.random.default_rng(7)
    S, H = 80, 48
    g, src = _geno(rng, S, H, 0.05)
    a = [int(x) for x in rng.choice(np.flatnonzero(src == 0), 9)]
    b = [int(x) for x in rng.choice(np.flatnonzero(src == 1), 6)]
    c = [int(x) for x in rng.choice(np.flatnonzero(src == 2), 12)]
    pops = [b, a, c, list(a), list(b)]
    wins = [(0, 4), (4, 20), (20, 60), (60, 80)]
    want = _case(g, wins, list(range(H)), pops, 1, delta, 0.0 if delta else 0.05)
    best = {int(np.argmin(o[1][k])) for o in want for k in range(H)}
    assert {0, 1} <= best and not {3, 4} & best
    if delta:
        assert {0, 1} <= {int(x) for o in want for x in o[0]}


@pytest.mark.parametrize("where", ["first", "middle", "last"])
@pytest.mark.parametrize("delta", [False, True])
def test_members_called_nowhere(where, delta):
    """a population of members with no call in the window has a nan mean: argmin takes the first nan, and sorted() keeps
    the nans where its comparisons leave them"""
    rng = np.random.default_rng(11)
    S, H, P = 60, 40, 5
    g, src = _geno(rng, S, H, 0.05)
    dead = [H - 3, H - 2, H - 1]
    g[:, dead] = -1
    g[:20, 5] = -1                                            # one more member called only in the later windows
    pops = [[int(x) for x in rng.choice(np.flatnonzero(src[:H - 3] == p % 4), int(rng.integers(2, 8)))]
            for p in range(P)]
    k = {"first": 0, "middle": 2, "last": P - 1}[where]
    pops[k] = list(dead)
    pops[(k + 1) % P].append(dead[0])                         # a nan inside a called population
    pops[(k + 3) % P].insert(0, 5)
    query = list(range(H))
    wins = [(0, 5), (5, 20), (20, 45), (45, 60)]
    _case(g, wins, query, pops, 1, delta, 0.02 if delta else 0.05)
    # the nan population only: the assignment is 0 under both rules wherever every mean is nan
    _case(g, wins, query, [list(dead), list(dead[::-1])], 1, delta, 0.02 if delta else 0.05)


@pytest.mark.parametrize("order", ["ascending", "descending", "interleaved", "descending_then_up", "nan_first"])
def test_delta_sort_orders(order):
    """means in every order count_run sees: a strictly descending run (reversed), a non-descending run, and runs that
    stop after two; population k's members differ from the query at k + 1 of every 10 sites"""
    S, P = 40, 6
    rng = np.random.default_rng(17)
    base, _ = _geno(rng, S, 1)
    alt = np.where(base == 0, 1, 0).astype(np.int8)
    cols = [base[:, 0]]
    for k in range(P):
        for r in range(3):                                    # three members per population, mismatches spread apart
            c = base[:, 0].copy()
            for w0 in range(0, S, 10):
                c[w0 + (np.arange(k + 1) * 3 + r) % 10] = alt[w0 + (np.arange(k + 1) * 3 + r) % 10, 0]
            cols.append(c)
    dead = len(cols)
    cols.append(np.full(S, -1, np.int8))
    g = np.stack(cols, axis=1).astype(np.int8)
    ranked = [[1 + 3 * k + r for r in range(3)] for k in range(P)]
    perm = {"ascending": [0, 1, 2, 3, 4, 5], "descending": [5, 4, 3, 2, 1, 0], "interleaved": [3, 0, 4, 1, 5, 2],
            "descending_then_up": [4, 2, 0, 5, 3, 1], "nan_first": [0, 1, 2, 3, 4, 5]}[order]
    pops = [ranked[k] for k in perm]
    if order == "nan_first":
        pops.insert(0, [dead])
    query = list(range(g.shape[1]))
    wins = [(0, 10), (10, 20), (0, 40)]
    want = _case(g, wins, query, pops, 1, delta=True, thr=0.05)
    if order != "nan_first":
        assert (want[0][0][0] == perm.index(0)) and (want[2][0][0] == perm.index(0))


def test_delta_thresholds():
    """0 (equal means are assigned), exactly the gap between the two lowest means of one query, and a negative one"""
    rng = np.random.default_rng(23)
    S, H, P = 60, 64, 4
    g, src = _geno(rng, S, H, 0.04)
    pops = [[int(x) for x in rng.choice(np.flatnonzero(src == p), 5)] for p in range(P)]
    pops.append(list(pops[2]))
    wins = [(0, 4), (4, 12), (12, 40), (40, 60)]
    query = list(range(H))
    base = _oracle(g, wins, query, pops, 1, True, 0.0)
    gaps = []
    for o in base:
        for k in range(H):
            s = sorted(list(o[1][k]))
            if s[1] - s[0] > 0:
                gaps.append(s[1] - s[0])
    gap = sorted(gaps)[len(gaps) // 2]
    for thr in (0.0, gap, np.nextafter(gap, 1.0), -0.25):
        want = _case(g, wins, query, pops, 1, True, thr, what=thr)
        at_gap = [o[0][k] for o in want for k in range(H) if np.diff(sorted(list(o[1][k]))[:2])[0] == gap]
        assert at_gap and all((a != NR) == (thr <= gap) for a in at_gap), thr


# ---- pair-path layouts ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [127, 128, 129, 255, 256, 257, 385])
@pytest.mark.parametrize("missing", ["genotype", "sample", "sample_broken"])
def test_pair_layouts(H, missing, monkeypatch):
    """queries and members in different pair tiles (reads through the upper triangle), a query list of 4k + 3 with
    repeats, queries that are members, a member with few calls; missing calls per genotype, per sample (the valid plane
    is kept once per sample when H is even) and per sample but for one genotype.  Both plane builders."""
    rng = np.random.default_rng(H)
    S = 90
    g, src = _geno(rng, S, H, 0.06, shared=missing != "genotype")
    if missing == "sample_broken":
        s = int(np.flatnonzero(g[:, 0] >= 0)[3])
        g[s, 0] = -1                                          # haplotype 0 missing where haplotype 1 is called
    sparse = H // 2
    few = rng.random(S) < 0.85                                # a few calls: nan distances, to itself included
    g[few, sparse] = -1
    if missing != "genotype":
        g[few, sparse ^ 1] = -1
    lo_tile, hi_tile = list(range(0, min(H, 40))), list(range(max(0, H - 40), H))
    pops = [[int(x) for x in rng.choice(lo_tile, 7)], [int(x) for x in rng.choice(hi_tile, 9)],
            [int(x) for x in rng.choice(H, 11)] + [sparse], [int(x) for x in rng.choice(lo_tile + hi_tile, 5)]]
    query = [int(x) for x in rng.choice(hi_tile, 9)] + [int(x) for x in rng.choice(lo_tile, 9)] + [sparse, pops[0][0],
                                                                                                    pops[1][0]]
    query += query[:2]                                        # 23 queries, two repeated
    assert len(query) % 4 == 3
    wins = [(0, 6), (6, 30), (30, 70), (70, 90), (10, 50)]
    want = {delta: _oracle(g, wins, query, pops, 3, delta, 0.02 if delta else 0.05) for delta in (False, True)}
    for popc in (False, True):
        if popc:
            monkeypatch.setenv("PG_K2_POPC", "1")
        for delta in (False, True):
            _check(_paint(g, wins, query, pops, 3, delta, 0.02 if delta else 0.05), want[delta], what=(popc, delta))


# ---- batches and statistics -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("delta", [False, True])
def test_batches_and_the_call_without_statistics(delta, monkeypatch):
    """small window batches over empty, single-site, overlapping and identical windows; the command line's call (no
    statistics, a different batch size) gives the same assignments; a non-default noresult"""
    monkeypatch.setenv("PG_PAIR_SCRATCH_MB", "1")
    rng = np.random.default_rng(41)
    S, H, P = 200, 160, 8
    g, src = _geno(rng, S, H, 0.04)
    pops = [[int(x) for x in rng.choice(np.flatnonzero(src == p % 4), int(rng.integers(3, 20)))] for p in range(P)]
    query = list(range(H))
    wins = [(0, 20), (20, 20), (5, 6), (10, 40), (10, 40), (30, 30), (35, 60), (100, 101), (60, 100), (0, 20),
            (199, 200), (150, 190), (140, 140), (160, 200)]
    thr = 0.01 if delta else 0.05
    want = _case(g, wins, query, pops, 2, delta, thr, noresult=-99)
    r = _paint(g, wins, query, pops, 2, delta, thr, noresult=-99, with_stats=False)
    assert set(r) == {"assign"}
    for w, o in enumerate(want):
        assert np.array_equal(r["assign"][w], o[0] if o is not None else np.full(H, -99)), w
    assigned = np.concatenate([o[0] for o in want if o is not None])
    assert (assigned == -99).any() and (assigned >= 0).any()


# ---- min_sites edges ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("min_sites", [1, 12, 13])
@pytest.mark.parametrize("delta", [False, True])
def test_min_sites_edges(min_sites, delta):
    """1; the window length (only pairs called at every site survive); above it (every distance nan: assignment 0)"""
    rng = np.random.default_rng(53)
    S, H, P = 80, 64, 4
    g, src = _geno(rng, S, H, 0.03)
    pops = [[int(x) for x in rng.choice(np.flatnonzero(src == p), 8)] for p in range(P)]
    wins = [(0, 5), (5, 17), (17, 29), (30, 50), (50, 50)]
    want = _case(g, wins, list(range(H)), pops, min_sites, delta, 0.01 if delta else 0.05)
    members = sorted({j for m in pops for j in m})
    for (lo, hi), o in zip(wins, want):
        if o is not None and hi - lo < min_sites:
            assert np.isnan(o[1]).all() and (o[0] == 0).all()
        if o is not None and hi - lo == min_sites:
            n = po.pair_counts(g[lo:hi])[1][:, members]
            assert (n == min_sites).any() and (n < min_sites).any()


# ---- the command line at large populations --------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES8, ids=[c["name"] for c in CASES8])
def test_cli_matches_large_population_fixture(case, tmp_path):
    assert run_cli(case, tmp_path, directory=DIR8) == expected(case, DIR8)
