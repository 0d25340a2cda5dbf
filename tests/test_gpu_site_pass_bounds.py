"""The site pass (csrc/k1.cu) at the boundaries where its behaviour changes, against oracle/dense_oracle.py:

  1. forced launch geometries (lanes per site, warps per team, sites per lane, ring depth, tile size) for ABBA-BABA, fourPop
     (all three modes) and per-site counts, on interleaved populations, unused columns and a population of > 255 haplotypes
  2. fourPop (all three modes) on tiny windows, windows ending inside a warp's sites and a last partial tile, at 1 and 4
     lanes per site
  3. window bounds on tile and CTA seams, S % T != 0, S < T
  4. the natural flush of the 32-bit popgen sums (acc_limit = (2^32 - 1) / maxN^2) with the large population not first
  5. wide rows (8, 16 and 32 lanes per site) up to the longest row the plan accepts, and the first row it refuses
  6. rows of 4 populations too long for the lane-per-population kernel, which fall back to the general one
  7. the slab seams of pg_site_counts, pg_site_target_freqs and pg_sfs
  8. more than 65535 windows (the grid-stride loop of k1_finalize) for ABBA-BABA and fourPop

Integer outputs (sites, pos_sum, sitesUsed, counts, histograms, first sites) are exact.  fp64 sums of ABBA / fourPop depend on
the summation order, so they are compared with the oracle at rtol 1e-9, and a ratio whose numerator cancels gets an absolute
floor scaled by the magnitude of the summed terms."""
import warnings

import numpy as np
import pytest

from helpers import assert_close
from oracle import dense_oracle as do

pytestmark = pytest.mark.gpu

KNOBS = ("PG_K1_G", "PG_K1_NW", "PG_K1_WPT", "PG_K1_I", "PG_K1_STAGES", "PG_K1_TILE_KB", "PG_K1_ACC_LIMIT", "PG_K1_LANEPOP",
         "PG_K1_NO_BYTES", "PG_COUNTS_NO_GATHER")
TOL = dict(rtol=1e-9, atol=1e-12)
FP_KEYS = do.FOURPOP_KEYS[:14]
FP_F4 = ("fhom", "D", "fd", "fdm")                         # numerator: sum of f4
FP_F4C = ("fhom'", "fd'", "fdm'", "fdh", "fdh2", "fh")       # numerator: sum of f4 + f4 of the complements
FP_MODES = (("default", {}), ("polarize", dict(polarize=True)), ("fixed", dict(fixed=True)))


@pytest.fixture(scope="module")
def eng():
    from genomics_general_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(autouse=True)
def _no_knobs(monkeypatch):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)


def set_knobs(monkeypatch, knobs):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in knobs.items():
        monkeypatch.setenv(k, v)


# ---- the library's geometry, restated --------------------------------------------------------------------------------
def pitch_for(H):
    c = max(1, (H + 15) // 16)
    return (c + 1 if c % 2 == 0 else c) * 16


def nw_default(H):
    """consumer warps per CTA of the general kernel: 12 for rows under 1 KiB, else 8 (k1.cu k1_nw_for)"""
    return 12 if pitch_for(H) < 1024 else 8


def table_bytes(hap_pop, P):
    """shared memory of the mask tables (k1.cu build_tables / table_bytes_of): one entry per chunk a population owns in
    part, or outside its longest run of fully-owned chunks"""
    H = len(hap_pop)
    chunks = pitch_for(H) // 16
    n_ent = 0
    for X in range(P):
        own = np.zeros(chunks * 16, dtype=bool)
        own[:H] = np.asarray(hap_pop) == X
        own = own.reshape(chunks, 16)
        full, anyc = own.all(axis=1), own.any(axis=1)
        best, run = 0, -1
        for c in range(chunks + 1):
            f = c < chunks and full[c]
            if f and run < 0:
                run = c
            if not f and run >= 0:
                best = max(best, c - run)
                run = -1
        n_ent += int(anyc.sum()) - best
    return n_ent * 20 + 64 + 512


def plan(S, hap_pop, P, nw=None, lanes=0):
    from genomics_general_b200.engine import k1_plan
    H = len(hap_pop)
    return k1_plan(S, H, nw=nw or nw_default(H), lanes=lanes, table_bytes=table_bytes(hap_pop, P))


# ---- inputs ----------------------------------------------------------------------------------------------------------
def synth(rng, S, hap_pop, P, all_missing=0.03, variable=0.6):
    """biallelic sites with independent frequencies per population; no partially missing site, so that popgen windows stay
    on the closed-form path; a fraction of sites is missing in every haplotype"""
    hap_pop = np.asarray(hap_pop)
    H = len(hap_pop)
    ref = rng.integers(0, 4, S)
    alt = (ref + rng.integers(1, 4, S)) % 4
    f = (rng.random((S, P + 1)) * (rng.random(S) < variable)[:, None]).astype(np.float32)
    col = np.where(hap_pop >= 0, hap_pop, P)
    g = np.where(rng.random((S, H), dtype=np.float32) < f[:, col], alt[:, None], ref[:, None]).astype(np.int8)
    g[rng.random(S) < all_missing] = -1
    return g


def interleaved_pops(rng, sizes, unused):
    hp = np.concatenate([np.full(n, x) for x, n in enumerate(sizes)] + [np.full(unused, -1)]).astype(np.int32)
    return rng.permutation(hp)


def contiguous_pops(sizes, gap=0):
    parts = []
    for x, n in enumerate(sizes):
        parts += [np.full(n, x), np.full(gap, -1)]
    return np.concatenate(parts).astype(np.int32)


# ---- comparisons with the oracle -------------------------------------------------------------------------------------
def ratio_floor(v, num, num_abs):
    """absolute tolerance of v = num / den when num is a sum of terms of total magnitude num_abs: 1e-9 relative to the
    terms, carried through 1 / den = v / num"""
    if not np.isfinite(v) or num == 0 or not np.isfinite(num):
        return 1e-12
    return max(1e-12, 1e-9 * num_abs * abs(v) / abs(num))


def oracle_abba(g, hp, sel, md, a, b, cache):
    key = ("abba", a, b, sel, md)
    if cache is None or key not in cache:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            want = do.abbababa(g[a:b], hp, *sel, md)
        if cache is None:
            return want
        cache[key] = want
    return cache[key]


def oracle_fourpop(g, hp, sel, md, kw, a, b, cache):
    key = ("fourpop", a, b, sel, md, tuple(sorted(kw)))
    if cache is None or key not in cache:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            want = do.four_pop(g[a:b], hp, *sel, md, **kw)
            p1, p2, p3, p4, _ = do.four_pop_sites(g[a:b], hp, *sel, md, **kw)
            f4, f4c = do._f4(p1, p2, p3, p4), do._f4c(p1, p2, p3, p4)
        sums = [(float(t.sum()), float(np.abs(t).sum())) for t in (f4, f4c)]
        if cache is None:
            return want, sums
        cache[key] = (want, sums)
    return cache[key]


def check_abba(r, g, hp, sel, md, lo, hi, pos, wins, what, cache=None):
    for w in wins:
        a, b = int(lo[w]), int(hi[w])
        assert r["sites"][w] == b - a and r["pos_sum"][w] == int(pos[a:b].sum(dtype=np.int64)), (what, w)
        want = oracle_abba(g, hp, sel, md, a, b, cache)
        tag = "%s w%d [%d,%d)" % (what, w, a, b)
        assert np.array_equal(r["sitesUsed"][w], want["sitesUsed"], equal_nan=True), tag
        assert_close([r["ABBA"][w], r["BABA"][w]], [want["ABBA"], want["BABA"]], tag, **TOL)
        num, num_abs = want["ABBA"] - want["BABA"], want["ABBA"] + want["BABA"]
        for k in ("D", "fd", "fdM"):
            assert_close(r[k][w], want[k], tag + " " + k, rtol=1e-9, atol=ratio_floor(want[k], num, num_abs))


def check_fourpop(r, g, hp, sel, md, kw, lo, hi, pos, wins, what, cache=None):
    for w in wins:
        a, b = int(lo[w]), int(hi[w])
        assert r["sites"][w] == b - a and r["pos_sum"][w] == int(pos[a:b].sum(dtype=np.int64)), (what, w)
        want, sums = oracle_fourpop(g, hp, sel, md, kw, a, b, cache)
        tag = "%s %s w%d [%d,%d)" % (what, kw, w, a, b)
        assert r["sitesUsed"][w] == want["sitesUsed"], tag
        for k in ("ABBA", "BABA", "ABAA", "BAAA"):
            assert_close(r[k][w], want[k], tag + " " + k, **TOL)
        for keys, (num, num_abs) in zip((FP_F4, FP_F4C), sums):
            for k in keys:
                assert_close(r[k][w], want[k], tag + " " + k, rtol=1e-9, atol=ratio_floor(want[k], num, num_abs))


def check_popgen(eng, g, hp, P, lo, hi, pos, wins, what, min_sites=1):
    eng.set_freqstats(True)
    r = eng.popgen(min_sites, 0.01)
    fq = eng.popgen_freqstats()
    eng.set_freqstats(False)
    for w in wins:
        a, b = int(lo[w]), int(hi[w])
        tag = "%s w%d [%d,%d)" % (what, w, a, b)
        assert r["sites"][w] == b - a and r["pos_sum"][w] == int(pos[a:b].sum(dtype=np.int64)), tag
        if b - a < min_sites:
            assert r["path"][w] == 0, tag
            continue
        assert r["path"][w] == 1, tag
        ok, pi, dxy, fst = do.group_dist_stats_closed_form(g[a:b], hp, P, min_sites, 0.01)
        assert ok, tag
        assert_close(r["pi"][w], pi, tag + " pi", **TOL)
        assert_close(r["dxy"][w], dxy, tag + " dxy", **TOL)
        assert_close(r["fst"][w], fst, tag + " fst", rtol=1e-8, atol=1e-12)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            f = do.group_freq_stats(g[a:b], hp, P)
        assert fq["l"][w] == f["l"][0], tag
        for key in ("S", "thetaPi", "thetaW", "TajD"):
            assert_close(fq[key][w], f[key], tag + " " + key, **TOL)
    return r, fq


def load(eng, g, pos, hp, P, lo, hi):
    eng.upload(g, pos)
    eng.set_pops(hp, P)
    eng.set_windows(lo, hi)


def launches(eng, name):
    t = eng.last_timings()
    return t[name]["launches"] if name in t else 0


# ======================================================================================================================
# 1. forced geometries for ABBA, fourPop and counts
# ======================================================================================================================
# knobs -> the geometry they must reach (checked through engine.k1_plan, which reads the same variables)
GEOMETRIES = [
    ({}, {}),
    ({"PG_K1_NW": "8"}, {}),
    ({"PG_K1_G": "2"}, {"lanes_per_site": 2}),
    ({"PG_K1_G": "4", "PG_K1_NW": "8"}, {"lanes_per_site": 4}),
    ({"PG_K1_G": "8", "PG_K1_WPT": "2"}, {"lanes_per_site": 8, "warps_per_tile": 2}),
    ({"PG_K1_STAGES": "2", "PG_K1_WPT": "1"}, {"stages": 2, "warps_per_tile": 1}),      # 12 teams on a 2-stage ring
    ({"PG_K1_I": "2"}, {"sites_per_lane": 2}),
    ({"PG_K1_TILE_KB": "4"}, {"warps_per_tile": 1}),      # 4 KiB tiles: one warp per tile, several lanes per row of 400 B
    ({"PG_K1_LANEPOP": "1"}, {}),
    ({"PG_K1_LANEPOP": "1", "PG_K1_WPT": "1"}, {}),
]


def _shape(name):
    rng = np.random.default_rng({"interleaved": 1, "unused": 2, "pop300": 3}[name])
    if name == "interleaved":       # populations interleaved sample by sample, unused samples among them
        hp = np.repeat(interleaved_pops(rng, (9, 7, 11, 8, 3), 4), 2).astype(np.int32)
        hp[hp == 4] = -1
    elif name == "unused":          # contiguous populations with unused columns between them
        hp = contiguous_pops((40, 33, 70, 50), gap=27)
    else:                           # one population of > 255 haplotypes: 16-bit count fields
        hp = contiguous_pops((20, 300, 17, 24), gap=3)
    return rng, hp


@pytest.mark.parametrize("shape", ["interleaved", "unused", "pop300"])
def test_geometry_matrix_abba_fourpop_counts(eng, shape, monkeypatch):
    rng, hp = _shape(shape)
    P, S = 4, 12000
    g = synth(rng, S, hp, P)
    pos = np.cumsum(rng.integers(1, 40, S)).astype(np.int32)
    lo = np.array([0, 0, 5, 37, 1000, 4000, 4095, 11999, 2500], dtype=np.int64)
    hi = np.array([S, 1, 37, 1000, 1001, 4100, 4097, S, 9000], dtype=np.int64)
    wins = range(len(lo))
    sel, md = (1, 0, 2, 3), 0.5
    counts_want = do.site_counts(g, hp, P)
    cache = {}                                           # the oracle's values do not depend on the geometry
    base = None
    for knobs, geo in GEOMETRIES:
        set_knobs(monkeypatch, knobs)
        nw = int(knobs.get("PG_K1_NW", nw_default(len(hp))))
        p = plan(S, hp, P, nw=nw)
        assert p["ok"], (knobs, p)
        for k, v in geo.items():
            assert p[k] == v, (knobs, k, p)
        if "PG_K1_TILE_KB" in knobs:
            assert p["tile_sites"] * p["pitch"] <= 4096 and (p["lanes_per_site"] > 1) == (p["pitch"] * 32 > 4096), p
        if "PG_K1_STAGES" in knobs:
            assert nw // p["warps_per_tile"] > p["stages"], p           # more teams than ring stages
        load(eng, g, pos, hp, P, lo, hi)
        r = eng.abbababa(*sel, md)
        assert launches(eng, "k1_abba") == 1
        check_abba(r, g, hp, sel, md, lo, hi, pos, wins, str(knobs), cache)
        fps = {}
        for mode, kw in FP_MODES:
            fps[mode] = eng.fourpop(*sel, md, **kw)
            check_fourpop(fps[mode], g, hp, sel, md, kw, lo, hi, pos, wins, str(knobs), cache)
        cnt = eng.site_counts()
        assert launches(eng, "k1_counts") == 1
        assert np.array_equal(cnt.astype(np.int64), counts_want), knobs
        if base is None:         # one geometry, run twice: bit-identical
            base = True
            r2 = eng.abbababa(*sel, md)
            f2 = eng.fourpop(*sel, md)
            for k in ("ABBA", "BABA", "D", "fd", "fdM", "sitesUsed"):
                assert np.array_equal(r[k], r2[k], equal_nan=True), k
            for k in FP_KEYS:
                assert np.array_equal(fps["default"][k], f2[k], equal_nan=True), k


# ======================================================================================================================
# 2. fourPop windows inside a warp's sites
# ======================================================================================================================
@pytest.mark.parametrize("lanes", [1, 4])
def test_fourpop_windows_inside_a_warp_match_the_oracle(eng, lanes, monkeypatch):
    rng = np.random.default_rng(20 + lanes)
    hp = contiguous_pops((11, 13, 9, 12), gap=2)
    P = 4
    S = 10007                                            # a last partial tile
    g = synth(rng, S, hp, P, variable=0.8)
    pos = np.arange(1, S + 1, dtype=np.int32)
    tiny_lo = np.arange(0, 3000, 3, dtype=np.int64)     # 2-site windows: every warp iteration crosses a segment
    lo = np.concatenate([tiny_lo, [3000, 3653, 3653, 8000, 0]]).astype(np.int64)
    hi = np.concatenate([tiny_lo + 2, [3653, 3685, 8000, S, S]]).astype(np.int64)      # ends inside a warp's 32 sites
    wins = list(range(0, len(tiny_lo), 7)) + list(range(len(tiny_lo), len(lo)))
    sel, md = (2, 0, 1, 3), 0.3
    set_knobs(monkeypatch, {"PG_K1_G": str(lanes)} if lanes > 1 else {})
    assert plan(S, hp, P)["lanes_per_site"] == lanes
    load(eng, g, pos, hp, P, lo, hi)
    cache = {}
    for mode, kw in FP_MODES:
        r = eng.fourpop(*sel, md, **kw)
        assert launches(eng, "k1_fourpop") == 1
        check_fourpop(r, g, hp, sel, md, kw, lo, hi, pos, wins, "lanes=%d" % lanes, cache)


# ======================================================================================================================
# 3. tile and CTA seams
# ======================================================================================================================
@pytest.mark.parametrize("case", ["many_ctas", "one_cta"])
def test_tile_and_cta_seams(eng, case, monkeypatch):
    rng = np.random.default_rng(7)
    hp = contiguous_pops((25, 25, 25, 25))
    P, H = 4, 100
    monkeypatch.setenv("PG_K1_NW", "8")                  # the plan below is for 8 consumer warps
    p = plan(10 ** 6, hp, P, nw=8)
    T = p["tile_sites"]
    if case == "many_ctas":
        S = (132 * 2 + 57) * T + 77                      # S % T != 0, tiles not divisible by the CTAs
        p = plan(S, hp, P, nw=8)
        nt, B = (S + T - 1) // T, p["ctas"]
        assert B == 132 and nt % B != 0 and S % T != 0
        starts = [b * nt // B * T for b in (1, 2, 3, 66, 130, 131)]        # first site of CTA b
        edges = sorted(set(starts + [T, 2 * T, 5 * T, (nt - 1) * T]))
    else:
        S = T - 212                                      # fewer sites than one tile: a single CTA
        assert plan(S, hp, P, nw=8)["ctas"] == 1
        edges = [1, 4, 31, 32, 100, S - 1]
    g = synth(rng, S, hp, P)
    pos = np.cumsum(rng.integers(1, 9, S)).astype(np.int32)
    lo, hi = [0, S - 1], [S, S]
    for e in edges:
        lo += [e - 1, e, e - 1, e, max(0, e - T)]
        hi += [e, e + 1, e + 1, min(S, e + T), e]
    lo, hi = np.array(lo, dtype=np.int64), np.array(hi, dtype=np.int64)
    wins = range(len(lo))
    load(eng, g, pos, hp, P, lo, hi)
    check_popgen(eng, g, hp, P, lo, hi, pos, wins, "seams")
    sel, md = (0, 1, 2, 3), 0.2
    check_abba(eng.abbababa(*sel, md), g, hp, sel, md, lo, hi, pos, wins, "seams")
    check_fourpop(eng.fourpop(*sel, md), g, hp, sel, md, {}, lo, hi, pos, wins, "seams")


# ======================================================================================================================
# 4. the natural flush of the 32-bit popgen sums
# ======================================================================================================================
def closed_form(Lp, N, sq, cross):
    """pi, dxy, fst of two populations from exact integer sums (oracle.group_dist_stats_closed_form's expressions)"""
    def pi_of(s, n):
        return ((n * n * Lp - s) / 2.0) / ((n * (n - 1) / 2.0) * Lp)
    pi = [pi_of(sq[0], N[0]), pi_of(sq[1], N[1])]
    dxy = (N[0] * N[1] * Lp - cross) / float(N[0] * N[1] * Lp)
    pi_t = pi_of(sq[0] + sq[1] + 2 * cross, N[0] + N[1])
    w = 1.0 * N[0] / (N[0] + N[1])
    return pi, dxy, 1 - (w * pi[0] + (1 - w) * pi[1]) / pi_t


def test_natural_32bit_flush_with_the_large_population_second(eng):
    rng = np.random.default_rng(11)
    N = (10, 28000)                                      # the large population is not population 0
    hp = contiguous_pops(N)
    H, P, S = len(hp), 2, 24000
    acc_limit = (2 ** 32 - 1) // (max(N) ** 2)
    p = plan(S, hp, P)
    assert p["ok"] and p["lanes_per_site"] == 32 and acc_limit == 5
    per_lane = S * p["lanes_per_site"] // (32 * 8 * 132)              # sites one lane adds on a 132-SM H100 (more on fewer SMs)
    assert per_lane >= 4 * acc_limit
    allele = rng.integers(0, 4, S).astype(np.int8)
    g = np.repeat(allele[:, None], H, axis=1)                        # monomorphic, complete ...
    var = np.sort(rng.choice(S, 400, replace=False))                 # ... except for a sparse set of variable sites
    alt = ((allele[var] + rng.integers(1, 4, len(var))) % 4).astype(np.int8)
    f = rng.random((len(var), 2))
    gv = np.where(rng.random((len(var), H)) < f[:, hp], alt[:, None], allele[var][:, None]).astype(np.int8)
    g[var] = gv
    pos = np.arange(1, S + 1, dtype=np.int32)
    load(eng, g, pos, hp, P, [0, 0], [S, S // 2])
    eng.set_freqstats(True)
    r = eng.popgen(1, 0.01)
    fq = eng.popgen_freqstats()
    eng.set_freqstats(False)
    for w, (a, b) in enumerate(((0, S), (0, S // 2))):
        sub = (var >= a) & (var < b)
        c = do.site_counts(gv[sub], hp, P)                           # [nvar, 2, 4]
        mono = (b - a) - int(sub.sum())
        sq = [mono * n * n + int((c[:, x, :] ** 2).sum()) for x, n in enumerate(N)]
        cross = mono * N[0] * N[1] + int((c[:, 0, :] * c[:, 1, :]).sum())
        pi, dxy, fst = closed_form(b - a, N, sq, cross)
        tag = "window %d" % w
        assert r["path"][w] == 1 and r["sites"][w] == b - a and r["pos_sum"][w] == int(pos[a:b].sum(dtype=np.int64)), tag
        assert_close(r["pi"][w], pi, tag + " pi", **TOL)
        assert_close(r["dxy"][w], [dxy], tag + " dxy", **TOL)
        assert_close(r["fst"][w], [fst], tag + " fst", rtol=1e-8, atol=1e-12)
        f = do.group_freq_stats(gv[sub], hp, P)                      # monomorphic sites add nothing to these
        assert fq["l"][w] == b - a, tag
        for key in ("S", "thetaPi", "thetaW", "TajD"):
            assert_close(fq[key][w], f[key], tag + " " + key, **TOL)


# ======================================================================================================================
# 5. wide rows, the longest accepted row and the first refused one
# ======================================================================================================================
def lanes_for(H):
    """ctx.cu pg_make_k1_plan: lanes per site until one lane walks at most 64 chunks and 32 / G rows fit 64 KiB"""
    G, pitch = 1, pitch_for(H)
    while G < 32 and (pitch // 16 // G > 64 or (32 // G) * pitch > 65536):
        G *= 2
    return G


def wide_layout(H):
    q = H // 4
    return contiguous_pops((q, q, q, H - 3 * q))


def longest_row():
    from genomics_general_b200.engine import k1_plan
    for H in range(29000, 16000, -1):
        hp = wide_layout(H)
        if k1_plan(10 ** 4, H, nw=8, table_bytes=table_bytes(hp, 4))["ok"]:
            return H
    raise AssertionError("no row length accepted")


HMAX = None


def _hmax():
    global HMAX
    if HMAX is None:
        HMAX = longest_row()
    return HMAX


@pytest.mark.parametrize("H", [5008, 8010, 16000, 16368, 16369, 20000, "max"])
def test_wide_rows_match_the_oracle(eng, H):
    H = _hmax() if H == "max" else H
    rng = np.random.default_rng(H)
    hp = wide_layout(H)
    P, S = 4, 1200
    p = plan(S, hp, P)
    assert p["ok"] and p["lanes_per_site"] == lanes_for(H) >= 8 and p["tile_sites"] % 4 == 0
    assert p["lanes_per_site"] == (16 if H in (16000, 16368, 16369) else (32 if H >= 20000 else 8)), p
    g = synth(rng, S, hp, P, variable=0.7)
    pos = np.cumsum(rng.integers(1, 5, S)).astype(np.int32)
    lo = np.array([0, 0, 400, 17], dtype=np.int64)
    hi = np.array([S, 400, S, 18], dtype=np.int64)
    wins = range(len(lo))
    load(eng, g, pos, hp, P, lo, hi)
    check_popgen(eng, g, hp, P, lo, hi, pos, wins, "H=%d" % H)
    sel, md = (0, 2, 1, 3), 0.5
    check_abba(eng.abbababa(*sel, md), g, hp, sel, md, lo, hi, pos, wins, "H=%d" % H)
    check_fourpop(eng.fourpop(*sel, md), g, hp, sel, md, {}, lo, hi, pos, wins, "H=%d" % H)
    assert np.array_equal(eng.site_counts().astype(np.int64), do.site_counts(g, hp, P))


def test_first_row_above_the_limit_is_refused_before_any_launch(eng):
    from genomics_general_b200._lib import PgError
    H = _hmax() + 1
    hp = wide_layout(H)
    assert not plan(64, hp, 4)["ok"]
    g = np.zeros((64, H), dtype=np.int8)
    load(eng, g, np.arange(1, 65, dtype=np.int32), hp, 4, [0], [64])
    n0 = eng.launch_count()
    for call in (lambda: eng.popgen(1, 0.01), lambda: eng.abbababa(0, 1, 2, 3, 0.5), lambda: eng.fourpop(0, 1, 2, 3, 0.5),
                 lambda: eng.site_counts()):
        with pytest.raises(PgError, match="too long"):
            call()
    assert eng.launch_count() == n0


# ======================================================================================================================
# 6. 4 populations on rows too long for the lane-per-population kernel
# ======================================================================================================================
def test_four_small_populations_on_rows_too_long_for_lane_per_population(eng):
    rng = np.random.default_rng(44)
    H, P, S = 14400, 4, 1500
    hp = np.full(H, -1, dtype=np.int32)
    for x in range(P):                                   # <= 255 haplotypes each, the rest of the row unused
        hp[x * 3600 + 5: x * 3600 + 5 + 200 + 10 * x] = x
    assert not plan(S, hp, P, nw=12, lanes=4)["ok"]       # the lane-per-population plan does not fit ...
    assert plan(S, hp, P)["ok"]                           # ... the general one does
    g = synth(rng, S, hp, P, variable=0.7)
    pos = np.arange(1, S + 1, dtype=np.int32)
    lo, hi = np.array([0, 100], dtype=np.int64), np.array([S, 700], dtype=np.int64)
    load(eng, g, pos, hp, P, lo, hi)
    check_popgen(eng, g, hp, P, lo, hi, pos, range(2), "H=14400")
    assert np.array_equal(eng.site_counts().astype(np.int64), do.site_counts(g, hp, P))
    for target in ("derived", "minor"):
        got, tie = eng.site_target_freqs(target)
        want, wtie = do.target_freqs(g, hp, P, target)
        if target == "minor":
            assert np.array_equal(tie, wtie)
            got, want = got[~wtie], want[~wtie]
        assert np.array_equal(got, want, equal_nan=True), target


# ======================================================================================================================
# 7. slab seams
# ======================================================================================================================
def sparse_sites(rng, S, seam, n=3000):
    """sorted distinctive sites: a random sample plus the neighbourhood of the seam and both ends"""
    extra = [0, S - 1] + [seam + d for d in (-2, -1, 0, 1, 2)]
    return np.unique(np.concatenate([rng.choice(S, n, replace=False), extra]))


def test_site_counts_slab_seam_gather(eng):
    P = 64                                               # more than 16 populations: the gather kernel
    slab = (1 << 30) // (P * 4 * 2)
    assert slab == 2097152
    rng = np.random.default_rng(64)
    site0 = 123
    S = site0 + slab + 300
    g = rng.integers(-1, 4, (S, P), dtype=np.int8)
    hp = np.arange(P, dtype=np.int32)                    # one haplotype per population
    eng.upload(g, None)
    eng.set_pops(hp, P)
    got = eng.site_counts(site0, S - site0)
    assert launches(eng, "k1_counts") == 2
    seam = site0 + slab
    assert np.array_equal(got[seam - site0 - 5: seam - site0 + 5].astype(np.int64), do.site_counts(g[seam - 5: seam + 5], hp, P))
    for k in range(0, S - site0, 1 << 18):
        sub, c = g[site0 + k: site0 + k + (1 << 18)], got[k: k + (1 << 18)]
        assert np.array_equal(c.sum(axis=2, dtype=np.int32), (sub >= 0).astype(np.int32)), k      # one-hot or empty ...
        assert np.array_equal(np.where(sub >= 0, c.argmax(axis=2), -1), sub), k                  # ... at the right allele


@pytest.mark.parametrize("P", [8, 20])
def test_target_freqs_slab_seam(eng, P):
    slab = (1 << 28) // (P * 4 * 2)
    assert slab == {8: 4194304, 20: 1677721}[P]
    rng = np.random.default_rng(P)
    S = slab + 500
    hp = np.repeat(np.arange(P, dtype=np.int32), 2)      # two haplotypes per population; the last one is the outgroup
    H = len(hp)
    D = sparse_sites(rng, S, slab)
    ref = rng.integers(0, 4, len(D))
    alt = (ref + rng.integers(1, 4, len(D))) % 4
    gd = np.where(rng.random((len(D), H)) < 0.4, alt[:, None], ref[:, None]).astype(np.int8)
    gd[:, -2:] = np.where(rng.random(len(D)) < 0.8, ref, alt)[:, None]             # a monomorphic outgroup, mostly
    gd[rng.random((len(D), H)) < 0.05] = -1
    g = np.full((S, H), -1, dtype=np.int8)               # every other site is missing everywhere: no target allele
    g[D] = gd
    eng.upload(g, None)
    eng.set_pops(hp, P)
    for target in ("derived", "minor"):
        for as_counts in (False, True):
            got, tie = eng.site_target_freqs(target, as_counts=as_counts)
            assert launches(eng, "k1_target_freqs") >= 2
            want, wtie = do.target_freqs(gd, hp, P, target, as_counts=as_counts)
            assert np.array_equal(tie[D], wtie) and not tie.sum() - wtie.sum()
            keep = ~wtie if target == "minor" else np.ones(len(D), dtype=bool)
            assert np.array_equal(got[D][keep], want[keep], equal_nan=True), (target, as_counts)
            rest = np.ones(S, dtype=bool)
            rest[D] = False
            assert np.all(got[rest] == 0) if as_counts else np.all(np.isnan(got[rest])), (target, as_counts)


def test_sfs_slab_seam_with_site_mask(eng):
    P = 8
    slab = (1 << 28) // (P * 4 * 2)
    rng = np.random.default_rng(88)
    S = slab + 700
    hp = np.repeat(np.arange(P, dtype=np.int32), 2)
    H = len(hp)
    D = sparse_sites(rng, S, slab)
    ref = rng.integers(0, 4, len(D))
    alt = (ref + rng.integers(1, 4, len(D))) % 4
    gd = np.where(rng.random((len(D), H)) < 0.4, alt[:, None], ref[:, None]).astype(np.int8)
    gd[:, -2:] = ref[:, None]                            # the outgroup carries the ancestral allele
    gd[rng.random(len(D)) < 0.1, 3] = -1                 # incomplete in-group sites do not count
    before = D < slab
    gd[before, 1] = ref[before]                          # before the seam population 0 never has 2 derived alleles ...
    at = np.searchsorted(D, slab)
    gd[at, 0:2] = alt[at]                                # ... the first site of the second slab opens that cell
    gd[at, 3] = ref[at]
    g = np.full((S, H), -1, dtype=np.int8)
    g[D] = gd
    mask = (rng.random(S) < 0.7).astype(np.uint8)
    mask[[slab - 1, slab, slab + 1]] = (1, 1, 0)
    eng.upload(g, None)
    eng.set_pops(hp, P)
    groups = [(0,), (1, 2)]
    hists, firsts, n = eng.sfs(7, groups, [2] * P, outgroup=7, site_mask=mask)
    assert launches(eng, "k1_sfs") >= 2
    tc, used = do.sfs_target_counts(gd, hp, 7, outgroup=7)
    used &= mask[D].astype(bool)
    assert n == int(used.sum())
    for grp, h, f in zip(groups, hists, firsts):
        want_h = np.zeros(h.shape, dtype=np.int64)
        want_f = np.full(h.shape, -1, dtype=np.int64)
        for s in np.where(used)[0]:
            cell = tuple(int(tc[s, x]) for x in grp)
            want_h[cell] += 1
            if want_f[cell] < 0:
                want_f[cell] = D[s]                      # absolute site index
        assert np.array_equal(h, want_h), grp
        assert np.array_equal(f, want_f), grp
    assert firsts[0][2] == slab


# ======================================================================================================================
# 8. more than 65535 windows
# ======================================================================================================================
def test_more_than_65535_windows_abba_and_fourpop(eng):
    rng = np.random.default_rng(65536)
    hp = contiguous_pops((6, 7, 5, 6))
    P, S, W = 4, 67000, 66500
    g = synth(rng, S, hp, P, variable=0.8)
    pos = np.arange(1, S + 1, dtype=np.int32)
    lo = np.arange(W, dtype=np.int64)
    hi = lo + 40
    wins = sorted(set(range(0, W, 1499)) | {65534, 65535, 65536, W - 1})
    load(eng, g, pos, hp, P, lo, hi)
    sel, md = (0, 1, 2, 3), 0.5
    r = eng.abbababa(*sel, md)
    check_abba(r, g, hp, sel, md, lo, hi, pos, wins, "W=%d" % W)
    check_fourpop(eng.fourpop(*sel, md), g, hp, sel, md, {}, lo, hi, pos, wins, "W=%d" % W)
