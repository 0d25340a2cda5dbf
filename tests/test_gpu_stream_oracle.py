"""The popgen stream pass (csrc/k1.cu uniform_prepare, uni_geometry, the k1_uni_* build kernels, k1_site_pass_packed<..., UNI>
with varied_mma, and the per-site prefixes k1_finalize adds) against oracle/dense_oracle.py, on its default path (no
PG_K1_UNIFORM_FORCE unless a case is about forcing):

  1. wide rows (3001 haplotypes up to the longest accepted row), 1 to 4 populations (one-plane rows, MMA K-loops of up to
     113 blocks) and 6 or 8 (three planes only), with the ring geometry each reaches; the engine's R across row widths;
     R = 1 and 2 rows per tile
  2. the largest counts through varied_mma's 16-bit pairs, and the first refused row
  3. the 32-bit flush inside the stream: forced flushes on loads where a warp provably takes one, and the natural limit of
     the widest rows, which the stream does not reach
  4. complete biallelic runs of every allele pair, and the class byte at wide rows
  5. the keep / drop decision at UNI_MIN_FRACTION
  6. window bounds on tile seams, on the seam of a tile's one-plane and three-plane rows and inside a 32-row MMA block,
     empty and nested windows, and more than 65535 windows
  7. positions near 2^31 - 1 across millions of sites
  8. missing data on the forced stream: the path of every window
  9. one engine reused across new data, populations, windows, appends, the popFreq toggle and PG_K1_UNI_BITS
 10. the bench's C2 and C5 shapes

Every case asserts that the stream ran (a silent fall-back to the packed pass over every row fails it), and, where the case
is about it, the one-plane row count, R and the ring.  sites and pos_sum are exact, pi / dxy / fst are compared with the
closed form and the popFreq columns with group_freq_stats at check_popgen's tolerances.  Where it is cheap the same load also
goes through four_passes, so that a failure tells the stream apart from every pass being wrong."""
import warnings

import numpy as np
import pytest

import test_gpu_site_pass_bounds as spb
from helpers import assert_close
from oracle import dense_oracle as do
from test_gpu_site_pass_bounds import (TOL, _hmax, check_popgen, contiguous_pops, interleaved_pops, plan, synth,
                                       wide_layout)
from test_gpu_uniform_bits import (KNOBS, PAIRS, PASSES, bits, four_passes, layout, mixed, run, sites, stream_rows,
                                   upload_stale)

pytestmark = pytest.mark.gpu


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


# ---- the stream's geometry, restated ---------------------------------------------------------------------------------
def _align(x, a):
    return (x + a - 1) // a * a


def packed_pitch(H):
    """bytes of a packed row: three planes of ceil(H / 32) words, padded to 16 bytes"""
    return (12 * ((H + 31) // 32) + 15) // 16 * 16


def stream_R(H):
    """R before uni_geometry's halving: a row per lane of a team of the packed plan (ctx.cu pg_make_k1_plan_rows at the
    packed pitch: lanes per site G, warps per team wpt; 12 consumer warps for rows under 1 KiB, else 8)"""
    pitch = packed_pitch(H)
    G, wpt, wmax = 1, 1, 4 if pitch < 1024 else 8
    while G < 32 and (pitch // 16 // G > 64 or (32 // G) * pitch > 65536):
        G *= 2
    while wpt < wmax and (32 * wpt * 2 // G) * pitch <= 65536:
        wpt *= 2
    while wpt < wmax and (32 * wpt // G) % 4:
        wpt *= 2
    return 32 // G * wpt, 32 // G


def ring_R(eng, words):
    """R of the stream the last popgen call read, solved from uniform_ring() (rows per tile at most, stages, stage bytes):
    with a budget of words a stage holds R + 1 three-plane rows and (R * pitch / 4 - 3) / wd one-plane rows' slots, with a
    budget of rows R of each"""
    cap, stages, sb = eng.uniform_ring()
    wd, pp = (eng.H + 31) // 32, packed_pitch(eng.H)
    for R in range(1, 0x8000):
        w = words and R >= 2
        rows, slots = (R + 1, (R * (pp // 4) - 3) // wd) if w else (R, R)
        if slots == cap and _align(rows * pp + _align(slots * 2, 16), 128) == sb:
            return R
    raise AssertionError(("no R gives this ring", eng.uniform_ring(), eng.H))


def assert_stream(eng, what, name="bits"):
    """the last popgen call read the varied-row stream: every varied site counted, the one-plane rows and words the classes
    give, a ring of at least 2 stages, and tiles that hold no more rows than the ring says; returns uniform_tiles()"""
    used, varied = eng.uniform_stream()
    assert used, (what, "the stream did not run")
    cls = eng.site_classes(0, eng.S)
    assert varied == int(np.count_nonzero((cls == 0) | (cls >= 6))), what
    stream_rows(eng, name)
    cap, stages, sb = eng.uniform_ring()
    assert stages >= 2 and cap >= 1 and sb > 0, (what, eng.uniform_ring())
    tiles = eng.uniform_tiles()
    assert tiles is not None and tiles[0] == cap, what
    site_lo = tiles[2]
    assert site_lo[0] == 0 and site_lo[-1] == eng.S and np.all(np.diff(site_lo) > 0) and np.all(np.diff(site_lo) <= tiles[1])
    return tiles


def freq_used(g, hp, P):
    """group_freq_stats over the haplotypes that belong to a population (the alignment popgenWindows reads)"""
    used = np.asarray(hp) >= 0
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return do.group_freq_stats(g[:, used], np.asarray(hp)[used], P)


def third_alleles(rng, g, frac):
    """a third allele in one haplotype of a share of the complete sites: three-plane rows"""
    H = g.shape[1]
    for s in np.flatnonzero(rng.random(g.shape[0]) < frac):
        if g[s, 0] < 0:
            continue
        absent = sorted(set(range(4)) - set(np.unique(g[s]).tolist()))
        g[s, rng.integers(0, H)] = absent[0]
    return g


def spread_pops(rng, H, P, inter):
    """P populations over H haplotypes with about 5 % unused: contiguous blocks with unused runs between them, or
    interleaved at random"""
    unused = max(1, H // 20)
    q = (H - unused) // P
    sizes = [q] * (P - 1) + [H - unused - q * (P - 1)]
    if inter:
        return interleaved_pops(rng, sizes, unused)
    hp = contiguous_pops(sizes, gap=unused // P)
    return np.concatenate([hp, np.full(H - len(hp), -1)]).astype(np.int32)


def even_pops(H, P):
    q = H // P
    return contiguous_pops([q] * (P - 1) + [H - q * (P - 1)])


LAYOUTS = ("inter", "contig", "even")


def wide_pops(rng, H, P, kind):
    """populations interleaved at random with about 5 % unused (inter), contiguous with unused runs between them (contig),
    or contiguous without unused columns (even).  Interleaved populations take a mask-table entry per 16 haplotypes each
    population touches (48 KiB at most), and near the longest row only the even layout leaves the ring its 2 stages: the
    cases below use each layout where the site pass takes it, and this asserts that it does"""
    hp = even_pops(H, P) if kind == "even" else spread_pops(rng, H, P, kind == "inter")
    assert spb.table_bytes(hp, P) <= 48 * 1024 and plan(64, hp, P)["ok"], (H, P, kind)
    assert np.any(hp < 0) == (kind != "even")
    return hp


def longest_for(P):
    """the longest row the site pass takes with P contiguous populations (_hmax() for P <= 4)"""
    H = _hmax()
    while not plan(64, even_pops(H, P), P)["ok"]:
        H -= 16
    return H


def passes(eng, monkeypatch, knobs=None):
    """four_passes; above 20000 haplotypes the byte pass refuses some layouts the packed passes run (populations of 10 and
    28000 haplotypes), so there the stream is compared with the three-plane stream and the packed pass only"""
    if eng.H <= 20000:
        return four_passes(eng, monkeypatch, knobs)
    res = {}
    for name in ("bits", "planes", "packed"):
        res[name], used = run(eng, monkeypatch, dict(knobs or {}, **PASSES[name]))
        assert used == (name != "packed"), name
    for name in ("planes", "packed"):
        for (ra, fa), (rb, fb) in zip(res["bits"], res[name]):
            for k in ra:
                assert np.array_equal(bits(ra[k]), bits(rb[k])), (name, knobs, k)
            for k in fa:
                assert np.array_equal(bits(fa[k]), bits(fb[k])), (name, knobs, k)


# ======================================================================================================================
# 1. wide rows
# ======================================================================================================================
WIDE = [(3001, 1, "contig", True), (3001, 6, "inter", False), (4096, 2, "inter", True), (4096, 8, "contig", False),
        (5008, 3, "contig", True), (5008, 4, "inter", False), (8010, 2, "inter", True), (8010, 4, "contig", False),
        (8010, 6, "contig", True), (16368, 2, "contig", False), (16368, 8, "contig", True), (16369, 1, "inter", False),
        (16369, 4, "contig", True), (20000, 1, "inter", True), (20000, 6, "contig", False), ("max", 4, "even", True),
        ("max", 2, "even", False), ("max", 8, "even", True), ("max", 1, "even", False), ("max", 3, "even", True)]


@pytest.mark.parametrize("H,P,kind,stale", WIDE, ids=["%s-%d-%s%s" % (h, p, k, "-stale" if t else "") for h, p, k, t in WIDE])
def test_wide_rows(eng, H, P, kind, stale, monkeypatch):
    """2 to 16 lanes per row (2 at 3001 .. 5008 haplotypes, 4 at 8010, 8 at 16368 .. 20000, 16 at the longest row), R = a
    row per lane of a team (32, 16, 8 and 4), one-plane rows on a budget of words and K-loops of up to 113 blocks at
    P <= 4, three planes at P = 6 and 8; every other case keeps a wider matrix's bytes past H"""
    H = longest_for(P) if H == "max" else H
    rng = np.random.default_rng(H * 10 + P)
    hp = wide_pops(rng, H, P, kind)
    S = int(np.clip(30_000_000 // H, 1000, 10000))
    g = third_alleles(rng, synth(rng, S, hp, P, variable=0.8), 0.05)
    pos = np.cumsum(rng.integers(1, 50, S)).astype(np.int32)
    lo = np.array([0, 0, S // 3, S // 2, 17, S - 1, 5], np.int64)
    hi = np.array([S, 1, 2 * S // 3, S, 18, S, 5 + S // 4], np.int64)
    if stale:
        upload_stale(eng, rng, g, pos)
    else:
        eng.upload(g, pos)
    eng.set_pops(hp, P)
    eng.set_windows(lo, hi)
    check_popgen(eng, g, hp, P, lo, hi, pos, range(len(lo)), "H=%d P=%d" % (H, P))
    tiles = assert_stream(eng, "H=%d P=%d" % (H, P))
    R, lanes = stream_R(H)
    assert lanes <= 16 and ring_R(eng, P <= 4) == R, (H, P, eng.uniform_ring(), R)
    assert len(tiles[2]) - 1 >= 40, len(tiles[2])
    if H == _hmax() and P <= 4:
        # the largest B operand (113 K-blocks of 256 bytes) beside the tables still leaves a ring of 2 or more stages
        assert (H + 31) // 32 == 897 and eng.uniform_ring()[1] >= 2
    passes(eng, monkeypatch)


@pytest.mark.parametrize("R", [1, 2])
@pytest.mark.parametrize("H,P", [("max", 4), ("max", 8), (20000, 2)])
def test_one_and_two_rows_per_tile(eng, R, H, P, monkeypatch):
    """R = 1 and 2 rows per tile with the budget of words off and Tmax 2048.  Without PG_K1_UNI_R they are not reached:
    R starts at a row per lane of a team and uni_geometry halves it no lower than a team's lanes (32 / G), and G stays at
    16 or below up to the longest row the plan accepts (asserted here), so R >= 2; the ring at R = lanes x warps per team
    holds 2 stages or more at every accepted row, so R = 2 is not reached either (test_ring_rows_follow_the_plan_across_widths
    checks both against the engine's own ring across row widths)"""
    hm = _hmax()
    assert all(stream_R(h)[1] >= 2 for h in range(1, hm + 1, 31)) and stream_R(hm)[0] == 4
    H = longest_for(P) if H == "max" else H
    rng = np.random.default_rng(H + 7 * R + P)
    hp = wide_pops(rng, H, P, "even" if H > 20000 else "contig")
    S = 900
    g = third_alleles(rng, synth(rng, S, hp, P, variable=0.8), 0.05)
    pos = np.cumsum(rng.integers(1, 50, S)).astype(np.int32)
    lo = np.array([0, 1, 100, 450, S - 2], np.int64)
    hi = np.array([S, 2, 460, S, S], np.int64)
    eng.upload(g, pos)
    eng.set_pops(hp, P)
    eng.set_windows(lo, hi)
    monkeypatch.setenv("PG_K1_UNI_R", str(R))
    monkeypatch.setenv("PG_K1_UNI_TMAX", "2048")
    check_popgen(eng, g, hp, P, lo, hi, pos, range(len(lo)), "R=%d H=%d" % (R, H))
    tiles = assert_stream(eng, "R=%d" % R)
    assert ring_R(eng, False) == R and tiles[0] == R and tiles[1] == 2048, eng.uniform_ring()
    assert np.all(np.diff(tiles[3]) <= R)
    passes(eng, monkeypatch, {"PG_K1_UNI_R": str(R), "PG_K1_UNI_TMAX": "2048"})


def test_ring_rows_follow_the_plan_across_widths(eng):
    """the engine's own R (solved from uniform_ring()) and warps per team (uniform_tile()) against stream_R at row widths
    either side of every change of stream_R up to the longest row, 4 populations: R is a row per lane of a team at every
    one (uni_geometry never halves it), and a team's lanes, R / wpt, are 2 or more, so R = 1 and 2 need PG_K1_UNI_R"""
    hm = _hmax()
    widths, prev = {4, hm}, None
    for h in range(4, hm + 1):
        cur = stream_R(h)
        if cur != prev:
            widths |= {h - 1, h}
        prev = cur
    widths |= set(np.linspace(4, hm, 12).astype(int).tolist())
    rng = np.random.default_rng(5)
    seen = set()
    for H in sorted(w for w in widths if w >= 4):
        g = sites(rng, rng.permutation(["u"] * 32 + ["b"] * 24 + ["t"] * 8), H)
        eng.upload(g, np.arange(1, 65, dtype=np.int32))
        eng.set_pops(even_pops(H, 4), 4)
        eng.set_windows(np.array([0], np.int64), np.array([64], np.int64))
        eng.popgen(1, 0.01)
        assert_stream(eng, "H=%d" % H)
        R, wpt = ring_R(eng, True), eng.uniform_tile()[1]
        assert (R, R // wpt) == stream_R(H) and R % wpt == 0 and R // wpt >= 2, (H, R, wpt, stream_R(H))
        seen.add(R)
    assert seen == {128, 64, 32, 16, 8, 4}, seen


# ======================================================================================================================
# 2. the largest counts through the 16-bit pairs
# ======================================================================================================================
@pytest.mark.parametrize("P", [1, 2])
def test_largest_counts_through_16bit_pairs(eng, P, monkeypatch):
    """varied_mma hands a lane two populations' counts as 16-bit halves of a word.  On the longest accepted row: P = 1 with
    every member carrying the higher code (k = N = H - 3, the 3 unused columns carrying the lower one), exactly one, all
    but one; P = 2 of 10 and H - 10 haplotypes with either population all on the higher code and the other all on the
    lower, and so on.  No row longer than the one accepted can be set up, so no count reaches 65536."""
    from genomics_general_b200.engine import k1_plan
    H = _hmax()
    assert H < 65536 and not plan(64, wide_layout(H + 1), 4)["ok"]
    assert not k1_plan(64, H + 1, nw=8, table_bytes=576)["ok"]      # not even with the smallest tables (one population)
    rng = np.random.default_rng(P)
    if P == 1:
        hp = np.zeros(H, np.int32)
        hp[-3:] = -1
    else:
        hp = contiguous_pops((10, H - 10))
    members = [np.flatnonzero(hp == x) for x in range(P)]
    S = 640
    g = np.empty((S, H), np.int8)
    for s in range(S):
        a, b = PAIRS[s % 6]
        row = np.full(H, a, np.int8)
        kind = (s // 6) % 6
        if kind == 5 or s % 4 == 3:                       # uniform rows, for the stream's share
            row[:] = b if s % 2 else a
        elif P == 1:
            m = members[0]
            if kind == 0:
                row[m] = b                                # k = N
            elif kind == 1:
                row[m[rng.integers(0, len(m))]] = b       # k = 1
            elif kind == 2:
                row[m] = b
                row[m[rng.integers(0, len(m))]] = a       # k = N - 1
            else:
                row[rng.random(H) < rng.random()] = b
                row[[0, 1]] = a, b
        else:
            if kind == 0:
                row[members[1]] = b                       # k = (0, N1)
            elif kind == 1:
                row[members[0]] = b                       # k = (N0, 0)
            elif kind == 2:
                row[members[0]] = b
                row[members[1]] = b
                row[members[1][rng.integers(0, H - 10)]] = a      # k = (N0, N1 - 1)
            elif kind == 3:
                row[members[1][rng.integers(0, H - 10)]] = b      # exactly one member
            else:
                row[rng.random(H) < rng.random()] = b
                row[[0, 1]] = a, b
        g[s] = row
    pos = np.arange(1, S + 1, dtype=np.int32)
    lo = np.array([0, 0, S // 2, 32, 95], np.int64)
    hi = np.array([S, S // 2, S, 64, 97], np.int64)
    eng.upload(g, pos)
    eng.set_pops(hp, P)
    eng.set_windows(lo, hi)
    check_popgen(eng, g, hp, P, lo, hi, pos, range(len(lo)), "P=%d" % P)
    assert_stream(eng, "P=%d" % P)
    assert eng.uniform_rows()[0] > 300
    passes(eng, monkeypatch)


# ======================================================================================================================
# 3. the 32-bit flush inside the stream
# ======================================================================================================================
def test_natural_32bit_limit_on_the_stream(eng, monkeypatch):
    """populations of 10 and 28000 haplotypes, the large one second (acc_limit 5), on a row of 28010 haplotypes that the
    stream carries as one plane: the stream matches the oracle at the natural limit, but does not flush there.  A warp
    flushes after acc_limit + 1 of its row blocks in one segment, and at this width a tile holds one 32-row block (R = 4
    on a budget of words), so every warp of every CTA (132 x 8 on an H100) would need 6 tiles of its own in a segment:
    about 200,000 varied rows, 6 billion genotypes.  The forced flushes are in test_forced_32bit_flush_in_the_stream;
    test_gpu_gram_bounds.py::test_natural_32bit_flush_on_one_cta reaches the natural flush on a stream capped at one CTA
    (PG_K1_UNI_CTAS=1)."""
    spb.test_natural_32bit_flush_with_the_large_population_second(eng)
    assert_stream(eng, "natural limit")
    assert ring_R(eng, True) == stream_R(28010)[0] == 4 and eng.uniform_rows()[0] > 300
    passes(eng, monkeypatch)


def warp_blocks(eng, H, P, gv):
    """per tile of the stream the last popgen call read: (first site, end site, row blocks a team's warps share out), with
    one-plane rows in blocks of 32 and three-plane rows in blocks of 32 / Gv (Gv lanes per row); and the warps per team"""
    _, _, site_lo, _ = eng.uniform_tiles()
    R, lanes = stream_R(H)
    cls = eng.site_classes(0, eng.S)
    spv = 32 // gv if gv else lanes
    out = []
    for a, b in zip(site_lo[:-1], site_lo[1:]):
        c = cls[a:b]
        n1 = int(np.count_nonzero(c >= 6)) if P <= 4 else 0
        n3 = int(np.count_nonzero((c == 0) | (c >= 6))) - n1
        out.append((int(a), int(b), -(-n1 // 32) + -(-n3 // spv)))
    return out, R // lanes


@pytest.mark.parametrize("acc", [1, 2])
@pytest.mark.parametrize("H,P,kind", [(20000, 2, "three"), (16369, 8, "three"), (400, 4, "one")])
def test_forced_32bit_flush_in_the_stream(eng, H, P, kind, acc, monkeypatch):
    """PG_K1_ACC_LIMIT = 1 and 2 on loads where the stream provably flushes: some tile lies inside one segment and holds at
    least wpt x (acc + 1) row blocks, which its team's wpt warps take in turn, so each of them adds acc + 1 blocks to the
    same sums and flushes them before the last (add_row's acc_limit step).  On wide rows the tiles are three-plane rows,
    one row per block (PG_K1_UNI_GV=32), populations of 10 and H - 10 or 8 populations; on a short row they are 32-row MMA
    blocks of one-plane rows (up to 13 of them in a tile at R = 128)."""
    rng = np.random.default_rng(H + acc)
    if kind == "three":
        hp = contiguous_pops((10, H - 10)) if P == 2 else wide_pops(rng, H, P, "contig")
        S = 24_000_000 // H
        g = synth(rng, S, hp, P, variable=0.75, all_missing=0.0)
        var = np.flatnonzero(np.any(g != g[:, :1], axis=1))
        g[var] = third_alleles(rng, g[var], 1.0)               # every varied row on three planes
        knobs = {"PG_K1_ACC_LIMIT": str(acc), "PG_K1_UNI_GV": "32"}
    else:
        hp = wide_pops(rng, H, P, "contig")
        S = 20000
        g = synth(rng, S, hp, P, variable=0.5, all_missing=0.02)
        knobs = {"PG_K1_ACC_LIMIT": str(acc)}
    pos = np.cumsum(rng.integers(1, 30, S)).astype(np.int32)
    lo = np.array([0, 0, S // 3, S - 7], np.int64)
    hi = np.array([S, S // 2, S, S], np.int64)
    eng.upload(g, pos)
    eng.set_pops(hp, P)
    eng.set_windows(lo, hi)
    for k, v in knobs.items():
        monkeypatch.setenv(k, v)
    check_popgen(eng, g, hp, P, lo, hi, pos, range(len(lo)), "acc=%d H=%d" % (acc, H))
    assert_stream(eng, "acc=%d" % acc)
    blocks, wpt = warp_blocks(eng, H, P, 32 if kind == "three" else 0)
    seams = np.unique(np.concatenate([lo, hi]))
    inside = [n for a, b, n in blocks if not np.any((seams > a) & (seams < b))]
    assert max(inside) >= wpt * (acc + 1), (max(inside), wpt, acc)
    passes(eng, monkeypatch, knobs)


# ======================================================================================================================
# 4. each allele pair
# ======================================================================================================================
def classes_vec(g):
    """the class byte of each row (test_gpu_uniform_bits.classes_np), vectorised for wide rows"""
    H = g.shape[1]
    called = (g >= 0).sum(axis=1)
    present = np.stack([(g == a).any(axis=1) for a in range(4)], axis=1)
    n_al = present.sum(axis=1)
    hi_bit = (present[:, 0] | present[:, 1]) & (present[:, 2] | present[:, 3])
    out = np.zeros(g.shape[0], np.uint8)
    out[called == 0] = 5
    one = (called == H) & (n_al == 1)
    out[one] = 1 + np.argmax(present[one], axis=1)
    out[(called == H) & (n_al == 2)] = np.where(hi_bit, 7, 6)[(called == H) & (n_al == 2)]
    return out


@pytest.mark.parametrize("H,P", [(5008, 4), (8010, 3), ("max", 2)])
def test_each_allele_pair(eng, H, P, monkeypatch):
    """runs of 96 complete biallelic sites (three MMA blocks) of each pair: {A,G}, {A,T}, {C,G} and {C,T} differ in the
    high code bit (PG_CLS_VARIED2_B1, plane B1), {A,C} and {G,T} in the low one only (PG_CLS_VARIED2, plane B0)"""
    H = _hmax() if H == "max" else H
    rng = np.random.default_rng(H + P)
    kinds = []
    for k in list(rng.permutation(6)) * 2:
        kinds += ["b%d" % k] * 96 + ["u"] * 40
    g = sites(rng, kinds, H)
    S = len(kinds)
    hp = wide_pops(rng, H, P, "even" if H > 20000 else "inter")
    pos = np.cumsum(rng.integers(1, 9, S)).astype(np.int32)
    lo = np.array([0, 0, 136, 500, 1000], np.int64)
    hi = np.array([S, 232, 272, 1100, S], np.int64)
    eng.upload(g, pos)
    eng.set_pops(hp, P)
    eng.set_windows(lo, hi)
    cls = eng.site_classes(0, S)
    want = classes_vec(g)
    assert np.array_equal(cls, want)
    for k, (a, b) in enumerate(PAIRS):
        rows = np.array([x == "b%d" % k for x in kinds])
        assert np.all(cls[rows] == (7 if (a ^ b) & 2 else 6)), (a, b)
    check_popgen(eng, g, hp, P, lo, hi, pos, range(len(lo)), "pairs H=%d" % H)
    assert_stream(eng, "pairs")
    assert eng.uniform_rows()[0] == 12 * 96
    passes(eng, monkeypatch)


# ======================================================================================================================
# 5. the keep / drop threshold
# ======================================================================================================================
@pytest.mark.parametrize("S", [4000, 4003])
@pytest.mark.parametrize("d", [-1, 0, 1])
def test_keep_drop_threshold(eng, S, d, monkeypatch):
    """ceil(S / 8) - 1, ceil(S / 8) and ceil(S / 8) + 1 sites that are not varied (a fifth of them missing in every
    haplotype, which counts as not varied): the stream is kept exactly when S - varied >= S / 8"""
    rng = np.random.default_rng(S * 3 + d)
    H, P = 120, 4
    u = -(-S // 8) + d
    kinds = np.array(["u"] * (u - u // 5) + ["m"] * (u // 5) + list(rng.choice(["b", "t"], S - u, p=[0.8, 0.2])))
    g = sites(rng, rng.permutation(kinds), H)
    hp = layout(rng, H, P, False)
    pos = np.cumsum(rng.integers(1, 9, S)).astype(np.int32)
    lo = np.array([0, 0, S // 3, S - 1, 7], np.int64)
    hi = np.array([S, S // 2, S, S, 7 + S // 8], np.int64)
    eng.upload(g, pos)
    eng.set_pops(hp, P)
    eng.set_windows(lo, hi)
    check_popgen(eng, g, hp, P, lo, hi, pos, range(len(lo)), "S=%d u=%d" % (S, u))
    used, varied = eng.uniform_stream()
    assert varied == S - u
    assert used == (S - varied >= S / 8), (S, u, used)
    if used:
        assert_stream(eng, "S=%d u=%d" % (S, u))
    else:
        assert eng.uniform_ring() == (0, 0, 0) and eng.uniform_rows() == (0, 0) and eng.uniform_tiles() is None


# ======================================================================================================================
# 6. window bounds on the stream's seams
# ======================================================================================================================
def test_window_bounds_on_stream_seams(eng):
    """window starts and ends on tile seams and a site either side, on the seam of a tile's one-plane and three-plane rows
    (its last one-plane site and first three-plane site), ending inside and at the edges of the tile's first 32-row MMA
    blocks; empty and nested windows.  New windows over the same data leave the tiles as they were."""
    rng = np.random.default_rng(66)
    H, P, S = 160, 4, 30000
    g = mixed(rng, S, H, (0.45, 0.03, 0.42, 0.1, 0.0))
    hp = layout(rng, H, P, True)
    pos = np.cumsum(rng.integers(1, 30, S)).astype(np.int32)
    eng.upload(g, pos)
    eng.set_pops(hp, P)
    eng.set_windows(np.array([0], np.int64), np.array([S], np.int64))
    check_popgen(eng, g, hp, P, [0], [S], pos, [0], "seams: whole")
    cap, Tmax, site_lo, row0 = assert_stream(eng, "seams")
    cls = eng.site_classes(0, S)
    nt = len(site_lo) - 1
    assert nt > 40
    lo, hi = [], []

    def win(a, b):
        a, b = max(0, min(S, a)), max(0, min(S, b))
        lo.append(min(a, b))
        hi.append(max(a, b))

    picked = sorted(set([1, 2, 3, nt // 2, nt // 2 + 1, nt - 2, nt - 1]))
    for t in picked:
        e = int(site_lo[t])
        for a, b in ((e - 1, e + 1), (e, e + 1), (e - 1, e), (e, e), (e - 5, e), (e, e + 5), (e - 1, e + 2)):
            win(a, b)
    for t in picked[:-1]:
        a, b = int(site_lo[t]), int(site_lo[t + 1])
        c = cls[a:b]
        one, three = a + np.flatnonzero(c >= 6), a + np.flatnonzero(c == 0)
        if len(one) and len(three):
            for s in (int(one[-1]), int(three[0])):          # the last one-plane site, the first three-plane one
                win(a, s)
                win(a, s + 1)
                win(s, b)
                win(s + 1, b)
        for k in (15, 16, 31, 32, 33, 63, 64):                # inside and at the edges of the tile's MMA blocks
            if k < len(one):
                win(a, int(one[k]))
                win(a, int(one[k]) + 1)
                win(int(one[k]), b)
        win(a, b)                                             # nested windows
        win(a + 1, b - 1)
        win(a + 2, b - 3)
        win(a - 3, b + 3)
    lo, hi = np.array(lo, np.int64), np.array(hi, np.int64)
    assert np.count_nonzero(lo == hi) >= len(picked)
    eng.set_windows(lo, hi)
    check_popgen(eng, g, hp, P, lo, hi, pos, range(len(lo)), "seams")
    cap2, Tmax2, site_lo2, row02 = assert_stream(eng, "seams")
    assert (cap2, Tmax2) == (cap, Tmax) and np.array_equal(site_lo2, site_lo) and np.array_equal(row02, row0)


def test_more_than_65535_windows_on_the_stream(eng):
    """70000 windows (some empty) over 3000 sites: k1_finalize's grid-stride loop and the prefixes it reads"""
    rng = np.random.default_rng(65537)
    H, P, S, W = 64, 2, 3000, 70000
    g = mixed(rng, S, H, (0.5, 0.05, 0.35, 0.1, 0.0))
    hp = layout(rng, H, P, True)
    pos = np.cumsum(rng.integers(1, 30, S)).astype(np.int32)
    lo = rng.integers(0, S, W).astype(np.int64)
    hi = np.minimum(lo + rng.integers(0, 40, W), S).astype(np.int64)
    wins = sorted(set(range(0, W, 997)) | {65534, 65535, 65536, W - 1} | set(np.flatnonzero(lo == hi)[:5].tolist()))
    eng.upload(g, pos)
    eng.set_pops(hp, P)
    eng.set_windows(lo, hi)
    r, _ = check_popgen(eng, g, hp, P, lo, hi, pos, wins, "W=%d" % W)
    assert_stream(eng, "W=%d" % W)
    assert np.array_equal(r["sites"], hi - lo)
    cs = np.concatenate([[0], np.cumsum(pos.astype(np.int64))])
    assert np.array_equal(r["pos_sum"], cs[hi] - cs[lo])


# ======================================================================================================================
# 7. positions near the int32 limit
# ======================================================================================================================
def test_positions_near_the_int32_limit(eng):
    """3 million sites at positions up to 2^31 - 1: the per-site position prefix (Widen) and pos_sum overflow 32 bits
    within a few sites"""
    rng = np.random.default_rng(31)
    S, H, P = 3_000_000, 12, 2
    base = rng.integers(0, 4, S).astype(np.int8)
    g = np.repeat(base[:, None], H, axis=1)
    var = np.flatnonzero(rng.random(S) < 0.45)
    alt = ((base[var] + rng.integers(1, 4, len(var))) % 4).astype(np.int8)
    g[var] = np.where(rng.random((len(var), H)) < 0.4, alt[:, None], base[var][:, None])
    g[rng.random(S) < 0.01] = -1
    pos = (np.int64(2 ** 31 - 1) - np.arange(S, dtype=np.int64)[::-1]).astype(np.int32)
    assert pos[-1] == 2 ** 31 - 1 and pos[0] > 2 ** 31 - 1 - S
    hp = np.array([0] * 5 + [-1] + [1] * 6, np.int32)
    lo = np.array([0, 0, S - 1, S // 3, 1_234_567], np.int64)
    hi = np.array([S, S // 2, S, S, 1_234_568], np.int64)
    eng.upload(g, pos)
    eng.set_pops(hp, P)
    eng.set_windows(lo, hi)
    r, _ = check_popgen(eng, g, hp, P, lo, hi, pos, range(len(lo)), "int32 positions")
    assert_stream(eng, "int32 positions")
    assert r["pos_sum"][0] == int(pos.astype(np.int64).sum()) > 2 ** 52


# ======================================================================================================================
# 8. missing data on the forced stream
# ======================================================================================================================
def test_missing_data_paths(eng, monkeypatch):
    """ragged sites (some but not all used haplotypes missing), sites missing everywhere, missing in the unused columns
    only and in the used ones only, on the stream forced whatever its uniform share: a window with a ragged site takes the
    pairwise path (path 2, checked with group_dist_stats), one without takes the closed form (path 1), an empty one path
    0.  The popFreq columns count only the sites complete in every used haplotype, on every path."""
    monkeypatch.setenv("PG_K1_UNIFORM_FORCE", "1")
    rng = np.random.default_rng(8)
    hp = contiguous_pops((40, 50, 45), gap=5)
    H, P, S = len(hp), 3, 6000
    used = hp >= 0
    g = mixed(rng, S, H, (0.3, 0.05, 0.5, 0.15, 0.0))
    ragged = rng.choice(S, 25, replace=False)
    for s in ragged:
        g[s, rng.choice(np.flatnonzero(used), 1 + rng.integers(0, 5))] = -1
    unused_only = rng.choice(np.setdiff1d(np.arange(S), ragged), 40, replace=False)
    g[unused_only[:, None], np.flatnonzero(~used)[None, :]] = -1
    used_only = rng.choice(np.setdiff1d(np.arange(S), np.concatenate([ragged, unused_only])), 40, replace=False)
    g[used_only[:, None], np.flatnonzero(used)[None, :]] = -1
    pos = np.cumsum(rng.integers(1, 30, S)).astype(np.int32)
    lo = list(range(0, S, 100)) + [0] + [int(s) for s in ragged[:5]] + [int(s) for s in unused_only[:5]] + \
        [int(s) for s in used_only[:5]] + [int(unused_only[0]) - 3, 10]
    hi = [min(S, a + 100) for a in range(0, S, 100)] + [S] + [int(s) + 1 for s in ragged[:5]] + \
        [int(s) + 1 for s in unused_only[:5]] + [int(s) + 1 for s in used_only[:5]] + [int(unused_only[0]) + 4, 10]
    lo, hi = np.array(lo, np.int64), np.array(hi, np.int64)
    eng.upload(g, pos)
    eng.set_pops(hp, P)
    eng.set_windows(lo, hi)
    eng.set_freqstats(True)
    r = eng.popgen(1, 0.01)
    fq = eng.popgen_freqstats()
    eng.set_freqstats(False)
    assert_stream(eng, "missing")
    nval = (g[:, used] >= 0).sum(axis=1)
    is_ragged = (nval > 0) & (nval < used.sum())
    paths = set()
    for w in range(len(lo)):
        a, b = int(lo[w]), int(hi[w])
        tag = "w%d [%d,%d)" % (w, a, b)
        assert r["sites"][w] == b - a and r["pos_sum"][w] == int(pos[a:b].sum(dtype=np.int64)), tag
        want_path = 0 if b == a else (2 if is_ragged[a:b].any() else 1)
        assert r["path"][w] == want_path, (tag, r["path"][w], want_path)
        paths.add(want_path)
        if want_path == 0:
            continue
        if want_path == 1:
            ok, pi, dxy, fst = do.group_dist_stats_closed_form(g[a:b], hp, P, 1, 0.01)
            assert ok, tag
        else:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                pi, dxy, fst = do.group_dist_stats(g[a:b], hp, P, 1, 0.01)
        assert_close(r["pi"][w], pi, tag + " pi", **TOL)
        assert_close(r["dxy"][w], dxy, tag + " dxy", **TOL)
        assert_close(r["fst"][w], fst, tag + " fst", rtol=1e-8, atol=1e-12)
        f = freq_used(g[a:b], hp, P)
        assert fq["l"][w] == f["l"][0], tag
        for key in ("S", "thetaPi", "thetaW", "TajD"):
            assert_close(fq[key][w], f[key], tag + " " + key, **TOL)
    assert paths == {0, 1, 2}
    passes(eng, monkeypatch)


# ======================================================================================================================
# 9. one engine reused
# ======================================================================================================================
def test_reuse_of_one_engine(eng, monkeypatch):
    """one engine through new data, populations 4 -> 8 -> 3 -> 4 (the one-plane rows off and on again), new windows, an
    append, a new matrix of the same shape with another uniform share, the popFreq toggle and PG_K1_UNI_BITS=0 and back.
    After each step: the oracle, and the stream, its rows, ring and tiles and every record field as a new engine, created
    for the comparison and loaded with the same state, has them"""
    from genomics_general_b200.engine import Engine
    rng = np.random.default_rng(99)
    H, S0, S1 = 300, 8000, 2500
    st = {}

    def compare(what, name="bits"):
        g, pos, hp, P, lo, hi = st["g"], st["pos"], st["hp"], st["P"], st["lo"], st["hi"]
        r, fq = check_popgen(eng, g, hp, P, lo, hi, pos, range(len(lo)), what)
        tiles = assert_stream(eng, what, name)
        with Engine(0) as new:
            new.upload(g, pos)
            new.set_pops(hp, P)
            new.set_windows(lo, hi)
            new.set_freqstats(True)
            r2 = new.popgen(1, 0.01)
            fq2 = new.popgen_freqstats()
            assert eng.uniform_stream() == new.uniform_stream(), what
            assert eng.uniform_rows() == new.uniform_rows() and eng.uniform_ring() == new.uniform_ring(), what
            t2 = new.uniform_tiles()
        assert tiles[:2] == t2[:2] and np.array_equal(tiles[2], t2[2]) and np.array_equal(tiles[3], t2[3]), what
        for k in ("pi", "dxy", "fst", "sites", "pos_sum", "path"):
            assert np.array_equal(r[k], r2[k], equal_nan=True), (what, k)
        for k in fq:
            assert np.array_equal(fq[k], fq2[k], equal_nan=True), (what, k)
        return r

    g = mixed(rng, S0 + S1, H, (0.5, 0.03, 0.35, 0.12, 0.0))
    pos = np.cumsum(rng.integers(1, 30, S0 + S1)).astype(np.int32)
    st.update(g=g[:S0], pos=pos[:S0], hp=layout(rng, H, 4, False), P=4)
    st.update(lo=np.array([0, 100, 4000, 7999], np.int64), hi=np.array([S0, 3000, 7000, S0], np.int64))
    eng.upload(st["g"], st["pos"])
    eng.set_pops(st["hp"], 4)
    eng.set_windows(st["lo"], st["hi"])
    compare("1 upload")
    for P, inter in ((8, True), (3, True), (4, True)):
        st.update(hp=layout(rng, H, P, inter), P=P)
        eng.set_pops(st["hp"], P)
        compare("2 set_pops %d" % P)
    lo = rng.integers(0, S0, 30).astype(np.int64)
    st.update(lo=lo, hi=np.minimum(lo + rng.integers(0, 2000, 30), S0).astype(np.int64))
    eng.set_windows(st["lo"], st["hi"])
    compare("3 set_windows")
    eng.append_sites(g[S0:], pos[S0:])
    st.update(g=g, pos=pos, lo=np.array([0, S0 - 5, 9000], np.int64), hi=np.array([S0 + S1, S0 + 5, S0 + S1], np.int64))
    eng.set_windows(st["lo"], st["hi"])
    compare("4 append_sites")
    g2 = mixed(rng, S0 + S1, H, (0.2, 0.0, 0.7, 0.1, 0.0))
    st.update(g=g2)
    eng.upload(g2, pos)
    eng.set_pops(st["hp"], st["P"])
    eng.set_windows(st["lo"], st["hi"])
    r_on = compare("5 a new matrix")
    r_off = eng.popgen(1, 0.01)                           # 6: popFreq off after on, then on again
    for k in ("pi", "dxy", "fst", "sites", "pos_sum", "path"):
        assert np.array_equal(r_on[k], r_off[k], equal_nan=True), k
    assert_stream(eng, "6 popFreq off")
    compare("6 popFreq on again")
    assert eng.uniform_rows()[0] > 0
    monkeypatch.setenv("PG_K1_UNI_BITS", "0")
    compare("7 PG_K1_UNI_BITS=0", "planes")
    assert eng.uniform_rows()[0] == 0
    monkeypatch.delenv("PG_K1_UNI_BITS")
    compare("7 cleared")
    assert eng.uniform_rows()[0] > 0


# ======================================================================================================================
# 10. the bench's C2 and C5 shapes
# ======================================================================================================================
@pytest.mark.parametrize("case", ["C2", "C5"])
def test_bench_shapes(eng, case):
    """C2: 4 populations x 50 diploid samples (H = 400), 50,000 bp windows (about 5,000 sites), -m 100, and windows of
    50,000 sites; C5: 8 x 100 (H = 1600), 5,000-site windows.  The synthetic matrix is filled on the device, and a sample
    of windows is checked against the oracle on the numpy twin of the generator"""
    from genomics_general_b200 import synth as gsynth
    from genomics_general_b200 import windows as gwin
    if case == "C2":
        spec, S = gsynth.SynthSpec(4, 50, 2, seed=20260923), 2_000_000
    else:
        spec, S = gsynth.SynthSpec(8, 100, 2, seed=20260928), 1_000_000
    eng.synth_fill(spec, S)
    _, pos = eng.download(0, S, want_geno=False)
    hp, P = spec.hap_pop(), spec.n_pops
    eng.set_pops(hp, P)
    if case == "C2":
        lo, hi = gwin.sliding_coord_windows(np.zeros(S, dtype=np.int32), ["chr1"], pos, 50000).ranges()
        lo, hi = np.asarray(lo, np.int64), np.asarray(hi, np.int64)
        lo, hi = np.concatenate([lo, [0, 1_234_567]]), np.concatenate([hi, [50_000, 1_284_567]])
    else:
        lo = np.arange(0, S, 5000, dtype=np.int64)
        hi = np.minimum(lo + 5000, S)
    W = len(lo)
    eng.set_windows(lo, hi)
    eng.set_freqstats(True)
    r = eng.popgen(100, 0.01)
    fq = eng.popgen_freqstats()
    eng.set_freqstats(False)
    assert_stream(eng, case)
    assert ring_R(eng, P <= 4) == stream_R(spec.n_haps)[0]
    assert np.all(r["path"][hi - lo >= 100] == 1)
    for w in sorted(set([0, 1, W // 2, W - 3, W - 2, W - 1]) | set(rng_pick(W))):
        a, b = int(lo[w]), int(hi[w])
        tag = "%s w%d [%d,%d)" % (case, w, a, b)
        g = gsynth.synth_genotypes(spec, a, b - a)
        assert r["sites"][w] == b - a and r["pos_sum"][w] == int(pos[a:b].sum(dtype=np.int64)), tag
        if b - a < 100:
            assert r["path"][w] == 0, tag
            continue
        ok, pi, dxy, fst = do.group_dist_stats_closed_form(g, hp, P, 100, 0.01)
        assert ok and r["path"][w] == 1, tag
        assert_close(r["pi"][w], pi, tag + " pi", **TOL)
        assert_close(r["dxy"][w], dxy, tag + " dxy", **TOL)
        assert_close(r["fst"][w], fst, tag + " fst", rtol=1e-8, atol=1e-12)
        f = freq_used(g, hp, P)
        assert fq["l"][w] == f["l"][0], tag
        for key in ("S", "thetaPi", "thetaW", "TajD"):
            assert_close(fq[key][w], f[key], tag + " " + key, **TOL)


def rng_pick(W, n=6):
    return np.random.default_rng(W).choice(W, min(n, W), replace=False).tolist()
