"""The varied-row stream's one-plane Gram (csrc/k1.cu k1_site_pass_packed<MODE, P, NW, true, true>, gram_counts, imma_u8,
gram_add, gram_flush) at the bounds its own tests do not reach:

  a. the natural fold: with every population of at most 255 haplotypes the Gram folds every glimit = 33,025 rows of a
     segment, and 33,025 rows of k = 255 put 2,147,450,625 in an s32 entry, 33,022 below 2^31 - 1.  On a grid capped at
     one CTA (PG_K1_UNI_CTAS=1) some warp provably holds more than 33,025 rows of one segment
  b. the per-row path's natural 32-bit flush (populations of 10 and 28,000), on the same capped grid
  c. wide rows (up to the longest accepted row) with small populations in the first word, the last K-block, across a
     K-block seam or spread over every K-block, at the width where the stream turns from 12 to 8 consumer warps
  d. count edges: k = 0, 1, N - 1 and N at N = 1, 2, 254 and 255, unequal population sizes in both orders, and
     populations fixed for either allele while others segregate
  e. every Gram instantiation ({POPGEN, POPGEN_FREQ} x padded P {2, 4} x NW {8, 12}) with segment cuts inside 32-row
     blocks, windows with gaps, forced folds, and the collapsed bookkeeping pass of more than 8 populations
  f. 1 to 3 CTAs with segments across CTA seams, and every warps-per-team value the plan takes

Every record field, the popFreq columns included, must be bit-identical to the same stream with the one-plane rows
summed row by row (PG_K1_NO_BYTES=1: varied_mma and add_row, the exact-integer reference of the Gram), the stream with
every varied row on three planes, the packed pass and the byte pass; sites and pos_sum match oracle/dense_oracle.py
exactly and the statistics at check_popgen's tolerances.  Each case asserts through Engine.uniform_launch() that the Gram
kernel it is about ran, on the grid and warps it is about."""
import numpy as np
import pytest

from test_gpu_site_pass_bounds import _hmax, check_popgen, contiguous_pops
from test_gpu_uniform_bits import PAIRS, bits, upload_stale

pytestmark = pytest.mark.gpu

KNOBS = ("PG_K1_BYTE_PASS", "PG_K1_NO_UNIFORM", "PG_K1_UNIFORM_FORCE", "PG_K1_UNI_BITS", "PG_K1_UNI_R", "PG_K1_UNI_GV",
         "PG_K1_UNI_TMAX", "PG_K1_STAGES", "PG_K1_ACC_LIMIT", "PG_K1_NW", "PG_K1_WPT", "PG_K1_NO_BYTES", "PG_K1_UNI_CTAS",
         "PG_K1_G", "PG_K1_I", "PG_K1_TILE_KB", "PG_K1_LANEPOP")
GLIMIT = max((2 ** 32 - 1) // 255 ** 2 // 2, 32)          # the Gram's fold at maxN = 255
PASSES = {"gram": {"PG_K1_UNIFORM_FORCE": "1"},
          "rows": {"PG_K1_UNIFORM_FORCE": "1", "PG_K1_NO_BYTES": "1"},
          "planes": {"PG_K1_UNIFORM_FORCE": "1", "PG_K1_UNI_BITS": "0"},
          "packed": {"PG_K1_NO_UNIFORM": "1"},
          "byte": {"PG_K1_BYTE_PASS": "1"}}


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
        monkeypatch.setenv(k, str(v))


def run(eng, monkeypatch, knobs):
    set_knobs(monkeypatch, knobs)
    out = []
    for freq in (False, True):
        eng.set_freqstats(freq)
        r = eng.popgen(1, 0.01)
        out.append((r, eng.popgen_freqstats() if freq else {}))
    eng.set_freqstats(False)
    return out, eng.uniform_launch()


def compare(eng, monkeypatch, knobs, nw, ctas=None, byte=True):
    """the Gram stream against the four other passes, bit for bit; the Gram kernel ran with nw consumer warps (and ctas
    CTAs), the row-by-row stream with the same grid but not the Gram"""
    names = [n for n in PASSES if byte or n != "byte"]
    res = {}
    for name in names:
        res[name], launch = run(eng, monkeypatch, dict(knobs, **PASSES[name]))
        if name in ("gram", "rows"):
            assert launch[1:] == (nw, int(name == "gram")), (name, knobs, launch)
            assert ctas is None or launch[0] == ctas, (name, knobs, launch)
        elif name != "planes":
            assert launch == (0, 0, 0), (name, launch)
    for name in names[1:]:
        for (ra, fa), (rb, fb) in zip(res["gram"], res[name]):
            for k in ra:
                assert np.array_equal(bits(ra[k]), bits(rb[k])), (name, knobs, k)
            for k in fa:
                assert np.array_equal(bits(fa[k]), bits(fb[k])), (name, knobs, k)


def oracle(eng, monkeypatch, g, hp, P, lo, hi, pos, knobs, what):
    set_knobs(monkeypatch, dict(knobs, **PASSES["gram"]))
    check_popgen(eng, g, hp, P, lo, hi, pos, range(len(lo)), what)
    assert eng.uniform_launch()[2] == 1, what


def load(eng, g, hp, P, lo, hi, pos, stale=False, rng=None):
    if stale:
        upload_stale(eng, rng, g, pos)
    else:
        eng.upload(g, pos)
    eng.set_pops(hp, P)
    eng.set_windows(np.asarray(lo, np.int64), np.asarray(hi, np.int64))


# ---- the stream's block-to-warp assignment, restated -----------------------------------------------------------------
def warp_blocks(eng, lo, hi):
    """per (CTA, warp) of the stream the last popgen call ran: its one-plane blocks in the order it takes them, each as the
    segment index of its rows.  CTA b takes tiles [b nt / B, (b + 1) nt / B); its tile it goes to team it % (NW / wpt), and
    block k of tile t to the team's warp (k + t) % wpt; a block is 32 one-plane rows of the tile, the last one shorter"""
    ctas, nw, _ = eng.uniform_launch()
    wpt = eng.uniform_tile()[1]
    _, _, site_lo, _ = eng.uniform_tiles()
    nt = len(site_lo) - 1
    one = np.flatnonzero(eng.site_classes(0, eng.S) >= 6)
    brk = np.unique(np.concatenate([lo, hi, [0, eng.S]]))
    seg = np.searchsorted(brk, one, side="right") - 1
    first = np.searchsorted(one, site_lo)
    out = {}
    for b in range(ctas):
        t0, t1 = b * nt // ctas, (b + 1) * nt // ctas
        for t in range(t0, t1):
            rows = seg[first[t]:first[t + 1]]
            for k in range(-(-len(rows) // 32)):
                w = ((t - t0) % (nw // wpt)) * wpt + (k + t) % wpt
                out.setdefault((b, w), []).append(rows[32 * k:32 * k + 32])
    return out


def gram_peak(blocks, glimit):
    """the most rows any warp's Gram holds with a fold every glimit rows (gram_add), a segment's rows at a time"""
    peak = 0
    for bl in blocks.values():
        gseg, grows = -1, 0
        for rows in bl:
            for s in np.unique(rows):
                n = int(np.count_nonzero(rows == s))
                if s != gseg:
                    gseg, grows = s, 0
                if grows + n > glimit:
                    grows = 0
                grows += n
                peak = max(peak, grows)
    return peak


def segment_rows(blocks):
    """the most one-plane rows a warp takes in one segment"""
    best = 0
    for bl in blocks.values():
        rows = np.concatenate(bl)
        best = max(best, int(np.bincount(rows).max()))
    return best


# ======================================================================================================================
# a. the natural fold at the s32 bound
# ======================================================================================================================
def fold_rows(rng, S, hp, P, data):
    """complete biallelic rows with k = 255 in every 255-haplotype population (or k in {253, 254, 255}) and the lower
    allele in the other haplotypes: one-plane rows whose Gram entries grow by up to 65,025 a row"""
    H = len(hp)
    pair = rng.integers(0, 6, S)
    a = np.array([p[0] for p in PAIRS], np.int8)[pair]        # a < b: k counts the haplotypes that carry b
    b = np.array([p[1] for p in PAIRS], np.int8)[pair]
    big = np.array([np.count_nonzero(hp == x) == 255 for x in range(P)])
    carrier = big[np.maximum(hp, 0)] & (hp >= 0)
    g = np.where(carrier[None, :], b[:, None], a[:, None]).astype(np.int8)
    if data == "mixed":
        for x in np.flatnonzero(big):
            m = np.flatnonzero(hp == x)
            for _ in range(2):                                    # up to two members back to the lower allele
                pick = rng.random(S) < 0.5
                col = m[rng.integers(0, len(m), S)]
                g[np.flatnonzero(pick), col[pick]] = a[pick]
    assert H == g.shape[1]
    return g


FOLD = [(2, 12, "k255"), (2, 8, "k255"), (2, 12, "mixed"), (2, 8, "mixed"), (4, 12, "k255"), (4, 8, "mixed")]


@pytest.mark.parametrize("P,nw,data", FOLD, ids=["P%d-nw%d-%s" % c for c in FOLD])
def test_natural_fold_at_the_s32_bound(eng, P, nw, data, monkeypatch):
    """one window over every site (one segment) and one CTA: some warp takes more than glimit rows of the segment, so the
    Gram folds at its natural bound; had it folded 32 rows later, some warp's Gram would have held more than glimit rows
    (asserted on the restated assignment), and an entry of 33,026 rows of k = 255 wraps the s32 accumulator.  At P = 2,
    12 warps, k = 255 the case is repeated on tiles of 128 rows with a window edge 2 rows into one warp's 1033rd block,
    so that its Gram reaches 33,024 + 2 rows of one segment: a fold one row later wraps it too"""
    rng = np.random.default_rng(P * 100 + nw + len(data))
    hp = contiguous_pops((255, 1)) if P == 2 else np.concatenate([contiguous_pops((255,) * 4), [-1]]).astype(np.int32)
    S = nw * 33_056 + 4000
    g = fold_rows(rng, S, hp, P, data)
    pos = np.arange(1, S + 1, dtype=np.int32)
    knobs = {"PG_K1_UNI_CTAS": 1, "PG_K1_NW": nw}
    load(eng, g, hp, P, [0], [S], pos)
    oracle(eng, monkeypatch, g, hp, P, [0], [S], pos, knobs, "fold P=%d nw=%d %s" % (P, nw, data))
    blocks = warp_blocks(eng, [0], [S])
    assert eng.uniform_launch() == (1, nw, 1) and len(blocks) == nw
    assert segment_rows(blocks) > GLIMIT
    assert gram_peak(blocks, GLIMIT) <= GLIMIT < gram_peak(blocks, GLIMIT + 32)
    compare(eng, monkeypatch, knobs, nw, 1)
    if (P, nw, data) != (2, 12, "k255"):
        return
    knobs["PG_K1_UNI_R"] = 128                                   # tiles of 4 full blocks: every block holds 32 rows
    set_knobs(monkeypatch, dict(knobs, **PASSES["gram"]))
    eng.popgen(1, 0.01)
    assert eng.uniform_launch() == (1, nw, 1)
    sites0 = warp_sites(eng)[(0, 0)]
    assert len(sites0) > 1033 * 32 and np.all(np.diff(sites0) > 0)
    cut = int(sites0[1032 * 32 + 2])                             # warp 0's 1033rd block: 2 rows before the cut
    lo, hi = [0, 0], [S, cut]
    eng.set_windows(np.array(lo, np.int64), np.array(hi, np.int64))
    oracle(eng, monkeypatch, g, hp, P, lo, hi, pos, knobs, "fold +1")
    blocks = warp_blocks(eng, lo, hi)
    assert gram_peak(blocks, GLIMIT) == GLIMIT - 1 and gram_peak(blocks, GLIMIT + 1) == GLIMIT + 1
    compare(eng, monkeypatch, knobs, nw, 1)


def warp_sites(eng):
    """per (CTA, warp): the sites of its one-plane rows in the order it takes them (warp_blocks with a segment per site)"""
    S = eng.S
    return {k: np.concatenate(v) for k, v in warp_blocks(eng, np.arange(S), np.arange(1, S + 1)).items()}


# ======================================================================================================================
# b. the per-row path's natural flush
# ======================================================================================================================
def test_natural_32bit_flush_on_one_cta(eng, monkeypatch):
    """populations of 10 and 28,000 haplotypes (acc_limit 5, the per-row sums: no Gram above 255) at H = 28,010, on one
    CTA: the restated assignment shows a warp taking acc_limit + 1 blocks of one segment, so add_row flushes its 32-bit
    sums at their natural limit"""
    rng = np.random.default_rng(28010)
    N = (10, 28000)
    hp = contiguous_pops(N)
    H, P, S = len(hp), 2, 1500
    acc_limit = (2 ** 32 - 1) // (max(N) ** 2)
    assert acc_limit == 5
    allele = rng.integers(0, 4, S).astype(np.int8)
    g = np.repeat(allele[:, None], H, axis=1)
    var = np.flatnonzero(rng.random(S) < 0.8)
    alt = ((allele[var] + rng.integers(1, 4, len(var))) % 4).astype(np.int8)
    f = rng.random((len(var), 2)) * 0.9 + 0.05
    g[var] = np.where(rng.random((len(var), H), dtype=np.float32) < f[:, hp], alt[:, None], allele[var][:, None])
    g[var, 0], g[var, -1] = allele[var], alt
    pos = np.arange(1, S + 1, dtype=np.int32)
    lo, hi = [0, 0, 333], [S, S // 2, 1001]
    load(eng, g, hp, P, lo, hi, pos)
    set_knobs(monkeypatch, {"PG_K1_UNI_CTAS": 1})
    check_popgen(eng, g, hp, P, lo, hi, pos, range(len(lo)), "natural flush")
    assert eng.uniform_launch() == (1, 8, 0)
    blocks = warp_blocks(eng, lo, hi)
    run_max = 0
    for bl in blocks.values():
        cur, prev = 0, None
        for rows in bl:
            s = int(rows[0]) if np.all(rows == rows[0]) else None
            cur = cur + 1 if s is not None and s == prev else 1
            prev = s
            run_max = max(run_max, cur)
    assert run_max >= acc_limit + 1, run_max
    res = {}                                                     # the byte pass refuses these rows
    for name in ("rows", "planes", "packed"):
        res[name], _ = run(eng, monkeypatch, dict(PASSES[name], PG_K1_UNI_CTAS=1))
    for name in ("planes", "packed"):
        for (ra, fa), (rb, fb) in zip(res["rows"], res[name]):
            for k in ra:
                assert np.array_equal(bits(ra[k]), bits(rb[k])), (name, k)
            for k in fa:
                assert np.array_equal(bits(fa[k]), bits(fb[k])), (name, k)


# ======================================================================================================================
# c. wide rows with small populations
# ======================================================================================================================
def place(rng, H, P, where):
    """P populations of 4 to 255 haplotypes, the rest unassigned: in word 0, in the last K-block (widened back to 8P
    haplotypes where it holds fewer), across the seam of K-blocks kb and kb + 1 (words 8 kb + 7 and 8 kb + 8), or a few
    haplotypes in every K-block"""
    hp = np.full(H, -1, np.int32)
    wd = (H + 31) // 32
    nkb = (wd + 7) // 8
    if where == "word0":
        cols = np.arange(min(32, H))
    elif where == "last":
        cols = np.arange(min(32 * 8 * (nkb - 1), H - 8 * P), H)
    elif where == "seam":
        kb = nkb // 2 - 1
        cols = np.arange(32 * (8 * kb + 7), min(H, 32 * (8 * kb + 9)))
    else:
        per = max(1, min(3, 255 // nkb // 1))
        cols = np.concatenate([rng.choice(np.arange(256 * k, min(H, 256 * (k + 1))), min(per * P, min(H, 256 * (k + 1)) - 256 * k),
                                          replace=False) for k in range(nkb)])
    cols = rng.permutation(cols)
    keep = cols[:max(P, len(cols) - len(cols) // 8)]            # a few columns of the region stay unassigned
    for i, c in enumerate(keep):
        hp[c] = i % P
    for x in range(P):
        assert 4 <= np.count_nonzero(hp == x) <= 255      # TajD is 0 / 0 at 3 haplotypes: its sign is rounding noise
    return hp


def wide_rows(rng, S, hp, P):
    """uniform rows, complete biallelic rows (one plane), rows fixed in every population but varied among the unassigned
    haplotypes, and three-plane rows"""
    H = len(hp)
    kinds = rng.choice(["u", "b", "f", "t"], S, p=[0.3, 0.45, 0.15, 0.1])
    pair = rng.integers(0, 6, S)
    a = np.array([p[0] for p in PAIRS], np.int8)[pair][:, None]
    b = np.array([p[1] for p in PAIRS], np.int8)[pair][:, None]
    fr = rng.random((S, P + 1)).astype(np.float32)
    fr[kinds == "f", :P] = rng.integers(0, 2, (int(np.count_nonzero(kinds == "f")), P))
    col = np.where(hp >= 0, hp, P)
    g = np.where(rng.random((S, H), dtype=np.float32) < fr[:, col], b, a).astype(np.int8)
    free = np.flatnonzero(hp < 0)
    rows = np.flatnonzero(kinds != "u")
    g[rows, free[0]] = a[rows, 0]
    g[rows, free[-1]] = b[rows, 0]
    u = np.flatnonzero(kinds == "u")
    g[u] = a[u]
    t = np.flatnonzero(kinds == "t")
    third = np.array([({0, 1, 2, 3} - set(p)).pop() for p in PAIRS], np.int8)[pair[t]]
    g[t, rng.integers(0, H, len(t))] = third
    return g


def accepted(eng, hp, P):
    """whether the popgen pass takes rows of len(hp) haplotypes with this layout (the shared memory its mask tables leave
    decides near the longest row)"""
    from genomics_general_b200._lib import PgError
    H = len(hp)
    eng.upload(np.zeros((8, H), np.int8), np.arange(1, 9, dtype=np.int32))
    eng.set_pops(hp, P)
    eng.set_windows(np.array([0], np.int64), np.array([8], np.int64))
    try:
        eng.popgen(1, 0.01)
    except PgError as e:
        assert "too long" in str(e), e
        return False
    return True


WIDE_H = [2688, 2689, 4097, 8192, 16369, "max"]
WHERE = ["word0", "last", "seam", "sparse"]
WIDE = [(h, w, 1 + (i + j) % 4) for i, h in enumerate(WIDE_H) for j, w in enumerate(WHERE)]


@pytest.mark.parametrize("H,where,P", WIDE, ids=["%s-%s-P%d" % c for c in WIDE])
def test_wide_rows_small_populations(eng, H, where, P, monkeypatch):
    """1 to 4 populations of at most 255 haplotypes inside rows of 2,688 to the longest accepted haplotypes: the Gram's K
    loop walks every K-block of the row and the A operand is at its largest; 12 consumer warps up to 2,688 haplotypes
    (packed rows under 1 KiB), 8 from 2,689 on.  "max" is the longest row the site pass takes with the case's layout
    (28,688 haplotypes with word 0's), less where its mask tables leave too little shared memory.  Every other case
    keeps a wider matrix's bytes past H"""
    longest, H = H == "max", _hmax() if H == "max" else H
    while True:                        # "max": the longest row the popgen pass takes with this layout
        rng = np.random.default_rng(H * 8 + P + len(where))
        hp = place(rng, H, P, where)
        if not longest or accepted(eng, hp, P):
            break
        H -= 32
    S = int(np.clip(12_000_000 // H, 400, 3000))
    g = wide_rows(rng, S, hp, P)
    pos = np.cumsum(rng.integers(1, 40, S)).astype(np.int32)
    lo = np.array([0, 0, S // 3, 17, S - 1, 5], np.int64)
    hi = np.array([S, S // 2, 2 * S // 3, 18 + S // 4, S, 5 + S // 5], np.int64)
    load(eng, g, hp, P, lo, hi, pos, stale=(H + len(where)) % 2 == 1, rng=rng)
    nw = 12 if 12 * ((H + 31) // 32) <= 1008 else 8
    assert nw == (12 if H <= 2688 else 8)
    oracle(eng, monkeypatch, g, hp, P, lo, hi, pos, {}, "wide H=%d %s P=%d" % (H, where, P))
    assert eng.uniform_launch()[1:] == (nw, 1)
    compare(eng, monkeypatch, {}, nw, byte=H <= 20000)      # above, the byte pass refuses some layouts the stream runs


# ======================================================================================================================
# d. count edges
# ======================================================================================================================
EDGES = [(255, 1), (1, 255), (7, 200), (200, 7), (2, 254), (254, 255, 1, 2), (1, 2, 254, 255)]


@pytest.mark.parametrize("sizes", EDGES, ids=["-".join(map(str, s)) for s in EDGES])
def test_count_edges(eng, sizes, monkeypatch):
    """k in {0, 1, N - 1, N} per population (so populations fixed for either allele beside segregating ones), at
    N = 1, 2, 254 and 255 and unequal sizes in both orders; popFreq's 0 < k < N test and the N_X S_Y / N_Y S_X terms of
    the cross sums depend on exactly these"""
    rng = np.random.default_rng(sum(sizes) * 7 + len(sizes))
    P = len(sizes)
    hp = np.concatenate([contiguous_pops(sizes, gap=2), [-1, -1, -1]]).astype(np.int32)
    hp = hp[rng.permutation(len(hp))]
    H, S = len(hp), 6000
    kinds = rng.random(S)
    pair = rng.integers(0, 6, S)
    a = np.array([p[0] for p in PAIRS], np.int8)[pair]
    b = np.array([p[1] for p in PAIRS], np.int8)[pair]
    g = np.repeat(a[:, None], H, axis=1)
    for x, n in enumerate(sizes):
        m = np.flatnonzero(hp == x)
        k = np.array([0, 1, n - 1, n])[rng.integers(0, 4, S)]
        rand = rng.random(S) < 0.2
        k[rand] = rng.integers(0, n + 1, int(rand.sum()))
        order = np.argsort(rng.random((S, n)), axis=1)
        take = np.arange(n)[None, :] < k[:, None]
        rows, j = np.nonzero(take)
        g[rows, m[order[rows, j]]] = b[rows]
    free = np.flatnonzero(hp < 0)
    g[:, free[0]], g[:, free[1]] = a, b                          # complete biallelic whatever the populations hold
    g[:, free[2]] = np.where(rng.random(S) < 0.5, a, b)
    g[kinds < 0.2] = a[kinds < 0.2, None]                        # uniform rows
    t = np.flatnonzero((kinds >= 0.2) & (kinds < 0.25))          # three-plane rows
    g[t, free[2]] = np.array([({0, 1, 2, 3} - set(p)).pop() for p in PAIRS], np.int8)[pair[t]]
    pos = np.cumsum(rng.integers(1, 20, S)).astype(np.int32)
    lo = np.array([0, 3, 100, 1000, 2500, S - 40], np.int64)
    hi = np.array([S, 45, 1071, 1033, 6000, S], np.int64)
    load(eng, g, hp, P, lo, hi, pos)
    oracle(eng, monkeypatch, g, hp, P, lo, hi, pos, {}, "edges %s" % (sizes,))
    compare(eng, monkeypatch, {}, 12)


# ======================================================================================================================
# e. the instantiation matrix
# ======================================================================================================================
MATRIX = [(P, nw) for P in (1, 2, 3, 4, 11) for nw in (12, 8)]


@pytest.mark.parametrize("P,nw", MATRIX, ids=["P%d-nw%d" % c for c in MATRIX])
def test_instantiations(eng, P, nw, monkeypatch):
    """{POPGEN, POPGEN_FREQ} (compare runs both) x padded P {2, 4} (P = 1, 3 pad up) x NW {8, 12}, and 11 populations
    (the collapsed bookkeeping pass, one population of their 255 haplotypes): windows that do not start at site 0, with
    gaps between them and cuts inside 32-row blocks, folds forced every 50 rows (PG_K1_ACC_LIMIT=100) and natural"""
    rng = np.random.default_rng(P * 13 + nw)
    H = 300
    if P == 11:
        hp = np.full(H, -1, np.int32)
        hp[rng.choice(H, 255, replace=False)] = np.arange(255) % P
    else:
        hp = np.full(H, -1, np.int32)
        cols = rng.choice(H, min(H - 20, 255 * P), replace=False)
        hp[cols] = np.arange(len(cols)) % P
    S = 9000
    g = wide_rows(rng, S, hp, P) if P <= 4 else wide_rows(rng, S, np.where(hp >= 0, 0, -1), 1)
    pos = np.cumsum(rng.integers(1, 30, S)).astype(np.int32)
    starts = np.sort(rng.choice(np.arange(7, S - 400), 25, replace=False))
    lo = starts.astype(np.int64)
    hi = np.minimum(lo + rng.integers(1, 700, len(lo)), S).astype(np.int64)
    lo, hi = np.concatenate([lo, [13]]), np.concatenate([hi, [S - 9]])
    load(eng, g, hp, P, lo, hi, pos)
    for knobs in ({"PG_K1_NW": nw, "PG_K1_ACC_LIMIT": 100}, {"PG_K1_NW": nw}):
        if P <= 4:
            oracle(eng, monkeypatch, g, hp, P, lo, hi, pos, knobs, "P=%d nw=%d %s" % (P, nw, knobs))
        compare(eng, monkeypatch, knobs, nw)
    if P == 11:
        set_knobs(monkeypatch, dict(PASSES["gram"], PG_K1_NW=nw))
        r = eng.popgen(1, 0.01)
        assert np.array_equal(r["sites"], hi - lo)
        cs = np.concatenate([[0], np.cumsum(pos.astype(np.int64))])
        assert np.array_equal(r["pos_sum"], cs[hi] - cs[lo])


# ======================================================================================================================
# f. grid and team geometry
# ======================================================================================================================
GRID = [(1, 12, 4), (2, 12, 2), (3, 12, 1), (3, 8, 8), (2, 8, 4), (1, 8, 2), (3, 8, 1)]


@pytest.mark.parametrize("ctas,nw,wpt", GRID, ids=["c%d-nw%d-wpt%d" % c for c in GRID])
def test_grid_and_teams(eng, ctas, nw, wpt, monkeypatch):
    """PG_K1_UNI_CTAS of 1, 2 and 3 with windows across the CTAs' tile ranges, and every warps-per-team value the plan
    takes at 12 and 8 consumer warps (PG_K1_WPT)"""
    rng = np.random.default_rng(ctas * 100 + nw * 10 + wpt)
    H, P = 200, 4
    hp = np.full(H, -1, np.int32)
    hp[rng.choice(H, 180, replace=False)] = np.arange(180) % P
    S = 12000
    g = wide_rows(rng, S, hp, P)
    pos = np.cumsum(rng.integers(1, 30, S)).astype(np.int32)
    lo = np.concatenate([np.arange(0, S, 997), [0, S // 3]]).astype(np.int64)
    hi = np.minimum(np.concatenate([np.arange(0, S, 997) + 1500, [S, 2 * S // 3 + 5]]), S).astype(np.int64)
    knobs = {"PG_K1_UNI_CTAS": ctas, "PG_K1_NW": nw, "PG_K1_WPT": wpt}
    load(eng, g, hp, P, lo, hi, pos)
    oracle(eng, monkeypatch, g, hp, P, lo, hi, pos, knobs, "grid %s" % knobs)
    assert eng.uniform_launch() == (ctas, nw, 1) and eng.uniform_tile()[1] == wpt
    _, _, site_lo, _ = eng.uniform_tiles()
    nt = len(site_lo) - 1
    seams = [int(site_lo[b * nt // ctas]) for b in range(1, ctas)]
    assert all(np.any((lo < s) & (hi > s)) for s in seams), seams
    compare(eng, monkeypatch, knobs, nw, ctas)
