"""The bit-sliced popgen site pass over the packed companion of the resident matrix (csrc/k1.cu k1_site_pass_packed) against
the byte pass (PG_K1_BYTE_PASS): both fold integer sums into the same slots, so every record field (the popFreq columns
included) must be bit-identical.  The cases cover rows around the 32-haplotype words (H = 1, 31, 32, 33, 400, 1600, 3000),
populations that split words, unused and single-haplotype columns, 0 / 2 / 50 % missing genotypes, 1 to 9 populations
(9: the site pass only keeps the books), forced flushes of the 32-bit sums, forced launch geometries and windows across tile
edges with S not a multiple of the tile.

The companion itself must unpack to the resident bytes after every way the matrix is written: upload, upload of a range,
appends (reallocating, and inside the capacity of an earlier, wider matrix), synth_fill and the text ingest."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KNOBS = ("PG_K1_BYTE_PASS", "PG_K1_ACC_LIMIT", "PG_K1_G", "PG_K1_NW", "PG_K1_WPT", "PG_K1_I", "PG_K1_STAGES", "PG_K1_TILE_KB",
         "PG_K1_LANEPOP", "PG_K1_NO_BYTES")


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


def genotypes(rng, S, H, miss):
    """mostly biallelic sites, a few third alleles, `miss` of the genotypes missing and 3 % of the sites missing entirely"""
    ref = rng.integers(0, 4, S)
    alt = (ref + rng.integers(1, 4, S)) % 4
    f = rng.random(S) * (rng.random(S) < 0.7)
    g = np.where(rng.random((S, H)) < f[:, None], alt[:, None], ref[:, None])
    third = rng.random((S, H)) < 0.02
    g[third] = (g[third] + 2) % 4
    g[rng.random((S, H)) < miss] = -1
    g[rng.random(S) < 0.03] = -1
    return g.astype(np.int8)


def layout(rng, H, P):
    """P populations in runs whose edges fall anywhere in a 32-haplotype word, ~10 % of the columns unused, and a few
    haplotypes swapped across the row (populations interleaved, single haplotypes inside another population's run)"""
    cuts = np.sort(rng.choice(np.arange(1, H), P - 1, replace=False)) if P > 1 else np.zeros(0, np.int64)
    hp = np.repeat(np.arange(P), np.diff(np.concatenate([[0], cuts, [H]]))).astype(np.int32)
    for h in rng.permutation(H)[:H // 10]:
        if np.count_nonzero(hp == hp[h]) > 1:
            hp[h] = -1
    for _ in range(H // 16):
        a, b = rng.integers(0, H, 2)
        hp[a], hp[b] = hp[b], hp[a]
    assert all(np.any(hp == x) for x in range(P))
    return hp


def windows(rng, S):
    """random windows, windows around the tile edges of the plans in use (multiples of 4 .. 384 sites), the whole range"""
    lo = rng.integers(0, S, 40)
    hi = np.minimum(lo + rng.integers(1, 900, 40), S)
    edges = [t * k for t in (8, 64, 128, 384) for k in (1, 3, 7) if t * k < S]
    lo = np.concatenate([lo, [e - 1 for e in edges], [0, S - 3]])
    hi = np.concatenate([hi, [e + 1 for e in edges], [S, S]])
    return lo.astype(np.int64), hi.astype(np.int64)


def bits(a):
    a = np.asarray(a)
    return a.view(np.uint64) if a.dtype == np.float64 else a


def both_passes(eng, g, pos, hp, P, lo, hi, knobs, monkeypatch, min_sites=3):
    out = {}
    for byte in (False, True):
        for k in KNOBS:
            monkeypatch.delenv(k, raising=False)
        for k, v in knobs.items():
            monkeypatch.setenv(k, v)
        if byte:
            monkeypatch.setenv("PG_K1_BYTE_PASS", "1")
        eng.upload(g, pos)
        assert eng.packed_rows(0, 1) is not None           # the companion exists: without the hook, the packed pass runs
        eng.set_pops(hp, P)
        eng.set_windows(lo, hi)
        for freq in (False, True):
            eng.set_freqstats(freq)
            r = eng.popgen(min_sites, 0.01)
            assert eng.last_timings()["k1_popgen"]["launches"] == 1
            out[byte, freq] = (r, eng.popgen_freqstats() if freq else {})
        eng.set_freqstats(False)
    for freq in (False, True):
        (a, fa), (b, fb) = out[False, freq], out[True, freq]
        for k in a:
            assert np.array_equal(bits(a[k]), bits(b[k])), (knobs, freq, k)
        for k in fa:
            assert np.array_equal(bits(fa[k]), bits(fb[k])), (knobs, freq, k)
    return out


CASES = [(1, 1, 0.0), (31, 3, 0.02), (31, 9, 0.0), (32, 2, 0.5), (32, 8, 0.02), (33, 5, 0.0), (33, 4, 0.5), (400, 4, 0.0),
         (400, 4, 0.02), (400, 9, 0.02), (400, 1, 0.5), (1600, 8, 0.0), (1600, 8, 0.02), (1600, 3, 0.5), (3000, 4, 0.0)]


@pytest.mark.parametrize("H,P,miss", CASES, ids=lambda v: str(v))
def test_packed_pass_matches_the_byte_pass(eng, H, P, miss, monkeypatch):
    rng = np.random.default_rng(H * 100 + P * 10 + int(miss * 100))
    S = 5003                                              # not a multiple of any tile
    g = genotypes(rng, S, H, miss)
    pos = np.cumsum(rng.integers(1, 50, S)).astype(np.int32)
    hp = layout(rng, H, P)
    lo, hi = windows(rng, S)
    out = both_passes(eng, g, pos, hp, P, lo, hi, {}, monkeypatch)
    r = out[False, False][0]
    assert np.array_equal(r["sites"], hi - lo)
    if miss == 0.0 and P <= 8:
        assert np.count_nonzero(r["path"] == 1) > 0         # windows on the closed-form path: the site pass's sums count


@pytest.mark.parametrize("knobs", [{"PG_K1_ACC_LIMIT": "1"}, {"PG_K1_ACC_LIMIT": "3"}, {"PG_K1_G": "2"},
                                   {"PG_K1_G": "8", "PG_K1_WPT": "2"}, {"PG_K1_NW": "8"}, {"PG_K1_I": "2"},
                                   {"PG_K1_STAGES": "2", "PG_K1_WPT": "1"}, {"PG_K1_TILE_KB": "4"}], ids=str)
def test_packed_pass_geometries_and_flushes(eng, knobs, monkeypatch):
    rng = np.random.default_rng(len(str(knobs)))
    H, P, S = 400, 4, 12007
    g = genotypes(rng, S, H, 0.0)
    pos = np.cumsum(rng.integers(1, 50, S)).astype(np.int32)
    hp = layout(rng, H, P)
    lo, hi = windows(rng, S)
    both_passes(eng, g, pos, hp, P, lo, hi, knobs, monkeypatch)


# ---- the companion ---------------------------------------------------------------------------------------------------
def unpack(rows, H):
    """uint32 [n, 3, wd] -> int8 [n, H] (A0 C1 G2 T3, -1 missing); no bit may be set past H or in a missing haplotype"""
    n, _, wd = rows.shape
    b = np.unpackbits(np.ascontiguousarray(rows).view(np.uint8), bitorder="little").reshape(n, 3, wd * 32)
    assert not b[:, :, H:].any()
    assert not (b[:, 1:, :H] & (1 - b[:, :1, :H])).any()
    code = b[:, 1, :H].astype(np.int8) + 2 * b[:, 2, :H].astype(np.int8)
    return np.where(b[:, 0, :H] == 1, code, -1).astype(np.int8)


def assert_companion(eng, what):
    g, _ = eng.download(0, eng.S, want_pos=False)
    rows = eng.packed_rows(0, eng.S)
    assert rows is not None, what
    assert np.array_equal(unpack(rows, eng.H), g), what


@pytest.mark.parametrize("H", [1, 33, 38, 400])
def test_companion_after_upload_range_and_append(eng, H):
    import ctypes as C
    from genomics_general_b200._lib import check
    rng = np.random.default_rng(H)
    g = genotypes(rng, 700, H, 0.1)
    pos = np.arange(1, 701, dtype=np.int32)
    wide = rng.integers(0, 4, size=(3000, 520)).astype(np.int8)         # no missing genotype: every byte nonzero
    eng.upload(wide, np.arange(1, 3001, dtype=np.int32))
    eng.upload(g[:200], pos[:200])
    assert_companion(eng, "upload")
    part = np.ascontiguousarray(g[150:190][::-1])
    check(eng._lib.pg_upload_range(eng._ctx, 20, 40, C.c_void_p(part.ctypes.data), None), "pg_upload_range")
    got, _ = eng.download(20, 40, want_pos=False)
    assert np.array_equal(got, part)
    assert_companion(eng, "upload_range")
    eng.append_sites(g[200:500], pos[200:500])          # inside the capacity the wider matrix left, past the zeroed slack
    assert_companion(eng, "append inside the capacity")
    eng.append_sites(g[500:], pos[500:])                # reallocates
    assert eng.S == 700
    assert_companion(eng, "append that reallocates")


def test_companion_after_synth_fill_and_text_ingest(eng, tmp_path):
    from genomics_general_b200 import geno_io, synth
    spec = synth.SynthSpec(3, 11, miss=0.05, seed=5)
    eng.synth_fill(spec, 4321)
    assert_companion(eng, "synth_fill")
    S = 2500
    g = synth.synth_genotypes(spec, 0, S)
    p = str(tmp_path / "c.geno")
    synth.write_geno(p, g, synth.synth_positions(S), ["c1"] * S, spec.sample_names(), ploidy=2, fmt="phased")
    geno_io.ingest_geno(eng, p, "phased")
    assert eng.S == S
    assert_companion(eng, "ingest_file")
    geno_io.ingest_geno(eng, open(p, "rb").read(), "phased")
    assert_companion(eng, "ingest_text")
