"""The packed popgen site pass with uniform sites elided (csrc/k1.cu uniform_prepare, k1_site_pass_packed<..., UNI>): a site whose
H haplotypes all carry one allele, or are all missing, is not streamed, and its counts follow from the population sizes.
Every record field (the popFreq columns included) must be bit-identical to the packed pass that streams every row
(PG_K1_NO_UNIFORM) and to the byte pass (PG_K1_BYTE_PASS).  The cases cover uniform fractions from 0 to 100 %, uniform-missing
sites, rows around the 32-haplotype words, unused columns (a site that varies only in a haplotype of no population is not
uniform), 1 to 9 populations, windows across tile edges, forced flushes and geometries, missing data with the stream forced
on (PG_K1_UNIFORM_FORCE), the rebuild after every way the matrix is written, and which data select the stream."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KNOBS = ("PG_K1_BYTE_PASS", "PG_K1_NO_UNIFORM", "PG_K1_UNIFORM_FORCE", "PG_K1_ACC_LIMIT", "PG_K1_G", "PG_K1_NW", "PG_K1_WPT",
         "PG_K1_I", "PG_K1_STAGES", "PG_K1_TILE_KB", "PG_K1_LANEPOP", "PG_K1_NO_BYTES")
PASSES = {"uniform": {}, "packed": {"PG_K1_NO_UNIFORM": "1"}, "byte": {"PG_K1_BYTE_PASS": "1"}}


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


def genotypes(rng, S, H, uniform, miss=0.0):
    """a `uniform` share of the sites carries one allele in every haplotype (a tenth of those: every haplotype missing);
    every other site has at least two alleles (H > 1), `miss` of their genotypes missing"""
    ref = rng.integers(0, 4, S)
    alt = (ref + rng.integers(1, 4, S)) % 4
    f = rng.random(S) * 0.5
    g = np.where(rng.random((S, H)) < f[:, None], alt[:, None], ref[:, None])
    g[rng.random((S, H)) < miss] = -1
    idx = np.arange(S)
    g[idx, idx % H] = alt                                  # not uniform
    uni = rng.random(S) < uniform
    g[uni] = ref[uni, None]
    g[uni & (rng.random(S) < 0.1)] = -1
    return g.astype(np.int8), uni


def layout(rng, H, P):
    """P populations in runs whose edges fall anywhere in a word, ~10 % of the columns unused, a few haplotypes swapped"""
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
    lo = rng.integers(0, S, 40)
    hi = np.minimum(lo + rng.integers(1, 900, 40), S)
    edges = [t * k for t in (8, 64, 128, 384, 512) for k in (1, 3, 7) if t * k < S]
    lo = np.concatenate([lo, [e - 1 for e in edges], [0, S - 3]])
    hi = np.concatenate([hi, [e + 1 for e in edges], [S, S]])
    return lo.astype(np.int64), hi.astype(np.int64)


def bits(a):
    a = np.asarray(a)
    return a.view(np.uint64) if a.dtype == np.float64 else a


def set_knobs(monkeypatch, knobs):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in knobs.items():
        monkeypatch.setenv(k, v)


def run(eng, monkeypatch, knobs, min_sites=3):
    """popgen records without and with the popFreq counters under `knobs`, and whether the stream was read"""
    set_knobs(monkeypatch, knobs)
    out = {}
    for freq in (False, True):
        eng.set_freqstats(freq)
        r = eng.popgen(min_sites, 0.01)
        assert eng.last_timings()["k1_popgen"]["launches"] == 1
        out[freq] = (r, eng.popgen_freqstats() if freq else {})
    eng.set_freqstats(False)
    return out, eng.uniform_stream()[0]


def assert_same(a, b, what):
    for freq in (False, True):
        (ra, fa), (rb, fb) = a[freq], b[freq]
        for k in ra:
            assert np.array_equal(bits(ra[k]), bits(rb[k])), (what, freq, k)
        for k in fa:
            assert np.array_equal(bits(fa[k]), bits(fb[k])), (what, freq, k)


def three_passes(eng, monkeypatch, knobs=None, force=True, expect_stream=True):
    knobs = dict(knobs or {})
    uk = dict(knobs, PG_K1_UNIFORM_FORCE="1") if force else knobs
    u, used = run(eng, monkeypatch, uk)
    assert used == expect_stream, knobs
    p, used_p = run(eng, monkeypatch, dict(knobs, PG_K1_NO_UNIFORM="1"))
    assert not used_p
    b, _ = run(eng, monkeypatch, dict(knobs, PG_K1_BYTE_PASS="1"))
    assert_same(u, p, ("uniform vs packed", knobs))
    assert_same(u, b, ("uniform vs byte", knobs))
    return u


def load(eng, rng, S, H, P, uniform, miss=0.0):
    g, uni = genotypes(rng, S, H, uniform, miss)
    pos = np.cumsum(rng.integers(1, 50, S)).astype(np.int32)
    eng.upload(g, pos)
    hp = layout(rng, H, P)
    eng.set_pops(hp, P)
    lo, hi = windows(rng, S)
    eng.set_windows(lo, hi)
    return g, pos, hp, lo, hi


@pytest.mark.parametrize("uniform", [0.0, 0.3, 0.7, 0.99, 1.0])
def test_uniform_fractions(eng, uniform, monkeypatch):
    rng = np.random.default_rng(int(uniform * 100) + 7)
    S, H, P = 5003, 400, 4
    _, _, _, lo, hi = load(eng, rng, S, H, P, uniform)
    out = three_passes(eng, monkeypatch)
    _, varied = eng.uniform_stream()
    assert abs((S - varied) / S - uniform) < 0.03
    # chosen from the observed fraction alone
    _, used = run(eng, monkeypatch, {})
    assert used == ((S - varied) >= S / 8)
    r = out[False][0]
    assert np.array_equal(r["sites"], hi - lo)
    if uniform < 1.0:
        assert np.count_nonzero(r["path"] == 1) > 0


CASES = [(1, 1, 0.5), (31, 3, 0.7), (31, 9, 0.7), (32, 2, 0.3), (32, 8, 0.7), (33, 5, 0.99), (33, 4, 0.7), (400, 1, 0.7),
         (400, 6, 0.7), (400, 9, 0.5), (1600, 8, 0.7), (1600, 3, 0.3)]


@pytest.mark.parametrize("H,P,uniform", CASES, ids=lambda v: str(v))
def test_shapes_and_populations(eng, H, P, uniform, monkeypatch):
    rng = np.random.default_rng(H * 100 + P * 10 + int(uniform * 10))
    load(eng, rng, 5003, H, P, uniform)                   # S not a multiple of any tile
    three_passes(eng, monkeypatch)


def test_variation_only_in_unused_columns(eng, monkeypatch):
    """a site that differs only in a haplotype of no population is varied (the class is over all H haplotypes) and is
    walked; the populations see it as uniform"""
    rng = np.random.default_rng(3)
    S, H, P = 3001, 96, 3
    hp = np.repeat(np.arange(P), H // P).astype(np.int32)
    hp[[5, 40, 95]] = -1
    g = np.repeat(rng.integers(0, 4, S)[:, None], H, axis=1).astype(np.int8)
    odd = rng.random(S) < 0.5
    g[odd, 40] = (g[odd, 40] + 1) % 4
    g[rng.random(S) < 0.2, 95] = -1
    eng.upload(g, np.arange(1, S + 1, dtype=np.int32))
    eng.set_pops(hp, P)
    lo, hi = windows(rng, S)
    eng.set_windows(lo, hi)
    three_passes(eng, monkeypatch, force=False)
    _, varied = eng.uniform_stream()
    assert varied == np.count_nonzero(np.any(g != g[:, :1], axis=1))


@pytest.mark.parametrize("knobs", [{"PG_K1_ACC_LIMIT": "1"}, {"PG_K1_ACC_LIMIT": "3"}, {"PG_K1_G": "2"},
                                   {"PG_K1_G": "8", "PG_K1_WPT": "2"}, {"PG_K1_NW": "8"}, {"PG_K1_I": "2"},
                                   {"PG_K1_STAGES": "2", "PG_K1_WPT": "1"}, {"PG_K1_TILE_KB": "4"}], ids=str)
def test_geometries_and_flushes(eng, knobs, monkeypatch):
    rng = np.random.default_rng(len(str(knobs)))
    load(eng, rng, 12007, 400, 4, 0.7)
    three_passes(eng, monkeypatch, knobs)


@pytest.mark.parametrize("H,P", [(400, 4), (33, 2), (1600, 8)])
def test_missing_data_with_the_stream_forced(eng, H, P, monkeypatch):
    rng = np.random.default_rng(H + P)
    load(eng, rng, 5003, H, P, 0.3, miss=0.02)
    three_passes(eng, monkeypatch)


# ---- rebuilds -------------------------------------------------------------------------------------------------------
def stream_matches(eng, monkeypatch, what, rebuilt=True):
    """the next popgen call rebuilds the stream (or, on unchanged data, adds no launch) and agrees with the packed pass"""
    set_knobs(monkeypatch, {"PG_K1_UNIFORM_FORCE": "1"})
    r = eng.popgen(3, 0.01)
    t = eng.last_timings()
    assert ("k1_uniform" in t) == rebuilt, what
    assert eng.uniform_stream()[0], what
    set_knobs(monkeypatch, {"PG_K1_NO_UNIFORM": "1"})
    p = eng.popgen(3, 0.01)
    for k in r:
        assert np.array_equal(bits(r[k]), bits(p[k])), (what, k)
    set_knobs(monkeypatch, {"PG_K1_UNIFORM_FORCE": "1"})


def test_rebuild_after_every_write(eng, monkeypatch, tmp_path):
    from genomics_general_b200 import geno_io, synth
    from genomics_general_b200._lib import check
    rng = np.random.default_rng(11)
    H, P = 100, 3
    g, uni = genotypes(rng, 900, H, 0.7)
    pos = np.arange(1, 901, dtype=np.int32)
    hp = layout(rng, H, P)
    wide = rng.integers(0, 4, size=(3000, 520)).astype(np.int8)
    eng.upload(wide, np.arange(1, 3001, dtype=np.int32))     # leaves capacity for the appends below

    def windows_all():
        lo = np.arange(0, eng.S, 37, dtype=np.int64)
        eng.set_windows(lo, np.minimum(lo + 50, eng.S))

    eng.upload(g[:300], pos[:300])
    eng.set_pops(hp, P)
    windows_all()
    stream_matches(eng, monkeypatch, "upload")
    stream_matches(eng, monkeypatch, "unchanged", rebuilt=False)
    # a range that turns uniform sites into varied ones, then back
    s0 = int(np.flatnonzero(uni[:300])[0])
    part = g[s0:s0 + 40].copy()
    part[:, 7] = (np.maximum(part[:, 7], 0) + 1) % 4
    check(eng._lib.pg_upload_range(eng._ctx, s0, 40, C.c_void_p(part.ctypes.data), None), "pg_upload_range")
    stream_matches(eng, monkeypatch, "upload_range: uniform -> varied")
    back = np.ascontiguousarray(g[s0:s0 + 40])
    check(eng._lib.pg_upload_range(eng._ctx, s0, 40, C.c_void_p(back.ctypes.data), None), "pg_upload_range")
    stream_matches(eng, monkeypatch, "upload_range: varied -> uniform")
    eng.append_sites(g[300:600], pos[300:600])                # inside the capacity
    windows_all()
    stream_matches(eng, monkeypatch, "append inside the capacity")
    eng.append_sites(g[600:], pos[600:])                      # reallocates
    assert eng.S == 900
    windows_all()
    stream_matches(eng, monkeypatch, "append that reallocates")
    spec = synth.SynthSpec(3, 20, miss=0.0, seed=5)
    eng.synth_fill(spec, 4321)
    eng.set_pops(spec.hap_pop(), 3)
    windows_all()
    stream_matches(eng, monkeypatch, "synth_fill")
    S = 2500
    gs = synth.synth_genotypes(spec, 0, S)
    p = str(tmp_path / "c.geno")
    synth.write_geno(p, gs, synth.synth_positions(S), ["c1"] * S, spec.sample_names(), ploidy=2, fmt="phased")
    geno_io.ingest_geno(eng, p, "phased")
    eng.set_pops(spec.hap_pop(), 3)
    windows_all()
    stream_matches(eng, monkeypatch, "ingest_file")
    geno_io.ingest_geno(eng, open(p, "rb").read(), "phased")
    eng.set_pops(spec.hap_pop(), 3)
    windows_all()
    stream_matches(eng, monkeypatch, "ingest_text")


def test_selection_follows_the_uniform_fraction(eng):
    """C2-like data (70 % of the sites uniform) take the stream; 2 % missing genotypes (almost no uniform site) do not"""
    from genomics_general_b200 import synth
    S = 200_000
    for miss, want in ((0.0, True), (0.02, False)):
        spec = synth.SynthSpec(4, 50, seed=9, miss=miss)
        eng.synth_fill(spec, S)
        eng.set_pops(spec.hap_pop(), 4)
        lo = np.arange(0, S, 5000, dtype=np.int64)
        eng.set_windows(lo, np.minimum(lo + 5000, S))
        eng.popgen(1, 0.01)
        used, varied = eng.uniform_stream()
        assert used == want, (miss, varied)
        if want:
            assert 0.6 < (S - varied) / S < 0.8
        else:
            assert (S - varied) / S < 0.05
