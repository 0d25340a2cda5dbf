"""GPU parity tests, second batch (pytest -m gpu): sampleHet, H12stats, freq.py --target columns and the masked
indPairDists through the C-ABI, against fixtures produced by the unmodified reference (oracle/make_golden2.py) and
against the oracle on seeded inputs.  Integer-derived outputs bit-exact; doubles at 1e-9 (contract 1e-6)."""
import hashlib
import json
import os

import numpy as np
import pytest

from helpers import GOLDEN, assert_close

pytestmark = pytest.mark.gpu

META = json.load(open(os.path.join(GOLDEN, "window_cases2.json")))
ARR = np.load(os.path.join(GOLDEN, "window_cases2.npz"))
IDS = [m["name"] for m in META]
CLI2 = json.load(open(os.path.join(GOLDEN, "cli_cases2.json")))
TOL = dict(rtol=1e-9, atol=1e-12)


@pytest.fixture(scope="module")
def eng():
    from genomics_general_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _load(eng, m, key="__g_aln"):
    g = ARR[m["name"] + key]
    hp = ARR[m["name"] + "__hap_pop"]
    L = g.shape[0]
    eng.upload(g, np.arange(1, L + 1, dtype=np.int32))
    eng.set_pops(hp, len(m["pop_names"]))
    eng.set_windows([0], [L])
    return g, hp, L


def _hap_ind(m):
    idx = {n: k for k, n in enumerate(m["sample_names"])}
    return np.array([idx[s] for s in m["hap_samples"]], dtype=np.int32)


@pytest.mark.parametrize("m", META, ids=IDS)
def test_ind_het_golden(eng, m):
    from oracle import dense_oracle as do
    g, hp, L = _load(eng, m)
    hi = _hap_ind(m)
    n = len(m["sample_names"])
    for key, masked in (("alone", 0), ("after_popDist", m["minSites"]), ("after_indPairDist", 0)):
        got = eng.ind_het(hi, n, min_sites=masked)[0]
        assert_close(got, do.sample_het(g, hi, n, masked_min_sites=masked or None), "oracle " + key, **TOL)
        if m["sampleHet"]:
            want = np.array([m["sampleHet"][key][s] for s in m["sample_names"]])
            assert_close(got, want, key, **TOL)


@pytest.mark.parametrize("m", META, ids=IDS)
def test_hapstats_golden(eng, m):
    g, hp, L = _load(eng, m)
    for key, want in m["H12stats"].items():
        state, md = key.rsplit("_", 1)
        masked = m["minSites"] if state == "after_popDist" else 0
        got = eng.hapstats(float(md), min_sites=masked, diag_nan=(state != "alone"))[0]
        for x, pn in enumerate(m["pop_names"]):
            assert_close(got[x], [want["H1_" + pn], want["H12_" + pn], want["H2_" + pn]], key + " " + pn, **TOL)


@pytest.mark.parametrize("m", META, ids=IDS)
def test_pairdist_masked_matches_oracle(eng, m):
    from oracle import dense_oracle as do
    g, hp, L = _load(eng, m)
    hi = _hap_ind(m)
    n = len(m["sample_names"])
    for ms in (0, m["minSites"], L + 1):
        got = eng.pairdist(hi, n, False, min_sites=ms)["dist"][0]
        assert_close(got, do.ind_pair_dists(g, hi, n, False, min_sites=ms or None), "min_sites=%d" % ms, **TOL)


@pytest.mark.parametrize("m", META, ids=IDS)
def test_target_freqs_golden(eng, m):
    g, hp, L = _load(eng, m)
    for target in ("derived", "minor"):
        for md in (0.0, 3.0):
            for asCounts in (False, True):
                want = ARR["%s__tf_%s_%g_%d" % (m["name"], target, md, int(asCounts))]
                got, tie = eng.site_target_freqs(target, 0, L, min_data=md, as_counts=asCounts)
                if target == "minor":
                    gold_tie = ARR[m["name"] + "__minor_tie"]
                    assert np.array_equal(tie, gold_tie)
                    got, want = got[~gold_tie], want[~gold_tie]     # the reference draws at random on ties
                assert got.shape == want.shape
                assert np.array_equal(np.isnan(got), np.isnan(want))
                assert np.array_equal(got[~np.isnan(got)], want[~np.isnan(want)]), (target, md, asCounts)   # bit-exact


def test_hapstats_and_het_many_windows_vs_oracle(eng):
    """Seeded low-diversity data, several windows (word-edge clipping), interleaved populations."""
    from oracle import dense_oracle as do
    rng = np.random.default_rng(99)
    L, H = 1000, 44
    hap_pop = np.repeat(rng.permutation(np.repeat([0, 1, 2, -1], [7, 8, 5, 2])), 2).astype(np.int32)
    base = rng.integers(0, 4, L)
    g = np.repeat(base[:, None], H, axis=1).astype(np.int8)
    mut = rng.random((L, H)) < 0.004
    g[mut] = (g[mut] + 1) % 4
    # copies of haplotypes -> real clusters
    for a, b in ((0, 5), (0, 9), (3, 20), (21, 33), (21, 40), (21, 41)):
        g[:, b] = g[:, a]
    g[rng.random((L, H)) < 0.03] = -1
    eng.upload(g, np.arange(1, L + 1, dtype=np.int32))
    eng.set_pops(hap_pop, 3)
    lo = np.array([0, 37, 300, 640, 999], dtype=np.int64)
    hi = np.array([37, 300, 640, 1000, 1000], dtype=np.int64)
    eng.set_windows(lo, hi)
    hap_ind = (np.arange(H) // 2).astype(np.int32)
    for md, ms, dn in ((0.0, 0, False), (0.0, 30, True), (0.01, 0, True), (0.02, 250, True)):
        got = eng.hapstats(md, min_sites=ms, diag_nan=dn)
        het = eng.ind_het(hap_ind, H // 2, min_sites=ms)
        for w in range(len(lo)):
            want = do.h12_stats(g[lo[w]:hi[w]], hap_pop, 3, md, ms or None, dn)
            assert_close(got[w], want, "h12 w%d md=%g ms=%d" % (w, md, ms), **TOL)
            assert_close(het[w], do.sample_het(g[lo[w]:hi[w]], hap_ind, H // 2, ms or None), "het w%d" % w, **TOL)


# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def inputs2(tmp_path_factory):
    from genomics_general_b200 import synth
    d = tmp_path_factory.mktemp("cli2")
    c = CLI2["four_pops"]["cfg"]
    spec = synth.SynthSpec(c["n_pops"], c["spp"], seed=c["seed"], miss=c["miss"])
    g = synth.synth_genotypes(spec, 0, c["S"])
    nsc = c["scaffolds"]
    per = c["S"] // nsc
    scafs, pos = [], []
    for k in range(nsc):
        n = per if k < nsc - 1 else c["S"] - per * (nsc - 1)
        scafs += ["chr%d" % (k + 1)] * n
        pos.append(synth.synth_positions(n, seed=c["seed"] + k))
    path = str(d / "four_pops.geno")
    synth.write_geno(path, g, np.concatenate(pos), scafs, spec.sample_names())
    pops = str(d / "four_pops.pops")
    with open(pops, "wt") as f:
        for i, n in enumerate(spec.sample_names()):
            f.write("%s pop%d\n" % (n, i // c["spp"]))
    popargs = []
    for p in spec.pop_names():
        popargs += ["-p", p]
    return dict(geno=path, pops=pops, popargs=popargs, dir=str(d))


def _table(text):
    lines = text.strip("\n").split("\n")
    hdr = lines[0].split(",")
    return hdr, [dict(zip(hdr, l.split(","))) for l in lines[1:]]


def _compare_by_column(ours, ref, n_prefix=5, atol=2e-8):
    """The reference's indHet column order is that of a Python set: compare by column name."""
    h1, r1 = _table(ours)
    h2, r2 = _table(ref)
    assert sorted(h1) == sorted(h2)
    assert len(r1) == len(r2)
    for a, b in zip(r1, r2):
        for k in h2[:n_prefix]:
            assert a[k] == b[k], (k, a[k], b[k])
        keys = h2[n_prefix:]
        assert_close([float(a[k]) for k in keys], [float(b[k]) for k in keys], "row " + a["start"], rtol=1e-6, atol=atol)


@pytest.mark.parametrize("key,extra", [
    ("popgen_indHet_alone", ["--windType", "sites", "-w", "300", "-m", "290", "--analysis", "indHet"]),
    ("popgen_popDist_indHet_hapStats", ["--windType", "sites", "-w", "300", "-m", "290", "--analysis", "popDist", "indHet",
                                        "hapStats", "--hapDist", "0.05"]),
    ("popgen_hapStats_alone", ["-w", "20000", "-m", "50", "--analysis", "hapStats", "--hapDist", "0.08"]),
    ("popgen_indPairDist_hapStats_indHet", ["-w", "20000", "-m", "50", "--analysis", "indPairDist", "hapStats", "indHet",
                                            "--hapDist", "0.08"]),
])
def test_popgenWindows_more_analyses_cli(inputs2, key, extra):
    from genomics_general_b200.cli import popgenWindows
    i = inputs2
    o = os.path.join(i["dir"], key + ".csv")
    popgenWindows.main(["-g", i["geno"], "-o", o, "-f", "phased", "-T", "1", "--popsFile", i["pops"], "--roundTo", "8"]
                       + extra + i["popargs"])
    _compare_by_column(open(o).read(), CLI2["four_pops"][key])


@pytest.mark.parametrize("key,extra", [
    ("freq_derived", ["--target", "derived"]),
    ("freq_derived_counts", ["--target", "derived", "--asCounts"]),
    ("freq_derived_keepnan_mindata", ["--target", "derived", "--keepNanLines", "--minData", "11"]),
    ("freq_derived_threshold", ["--target", "derived", "--threshold", "0.5"]),
])
def test_freq_target_cli_bit_exact(inputs2, key, extra):
    from genomics_general_b200.cli import freq
    i = inputs2
    o = os.path.join(i["dir"], key + ".tsv")
    freq.main(["-g", i["geno"], "-o", o, "-f", "phased", "-t", "1", "--popsFile", i["pops"]] + extra + i["popargs"])
    txt = open(o).read().splitlines()
    res = CLI2["four_pops"]
    assert txt[:300] == res[key + "_head"]
    assert len(txt) == res[key + "_nlines"]
    assert hashlib.sha256(("\n".join(txt) + "\n").encode()).hexdigest() == res[key + "_sha256"]


@pytest.mark.parametrize("m", [m for m in META if m["sampleHet"]], ids=[m["name"] for m in META if m["sampleHet"]])
def test_alignment_api_cache_states(m):
    """genomics-compatible Alignment: sampleHet / H12stats after groupDistStats see the in-place masked matrix."""
    import warnings
    from genomics_general_b200 import genomics as G
    g = ARR[m["name"] + "__g_aln"]
    hp = ARR[m["name"] + "__hap_pop"]
    groups = [m["pop_names"][x] if x >= 0 else None for x in hp]

    def new():
        return G.Alignment(g, names=m["hap_names"], groups=groups, sampleNames=m["hap_samples"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        a = new()
        het = a.sampleHet()
        assert_close([het[s] for s in m["sample_names"]], [m["sampleHet"]["alone"][s] for s in m["sample_names"]], "alone", **TOL)
        h = a.H12stats(maxDist=0.02)
        assert_close([h[k] for k in sorted(h)], [m["H12stats"]["alone_0.02"][k] for k in sorted(h)], "h12 alone", **TOL)
        a = new()
        a.groupDistStats(doPairs=True, minSites=m["minSites"], minData=0.01)
        het = a.sampleHet()
        assert_close([het[s] for s in m["sample_names"]], [m["sampleHet"]["after_popDist"][s] for s in m["sample_names"]],
                     "after_popDist", **TOL)
        h = a.H12stats(maxDist=0.02)
        assert_close([h[k] for k in sorted(h)], [m["H12stats"]["after_popDist_0.02"][k] for k in sorted(h)], "h12 masked", **TOL)
        a = new()
        a.indPairDists()
        h = a.H12stats(maxDist=0.1)
        assert_close([h[k] for k in sorted(h)], [m["H12stats"]["after_indPairDist_0.1"][k] for k in sorted(h)], "h12 diag", **TOL)


# ------------------------------------------------------------------------------------------------
# fourPop (genomics.py:1585-1643)
# ------------------------------------------------------------------------------------------------
FP_KEYS = ('fhom', "fhom'", 'D', 'fd', "fd'", 'fdm', "fdm'", 'fdh', 'fdh2', 'fh', "ABBA", "BABA", "ABAA", "BAAA")
FP_META = [m for m in META if "fourPop" in m]


@pytest.mark.parametrize("m", FP_META, ids=[m["name"] for m in FP_META])
def test_fourpop_golden(eng, m):
    for key, want in m["fourPop"].items():
        notie = key.startswith(("default", "perm"))
        g, hp, L = _load(eng, m, "__g_aln_notie" if notie else "__g_aln")
        if key.startswith("perm"):
            sel, md, kw = (2, 0, 1, 3), 0.4, {}
        else:
            mode, md = key.rsplit("_", 1)
            sel, md, kw = (0, 1, 2, 3), float(md), ({} if mode == "default" else {mode: True})
        r = eng.fourpop(*sel, md, **kw)
        assert r["sites"][0] == L
        assert r["sitesUsed"][0] == want["sitesUsed"], key
        assert_close([r[k][0] for k in FP_KEYS], [want[k] for k in FP_KEYS], key, rtol=1e-9, atol=1e-12)


def test_fourpop_windows_vs_oracle(eng):
    """Many windows (with overlap), 2 % missing data, every mode and several minData values."""
    from genomics_general_b200 import synth
    from oracle import dense_oracle as do
    spec = synth.SynthSpec(4, 7, miss=0.02, seed=31)
    S = 30000
    g = synth.synth_genotypes(spec, 0, S)
    hp = spec.hap_pop()
    # exactly-tied sites are implementation-defined in the reference's default mode: blank them
    tot = np.stack([(g == a).sum(axis=1) for a in range(4)], axis=1)
    srt = np.sort(tot, axis=1)
    g[(srt[:, 2] > 0) & (srt[:, 2] == srt[:, 3])] = -1
    eng.upload(g, synth.synth_positions(S, seed=31))
    eng.set_pops(hp, 4)
    lo = np.arange(0, S - 3000, 1500, dtype=np.int64)
    hi = lo + 3000
    eng.set_windows(lo, hi)
    import warnings
    for kw in ({}, dict(polarize=True), dict(fixed=True)):
        for md in (0.0, 0.6, 1.0):
            r = eng.fourpop(1, 0, 2, 3, md, **kw)
            for w in range(0, len(lo), 3):
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    want = do.four_pop(g[lo[w]:hi[w]], hp, 1, 0, 2, 3, md, **kw)
                assert r["sitesUsed"][w] == want["sitesUsed"]
                assert_close([r[k][w] for k in FP_KEYS], [want[k] for k in FP_KEYS], "%s md=%g w=%d" % (kw, md, w),
                             rtol=1e-9, atol=1e-12)


def test_fourpop_api_mirror(eng):
    from genomics_general_b200 import genomics as G
    m = FP_META[0]
    g = ARR[m["name"] + "__g_aln"]
    hp = ARR[m["name"] + "__hap_pop"]
    groups = [m["pop_names"][x] if x >= 0 else None for x in hp]
    a = G.Alignment(g, names=m["hap_names"], groups=groups, sampleNames=m["hap_samples"])
    r = G.fourPop(a, "pop0", "pop1", "pop2", "pop3", 0.5, polarize=True)
    want = m["fourPop"]["polarize_0.5"]
    assert r["sitesUsed"] == want["sitesUsed"]
    assert_close([r[k] for k in FP_KEYS], [want[k] for k in FP_KEYS], "api", rtol=1e-9, atol=1e-12)


@pytest.mark.parametrize("key,notie,extra", [
    ("fourPopWindows_default", True, ["-w", "20000", "-m", "50", "--minData", "0.5"]),
    ("fourPopWindows_polarize", False, ["-w", "20000", "-m", "50", "--minData", "0.5", "--polarize"]),
    ("fourPopWindows_fixed_sites", False, ["--windType", "sites", "-w", "1000", "--overlap", "250", "-m", "20", "--minData", "0.9",
                                           "--fixed", "--writeFailedWindows", "--addWindowID"]),
])
def test_fourPopWindows_cli(inputs2, key, notie, extra):
    from genomics_general_b200 import geno_io, synth
    from genomics_general_b200.cli import fourPopWindows
    i = inputs2
    path = i["geno"]
    if notie:       # the default-mode fixture ran on the input with exactly-tied sites blanked (make_golden2.py)
        c = CLI2["four_pops"]["cfg"]
        spec = synth.SynthSpec(c["n_pops"], c["spp"], seed=c["seed"], miss=c["miss"])
        g = synth.synth_genotypes(spec, 0, c["S"])
        g[np.array(CLI2["four_pops"]["fourpop_tied_sites"], dtype=np.int64)] = -1
        gd = geno_io.parse_geno(path, geno_format="phased")
        path = os.path.join(i["dir"], "notie.geno")
        synth.write_geno(path, g, gd.pos, [gd.scaf_names[k] for k in gd.scaf_ids], spec.sample_names())
    o = os.path.join(i["dir"], key + ".csv")
    fourPopWindows.main(["-g", path, "-o", o, "-f", "phased", "-T", "1", "--popsFile", i["pops"], "-P1", "pop0", "-P2", "pop1",
                         "-P3", "pop2", "-O", "pop3"] + extra)
    npre = 7 if "--addWindowID" in extra else 6
    _compare_by_column(open(o).read(), CLI2["four_pops"][key], n_prefix=npre, atol=1.0001e-4)


def test_pairdist_cat_equals_one_window(eng):
    """--windType cat: chunked int64 accumulation over the site axis == the one-window pair matrix, bit for bit."""
    from genomics_general_b200 import synth
    from oracle import dense_oracle as do
    spec = synth.SynthSpec(3, 5, miss=0.05, seed=12)
    for S in (1000, 32768, 70001):
        g = synth.synth_genotypes(spec, 0, S)
        H = g.shape[1]
        hap_ind = (np.arange(H) // 2).astype(np.int32)
        hap_ind[-2:] = -1                                  # one sample left out (--samples subset)
        eng.upload(g, None)
        eng.set_windows([0], [S])
        for inc in (False, True):
            got, tot = eng.pairdist_cat(hap_ind, H // 2 - 1, inc)
            assert tot == S
            ref = eng.pairdist(hap_ind, H // 2 - 1, inc)["dist"][0]
            assert np.array_equal(got, ref, equal_nan=True)
        if S == 1000:
            assert_close(got, do.ind_pair_dists(g, hap_ind, H // 2 - 1, True), "oracle", **TOL)


# ------------------------------------------------------------------------------------------------
# K1 instantiations: byte-packed IDP.4A statistics vs the general path, 8 vs 12 consumer warps, early 32-bit flushes
# ------------------------------------------------------------------------------------------------
K1_KNOBS = [{}, {"PG_K1_NO_BYTES": "1"}, {"PG_K1_NW": "8"}, {"PG_K1_NO_BYTES": "1", "PG_K1_NW": "8"}, {"PG_K1_ACC_LIMIT": "3"},
            {"PG_K1_ACC_LIMIT": "1", "PG_K1_NO_BYTES": "1"}, {"PG_K1_G": "2"}, {"PG_K1_G": "4", "PG_K1_NO_BYTES": "1"},
            {"PG_K1_LANEPOP": "0"}, {"PG_K1_LANEPOP": "1"}, {"PG_K1_LANEPOP": "1", "PG_K1_NW": "8"},
            {"PG_K1_LANEPOP": "1", "PG_K1_ACC_LIMIT": "2"}, {"PG_K1_LANEPOP": "1", "PG_K1_WPT": "1"}]


def _popgen_fields(eng, pops):
    """Every record field of popgen with the popFreq counters on, then the closed-form fields again with them off."""
    eng.set_freqstats(True)
    r = eng.popgen(*pops)
    fq = eng.popgen_freqstats()
    eng.set_freqstats(False)
    r2 = eng.popgen(*pops)
    for k in ("pi", "dxy", "fst"):
        assert np.array_equal(r2[k], r[k], equal_nan=True), k
    return [r[k] for k in sorted(r)] + [fq[k] for k in sorted(fq)]


@pytest.mark.parametrize("shape", [(2, 9), (3, 20), (5, 7), (8, 13), (2, 150), (8, 100), (4, 127)], ids=lambda s: "%dx%d" % s)
def test_k1_variants_are_bit_identical_and_match_the_oracle(eng, shape, monkeypatch):
    """The byte pass's popgen and counts instantiations (PG_K1_BYTE_PASS: popgen otherwise takes the packed companion) agree
    bit for bit across the knobs that pick them, with the oracle, and with the default packed pass."""
    from genomics_general_b200 import synth
    from oracle import dense_oracle as do
    P, spp = shape
    spec = synth.SynthSpec(P, spp, miss=0.0, seed=100 + P)
    S = 20000
    g = synth.synth_genotypes(spec, 0, S)
    g[::97] = -1                                          # all-missing sites keep windows on the closed-form path
    hp = spec.hap_pop()
    pos = synth.synth_positions(S, seed=4)
    lo = np.array([0, 10, 4000, 4001, 9000, 15000], dtype=np.int64)
    hi = np.array([10, 4000, 4001, 9000, 15000, 20000], dtype=np.int64)
    base = None
    for knobs in K1_KNOBS:
        for k in ("PG_K1_NO_BYTES", "PG_K1_NW", "PG_K1_ACC_LIMIT", "PG_K1_G", "PG_K1_LANEPOP", "PG_K1_WPT", "PG_K1_BYTE_PASS"):
            monkeypatch.delenv(k, raising=False)
        monkeypatch.setenv("PG_K1_BYTE_PASS", "1")
        for k, v in knobs.items():
            monkeypatch.setenv(k, v)
        eng.upload(g, pos)
        eng.set_pops(hp, P)
        eng.set_windows(lo, hi)
        eng.set_freqstats(True)
        r = eng.popgen(1, 0.01)
        fq = eng.popgen_freqstats()
        eng.set_freqstats(False)
        r2 = eng.popgen(1, 0.01)
        assert np.all(r["path"] == 1)
        cnt = eng.site_counts(17, 3000)
        cur = [r["pi"], r["dxy"], r["fst"], fq["S"], fq["thetaPi"], fq["thetaW"], fq["TajD"], fq["l"], cnt]
        for a, b in zip([r2["pi"], r2["dxy"], r2["fst"]], cur[:3]):
            assert np.array_equal(a, b, equal_nan=True)
        if base is None:
            base = cur
            assert np.array_equal(cnt.astype(np.int64), do.site_counts(g[17:3017], hp, P))
            for w in (1, 3, 5):
                ok, pi, dxy, fst = do.group_dist_stats_closed_form(g[lo[w]:hi[w]], hp, P, 1, 0.01)
                assert ok
                assert_close(r["pi"][w], pi, "pi", **TOL)
                assert_close(r["dxy"][w], dxy, "dxy", **TOL)
                assert_close(r["fst"][w], fst, "fst", rtol=1e-8, atol=1e-12)
                f = do.group_freq_stats(g[lo[w]:hi[w]], hp, P)
                for key in ("S", "thetaPi", "thetaW", "TajD"):
                    assert_close(fq[key][w], f[key], key, **TOL)
        else:
            for a, b in zip(cur, base):
                assert np.array_equal(a, b, equal_nan=True), knobs
    byte_fields = _popgen_fields(eng, (1, 0.01))
    monkeypatch.delenv("PG_K1_BYTE_PASS")
    for k in ("PG_K1_NO_BYTES", "PG_K1_NW", "PG_K1_ACC_LIMIT", "PG_K1_G", "PG_K1_LANEPOP", "PG_K1_WPT"):
        monkeypatch.delenv(k, raising=False)
    assert eng.packed_rows(0, 1) is not None           # the companion exists: without PG_K1_BYTE_PASS, the packed pass runs
    for a, b in zip(_popgen_fields(eng, (1, 0.01)), byte_fields):
        assert np.array_equal(a, b, equal_nan=True), "packed pass"


def test_seq_nonnan_bit_exact(eng):
    """Alignment.seqNonNan per window (the --minPerInd gate of distMat.py:40)."""
    from genomics_general_b200 import synth
    spec = synth.SynthSpec(3, 6, miss=0.07, seed=21)
    S = 5000
    g = synth.synth_genotypes(spec, 0, S)
    eng.upload(g, None)
    lo = np.array([0, 0, 31, 32, 33, 1000, 4999, 2500], dtype=np.int64)
    hi = np.array([0, 5000, 64, 33, 97, 3000, 5000, 2500], dtype=np.int64)
    eng.set_windows(lo, hi)
    got = eng.seq_nonnan()
    want = np.stack([(g[a:b] >= 0).sum(axis=0) for a, b in zip(lo, hi)])
    assert np.array_equal(got, want)


# ------------------------------------------------------------------------------------------------
# sfs.py (genotype input)
# ------------------------------------------------------------------------------------------------
def _sfs_keys():
    d = CLI2["four_pops"]
    return [k for k in d if k.startswith("sfs_") and not k.startswith(("sfs_base", "sfs_target")) and k + "_args" in d]


@pytest.mark.parametrize("key", _sfs_keys())
def test_sfs_engine_and_cli_match_the_reference_text(eng, key, tmp_path, capsys):
    from genomics_general_b200 import synth
    from genomics_general_b200.cli import sfs as sfs_cli
    from oracle import dense_oracle as do
    from test_oracle_golden2 import sfs_inputs, sfs_plan
    d = CLI2["four_pops"]
    spec, g, scaf = sfs_inputs()
    extra = d[key + "_args"]
    inpops, outgroup, groups, keep = sfs_plan(extra)
    order = inpops + ([outgroup] if outgroup else [])
    remap = {int(p[3:]): k for k, p in enumerate(order)}
    hp = np.array([remap[x] for x in spec.hap_pop()], dtype=np.int32)
    mask = None
    if keep is not None:
        mask = np.isin(scaf, keep[1]) if keep[0] else ~np.isin(scaf, keep[1])
    gi = [tuple(inpops.index(p) for p in grp) for grp in groups]
    eng.upload(g, None)
    eng.set_pops(hp, len(order))
    sizes = [int((hp == x).sum()) for x in range(len(order))]
    hists, firsts, n = eng.sfs(len(inpops), gi, sizes, outgroup=len(inpops) if outgroup else -1, site_mask=mask)
    chains, n_or = do.sfs(g, hp, len(inpops), gi, outgroup=len(inpops) if outgroup else -1, site_mask=mask)
    assert n == n_or
    text = "".join("\n".join("\t".join(str(x) for x in row) for row in sfs_cli.ordered_chains(h, f)) + "\n"
                   for h, f in zip(hists, firsts))
    assert text == d[key]                                   # the unmodified script's own stdout, byte for byte
    # the command line on a .geno file
    c = d["sfs_cfg"]
    path = str(tmp_path / "sfs.geno")
    scaf_names = ["chr%d" % (k + 1) for k in scaf]
    synth.write_geno(path, g, synth.synth_positions(c["S"], seed=c["seed"]), scaf_names, spec.sample_names())
    pops = str(tmp_path / "sfs.pops")
    with open(pops, "wt") as f:
        for i, nm in enumerate(spec.sample_names()):
            f.write("%s pop%d\n" % (nm, i // c["spp"]))
    capsys.readouterr()
    sfs_cli.main(["-i", path, "--inputType", "genotypes", "--popsFile", pops, "--pipe", "-p", "pop0", "-p", "pop1", "-p", "pop2",
                  "-p", "pop3"] + extra)
    assert capsys.readouterr().out == d[key]


def test_popgenWindows_haplo_and_pairs_formats_cli(inputs2, tmp_path):
    """-f haplo (ploidy 1) and -f pairs through the device tokenizer, against the reference script's rows."""
    from genomics_general_b200 import geno_io, synth
    from genomics_general_b200.cli import popgenWindows
    d = CLI2["four_pops"]
    c = d["haplo_cfg"]
    spec = synth.SynthSpec(c["n_pops"], c["spp"], ploidy=1, seed=c["seed"], miss=c["miss"])
    g = synth.synth_genotypes(spec, 0, c["S"])
    hpath = str(tmp_path / "haplo.geno")
    synth.write_geno(hpath, g, synth.synth_positions(c["S"], seed=c["seed"]), ["chr1"] * c["S"], spec.sample_names(), ploidy=1,
                     fmt="haplo")
    hpops = str(tmp_path / "haplo.pops")
    with open(hpops, "wt") as f:
        for i, n in enumerate(spec.sample_names()):
            f.write("%s pop%d\n" % (n, i // c["spp"]))
    o = str(tmp_path / "o.csv")
    base = ["-o", o, "-T", "1", "--roundTo", "9", "-w", "20000", "-m", "50"]
    popgenWindows.main(base + ["-g", hpath, "-f", "haplo", "--popsFile", hpops, "-p", "pop0", "-p", "pop1", "-p", "pop2"])
    _compare_by_column(open(o).read(), d["popgen_haplo"], atol=2e-9)
    # pairs: the four_pops input re-written without separators
    gd = geno_io.parse_geno(inputs2["geno"], geno_format="phased")
    ppath = str(tmp_path / "pairs.geno")
    synth.write_geno(ppath, gd.geno, gd.pos, [gd.scaf_names[k] for k in gd.scaf_ids], gd.names, fmt="pairs")
    popgenWindows.main(base + ["-g", ppath, "-f", "pairs", "--popsFile", inputs2["pops"]] + inputs2["popargs"])
    _compare_by_column(open(o).read(), d["popgen_pairs"], atol=2e-9)


def test_many_small_populations_counts_and_target_freqs(eng, monkeypatch):
    """freq.py --indFreqs: one population per individual (more than 64 populations) — gather kernel vs site passes vs oracle."""
    from genomics_general_b200 import synth
    from oracle import dense_oracle as do
    spec = synth.SynthSpec(5, 17, miss=0.05, seed=77)          # 85 individuals
    S = 3000
    g = synth.synth_genotypes(spec, 0, S)
    H = g.shape[1]
    hp = (np.arange(H) // 2).astype(np.int32)                  # population = individual
    hp[-4:] = -1                                               # two individuals left out
    P = int(hp.max()) + 1
    eng.upload(g, None)
    eng.set_pops(hp, P)
    want = do.site_counts(g, hp, P)
    a = eng.site_counts()
    monkeypatch.setenv("PG_COUNTS_NO_GATHER", "1")
    b = eng.site_counts()
    monkeypatch.delenv("PG_COUNTS_NO_GATHER")
    assert np.array_equal(a.astype(np.int64), want) and np.array_equal(a, b)
    v, tie = eng.site_target_freqs("derived")
    wv, _ = do.target_freqs(g, hp, P, "derived")
    assert np.array_equal(v, wv, equal_nan=True)


@pytest.mark.parametrize("P", [3, 4, 6, 8])
def test_lane_per_population_with_interleaved_columns(eng, P, monkeypatch):
    """k1_site_pass_lp forced on a layout it is not tuned for: populations interleaved column by column, unused
    haplotypes, unequal sizes (masked chunks only, P padded to 4 / 8).  Popgen runs on the byte pass (PG_K1_BYTE_PASS), and
    the default packed pass must give the same record fields bit for bit."""
    from genomics_general_b200 import synth
    from oracle import dense_oracle as do
    rng = np.random.default_rng(50 + P)
    sizes = rng.integers(3, 40, P)
    hp = np.concatenate([np.full(n, x) for x, n in enumerate(sizes)] + [np.full(5, -1)]).astype(np.int32)
    hp = rng.permutation(hp)
    H, S = len(hp), 9000
    ref = rng.integers(0, 4, S)
    alt = (ref + rng.integers(1, 4, S)) % 4
    freq = rng.random((S, P + 1)) * (rng.random(S) < 0.4)[:, None]
    g = np.where(rng.random((S, H)) < freq[:, hp], alt[:, None], ref[:, None]).astype(np.int8)
    g[rng.random(S) < 0.1] = -1
    pos = np.cumsum(rng.integers(1, 30, S)).astype(np.int32)
    lo = np.arange(0, S, 750, dtype=np.int64)
    hi = np.minimum(lo + 1000, S)                       # overlapping windows
    res = []
    monkeypatch.setenv("PG_K1_BYTE_PASS", "1")
    for lp in ("0", "1"):
        monkeypatch.setenv("PG_K1_LANEPOP", lp)
        eng.upload(g, pos)
        eng.set_pops(hp, P)
        eng.set_windows(lo, hi)
        eng.set_freqstats(True)
        r = eng.popgen(10, 0.01)
        fq = eng.popgen_freqstats()
        eng.set_freqstats(False)
        res.append([r["pi"], r["dxy"], r["fst"], r["sites"], r["pos_sum"], r["path"], fq["S"], fq["thetaPi"], eng.site_counts()])
    byte_fields = _popgen_fields(eng, (10, 0.01))
    monkeypatch.delenv("PG_K1_LANEPOP")
    monkeypatch.delenv("PG_K1_BYTE_PASS")
    for a, b in zip(*res):
        assert np.array_equal(a, b, equal_nan=True)
    assert eng.packed_rows(0, 1) is not None           # the companion exists: without PG_K1_BYTE_PASS, the packed pass runs
    for a, b in zip(_popgen_fields(eng, (10, 0.01)), byte_fields):
        assert np.array_equal(a, b, equal_nan=True), "packed pass"
    assert np.all(res[0][5] == 1)
    assert np.array_equal(res[1][8].astype(np.int64), do.site_counts(g, hp, P))
    for w in (0, 5, len(lo) - 1):
        ok, pi, dxy, fst = do.group_dist_stats_closed_form(g[lo[w]:hi[w]], hp, P, 10, 0.01)
        assert ok
        assert_close(res[1][0][w], pi, "pi", **TOL)
        assert_close(res[1][1][w], dxy, "dxy", **TOL)


def test_haploid_samples_in_a_phased_file_cli(inputs2, tmp_path):
    """--haploid: the named samples carry one-letter tokens (ploidy 1) — popgenWindows and ABBABABAwindows rows against the
    reference scripts' own output on the same mixed-ploidy file."""
    from genomics_general_b200 import geno_io
    from genomics_general_b200.cli import ABBABABAwindows, popgenWindows
    d = CLI2["four_pops"]
    hap = d["popgen_phased_haploid_samples"]
    gd = geno_io.parse_geno(inputs2["geno"], geno_format="phased")
    lut = np.array(list("ACGTN"))
    ch = lut[np.where(gd.geno < 0, 4, gd.geno)]
    mpath = str(tmp_path / "mixed.geno")
    hap_idx = {gd.names.index(n) for n in hap}
    with open(mpath, "wt") as f:
        f.write("#CHROM\tPOS\t" + "\t".join(gd.names) + "\n")
        for s in range(gd.n_sites):
            toks = [ch[s, 2 * k] if k in hap_idx else ch[s, 2 * k] + "/" + ch[s, 2 * k + 1] for k in range(len(gd.names))]
            f.write("%s\t%d\t%s\n" % (gd.scaf_names[gd.scaf_ids[s]], gd.pos[s], "\t".join(toks)))
    o = str(tmp_path / "o.csv")
    popgenWindows.main(["-o", o, "-T", "1", "--roundTo", "9", "-w", "20000", "-m", "50", "-g", mpath, "-f", "phased",
                        "--popsFile", inputs2["pops"], "--haploid", ",".join(hap)] + inputs2["popargs"])
    _compare_by_column(open(o).read(), d["popgen_phased_haploid"], atol=2e-9)
    ABBABABAwindows.main(["-w", "20000", "-m", "50", "-g", mpath, "-o", o, "-f", "phased", "-T", "1", "--popsFile", inputs2["pops"],
                          "--minData", "0.5", "--haploid", ",".join(hap), "-P1", "pop0", "-P2", "pop1", "-P3", "pop2", "-O", "pop3"])
    _compare_by_column(open(o).read(), d["abba_phased_haploid"], n_prefix=6, atol=1.0001e-4)


def test_freq_target_minor_cli_rows_without_ties(inputs2):
    """freq.py --target minor: byte-identical rows wherever the reference's choice is not random (no exact tie)."""
    from genomics_general_b200 import synth
    from genomics_general_b200.cli import freq
    d = CLI2["four_pops"]
    c = d["cfg"]
    spec = synth.SynthSpec(c["n_pops"], c["spp"], seed=c["seed"], miss=c["miss"])
    g = synth.synth_genotypes(spec, 0, c["S"])
    tot = np.stack([(g == a).sum(axis=1) for a in range(4)], axis=1)
    srt = np.sort(tot, axis=1)
    tied = (srt[:, 2] > 0) & (srt[:, 2] == srt[:, 3]) & (srt[:, 1] == 0)
    o = os.path.join(inputs2["dir"], "minor.tsv")
    freq.main(["-g", inputs2["geno"], "-o", o, "-f", "phased", "-t", "1", "--popsFile", inputs2["pops"], "--target", "minor",
               "--keepNanLines"] + inputs2["popargs"])
    ours = open(o).read().splitlines()
    ref = d["freq_minor_keepnan"]
    assert len(ours) == len(ref) == c["S"] + 1 and ours[0] == ref[0]
    same = [a == b for a, b in zip(ours[1:], ref[1:])]
    assert all(s or t for s, t in zip(same, tied)), "a row without a tie differs"
    assert tied.sum() > 0 and sum(same) >= c["S"] - int(tied.sum())



def _sfs_table_keys():
    d = CLI2["four_pops"]
    return [k for k in d if k.startswith(("sfs_base", "sfs_target")) and k + "_args" in d]


@pytest.mark.parametrize("key", _sfs_table_keys())
def test_sfs_from_count_tables_matches_the_reference_pipeline(eng, key, tmp_path, capsys):
    """freq.py -> sfs.py, both ours, against the same pipeline of the reference scripts (byte-identical spectra)."""
    from genomics_general_b200 import synth
    from genomics_general_b200.cli import freq as freq_cli, sfs as sfs_cli
    from test_oracle_golden2 import sfs_inputs, sfs_table_plan, sfs_tables
    d = CLI2["four_pops"]
    c = d["sfs_cfg"]
    spec, g, scaf = sfs_inputs()
    base, target, _ = sfs_tables()
    kind, order, n_in, og, groups, inpops, excl = sfs_table_plan(key)
    cols = [int(p[3:]) for p in order]
    mask = ~np.isin(scaf, excl) if excl else None
    gi = [tuple(inpops.index(p) for p in grp) for grp in groups]
    table = base[:, cols, :] if kind == "base" else target[:, cols]
    hists, firsts, _ = eng.sfs_tables(kind, table, n_in, gi, outgroup=og, site_mask=mask)
    text = "".join("\n".join("\t".join(str(x) for x in row) for row in sfs_cli.ordered_chains(h, f)) + "\n"
                   for h, f in zip(hists, firsts))
    assert text == d[key]
    # the command lines: our freq.py writes the table, our sfs.py reads it
    path = str(tmp_path / "sfs.geno")
    synth.write_geno(path, g, synth.synth_positions(c["S"], seed=c["seed"]), ["chr%d" % (k + 1) for k in scaf], spec.sample_names())
    pops = str(tmp_path / "sfs.pops")
    with open(pops, "wt") as f:
        for i, nm in enumerate(spec.sample_names()):
            f.write("%s pop%d\n" % (nm, i // c["spp"]))
    tab = str(tmp_path / "table.tsv")
    fa = ["-g", path, "-o", tab, "-f", "phased", "-t", "1", "--popsFile", pops, "-p", "pop0", "-p", "pop1", "-p", "pop2", "-p", "pop3"]
    freq_cli.main(fa if kind == "base" else fa + ["--target", "derived", "--asCounts", "--keepNanLines"])
    capsys.readouterr()
    sfs_cli.main(["-i", tab, "--pipe"] + d[key + "_args"])
    assert capsys.readouterr().out == d[key]
