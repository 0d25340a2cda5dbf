"""filterGenotypes.py's kernels (csrc/filter.cu) at the limits the reference fixtures do not reach, against the numpy
restatement oracle/filter_oracle.py (itself checked against the reference's siteTest / asList in test_filter_cpu.py):

  1. k_filter_emit across the output formats, the input formats with and without --partialToMissing, ploidies 1 to 8 mixed
     in one file with phased separators of every kind, and 1 to 203 selected samples (more than one 32-sample step of the
     warp scan), taken out of column order with unselected columns between them
  2. the slabs of pg_filter_emit: caps of exactly k whole rows and one byte less, a row larger than the buffer,
     row0 == n_kept, and the offset cache across format changes and across a second pg_filter on the same ingest
  3. grid-stride passes: more sites than one grid of k_filter_sites covers and more kept rows than one grid of k_filter_emit
     (132 SMs x 32 CTAs x 8 warps = 33 792), and k_filter_thin, one thread per pod, with pods of 1, 3, 256 and 257 sites
     (274, 92, 2 and 2 blocks of 256 threads)
  4. k_filter_sites at 64 populations (and the refusal of 65), and its fp64 predicates exactly on their thresholds and one
     ulp to either side, with the IEEE edges of maxHet and nearlyFixedDiff
  5. the text layout of data lines (leading blanks, runs of blanks, CRLF, a last line without a newline, comment and blank
     lines, positions written 0012 and +12), on the engine and through the command line

Text is compared byte for byte; counts, flags and verdicts exactly."""
import random
import types

import numpy as np
import pytest

from oracle import filter_oracle as fo

pytestmark = pytest.mark.gpu

FL_TIE, FL_PARTIAL, FL_NOALLELE = 1, 2, 4
SEPS = "|/:"
JUNK = ("NA", ".", "x", "A|T|G|C", "ACGTACGTAC", "0/1")      # unselected columns: never read, so never checked


@pytest.fixture(scope="module")
def eng():
    from genomics_general_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


# ---- generated .geno data ----------------------------------------------------------------------------------------------
class Geno:
    """data lines of a .geno body and the sample tables the command line builds for them (cols: genotype column of every
    selected sample, in output order)"""

    def __init__(self, body, lines, fmt, cols, ploidy, n_cols):
        self.body, self.lines, self.fmt, self.cols, self.ploidy = body, lines, fmt, list(cols), list(ploidy)
        self.hap0 = np.concatenate([[0], np.cumsum(ploidy)[:-1]]).astype(np.int32)
        self.H = int(sum(ploidy))
        self.col_hap = np.full(n_cols, -1, np.int32)
        self.col_pl = np.ones(n_cols, np.int8)
        for k, c in enumerate(cols):
            self.col_hap[c] = self.hap0[k]
            self.col_pl[c] = ploidy[k]


def mixed_ploidy(rng, n):
    pl = [1 + (k + n) % 8 for k in range(n)]
    rng.shuffle(pl)
    return pl


def random_alleles(rng, ploidy, miss, partial, all_missing):
    """alleles of one site, one list per sample; 'N' is a missing allele"""
    if rng.random() < all_missing:
        return [["N"] * pl for pl in ploidy]
    pool = rng.sample("ACGT", rng.choice([1, 2, 2, 3, 4]))
    m = rng.choice(miss)
    out = []
    for pl in ploidy:
        al = [rng.choice(pool) for _ in range(pl)]
        r = rng.random()
        if r < m:
            al = ["N"] * pl
        elif partial and pl > 1 and r < 2 * m:
            al[rng.randrange(pl)] = "N"
        out.append(al)
    return out


def token(rng, al, fmt):
    if fmt == "diplo":
        return "N" if "N" in al else fo.PAIR_DIPLO["".join(sorted(al))]
    if fmt == "alleles":
        return "".join(al)
    if len(al) == 1:
        return al[0]
    if rng.random() < 0.3:          # separators that differ inside one token: the first one is the sample's phase character
        seps = [rng.choice(SEPS) for _ in al[1:]]
    else:
        seps = [rng.choice(SEPS)] * (len(al) - 1)
    return al[0] + "".join(s + a for s, a in zip(seps, al[1:]))


def make_geno(seed, S, ploidy, fmt="phased", n_extra=0, miss=(0.0, 0.05, 0.3), partial=True, all_missing=0.02,
              scaf_every=37, sites=None):
    """S data lines; the selected samples sit in shuffled columns among n_extra unselected ones.  Every line has its own
    position, so (scaffold, position) names a line.  sites: alleles of every site instead of random ones."""
    rng = random.Random(seed)
    n = len(ploidy)
    n_cols = n + n_extra
    cols = rng.sample(range(n_cols), n)
    if n > 1 and cols == sorted(cols):
        cols.reverse()
    lines = []
    for i in range(S):
        al = sites[i] if sites is not None else random_alleles(rng, ploidy, miss, partial, all_missing)
        toks = [rng.choice(JUNK) for _ in range(n_cols)]
        for k, c in enumerate(cols):
            toks[c] = token(rng, al[k], fmt)
        lines.append("\t".join(["chr%d" % (i // scaf_every), str(2 * i + 1)] + toks))
    return Geno(("\n".join(lines) + "\n").encode(), lines, fmt, cols, ploidy, n_cols)


def tokens_geno(rows, ploidy):
    """phased lines from explicit tokens, every sample selected in column order"""
    lines = ["t\t%d\t%s" % (i + 1, "\t".join(r)) for i, r in enumerate(rows)]
    return Geno(("\n".join(lines) + "\n").encode(), lines, "phased", range(len(ploidy)), ploidy, len(ploidy))


def relabel(g, scaf, pos):
    """g with new scaffold names and positions (the genotype columns stay)"""
    g.lines = ["%s\t%s\t%s" % (sc, p, ln.split("\t", 2)[2]) for ln, sc, p in zip(g.lines, scaf, pos)]
    g.body = ("\n".join(g.lines) + "\n").encode()
    return g


def spec_of(g, **kw):
    spec = dict(samp_hap0=g.hap0, samp_ploidy=np.array(g.ploidy, np.int8), pops=[])
    spec.update(kw)
    return spec


# ---- the engine, as the command line drives it -------------------------------------------------------------------------
def ingest(eng, g, include=None, exclude=None):
    """strict ingest of g's body; (contig mask, scaffold id of every site) as filterGenotypes.main builds them"""
    from genomics_general_b200.cli.filterGenotypes import FMT_CODE, _scaffolds
    eng.set_strict_ingest(True)
    S = eng.ingest_text(g.body, FMT_CODE[g.fmt], g.col_hap, g.col_pl, g.H)
    assert S == len(g.lines)
    pos, newsc, off = eng.ingest_meta(S, release=False)
    names, run_of = _scaffolds(g.body, newsc, off)
    cmask = None
    if include is not None or exclude is not None:
        ok = np.array([(include is None or n in include) and (exclude is None or n not in exclude) for n in names], np.uint8)
        cmask = ok[run_of]
    ids = {}
    run_id = np.array([ids.setdefault(n, len(ids)) for n in names], dtype=np.int32)
    return cmask, run_id[run_of]


def emit(eng, nk, fmt, freq_order=False, cap=1 << 24):
    """every kept row through pg_filter_emit with a buffer of cap bytes: (bytes, [(rows, bytes) of every call])"""
    buf = np.zeros(max(cap, 1), np.uint8)
    out, calls, row = [], [], 0
    while row < nk:
        rows, nb = eng.filter_emit(fmt, freq_order, row, buf, cap)
        assert rows > 0
        calls.append((rows, nb))
        out.append(buf[:nb].tobytes())
        row += rows
    return b"".join(out), calls


def run(eng, g, spec, fmt, freq_order=False, cap=1 << 24, include=None, exclude=None, ing=None):
    """set_strict_ingest, ingest_text, ingest_meta, filter and the emit loop on one engine"""
    cmask, scaf = ing if ing is not None else ingest(eng, g, include, exclude)
    nk, flags = eng.filter(spec, contig_mask=cmask, scaf_id=scaf)
    text, calls = emit(eng, nk, fmt, freq_order, cap)
    return types.SimpleNamespace(bytes=text, calls=calls, n_kept=nk, flags=flags, stats=eng.filter_stats())


# ---- the oracle --------------------------------------------------------------------------------------------------------
def genotypes(g, s, spec):
    toks = g.lines[s].split()[2:]
    return [fo.genotype(toks[c], g.fmt, spec.get("partial_to_missing")) for c in g.cols]


def site_flags(gts):
    c = fo.counts(gts)
    partial = any(fo.is_missing(al) and any(a != "N" for a in al) for al, _ in gts)
    return (FL_TIE if fo.is_tied(c) else 0) | (FL_PARTIAL if partial else 0) | (FL_NOALLELE if c.sum() == 0 else 0)


def expect(g, spec, fmt, freq_order=False, include=None, exclude=None):
    """filter_lines over g's data lines: the rows, the sites they come from and the OR of those sites' flags"""
    rows = fo.filter_lines(g.lines, g.fmt, g.cols, spec["pops"], spec, fmt, "freq" if freq_order else None, include, exclude)
    where = {tuple(ln.split()[:2]): s for s, ln in enumerate(g.lines)}
    kept = [where[tuple(r.split("\t", 2)[:2])] for r in rows]
    flags = 0
    for s in kept:
        flags |= site_flags(genotypes(g, s, spec))
    return types.SimpleNamespace(bytes="".join(rows).encode(), rows=[r.encode() for r in rows], kept=kept, flags=flags)


def oracle_stats(g, spec):
    """what pg_filter_stats returns, per site, from the oracle"""
    pops = spec["pops"]
    S, P = len(g.lines), len(pops)
    st = dict(called=np.zeros(S, np.int64), het=np.zeros(S, np.int64), counts=np.zeros((S, 4), np.int64),
              pop_called=np.zeros((S, P), np.int64), pop_mask=np.zeros((S, P), np.int64), flags=np.zeros(S, np.int64),
              keep=np.zeros(S, np.int64))
    for s in range(S):
        gts = genotypes(g, s, spec)
        st["called"][s] = sum(not fo.is_missing(al) for al, _ in gts)
        st["het"][s] = sum(len(set(al)) > 1 for al, _ in gts)
        st["counts"][s] = fo.counts(gts)
        for p, m in enumerate(pops):
            st["pop_called"][s, p] = sum(not fo.is_missing(gts[i][0]) for i in m)
            st["pop_mask"][s, p] = sum(1 << a for a in np.flatnonzero(fo.counts(gts, m) > 0))
        st["flags"][s] = site_flags(gts)
        st["keep"][s] = True if spec.get("no_test") else fo.site_test(gts, pops, spec)
    return st


def assert_same_text(got, want):
    if got != want:
        g, w = got.split(b"\n"), want.split(b"\n")
        i = next((i for i, (a, b) in enumerate(zip(g, w)) if a != b), min(len(g), len(w)))
        pytest.fail("output row %d differs (%d bytes vs %d expected):\n  got  %r\n  want %r" %
                    (i, len(got), len(want), g[i] if i < len(g) else None, w[i] if i < len(w) else None))


def assert_stats(got, want, keys):
    for k in keys:
        a, b = np.asarray(got[k]).astype(np.int64), want[k]
        if not np.array_equal(a, b):
            s = int(np.flatnonzero((a != b).reshape(len(a), -1).any(axis=1))[0])
            pytest.fail("%s of site %d: %s, expected %s" % (k, s, a[s], b[s]))


def check(r, want):
    assert r.n_kept == len(want.kept)
    assert list(np.flatnonzero(r.stats["final"])) == want.kept
    assert r.flags == want.flags
    assert_same_text(r.bytes, want.bytes)


# ---- 1. emission against filter_lines ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mixed():
    """24 samples of ploidy 1 to 8 (three of each) among 7 unselected columns"""
    return make_geno(11, 900, mixed_ploidy(random.Random(11), 24), n_extra=7)


@pytest.mark.parametrize("fmt, freq_order", [("phased", False), ("bases", False), ("bases", True), ("alleles", False),
                                             ("alleles", True), ("coded", False), ("count", False)])
def test_output_formats(eng, mixed, fmt, freq_order):
    spec = spec_of(mixed, min_calls=2, max_het=0.95, min_freq=0.02)
    want = expect(mixed, spec, fmt, freq_order)
    assert 300 < len(want.kept) < len(mixed.lines)
    assert want.flags == FL_TIE | FL_PARTIAL        # tied counts and partly missing genotypes are emitted too
    check(run(eng, mixed, spec, fmt, freq_order), want)


@pytest.mark.parametrize("fmt, flag", [("diplo", FL_PARTIAL), ("count", FL_NOALLELE)])
def test_formats_the_command_line_refuses(eng, fmt, flag):
    """-of diplo with a partly missing kept genotype and -of count on a kept site without a called allele are refused by
    the command line on the flag bit pg_filter returns; with --partialToMissing / --minCalls 1 they are emitted"""
    g = make_geno(12, 700, [2] * 19, n_extra=3, all_missing=0.05)
    loose = spec_of(g, min_calls=0, min_alleles=0) if fmt == "count" else spec_of(g, min_calls=1)
    want = expect(g, loose, "phased")
    ing = ingest(eng, g)
    nk, flags = eng.filter(loose, contig_mask=ing[0], scaf_id=ing[1])
    assert flags == want.flags and flags & flag
    assert nk == len(want.kept) and list(np.flatnonzero(eng.filter_stats()["final"])) == want.kept
    spec = spec_of(g, partial_to_missing=True) if fmt == "diplo" else spec_of(g, min_calls=1)
    want = expect(g, spec, fmt)
    assert not want.flags & flag
    check(run(eng, g, spec, fmt, ing=ing), want)


@pytest.mark.parametrize("p2m", [False, True])
@pytest.mark.parametrize("fmt_in", ["phased", "diplo", "alleles"])
def test_input_formats(eng, fmt_in, p2m):
    rng = random.Random(13)
    ploidy = [2] * 21 if fmt_in == "diplo" else mixed_ploidy(rng, 21)
    g = make_geno(14 + len(fmt_in), 800, ploidy, fmt=fmt_in, n_extra=5)
    spec = spec_of(g, min_calls=2, max_het=0.8, min_freq=0.05, partial_to_missing=p2m)
    ing = ingest(eng, g)
    outs = [("phased", False), ("coded", False), ("alleles", True)] + ([("diplo", False)] if fmt_in == "diplo" else [])
    for fmt, freq_order in outs:
        want = expect(g, spec, fmt, freq_order)
        assert len(want.kept) > 100
        check(run(eng, g, spec, fmt, freq_order, ing=ing), want)


@pytest.mark.parametrize("n_samp", [1, 31, 32, 33, 64, 65, 203])
def test_sample_counts(eng, n_samp):
    """samples are formatted 32 at a time behind a warp scan of their lengths; the running offset carries over the steps"""
    rng = random.Random(n_samp)
    g = make_geno(100 + n_samp, 240 if n_samp > 100 else 400, mixed_ploidy(rng, n_samp), n_extra=n_samp // 3 + 2)
    spec = spec_of(g, min_calls=1)
    ing = ingest(eng, g)
    for fmt in ("alleles", "phased"):
        want = expect(g, spec, fmt)
        assert len(want.kept) > 100
        check(run(eng, g, spec, fmt, ing=ing), want)


# ---- 2. slabs and the emit API ----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def seam():
    """rows of unequal length: scaffold names of 1 to 40 characters and positions of 1 to 9 digits"""
    rng = random.Random(21)
    g = make_geno(21, 300, mixed_ploidy(rng, 13), n_extra=2)
    names = ["s%d" % k + "_" * rng.randint(0, 38) for k in range(300 // 37 + 1)]
    pos = np.cumsum([rng.choice([1, 9, 90, 900, 9000, 90000, 900000, 9000000]) for _ in range(300)])
    return relabel(g, [names[i // 37] for i in range(300)], pos)


def slabs(lens, cap):
    """(rows, bytes) of every call that a buffer of cap bytes gives, or the row that does not fit at all"""
    calls, r = [], 0
    while r < len(lens):
        n = nb = 0
        while r + n < len(lens) and nb + lens[r + n] <= cap:
            nb += lens[r + n]
            n += 1
        if n == 0:
            return calls, r
        calls.append((n, nb))
        r += n
    return calls, None


def test_caps_of_whole_rows_and_one_byte_less(eng, seam):
    from genomics_general_b200._lib import PgError
    spec = spec_of(seam, min_calls=1, max_het=0.9)
    want = expect(seam, spec, "alleles")
    lens = [len(r) for r in want.rows]
    assert len(set(lens)) >= 8
    ing = ingest(eng, seam)
    nk, _ = eng.filter(spec, contig_mask=ing[0], scaf_id=ing[1])
    assert nk == len(lens)
    for k in (1, 2, 3, 17, nk // 2, nk - 1, nk):
        for cap in (sum(lens[:k]), sum(lens[:k]) - 1):
            calls, stuck = slabs(lens, cap)
            if stuck is None:
                text, got = emit(eng, nk, "alleles", cap=cap)
                assert got == calls, (k, cap)
                assert got[0][0] == (k if cap == sum(lens[:k]) else k - 1)
                assert_same_text(text, want.bytes)
            else:
                with pytest.raises(PgError, match=r"row %d needs %d bytes, more than the %d of the buffer" %
                                   (stuck, lens[stuck], cap)):
                    emit(eng, nk, "alleles", cap=cap)


def test_row_larger_than_the_buffer_and_row0_at_the_end(eng, seam):
    from genomics_general_b200._lib import PgError
    spec = spec_of(seam, min_calls=1)
    want = expect(seam, spec, "phased")
    lens = [len(r) for r in want.rows]
    ing = ingest(eng, seam)
    nk, _ = eng.filter(spec, contig_mask=ing[0], scaf_id=ing[1])
    buf = np.zeros(1 << 16, np.uint8)
    for r in (0, nk // 3, nk - 1):
        with pytest.raises(PgError, match=r"row %d needs %d bytes, more than the %d of the buffer" % (r, lens[r], lens[r] - 1)):
            eng.filter_emit("phased", False, r, buf, lens[r] - 1)
        assert eng.filter_emit("phased", False, r, buf, lens[r]) == (1, lens[r])
        assert buf[:lens[r]].tobytes() == want.rows[r]
    assert eng.filter_emit("phased", False, nk, buf, len(buf)) == (0, 0)
    assert eng.filter_emit("coded", False, nk, buf, len(buf)) == (0, 0)


def test_offset_cache_across_formats_and_filters(eng, seam):
    spec = spec_of(seam, min_calls=1)
    ing = ingest(eng, seam)
    nk, _ = eng.filter(spec, contig_mask=ing[0], scaf_id=ing[1])
    for fmt, freq_order in [("alleles", False), ("coded", False), ("alleles", False), ("alleles", True), ("bases", True),
                            ("alleles", False)]:
        want = expect(seam, spec, fmt, freq_order)
        text, _ = emit(eng, nk, fmt, freq_order, cap=4096)
        assert_same_text(text, want.bytes)
    # a second filter on the same ingest, emitted in the format the offsets were last computed for
    spec2 = spec_of(seam, min_calls=10, max_het=0.5)
    want = expect(seam, spec2, "alleles")
    assert 10 < len(want.kept) < nk
    check(run(eng, seam, spec2, "alleles", cap=4096, ing=ing), want)


# ---- 3. grid-stride passes ---------------------------------------------------------------------------------------------
def test_grid_stride_over_sites_and_kept_rows(eng):
    g = make_geno(31, 150_000, [2, 3, 1, 2, 2], scaf_every=1000)
    spec = spec_of(g, min_calls=3, max_het=0.7)
    want = expect(g, spec, "phased")
    assert len(want.kept) > 40_000
    r = run(eng, g, spec, "phased", cap=len(want.bytes))
    assert r.calls == [(len(want.kept), len(want.bytes))]        # one write pass over every kept row
    check(r, want)
    assert_stats(r.stats, oracle_stats(g, spec), ("called", "het", "counts", "flags", "keep"))


@pytest.fixture(scope="module")
def thin_geno():
    """70 000 sites, scaffolds of 97 sites (so they change inside pods), positions 1 to 20 apart"""
    rng = random.Random(41)
    g = make_geno(41, 70_000, [2, 1, 2], scaf_every=97)
    pos = np.cumsum([rng.randint(1, 20) for _ in range(len(g.lines))])
    return relabel(g, [ln.split("\t", 1)[0] for ln in g.lines], pos)


@pytest.mark.parametrize("pod", [1, 3, 256, 257])
def test_thin_pods_across_blocks(eng, thin_geno, pod):
    """70 000 pods of 1 site span 274 blocks and 23 334 pods of 3 span 92; pods of 256 and 257 span 2 blocks, the second
    one partly full.  With pods of 1 no row is written: a pod's first site only sets the scaffold and position to measure
    from (filterGenotypes.py:41-44), so this case checks that every site comes out dropped."""
    g = thin_geno
    exclude = {"chr3", "chr250", "chr251"}
    spec = spec_of(g, min_calls=2, thin_dist=25, pod_size=pod)
    want = expect(g, spec, "phased", exclude=exclude)
    assert pod == 1 or len(want.kept) > 5000
    check(run(eng, g, spec, "phased", exclude=exclude), want)


# ---- 4. the site filter at its limits ----------------------------------------------------------------------------------
def split_sites(rng, ploidy, half, S):
    """random sites, and sites where the first `half` samples hold one allele and the others another"""
    sites = []
    for i in range(S):
        if i % 3:
            sites.append(random_alleles(rng, ploidy, (0.0, 0.1), True, 0.02))
            continue
        x, y = rng.sample("ACGT", 2)
        sites.append([[("N" if rng.random() < 0.1 else (x if k < half else y))] * pl for k, pl in enumerate(ploidy)])
        if i % 2:                                           # one minority allele: nearly fixed
            sites[-1][rng.randrange(len(ploidy))][0] = rng.choice("ACGT")
    return sites


PER_POP = ("min_pop_calls", "min_pop_alleles", "max_pop_alleles")


def per_pop_thresholds(pops, rng):
    """--minPopCalls and --min/maxPopAlleles that every population can meet, tight for a few populations on both sides of
    32 and loose for the rest, so that the verdicts depend on which population each threshold belongs to"""
    mpc = [0] * 64
    for p in (3, 37, 50, 61):
        mpc[p] = len(pops[p]) - p % 2                   # every member called, or all but one
    mpa, xpa = [0] * 64, [4] * 64
    for p, lo, hi in ((10, 1, 2), (37, 2, 4), (50, 0, 2)):
        mpa[p], xpa[p] = lo, hi
    if not pops[16]:
        mpa[16], xpa[16] = 1, 3                         # an empty list: the alleles of every sample
    loose_lo = [rng.choice([0, 1]) for _ in pops]       # at most what fixedDiffs asks of a population anyway
    loose_hi = [rng.choice([1, 2, 4]) for _ in pops]
    return mpc, (mpa, xpa), (loose_lo, loose_hi)


@pytest.mark.parametrize("with_empty", [False, True])
def test_64_populations(eng, with_empty):
    rng = random.Random(64 + with_empty)
    n = 40
    ploidy = [rng.choice([1, 2, 2, 3]) for _ in range(n)]
    S = 360
    g = make_geno(65, S, ploidy, n_extra=4, sites=split_sites(rng, ploidy, n // 2, S))
    # overlapping member lists inside each half of the samples; with_empty: some lists are empty (every sample)
    pops = [rng.sample(range(0, n // 2) if p < 32 else range(n // 2, n), rng.randint(2, n // 2)) for p in range(64)]
    if with_empty:
        for p in (5, 16, 40, 63):
            pops[p] = []
    mpc, (mpa, xpa), (loose_lo, loose_hi) = per_pop_thresholds(pops, rng)
    ing = ingest(eng, g)
    specs = [dict(min_pop_calls=mpc),
             dict(min_pop_alleles=mpa, max_pop_alleles=xpa),
             dict(fixed_diffs=True),
             dict(nearly_fixed_diff=0.6),
             dict(min_calls=0, min_pop_calls=mpc, min_pop_alleles=loose_lo, max_pop_alleles=loose_hi, fixed_diffs=True,
                  nearly_fixed_diff=0.9)]
    for kw in specs:
        spec = spec_of(g, pops=pops, **kw)
        want = expect(g, spec, "phased")
        if kw.get("fixed_diffs") and with_empty:
            # an empty list stands for every sample, so that population holds every allele of a varied site
            assert want.kept == []
        else:
            assert 10 < len(want.kept) < S - 10
        # the test can tell population p's thresholds from those of another population
        for other in ([p & 31 for p in range(64)], [63 - p for p in range(64)]):
            if any(k in kw for k in PER_POP) and want.kept:
                moved = dict(spec, **{k: [spec[k][q] for q in other] for k in PER_POP if k in kw})
                assert expect(g, moved, "phased").kept != want.kept
        r = run(eng, g, spec, "phased", ing=ing)
        assert_stats(r.stats, oracle_stats(g, spec), ("pop_called", "pop_mask", "keep"))
        check(r, want)
    from genomics_general_b200._lib import PgError
    with pytest.raises(PgError, match=r"pg_filter: 65 populations \(at most 64\)"):
        eng.filter(spec_of(g, pops=pops + [[0]]), contig_mask=ing[0], scaf_id=ing[1])


def probe(eng, g, spec, site, verdict):
    """pg_filter with spec: every site's verdict equals the oracle's, and `site`'s is `verdict`"""
    ing = ingest(eng, g)
    eng.filter(spec, contig_mask=ing[0], scaf_id=ing[1])
    keep = eng.filter_stats()["keep"].astype(bool)
    want = [fo.site_test(genotypes(g, s, spec), spec["pops"], spec) for s in range(len(g.lines))]
    assert want[site] == verdict, "the probe is not where it should be"
    assert list(keep) == want, (site, {k: v for k, v in spec.items() if k not in ("samp_hap0", "samp_ploidy")})


def around(x):
    """x, one ulp below, one ulp above"""
    return x, float(np.nextafter(x, -np.inf)), float(np.nextafter(x, np.inf))


MINOR = [(1, 2), (1, 3), (1, 4), (1, 5), (2, 5), (1, 6), (1, 7), (2, 7), (3, 7), (3, 8), (1, 10), (3, 10), (1, 12), (5, 12)]


def test_minor_frequency_on_its_thresholds(eng):
    """second / n >= minFreq and <= maxFreq in fp64: k of n called haploid alleles, the rest of 12 missing"""
    g = tokens_geno([["T"] * k + ["A"] * (n - k) + ["N"] * (12 - n) for k, n in MINOR], [1] * 12)
    for site, (k, n) in enumerate(MINOR):
        at, below, above = around(k / n)
        for thr, min_ok, max_ok in ((at, True, True), (below, True, False), (above, False, True)):
            probe(eng, g, spec_of(g, min_freq=thr), site, min_ok)
            probe(eng, g, spec_of(g, max_freq=thr), site, max_ok)


HET = [(1, 2), (1, 3), (2, 3), (1, 4), (3, 4), (1, 5), (2, 7), (5, 12), (1, 12), (12, 12)]


def test_het_fraction_on_its_thresholds_and_ieee_edges(eng):
    """het / called > maxHet drops: h het of c called diploid samples; and the sites without a called sample"""
    rows = [["A/T"] * h + ["A/A"] * (c - h) + ["N/N"] * (12 - c) for h, c in HET]
    rows.append(["A/N", "T/N"] + ["N/N"] * 10)          # two alleles, no called sample: 2 / 0 = inf, dropped
    rows.append(["A/N", "A/N"] + ["N/N"] * 10)          # one allele: maxHet is not evaluated
    rows.append(["N/N"] * 12)                           # no allele at all
    g = tokens_geno(rows, [2] * 12)
    base = dict(min_calls=0, min_alleles=0)
    for site, (h, c) in enumerate(HET):
        at, below, above = around(h / c)
        for thr, ok in ((at, True), (below, False), (above, True)):
            probe(eng, g, spec_of(g, max_het=thr, **base), site, ok)
    inf_site = len(HET)
    for thr in (0.0, 1.0, 1e308):
        probe(eng, g, spec_of(g, max_het=thr, **base), inf_site, False)
        probe(eng, g, spec_of(g, max_het=thr, **base), inf_site + 1, True)
        probe(eng, g, spec_of(g, max_het=thr, **base), inf_site + 2, True)
    probe(eng, g, spec_of(g, max_het=float("inf"), **base), inf_site, True)     # inf > inf is false
    # 0 / 0 cannot reach the predicate: with more than one allele, a sample that carries an allele is called or het


NFD = [("AAAN", "ATTN", "NNNN"), ("AAAT", "ATTT", "AATT"), ("AATN", "ATTT", "CCCC"), ("ATTN", "AAAA", "TTTT"),
       ("AAGN", "AGGN", "AAAA"), ("ACGT", "AACC", "GGTT"), ("ATNN", "AATN", "AAAT"), ("NNNN", "AAAA", "AAAA"),
       ("NNNN", "AAAA", "NNNN")]


def test_nearly_fixed_diff_on_its_thresholds(eng):
    """some |f_i - f_j| >= nearlyFixedDiff keeps; a population without a called allele leaves its pairs out"""
    g = tokens_geno([list("".join(r)) for r in NFD], [1] * 12)
    pops = [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9, 10, 11]]
    for site in range(len(NFD)):
        gts = genotypes(g, site, {})
        pf = [fo.freqs(fo.counts(gts, m)) for m in pops]
        d = np.concatenate([np.abs(pf[i] - pf[j]) for i in range(3) for j in range(i + 1, 3)])
        if np.isnan(d).all():                           # no pair with called alleles on both sides: never kept
            probe(eng, g, spec_of(g, pops=pops, nearly_fixed_diff=0.0), site, False)
            continue
        at, below, above = around(float(np.nanmax(d)))
        for thr, ok in ((at, True), (below, True), (above, False)):
            probe(eng, g, spec_of(g, pops=pops, nearly_fixed_diff=thr), site, ok)


# ---- 5. text layout ----------------------------------------------------------------------------------------------------
def layout_geno(seed, S=400):
    """data lines that start with blanks, runs of blanks between fields, LF and CRLF ends, comment and blank lines between
    data lines, positions written 0012 / +12 / +0012, and a last line without a newline"""
    rng = random.Random(seed)
    ploidy = [2, 1, 3, 2]
    body, lines = [], []
    for i in range(S):
        if rng.random() < 0.15:
            body.append(rng.choice(["# a comment", "#", "", "   ", "\t \t", "\r"]) + rng.choice(["\n", "\r\n"]))
        al = random_alleles(rng, ploidy, (0.0, 0.2), True, 0.0)
        toks = [token(rng, a, "phased") for a in al]
        pos = rng.choice(["%d", "%04d", "+%d", "+%04d"]) % (3 * i + 12)
        lead = [" ", "\t", "  \t "][i] if i < 3 else rng.choice(["", "", " ", "\t", "  \t ", "\t\t"])
        fields = ["chr%d" % (i // 60), pos] + toks
        text = lead + fields[0] + "".join(rng.choice(["\t", "\t", " ", "  ", "\t \t", " \t"]) + f for f in fields[1:])
        end = rng.choice(["\n", "\n", "\r\n", " \n", "\t\r\n"])
        body.append(text + (end if i < S - 1 else ""))
        lines.append(text + end)
    return Geno("".join(body).encode(), lines, "phased", range(4), ploidy, 4)


def test_text_layout_on_the_engine(eng):
    g = layout_geno(51)
    assert not g.body.endswith(b"\n")
    spec = spec_of(g, min_calls=3)
    ing = ingest(eng, g)
    for fmt in ("phased", "coded"):
        want = expect(g, spec, fmt)
        assert len(want.kept) > 100
        check(run(eng, g, spec, fmt, ing=ing), want)


@pytest.mark.parametrize("args", [["--minCalls", "3"], ["-of", "alleles", "--alleleOrder", "freq", "--exclude", "chr2"]])
def test_text_layout_through_the_command_line(tmp_path, monkeypatch, args):
    """the command line on the GPU engine and on the oracle-backed engine write the same bytes"""
    from genomics_general_b200.cli import filterGenotypes as F
    from oracle_engine_filter import FilterOracleEngine, HostArray
    g = layout_geno(52)
    path = tmp_path / "layout.geno"
    path.write_bytes(b"#CHROM\tPOS\ts0\ts1\ts2\ts3\r\n" + g.body)
    F.main(["-i", str(path), "-o", str(tmp_path / "gpu.out")] + args)
    with monkeypatch.context() as m:
        m.setattr(F, "Engine", FilterOracleEngine)
        m.setattr(F, "PinnedArray", HostArray)
        F.main(["-i", str(path), "-o", str(tmp_path / "oracle.out")] + args)
    got, ref = (tmp_path / "gpu.out").read_bytes(), (tmp_path / "oracle.out").read_bytes()
    spec = spec_of(g, min_calls=int(args[1]) if args[0] == "--minCalls" else 1)
    want = expect(g, spec, "alleles" if "alleles" in args else "phased", "freq" in args,
                  exclude={"chr2"} if "--exclude" in args else None)
    assert ref == b"#CHROM\tPOS\ts0\ts1\ts2\ts3\n" + want.bytes
    assert_same_text(got, ref)
