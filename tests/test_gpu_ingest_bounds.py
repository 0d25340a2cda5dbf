"""The device .geno tokenizer (pg_ingest_text / pg_ingest_file / pg_ingest_file_range, csrc/ingest.cu) at the edges of its
geometry, against the grammar in plain Python (oracle/geno_oracle.py) and, at sizes the oracle cannot reach, against the
host tokenizer (pg_geno_parse), which tests/test_geno_grammar_cpu.py pins to the oracle.

  1. the line index: line starts at the 4 096-byte blocks and 16-byte thread segments of k_count_starts / k_write_starts,
     '\\n' as a block's last byte, leading-blank and comment lines across a block seam, a final line that ends a block with
     and without '\\n', every text length mod 4;
  2. the warp steps of k_parse_lines: line starts at every offset mod 4, fields starting at the first and the last byte of a
     128-byte step, tokens across steps, lines of more than 32 steps, a '\\n' opening a step, fields past the header's
     columns, tokens of 2 * ploidy + 1 and + 2 characters;
  3. the grid-stride loops of k_parse_lines and k_scaffold_flags, with scaffold changes on both sides of the flag grid;
  4. the double-buffered slabs of the host-to-device copy: a text over two slabs from memory, from a file with a header
     offset and from a byte range inside the file, with 1 and 7 staging threads;
  5. one engine reused: a shorter text after a longer one, strict levels 1 -> 0 -> 2, an ingest after the upload of a wider
     matrix, and the packed companion after an ingest equal to the one after an upload;
  6. strict levels 1 and 2 on every token kind and width;
  7. errors: the same line and kind as the host, the first of several bad lines on different warps, every error code;
  8. popgen on a >1 M-line ingest equal, bit for bit, to popgen after the upload of the host-parsed matrix.
Every case checks geno, pos, new_scaffold and line_off (or the error), the passes that ran (eng.last_timings()) and, where
it aims at a seam, that the geometry of the ingest (eng.ingest_geometry()) put the case past it.

Not covered: the device flags a new scaffold where the 64-bit FNV-1a hashes of two scaffold names differ, not their bytes;
two names with the same hash would read as one scaffold.  No such collision is built here."""
import os

import numpy as np
import pytest

from genomics_general_b200._lib import PgError
from geno_text import FMT, columns_of, device_maps, error_of, host_parse, random_take, random_text
from oracle import geno_oracle as go

pytestmark = pytest.mark.gpu

PASSES = {"text_h2d", "ingest_index", "ingest_parse"}


@pytest.fixture(scope="module")
def eng():
    from genomics_general_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def geom(eng):
    """the geometry constants of the ingest, read from the device after a one-line ingest"""
    import torch
    col_hap, col_pl, H = device_maps([(0, 1)], 1)
    eng.ingest_text(b"c 1 A\n", FMT["haplo"], col_hap, col_pl, H)
    eng.ingest_meta(1)
    g = eng.ingest_geometry()
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    assert g["parse_warps"] == 8 and g["flag_threads"] == 256 and g["slabs"] == 1
    g["sm_count"] = sm
    g["parse_grid_lines"] = sm * 64 * 8          # k_parse_lines: at most sm_count * 64 blocks of 8 warps, one line per warp
    g["flag_grid_lines"] = 4096 * 256            # k_scaffold_flags: at most 4 096 blocks of 256 threads
    return g


def dev_parse(eng, body, fmt, take, n_cols, strict=0, via=None):
    """the device tokenizer on body -> (geno, pos, new_scaffold, line_off) or the error (kind, line, column)"""
    col_hap, col_pl, H = device_maps(take, n_cols)
    eng.set_strict_ingest(strict)
    try:
        S = via(col_hap, col_pl, H) if via else eng.ingest_text(body, FMT[fmt], col_hap, col_pl, H)
    except PgError as e:
        return error_of(str(e))
    finally:
        eng.set_strict_ingest(0)
    assert PASSES <= set(eng.last_timings()) or S == 0
    pos, newsc, off = eng.ingest_meta(S)
    g = eng.download(0, S)[0] if S else np.zeros((0, H), np.int8)
    return g, pos, newsc, off


def assert_dev_is(got, want):
    """got: dev_parse's result; want: an oracle Parsed, a host result tuple or an error tuple"""
    if isinstance(want, go.Parsed):
        want = want.error if want.error is not None else (want.geno, want.pos, want.new_scaffold, want.line_off)
    if isinstance(want[0], str):
        assert got == want
        return
    assert not isinstance(got[0], str), got
    for name, a, b in zip(("geno", "pos", "new_scaffold", "line_off"), got, want):
        assert a.shape == b.shape and np.array_equal(a, b), name


def check_oracle(eng, body, fmt, take, n_cols, strict=0):
    want = go.parse(body, fmt, columns_of(take), strict)
    assert_dev_is(dev_parse(eng, body, fmt, take, n_cols, strict), want)
    return want


def line_of(i, n, pad=" "):
    """a phased line of one diploid sample, n bytes long with its '\\n' (n >= 12), padded with blanks at the end"""
    s = "s%d %d %s|%s" % (i % 7, i, "ACGTN"[i % 5], "ACGTN"[(i // 5) % 5])
    assert len(s) + 1 <= n, (s, n)
    return s + pad * (n - 1 - len(s)) + "\n"


# ---- 1. the line index -----------------------------------------------------------------------------------------------------
def test_line_index_block_and_segment_seams(eng, geom):
    B = geom["index_block_bytes"]
    rng = np.random.default_rng(1)
    out, n = [], 0

    def put(s):
        nonlocal n
        out.append(s)
        n += len(s)

    def fill_to(target):
        """lines of 16..200 bytes, the last ones sized so that the next byte written is at `target`"""
        while target - n > 400:
            put(line_of(len(out), int(rng.integers(16, 201))))
        if target - n > 200:
            put(line_of(len(out), (target - n) // 2))
        put(line_of(len(out), target - n))

    for k in range(1, 6):
        fill_to(k * B)                                             # a line starts at 4096 k
        if k == 2:
            put("   \t" + line_of(len(out), 40))                   # a leading-blank line across nothing: starts at the seam
        if k == 3:
            fill_to(k * B + 16 * 7)                                 # a start at 16 k inside the block
    fill_to(6 * B - 30)                                            # a comment line across the seam of block 6
    put("# comment across the seam " + "x" * 20 + "\n")
    fill_to(7 * B - 20)                                            # a leading-blank line across the seam of block 7
    put("  \t " + line_of(len(out), 60))
    fill_to(8 * B - 1)                                             # '\n' is the last byte of block 7
    put("\n")
    fill_to(9 * B - 20)
    for k in range(1, 40):
        fill_to(9 * B + 16 * k)                                     # starts at consecutive 16-byte segments
    body = "".join(out).encode()
    assert body[8 * B - 1:8 * B] == b"\n" and body[6 * B - 30:6 * B - 29] == b"#"
    take = [(0, 2)]
    check_oracle(eng, body, "phased", take, 1)
    # the final line ends exactly at a block end, with and without its '\n'
    for end in (b"", b"\n"):
        text = body + line_of(0, 10 * B - len(body) + (0 if end else 1)).encode()
        text = text if end else text[:-1]
        assert len(text) == 10 * B
        check_oracle(eng, text, "phased", take, 1)
    # every text length mod 4, and texts shorter than 4 bytes
    for extra in (b"", b" ", b"  ", b"\t\r\n"):
        for cut in range(0, 4):
            text = body[:len(body) - cut] + extra
            check_oracle(eng, text, "phased", take, 1)
    for tiny in (b"", b"\n", b"#\n", b" \t\n", b"c", b"c 1", b"c 1 "):
        check_oracle(eng, tiny, "phased", take, 1)


# ---- 2. the warp steps -----------------------------------------------------------------------------------------------------
def field_starts(body):
    """(line start, [field starts]) of every data line"""
    out = []
    for off, line in go.data_lines(body):
        st = [off + j for j in range(len(line)) if line[j:j + 1] not in go.BLANKS and (j == 0 or line[j - 1:j] in go.BLANKS)]
        out.append((off, st))
    return out


def test_warp_steps(eng):
    rng = np.random.default_rng(2)
    take = random_take(rng, 30, 20, [1, 2, 3, 5, 8])
    body = random_text(rng, "phased", 1500, 30, take, runs=(1, 9))
    want = check_oracle(eng, body, "phased", take, 30)
    assert want.error is None
    # the text reached the step edges it aims at
    starts = field_starts(body)
    mods = {(s - (l0 & ~3)) % 128 for l0, st in starts for s in st}
    assert {0, 127} <= mods
    assert {l0 % 4 for l0, _ in starts} == {0, 1, 2, 3}
    # lines whose '\n' is the first byte of their second or third step, after starts at every offset mod 4
    out, n = [], 0
    for i in range(400):
        ln = line_of(i, int(rng.integers(16, 40))) if i % 2 else line_of(i, 129 + 128 * (i % 4 == 2) - n % 4)
        out.append(ln)
        n += len(ln)
    body = "".join(out).encode()
    ends = [(body.find(b"\n", l0) - (l0 & ~3)) for l0, _ in field_starts(body)]
    assert ends.count(128) > 50 and ends.count(256) > 50
    check_oracle(eng, body, "phased", [(0, 2)], 1)


def test_lines_of_more_than_32_steps(eng):
    rng = np.random.default_rng(3)
    take = random_take(rng, 1500, 1500, [2])
    body = random_text(rng, "phased", 40, 1500, take, runs=(1, 2))
    assert min(len(l) for _, l in go.data_lines(body)) > 32 * 128
    check_oracle(eng, body, "phased", take, 1500)
    # only a few of the columns, far into the line, and fields past the header's columns
    take = [(1499, 2), (3, 2), (1200, 2)]
    check_oracle(eng, body, "phased", take, 1500)
    check_oracle(eng, body, "phased", [(1299, 2), (3, 2), (1200, 2)], 1300)
    check_oracle(eng, body, "phased", [(2, 2), (0, 2)], 3)


@pytest.mark.parametrize("fmt", ["phased", "pairs"])
def test_token_widths_at_the_length_cut(eng, fmt):
    for pl in range(1, 9):
        for extra in (0, 1, 2):
            w = (2 * pl - 1 if fmt == "phased" else pl) if extra == 0 else 2 * pl + extra
            if fmt == "phased":
                tok = "".join("ACGT"[(i // 2) % 4] if i % 2 == 0 else "|" for i in range(w))
            else:
                tok = "".join("ACGT"[i % 4] for i in range(w))
            body = ("c 1 %s A\nc 2 %s A\n" % (tok, tok)).encode()
            want = check_oracle(eng, body, fmt, [(0, pl)], 2)
            assert (want.error is None) == (extra == 0), (pl, extra, want.error)


# ---- 3 and 8. the grids, at scale ------------------------------------------------------------------------------------------
def numpy_phased_text(rng, S, n_samp, scaf_at, pad_max=3):
    """S phased lines of n_samp diploid samples built with numpy: scaffold names change at the line indices scaf_at, every
    line gets 0..pad_max trailing blanks so that line lengths vary.  -> (bytes, geno int8 [S, 2 n_samp], pos int32 [S])"""
    geno = rng.integers(-1, 4, size=(S, 2 * n_samp)).astype(np.int8)
    pos = np.cumsum(rng.integers(1, 50, size=S)).astype(np.int32)
    ch = np.frombuffer(b"ACGTN", np.uint8)[np.where(geno < 0, 4, geno)]
    scaf = np.searchsorted(np.asarray(scaf_at), np.arange(S), side="right")
    W = 6 + 1 + 10 + n_samp * 4 + pad_max + 1
    buf = np.zeros((S, W), np.uint8)                       # 0 = no byte
    buf[:, 0:4] = np.frombuffer(b"scaf", np.uint8)
    buf[:, 4] = ord("A") + scaf % 26
    buf[:, 5] = ord("A") + scaf // 26 % 26
    buf[:, 6] = ord("\t")
    p = pos.astype(np.int64)
    for d in range(10):
        buf[:, 16 - d] = ord("0") + (p // 10 ** d) % 10
    for k in range(n_samp):
        o = 17 + 4 * k
        buf[:, o] = ord("\t")
        buf[:, o + 1] = ch[:, 2 * k]
        buf[:, o + 2] = ord("|")
        buf[:, o + 3] = ch[:, 2 * k + 1]
    pad = rng.integers(0, pad_max + 1, size=S)
    for j in range(pad_max):
        buf[:, 17 + 4 * n_samp + j] = np.where(j < pad, ord(" "), 0)
    buf[:, -1] = ord("\n")
    flat = buf.ravel()
    return flat[flat != 0].tobytes(), geno, pos


@pytest.fixture(scope="module")
def big(geom):
    """a text of more lines than one k_scaffold_flags grid covers and more bytes than two slabs, scaffold changes on both
    sides of the flag grid seam and at the parse grid seam"""
    rng = np.random.default_rng(8)
    F, P = geom["flag_grid_lines"], geom["parse_grid_lines"]
    n_samp = 36
    line = 17 + 4 * n_samp + 2.5
    S = max(F + 5000, int(2.2 * geom["slab_bytes"] / line))
    scaf_at = sorted({1, 1000, P - 1, P, P + 1, F - 2, F - 1, F, F + 1, F + 3, S - 1})
    body, g, pos = numpy_phased_text(rng, S, n_samp, scaf_at)
    assert len(body) > 2 * geom["slab_bytes"] and S > F
    return dict(body=body, geno=g, pos=pos, n_samp=n_samp, S=S, scaf_at=scaf_at)


def test_grids_past_one_parse_grid(eng, geom):
    rng = np.random.default_rng(9)
    S = geom["parse_grid_lines"] + 3000
    body, g, pos = numpy_phased_text(rng, S, 2, [S // 2, geom["parse_grid_lines"]])
    take = [(1, 2), (0, 2)]
    got = dev_parse(eng, body, "phased", take, 2)
    gm = eng.ingest_geometry()
    assert gm["parse_warps"] == geom["parse_grid_lines"] and S > gm["parse_warps"]
    assert_dev_is(got, host_parse(body, "phased", take, threads=4))
    assert np.array_equal(got[0], g[:, [2, 3, 0, 1]]) and np.array_equal(got[1], pos)


def test_grids_and_slabs_at_scale(eng, geom, big, tmp_path):
    body, S = big["body"], big["S"]
    take = [(k, 2) for k in range(big["n_samp"])]
    host = host_parse(body, "phased", take, threads=8)
    assert np.array_equal(host[0], big["geno"]) and np.array_equal(host[1], big["pos"])
    flags = np.zeros(S, np.int8)
    flags[0] = 1
    flags[[a for a in big["scaf_at"] if a < S]] = 1
    assert np.array_equal(host[2], flags)
    slab = geom["slab_bytes"]
    seams = [k * slab for k in range(1, len(body) // slab + 1)]
    starts = host[3]
    for s in seams:                                        # a line straddles every slab seam
        i = np.searchsorted(starts, s)
        assert i < S and starts[i] != s
    path = str(tmp_path / "big.geno")
    header = b"#CHROM\tPOS\t" + b"\t".join(b"s%d" % k for k in range(big["n_samp"])) + b"\n"
    with open(path, "wb") as f:
        f.write(header)
        f.write(body)
    lo_line = 12345
    byte_lo = int(starts[lo_line])
    col_hap, col_pl, H = device_maps(take, big["n_samp"])
    old = os.environ.get("PG_INGEST_THREADS")
    try:
        for threads in ("1", "7"):
            os.environ["PG_INGEST_THREADS"] = threads
            got = dev_parse(eng, body, "phased", take, big["n_samp"])
            gm = eng.ingest_geometry()
            assert gm["slabs"] >= 3 and gm["flag_threads"] == geom["flag_grid_lines"] and S > gm["flag_threads"]
            assert_dev_is(got, host)
            got = dev_parse(eng, None, "phased", take, big["n_samp"],
                            via=lambda ch, cp, h: eng.ingest_file(path, len(header), FMT["phased"], ch, cp, h))
            assert eng.ingest_geometry()["slabs"] >= 3
            assert_dev_is(got, host)
            got = dev_parse(eng, None, "phased", take, big["n_samp"],
                            via=lambda ch, cp, h: eng.ingest_file_range(path, len(header) + byte_lo, -1, FMT["phased"], ch, cp, h))
            assert eng.ingest_geometry()["slabs"] >= 3
            ng = host[2][lo_line:].copy()
            ng[0] = 1
            assert_dev_is(got, (host[0][lo_line:], host[1][lo_line:], ng, host[3][lo_line:] - byte_lo))
    finally:
        if old is None:
            os.environ.pop("PG_INGEST_THREADS", None)
        else:
            os.environ["PG_INGEST_THREADS"] = old


def test_popgen_on_a_large_ingest_equals_popgen_on_the_upload(eng, big):
    body, S, n = big["body"], big["S"], big["n_samp"]
    take = [(k, 2) for k in range(n)]
    col_hap, col_pl, H = device_maps(take, n)
    hap_pop = np.repeat(np.arange(4), H // 4).astype(np.int32)
    lo = np.arange(0, S, 50000, dtype=np.int64)
    hi = np.minimum(lo + 50000, S)
    eng.ingest_text(body, FMT["phased"], col_hap, col_pl, H)
    eng.ingest_meta(S)
    eng.set_pops(hap_pop, 4)
    eng.set_windows(lo, hi)
    a = eng.popgen(100, 0.01)
    eng.upload(host_parse(body, "phased", take, threads=8)[0], big["pos"])
    eng.set_pops(hap_pop, 4)
    eng.set_windows(lo, hi)
    b = eng.popgen(100, 0.01)
    for k in ("pi", "dxy", "fst", "sites", "pos_sum", "path"):
        assert np.array_equal(a[k], b[k], equal_nan=True), k


# ---- 5. reuse of one engine ------------------------------------------------------------------------------------------------
def test_reuse_of_one_engine(eng, geom):
    rng = np.random.default_rng(5)
    take = random_take(rng, 9, 6, [1, 2, 3])
    long_body = random_text(rng, "phased", 3000, 9, take)
    short_body = random_text(rng, "phased", 50, 9, take)
    check_oracle(eng, long_body, "phased", take, 9)
    check_oracle(eng, short_body, "phased", take, 9)
    # strict 1 -> 0 -> 2 on one context
    strict_take = [(0, 2), (2, 2)]
    sbody = b"c 1 A|T x G/C\nc 2 N|N x A|A\nc 3 A|? x G|G\n"
    for level in (1, 0, 2):
        check_oracle(eng, sbody, "phased", strict_take, 3, strict=level)
    # an ingest after the upload of a wider matrix
    eng.upload(rng.integers(-1, 4, size=(5000, 300)).astype(np.int8), np.arange(5000, dtype=np.int32))
    check_oracle(eng, short_body, "phased", take, 9)


def test_packed_companion_after_an_ingest_equals_the_upload(eng):
    rng = np.random.default_rng(6)
    take = random_take(rng, 20, 13, [1, 2, 3, 5])
    H = sum(pl for _, pl in take)
    assert H % 32
    body = random_text(rng, "phased", 2000, 20, take)
    g, pos, _, _ = dev_parse(eng, body, "phased", take, 20)
    S = len(pos)
    packed, cls = eng.packed_rows(0, S), eng.site_classes(0, S)
    assert packed is not None
    eng.upload(g, pos)
    assert np.array_equal(eng.packed_rows(0, S), packed)
    c2 = eng.site_classes(0, S)
    assert (cls is None) == (c2 is None) and (cls is None or np.array_equal(cls, c2))


# ---- 6. strict levels ------------------------------------------------------------------------------------------------------
STRICT_TOKENS = {
    "phased": ["A", "A|T", "A/T", "A|T|G", "A|T|", "N|N", "a|T", "A|x", "A?T", "-|-", "A|T|G|C|A|C|G|T", "ACGT"],
    "pairs": ["A", "AT", "ATG", "NN", "aT", "A-", "ACGTACGT"],
    "diplo": ["A", "K", "N", "k", "X", "AT", "-"],
    "haplo": ["A", "N", "a", "AT", "-", "x"],
}


@pytest.mark.parametrize("fmt", sorted(STRICT_TOKENS))
@pytest.mark.parametrize("strict", [1, 2])
def test_strict_levels_on_every_token_kind_and_width(eng, fmt, strict):
    pls = {"phased": (1, 2, 3, 4, 8), "pairs": (1, 2, 3, 8), "diplo": (1, 2, 3), "haplo": (1, 2)}[fmt]
    seen = set()
    for pl in pls:
        for tok in STRICT_TOKENS[fmt]:
            body = ("c 1 %s %s\nc 2 %s %s\n" % (tok, tok, tok, tok)).encode()
            want = check_oracle(eng, body, fmt, [(1, pl)], 2, strict=strict)
            seen.add(None if want.error is None else want.error[0])
    assert None in seen and "ploidy" in seen and ("char" in seen) == (strict == 1)


# ---- 7. errors -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad,kind,strict", [
    (b"c", "no_pos", 0), (b"c x A|T C|G", "pos", 0), (b"c -", "pos", 0), (b"c 3000000000 A|T C|G", "range", 0),
    (b"c -2147483649 A|T C|G", "range", 0), (b"c 99999999999999999999999 A|T C|G", "range", 0),
    (b"c 1 A C|G", "ploidy", 0), (b"c 1 A|T C|G|T", "ploidy", 0), (b"c 1 A|T", "columns", 0), (b"c 1", "columns", 0),
    (b"c 1 A|T C|x", "char", 1), (b"c 1 A|T C|", "ploidy", 2), (b"c x A T", "pos", 0), (b"c 3000000000 A|T C", "range", 0),
    (b"c 1 A|T C|?", "char", 1)])
def test_error_kinds_match_the_host_and_the_oracle(eng, bad, kind, strict):
    good = b"c 1 A|T C|G\n"
    body = good * 300 + bad + b"\n" + good * 300
    take = [(0, 2), (1, 2)]
    want = check_oracle(eng, body, "phased", take, 2, strict=strict)
    assert want.error[:2] == (kind, 301)
    if strict == 0:
        with pytest.raises(PgError) as e:
            host_parse(body, "phased", take)
        assert error_of(str(e.value)) == want.error


def test_first_of_several_bad_lines_on_different_warps(eng, geom):
    rng = np.random.default_rng(7)
    S = geom["parse_grid_lines"] + 5000
    body, _, _ = numpy_phased_text(rng, S, 2, [10])
    lines = body.split(b"\n")
    take = [(0, 2), (1, 2)]
    first = S // 2 + 123
    bad = {S - 10: b"c x A|T C|G", geom["parse_grid_lines"] + 7: b"c 1 A|T", first + 5000: b"c 1 A C|G",
           first: b"c 1 A|T C|G|T", S - 3: b"c"}
    for i, b in bad.items():
        lines[i] = b
    body = b"\n".join(lines)
    got = dev_parse(eng, body, "phased", take, 2)
    assert got == ("ploidy", first + 1, 2)
    with pytest.raises(PgError) as e:
        host_parse(body, "phased", take)
    assert error_of(str(e.value)) == got
