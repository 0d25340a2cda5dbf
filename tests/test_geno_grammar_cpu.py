"""The host .geno tokenizer (pg_geno_parse, csrc/geno_parse.cpp) against the grammar in plain Python (oracle/geno_oracle.py).

The host tokenizer serves the drop-in API and every file too large for device memory, and the device tokenizer's tests
take it as their reference at sizes the oracle cannot reach, so it is pinned here, without a GPU:
  - misreads it once had: a blank run that fits the fixed-width fast path's grid, a token longer than 8 alleles, a position
    outside int32, junk after the position digits;
  - seeded random texts in every format, ploidies 1-8 mixed in one file, requested columns in and out of file order, blank
    runs of 1-9 characters between fields (fast path hit and missed), comment and blank lines, CRLF, no final newline;
  - one thread and several on bodies over 4 MiB, where the line index is split between threads;
  - errors: the same data line, kind and column as the oracle, the first bad line when there are several."""
import numpy as np
import pytest

from genomics_general_b200._lib import PgError
from geno_text import columns_of, error_of, host_parse, random_take, random_text, token
from oracle import geno_oracle as go


def assert_host_is_oracle(body, fmt, take, strict=0, threads=1):
    want = go.parse(body, fmt, columns_of(take), strict)
    if want.error is not None:
        with pytest.raises(PgError) as e:
            host_parse(body, fmt, take, threads)
        assert error_of(str(e.value)) == want.error, (str(e.value), want.error)
        return want
    geno, pos, newsc, off = host_parse(body, fmt, take, threads)
    assert np.array_equal(geno, want.geno)
    assert np.array_equal(pos, want.pos)
    assert np.array_equal(newsc, want.new_scaffold)
    assert np.array_equal(off, want.line_off)
    return want


# ---- misreads of the host tokenizer ----------------------------------------------------------------------------------------
def test_blank_run_fitting_the_diplo_grid_is_a_separator():
    # "A   C" is 5 bytes: the grid of two 1-byte tokens and one separator would read it as A, blank
    w = assert_host_is_oracle(b"chr1 100 A   C\n", "diplo", [(0, 2), (1, 2)])
    assert w.geno.tolist() == [[0, 0, 1, 1]]


def test_blank_run_fitting_the_phased_grid_is_a_separator():
    # file columns 0 and 2 of "A|T\t\t\t\tG|C\tT|T": 15 bytes = the grid of four 3-byte tokens, whose column 2 is "G|C"
    w = assert_host_is_oracle(b"chr1 100 A|T\t\t\t\tG|C\tT|T\n", "phased", [(0, 2), (2, 2)])
    assert w.geno.tolist() == [[0, 3, 3, 3]]
    for fmt, line in (("pairs", b"c 1 AT    GC TT\n"), ("haplo", b"c 1 A   G T\n")):
        pl = 2 if fmt == "pairs" else 1
        assert_host_is_oracle(line, fmt, [(0, pl), (2, pl)])


@pytest.mark.parametrize("fmt", ["phased", "pairs"])
def test_token_of_more_alleles_than_the_ploidy_is_refused(fmt):
    for n in (9, 10, 17):
        tok = "|".join("ACGT"[i % 4] for i in range(n)) if fmt == "phased" else "".join("ACGT"[i % 4] for i in range(n))
        body = ("c 5 %s\n" % tok).encode()
        w = assert_host_is_oracle(body, fmt, [(0, 8)])
        assert w.error == ("ploidy", 1, 1)
    assert assert_host_is_oracle(b"c 5 " + (b"A|C|G|T|A|C|G|T" if fmt == "phased" else b"ACGTACGT") + b"\n", fmt,
                                 [(0, 8)]).error is None


@pytest.mark.parametrize("p,ok", [("3000000000", False), ("2147483647", True), ("2147483648", False), ("-2147483648", True),
                                  ("-2147483649", False), ("+2147483647", True), ("99999999999999999999999999", False),
                                  ("00000000000000000000000012", True), ("4294967296", False), ("-0", True)])
def test_position_outside_int32_is_refused(p, ok):
    body = ("c 1 A|T\nc %s A|T\nc 3 A|T\n" % p).encode()
    w = assert_host_is_oracle(body, "phased", [(0, 2)])
    assert (w.error is None) == ok
    if not ok:
        assert w.error == ("range", 2, 0)


def test_junk_after_the_position_digits_is_not_a_genotype_column():
    w = assert_host_is_oracle(b"c 12x A|T C|G\nc 13 A|T C|G\n", "phased", [(0, 2), (1, 2)])
    assert w.pos.tolist() == [12, 13] and w.geno.tolist() == [[0, 3, 1, 2]] * 2


# ---- random texts --------------------------------------------------------------------------------------------------------
FORMAT_PLOIDIES = {"phased": range(1, 9), "pairs": range(1, 9), "diplo": (1, 2), "haplo": (1,)}


@pytest.mark.parametrize("fmt", sorted(FORMAT_PLOIDIES))
@pytest.mark.parametrize("seed", range(4))
def test_random_texts_equal_the_oracle(fmt, seed):
    rng = np.random.default_rng(100 * seed + len(fmt))
    n_cols = int(rng.integers(1, 12))
    take = random_take(rng, n_cols, int(rng.integers(1, n_cols + 1)), list(FORMAT_PLOIDIES[fmt]), shuffle=seed % 2 == 0)
    body = random_text(rng, fmt, 400, n_cols, take, sep="|/"[seed % 2])
    assert go.parse(body, fmt, columns_of(take)).error is None
    assert_host_is_oracle(body, fmt, take)


@pytest.mark.parametrize("fmt", sorted(FORMAT_PLOIDIES))
def test_fixed_width_texts_with_blank_runs_equal_the_oracle(fmt):
    """uniform ploidy (the fast path's case) with single-blank separators on most lines and blank runs of 1-3 on others, so
    that many lines fit the grid by length alone"""
    rng = np.random.default_rng(7 + len(fmt))
    pl = 1 if fmt == "haplo" else 2
    n_cols = 6
    for take in ([(c, pl) for c in range(n_cols)], [(4, pl), (1, pl), (2, pl)], [(5, pl)]):
        lines = []
        for s in range(600):
            toks = [token(rng, fmt, pl) for _ in range(n_cols)]
            seps = ["\t" if s % 3 == 0 or rng.random() < 0.6 else " " * int(rng.integers(1, 4)) for _ in toks]
            lines.append("c%d\t%d" % (s // 200, s) + "".join(x + t for x, t in zip(seps, toks)))
        body = ("\n".join(lines) + "\n").encode()
        assert_host_is_oracle(body, fmt, take)


def test_layout_lines_crlf_and_final_newline():
    rng = np.random.default_rng(3)
    take = [(2, 2), (0, 3), (4, 1)]
    body = random_text(rng, "phased", 300, 5, take)
    for text in (body, body.rstrip(b"\n"), body + b"\n\n  \t\n# trailing comment", b"\n\n" + body, body.replace(b"\n", b"\r\n")):
        assert_host_is_oracle(text, "phased", take)
    assert_host_is_oracle(b"", "phased", take)
    assert_host_is_oracle(b"# only a comment\n\t \n", "phased", take)


@pytest.mark.parametrize("fmt", ["phased", "diplo"])
def test_threads_split_a_large_body(fmt):
    rng = np.random.default_rng(11)
    take = [(1, 2), (0, 2)] if fmt == "diplo" else [(3, 2), (0, 1), (1, 4)]
    parts, size = [], 0
    while size < (4 << 20) + 12345:
        p = random_text(rng, fmt, 2000, 4, take, runs=(1, 3), scaffolds=3)
        p = p if p.endswith(b"\n") else p + b"\n"
        parts.append(p)
        size += len(p)
    body = b"".join(parts)
    want = assert_host_is_oracle(body, fmt, take, threads=1)
    for threads in (3, 8):
        geno, pos, newsc, off = host_parse(body, fmt, take, threads)
        assert np.array_equal(geno, want.geno) and np.array_equal(pos, want.pos)
        assert np.array_equal(newsc, want.new_scaffold) and np.array_equal(off, want.line_off)


# ---- errors ---------------------------------------------------------------------------------------------------------------
BAD_LINES = [
    (b"c", "no_pos"), (b"  c  \r", "no_pos"), (b"c x A|T C|G", "pos"), (b"c - A|T C|G", "pos"), (b"c +x A|T C|G", "pos"),
    (b"c 2147483648 A|T C|G", "range"), (b"c 1 A C|G", "ploidy"), (b"c 1 A|T C|G|T", "ploidy"), (b"c 1 A|T|", "columns"),
    (b"c 1 A|T", "columns"), (b"c 1", "columns"), (b"c 1 A|T C|G|A", "ploidy"),
]


@pytest.mark.parametrize("bad,kind", BAD_LINES)
def test_error_names_the_line_kind_and_column(bad, kind):
    good = b"c 1 A|T C|G\n"
    body = good * 5 + bad + b"\n" + good * 3
    w = assert_host_is_oracle(body, "phased", [(0, 2), (1, 2)])
    assert w.error[:2] == (kind, 6)


def test_first_of_several_bad_lines_is_reported():
    rng = np.random.default_rng(5)
    take = [(0, 2), (2, 2)]
    lines = random_text(rng, "phased", 3000, 3, take, decorate=False).split(b"\n")
    for i, bad in ((1700, b"c 1 A|T|G x C|G"), (900, b"c -"), (2500, b"c 1 A")):
        lines[i] = bad
    body = b"\n".join(lines)
    w = assert_host_is_oracle(body, "phased", take, threads=1)
    assert w.error == ("pos", 901, 0)


@pytest.mark.parametrize("fmt,pl,tok", [("diplo", 3, "A"), ("haplo", 2, "A"), ("pairs", 3, "AC"), ("pairs", 2, "ACG"),
                                        ("phased", 1, "A|C")])
def test_ploidy_errors_of_every_format(fmt, pl, tok):
    body = ("c 1 %s %s\n" % (tok, tok)).encode()
    assert assert_host_is_oracle(body, fmt, [(1, pl)]).error == ("ploidy", 1, 2)
