"""genoToSeq's device index and transpose (pg_seq_*) against the plain Python statement (tests/oracle_engine_seq.py) on
seeded inputs at the transpose's edges: site counts off the 256-site tile and a single site, 1 and 33+ sequences, tokens of
width 1-15, --splitPhased ploidies 1-8, a sequence cut over many small slabs, thousands of one-site windows, lines longer
than one 128-byte warp step, comment lines, CRLF, and the first offending line and column of the index."""
import random

import numpy as np
import pytest

from oracle_engine_seq import SeqOracleEngine

pytestmark = pytest.mark.gpu

BASES = "ACGTNacgtn-RYKMSW"


@pytest.fixture(scope="module")
def eng():
    from genomics_general_b200.engine import Engine
    with Engine(0) as e:
        yield e


def make_text(rng, S, widths, crlf=False, comments=False, scaffolds=1):
    lines = []
    for s in range(S):
        if comments and s % 7 == 3:
            lines.append("# comment %d" % s)
        toks = ["".join(rng.choice(BASES) for _ in range(w)) for w in widths]
        lines.append("\t".join(["sc%d" % (s * scaffolds // max(S, 1)), str(10 + 3 * s)] + toks))
    nl = "\r\n" if crlf else "\n"
    return (nl.join(lines) + nl).encode()


def both(eng, text, col_slot, slot_width, exact, fmt, nto, names, seq_slot, seq_byte, seq_width, lo, hi, cap):
    """(index error, meta, emitted bytes) from the device and from the oracle"""
    res = []
    for e in (eng, SeqOracleEngine()):
        S, err = e.seq_index(col_slot, slot_width, exact, data=text)
        if err[0]:
            res.append((S, err, None, None))
            continue
        meta = e.seq_meta(S)
        R, wb = e.seq_plan(fmt, nto, names, seq_slot, seq_byte, seq_width, lo, hi)
        buf = np.zeros(cap, np.uint8)
        out, row, part, calls = [], 0, -1, 0
        while row < R:
            row, part, nb = e.seq_emit(row, part, buf, cap)
            out.append(bytes(buf[:nb]))
            calls += 1
        res.append((S, err, [m.tolist() for m in meta], (b"".join(out), wb.tolist(), calls)))
    return res


def whole(n_cols, widths, split_pl=None):
    col_slot = np.arange(n_cols, dtype=np.int32)
    if split_pl is None:
        names = ["s%d" % c for c in range(n_cols)]
        return col_slot, names, list(range(n_cols)), [0] * n_cols, list(widths)
    names, sl, sb = [], [], []
    for c, p in enumerate(split_pl):
        for a in range(p):
            names.append("s%d_%s" % (c, "ABCDEFGH"[a]))
            sl.append(c)
            sb.append(2 * a)
    return col_slot, names, sl, sb, [1] * len(names)


@pytest.mark.parametrize("S", [1, 2, 255, 256, 257, 1000])
@pytest.mark.parametrize("n_cols", [1, 33, 70])
@pytest.mark.parametrize("fmt", ["fasta", "phylip"])
def test_site_counts_sequences_and_widths(eng, S, n_cols, fmt):
    rng = random.Random(S * 131 + n_cols)
    widths = [rng.randint(1, 15) for _ in range(n_cols)]
    text = make_text(rng, S, widths)
    col_slot, names, sl, sb, sw = whole(n_cols, widths)
    d, o = both(eng, text, col_slot, np.array(widths, np.int32), True, fmt, S % 2 == 0, names, sl, sb, sw,
                [0], [S], 1 << 20)
    assert d == o


@pytest.mark.parametrize("ploidy", range(1, 9))
def test_split_ploidies(eng, ploidy):
    rng = random.Random(ploidy)
    n_cols = 9
    pls = [ploidy] * n_cols
    text = make_text(rng, 300, [2 * p - 1 for p in pls], comments=True)
    col_slot, names, sl, sb, sw = whole(n_cols, None, pls)
    d, o = both(eng, text, col_slot, np.array([2 * p - 1 for p in pls], np.int32), True, "phylip", True, names, sl, sb, sw,
                [0, 100], [300, 170], 1 << 20)
    assert d == o


def test_sequence_over_many_small_slabs(eng):
    rng = random.Random(5)
    text = make_text(rng, 5000, [3, 1], crlf=True)
    col_slot, names, sl, sb, sw = whole(2, [3, 1])
    d, o = both(eng, text, col_slot, np.array([3, 1], np.int32), True, "fasta", False, names, sl, sb, sw, [0, 10], [5000, 4000],
                301)
    assert d == o
    assert d[3][2] > 50                         # the rows went out in many slabs


def test_thousands_of_one_site_windows(eng):
    rng = random.Random(6)
    S = 4000
    text = make_text(rng, S, [3] * 40, scaffolds=3)
    col_slot, names, sl, sb, sw = whole(40, None, [2] * 40)
    lo = np.arange(S, dtype=np.int64)
    d, o = both(eng, text, col_slot, np.array([3] * 40, np.int32), True, "phylip", False, names, sl, sb, sw, lo, lo + 1,
                64 << 20)
    assert d == o
    assert d[3][2] == 1                         # one slab: every window in one launch of the transpose


def test_long_lines_subset_of_columns(eng):
    """lines of several warp steps; only some columns have slots (-S), exactness off"""
    rng = random.Random(7)
    widths = [rng.randint(1, 9) for _ in range(120)]
    text = make_text(rng, 77, widths, crlf=True, comments=True)
    take = [119, 3, 64, 3]
    slots = sorted(set(take))
    col_slot = np.full(120, -1, np.int32)
    for s, c in enumerate(slots):
        col_slot[c] = s
    names = ["n%d" % c for c in take]
    d, o = both(eng, text, col_slot, np.array([widths[c] for c in slots], np.int32), False, "fasta", True, names,
                [int(col_slot[c]) for c in take], [0] * 4, [widths[c] for c in take], [0, 5], [77, 6], 1 << 20)
    assert d == o


@pytest.mark.parametrize("bad, err", [
    ("c\t2\tA|T\tGG\tC|C", (4, 4, 2)),
    ("c\t2\tA|T\tG|G", (6, 4, 3)),
    ("c\t2x\tA|T\tG|G\tC|C", (1, 4, 0)),
    ("c", (2, 4, 0)),
    ("c\t2\tA|T\tG|G\tC|C\tA|A", (6, 4, 5)),
    ("c\t2\tA|TT\tGG\tC|C", (4, 4, 1)),
])
def test_first_error_names_the_line_and_column(eng, bad, err):
    good = "c\t1\tA|T\tG|G\tC|C"
    lines = [good] * 3 + ["#x", bad] + [good] * 200 + [bad.replace("c\t2", "c\t9")]
    text = ("\n".join(lines) + "\n").encode()
    for e in (eng, SeqOracleEngine()):
        S, got = e.seq_index(np.arange(3, dtype=np.int32), np.array([3, 3, 3], np.int32), True, data=text)
        assert got == err
