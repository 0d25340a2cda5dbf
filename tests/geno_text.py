"""Shared pieces of the .geno tokenizer tests: random texts, the host tokenizer called as the library exposes it, the
column maps of the device tokenizer and the error a tokenizer reported, read back from its message."""
import ctypes as C
import re

import numpy as np

from genomics_general_b200 import _lib
from genomics_general_b200._lib import check

FMT = {"phased": 0, "diplo": 1, "pairs": 2, "haplo": 3}
BLANKS = " \t\r\v\f"
DIPLO_OF = {"AA": "A", "CC": "C", "GG": "G", "TT": "T", "GT": "K", "TG": "K", "AC": "M", "CA": "M", "CG": "S", "GC": "S",
            "AG": "R", "GA": "R", "AT": "W", "TA": "W", "CT": "Y", "TC": "Y"}
ALLELES = "ACGTACGTACGTNacgn-?."        # mostly bases; missing, lower case and other characters now and then


def columns_of(take):
    """take: [(file genotype column, ploidy)] in output order -> the oracle's {column: (first haplotype, ploidy)}"""
    out, h = {}, 0
    for c, pl in take:
        out[c] = (h, pl)
        h += pl
    return out


def device_maps(take, n_cols):
    """col_hap, col_ploidy, H of pg_ingest_text for the same request"""
    col_hap = np.full(n_cols, -1, np.int32)
    col_pl = np.ones(n_cols, np.int8)
    for c, (h, pl) in columns_of(take).items():
        col_hap[c], col_pl[c] = h, pl
    return col_hap, col_pl, int(sum(pl for _, pl in take))


def host_parse(body: bytes, fmt, take, threads=1):
    """pg_geno_parse on body -> (geno, pos, new_scaffold, line_off); raises PgError as the library reports it"""
    L = _lib.lib()
    n = C.c_int64(0)
    check(L.pg_geno_count_lines(body, len(body), C.byref(n)), "pg_geno_count_lines")
    S = int(n.value)
    H = int(sum(pl for _, pl in take))
    col_take = np.array([c for c, _ in take], np.int32)
    pl = np.array([p for _, p in take], np.int8)
    geno = np.empty((S, H), np.int8)
    pos = np.empty(S, np.int32)
    newsc = np.empty(S, np.int8)
    off = np.empty(S, np.int64)
    check(L.pg_geno_parse(body, len(body), FMT.get(fmt, fmt), len(take), col_take.ctypes.data_as(C.c_void_p),
                          pl.ctypes.data_as(C.c_void_p), H, S, geno.ctypes.data_as(C.c_void_p), pos.ctypes.data_as(C.c_void_p),
                          newsc.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p), int(threads)), "pg_geno_parse")
    return geno, pos, newsc, off


_ERRORS = (("no_pos", r"data line (\d+): no position field"),
           ("pos", r"data line (\d+): position is not an integer"),
           ("range", r"data line (\d+): position outside the int32 range"),
           ("ploidy", r"data line (\d+), genotype column (\d+): .*ploidy"),
           ("char", r"data line (\d+), genotype column (\d+): a character other than"),
           ("columns", r"data line (\d+): (\d+) genotype columns"))


def error_of(msg: str):
    """(kind, data line, column) of a tokenizer's error message, in the oracle's terms"""
    for kind, pat in _ERRORS:
        m = re.search(pat, msg)
        if m:
            g = [int(x) for x in m.groups()]
            return kind, g[0], g[1] if len(g) > 1 else 0
    raise AssertionError("unrecognised tokenizer error: " + msg)


def token(rng, fmt, pl, sep="|"):
    """a well-formed token of ploidy pl (its characters may still read as missing)"""
    al = [ALLELES[i] for i in rng.integers(0, len(ALLELES), pl)]
    if fmt == "phased":
        return sep.join(al)
    if fmt == "pairs":
        return "".join(al)
    if fmt == "haplo":
        return al[0]
    if pl == 1 and rng.random() < 0.5:
        return "ACGT"[int(rng.integers(0, 4))]
    return DIPLO_OF.get(al[0].upper() + al[1 % pl].upper(), "N" if rng.random() < 0.7 else al[0])


def blank_run(rng, lo=1, hi=9):
    return "".join(BLANKS[i] for i in rng.integers(0, len(BLANKS), int(rng.integers(lo, hi + 1))))


def random_text(rng, fmt, S, n_cols, take, runs=(1, 9), scaffolds=4, decorate=True, sep="|"):
    """S data lines of n_cols genotype columns; the requested columns carry well-formed tokens of their ploidy, the others
    junk.  Separators are blank runs of runs[0]..runs[1] characters (other than '\\n'); with decorate, comment lines,
    blank lines, leading blanks and CRLF endings are mixed in and the final newline may be missing."""
    want = dict(take)
    lines = []
    pos = 0
    for s in range(S):
        if decorate and rng.random() < 0.03:
            lines.append("#" + blank_run(rng) + "comment A|T 12")
        if decorate and rng.random() < 0.03:
            lines.append(blank_run(rng, 0, 4))
        pos += int(rng.integers(0, 3000))
        sc = "scaf%d" % min(scaffolds - 1, s * scaffolds // S)
        toks = [token(rng, fmt, want[c], sep) if c in want else "xy"[: int(rng.integers(1, 3))] for c in range(n_cols)]
        if rng.random() < 0.05:
            toks.append("extra")
        fields = [sc, str(pos) + ("" if rng.random() < 0.9 else "junk")] + toks
        line = "".join(f + blank_run(rng, *runs) for f in fields[:-1]) + fields[-1]
        if decorate and rng.random() < 0.05:
            line = blank_run(rng) + line
        if decorate and rng.random() < 0.1:
            line += "\r"
        lines.append(line)
    tail = "\n" if not decorate or rng.random() < 0.5 else ""
    return ("\n".join(lines) + tail).encode()


def random_take(rng, n_cols, n_take, ploidies, shuffle=True):
    cols = [int(c) for c in rng.choice(n_cols, n_take, replace=False)]
    if not shuffle:
        cols.sort()
    return [(c, int(ploidies[int(rng.integers(0, len(ploidies)))])) for c in cols]
