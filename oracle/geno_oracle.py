"""CHECKER ONLY — the .geno grammar in plain Python, one data line at a time.  The host tokenizer (csrc/geno_parse.cpp,
pg_geno_parse) and the device tokenizer (csrc/ingest.cu, pg_ingest_text) are compared with it; the product never imports it.

The rules are the reference's reader (genomics.py:1884-1904 parseGenoLine: str.split on runs of blanks; 390-396 splitSeq:
characters 0, 2, 4, ... of a phased token; 1111: the allele count must equal the sample's ploidy; 407 forceHomo) and what
this project states on top of it:
  - blanks are ' ' '\\t' '\\r' '\\v' '\\f'; a line ends at '\\n' (or at the end of the text);
  - a data line is a line whose first byte is not '#' and which holds a non-blank byte; fields are runs of non-blanks;
  - field 0 is the scaffold, field 1 the position: an optional sign and at least one digit, anything after the leading digits
    is ignored ("12x" reads 12), and the value must lie in [-2**31, 2**31 - 1];
  - field 2 + c is genotype column c.  phased: alleles are characters 0, 2, 4, ...; pairs: every character; diplo: one IUPAC
    letter -> two alleles (a haploid diplo sample keeps homozygous calls only); haplo: the first character.  The allele
    count must equal the ploidy (diplo: ploidy 1 or 2, haplo: ploidy 1).  A C G T -> 0 1 2 3, any other character missing;
  - strict 1 (filterGenotypes): a token is exactly as wide as the ploidy asks (phased 2 * ploidy - 1, pairs and haplo
    ploidy, diplo one letter and diploid samples only) and holds only A C G T N at its allele characters (diplo: a letter of
    DIPLOTYPES); the phase character (character 1 of a phased token of ploidy >= 2, else '/') is recorded per sample.
    strict 2 (distPaint) checks the width only;
  - new_scaffold is 1 where the scaffold field's bytes differ from the previous data line's.
The first bad data line is the error; inside it the position comes first, then the wanted genotype columns in file order,
then the check that every wanted column was present."""
from __future__ import annotations

import re
from dataclasses import dataclass

import numpy as np

FORMATS = {"phased": 0, "diplo": 1, "pairs": 2, "haplo": 3}
BLANKS = b" \t\r\v\f"
BASE = {ord("A"): 0, ord("C"): 1, ord("G"): 2, ord("T"): 3}
DIPLO = dict(zip(b"ACGKMNSRTWY", ("AA", "CC", "GG", "GT", "AC", "NN", "CG", "AG", "TT", "AT", "CT")))
ACGTN = set(b"ACGTN")
INT32_MIN, INT32_MAX = -(1 << 31), (1 << 31) - 1
_FIELD = re.compile(rb"[^ \t\r\v\f\n]+")


@dataclass
class Parsed:
    geno: np.ndarray          # int8 [S, H]: A0 C1 G2 T3, -1 missing
    pos: np.ndarray           # int32 [S]
    new_scaffold: np.ndarray  # int8 [S]
    line_off: np.ndarray      # int64 [S]: byte offset of each data line in the text
    phase: np.ndarray         # uint8 [S, H]: phase character at each sample's first haplotype (strict 1 only, else 0)
    error: tuple | None       # (kind, data line 1-based, column): kind in no_pos, pos, range, ploidy, char, columns;
                              # column = 1-based genotype column (ploidy, char), genotype columns of the line (columns), else 0


def data_lines(text: bytes):
    """(byte offset, line bytes without '\\n') of every data line"""
    out = []
    off = 0
    for line in text.split(b"\n"):
        if line[:1] != b"#" and any(c not in BLANKS for c in line):
            out.append((off, line))
        off += len(line) + 1
    return out


def read_position(field: bytes):
    """-> (value, None) or (None, error kind)"""
    i = 0
    neg = False
    if field[:1] in (b"-", b"+"):
        neg = field[:1] == b"-"
        i = 1
    j = i
    while j < len(field) and 48 <= field[j] <= 57:
        j += 1
    if j == i:
        return None, "pos"
    v = int(field[i:j])
    v = -v if neg else v
    if v < INT32_MIN or v > INT32_MAX:
        return None, "range"
    return v, None


def read_token(tok: bytes, fmt: int, pl: int, strict: int):
    """-> (allele codes, phase character, None) or (None, None, error kind)"""
    if strict:
        want = 2 * pl - 1 if fmt == 0 else (1 if fmt == 1 else pl)
        if len(tok) != want or (fmt == 1 and pl != 2):
            return None, None, "ploidy"
    phase = None
    if strict == 1:
        if fmt == 1:
            ok = tok[0] in DIPLO
        else:
            ok = all(tok[2 * a if fmt == 0 else a] in ACGTN for a in range(pl))
        if not ok:
            return None, None, "char"
        phase = tok[1] if fmt == 0 and pl >= 2 else ord("/")
    if fmt == 0:
        al = list(tok[0::2])
    elif fmt == 2:
        al = list(tok)
    elif fmt == 1:
        pair = DIPLO.get(tok[0], "NN").encode()
        if pl == 1:                                     # forceHomo
            al = [pair[0] if pair[0] == pair[1] else ord("N")]
        else:
            al = list(pair)
    else:
        if pl != 1:
            return None, None, "ploidy"
        al = [tok[0]]
    if len(al) != pl:
        return None, None, "ploidy"
    return [BASE.get(c, -1) for c in al], phase, None


def parse(text: bytes, fmt, columns: dict, strict: int = 0) -> Parsed:
    """text: data lines (no header line); fmt: name or code; columns: {genotype column: (first haplotype, ploidy)} of the
    wanted columns (their ploidies tile the haplotypes 0 .. H-1)."""
    fmt = FORMATS.get(fmt, fmt)
    H = sum(pl for _, pl in columns.values())
    lines = data_lines(text)
    S = len(lines)
    geno = np.full((S, H), -1, dtype=np.int8)
    pos = np.zeros(S, dtype=np.int32)
    newsc = np.zeros(S, dtype=np.int8)
    off = np.zeros(S, dtype=np.int64)
    phase = np.zeros((S, H), dtype=np.uint8)
    error = None
    prev = None
    for s, (o, line) in enumerate(lines):
        off[s] = o
        fields = _FIELD.findall(line)
        newsc[s] = 1 if fields[0] != prev else 0
        prev = fields[0]
        if len(fields) < 2:
            error = ("no_pos", s + 1, 0)
            break
        v, kind = read_position(fields[1])
        if kind:
            error = (kind, s + 1, 0)
            break
        pos[s] = v
        toks = fields[2:]
        for c in sorted(columns):
            if c >= len(toks):
                continue
            hap0, pl = columns[c]
            al, ph, kind = read_token(toks[c], fmt, pl, strict)
            if kind:
                error = (kind, s + 1, c + 1)
                break
            geno[s, hap0:hap0 + pl] = al
            if ph is not None:
                phase[s, hap0] = ph
        if error is None and any(c >= len(toks) for c in columns):
            error = ("columns", s + 1, len(toks))
        if error:
            break
    return Parsed(geno, pos, newsc, off, phase, error)
