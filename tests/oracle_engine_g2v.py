"""TEST INFRASTRUCTURE — the genoToVCF methods of the Engine (pg_g2v_*) restated in plain Python (str.split() of every data
line, one bytes object per output row), so that the CPU tests run the command line's host logic (flags, header, FASTA map,
chunks, slabs, messages) without a GPU, and the GPU tests have a statement to compare the device with.  Never imported by the
product."""
import re

import numpy as np

POS = re.compile(rb"[+-]?[0-9]+")
PAIRS = dict(zip("ACGKMNSRTWY", ("AA", "CC", "GG", "GT", "AC", "NN", "CG", "AG", "TT", "AT", "CT")))
BLANK = b" \t\r\x0b\x0c"                      # the line index's blanks (ingest.cu is_ws_dev)


def data_lines(text):
    """(offset, line) of every data line as the device's line index takes them: not '#', not blank"""
    out, at = [], 0
    for raw in text.split(b"\n"):
        if raw and raw[0] != ord("#") and raw.strip(BLANK):
            out.append((at, raw))
        at += len(raw) + 1
    return out


def alleles(tok, fmt):
    """(alleles, phase) of a token (genomics.py Genotype.__init__), None for a bad diplo token"""
    if fmt == 0:
        return list(tok[::2]), (tok[1] if len(tok) > 1 and len(tok) % 2 == 1 else "/")
    if fmt == 2:
        return list(tok), "/"
    return (list(PAIRS[tok]), "/") if tok in PAIRS else None


def site(raw, fmt, col_prev, sel_col, seq):
    """(row bytes, None) or (None, (column, code)) of one data line; seq(scaffold) -> reference sequence, or None without
    one (a KeyError where the scaffold is missing)"""
    errs = []
    if any(b >= 0x80 for b in raw):
        errs.append((0, 5))
    if b"\r" in raw[:-1]:
        errs.append((0, 6))
    toks = raw.decode("latin-1").split()
    if len(toks) < 2:
        return None, min(errs + [(0, 2)])
    if len(toks) == 2:
        errs.append((0, 4))
    p = toks[1].encode("latin-1")
    pos = 0
    if not POS.fullmatch(p):
        errs.append((0, 1))
    else:
        pos = int(p)
        if not -(1 << 63) <= pos < (1 << 63):
            errs.append((0, 3))
    g = toks[2:]
    counts = [0, 0, 0, 0]
    gts = []
    for k, c in enumerate(sel_col):
        while c >= len(g):
            c = col_prev[c]
        if c < 0:
            errs.append((k + 1, 7))
            continue
        a = alleles(g[c], fmt)
        if a is None:
            errs.append((k + 1, 8))
            continue
        gts.append(a)
        if all(x in "ACGTN" for x in a[0]):
            for x in a[0]:
                if x != "N":
                    counts["ACGT".index(x)] += 1
    L = [b for _, _, b in sorted((-n, -i, b) for i, (b, n) in enumerate(zip("ACGT", counts)) if n > 0)] or ["N"]
    if seq is not None:
        s = seq(toks[0])
        if s is None:
            errs.append((len(sel_col) + 1, 9))
        elif not -len(s) <= pos - 1 < len(s):
            errs.append((len(sel_col) + 1, 10))
        else:
            r = s[pos - 1]
            L = [r] + [b for b in L if b != r]
    if errs:
        return None, min(errs)
    fields = []
    for al, ph in gts:
        fields.append(ph.join(str(L.index(x)) if all(y in L for y in al) else "." for x in al))
    row = [toks[0], str(pos), ".", L[0], ",".join(L[1:]) or ".", ".", ".", ".", "GT"] + fields
    return ("\t".join(row) + "\n").encode("latin-1"), None


class G2vOracleEngine:
    def __init__(self, device=0):
        self.seqs = []

    def __enter__(self):
        return self

    def __exit__(self, *a):
        pass

    def last_timings(self):
        return {}

    def g2v_ref_load(self, text):
        self.fa = text
        return np.array([i for i, b in enumerate(text) if b == ord(">")], np.int64)

    def g2v_ref_index(self, lo, hi):
        self.seqs = [self.fa[a:b].replace(b"\n", b"").replace(b"\r", b"").replace(b" ", b"").decode()
                     for a, b in zip(lo, hi)]
        return np.array([len(s) for s in self.seqs], np.int64)

    def g2v_spec(self, fmt, col_slot, col_prev, sel_col, use_ref):
        self.fmt, self.col_prev, self.sel_col, self.use_ref = fmt, list(col_prev), list(sel_col), use_ref

    def g2v_chunk(self, text):
        self.lines = data_lines(text)
        first = [(raw.decode("latin-1").split() or [None])[0] for _, raw in self.lines]
        self.run_line = [i for i in range(len(first)) if i == 0 or first[i] != first[i - 1]]
        return len(self.lines), np.array(self.run_line, np.int64), np.array([self.lines[i][0] for i in self.run_line],
                                                                               np.int64)

    def g2v_sites(self, run_rec):
        run_of = np.searchsorted(self.run_line, np.arange(len(self.lines)), side="right") - 1
        self.rows = []
        for i, (off, raw) in enumerate(self.lines):
            seq = None
            if self.use_ref:
                r = int(run_rec[run_of[i]])
                seq = (lambda s: (lambda name: s))(self.seqs[r] if r >= 0 else None)
            row, err = site(raw, self.fmt, self.col_prev, self.sel_col, seq)
            if err is not None:
                self.out = b"".join(self.rows)
                return len(self.rows), len(self.out), (err[1], i, err[0], off)
            self.rows.append(row)
        self.out = b"".join(self.rows)
        return len(self.rows), len(self.out), (0, 0, 0, 0)

    def g2v_emit(self, at, buf, cap):
        piece = self.out[at:at + cap]
        buf[:len(piece)] = np.frombuffer(piece, np.uint8)
        return len(piece)
