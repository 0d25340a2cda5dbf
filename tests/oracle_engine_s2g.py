"""TEST INFRASTRUCTURE — the seqToGeno methods of the Engine (pg_s2g_*) restated in plain Python (str.split() of every
line, one bytes object per output row), so that the CPU tests run the command line's host logic (flags, refusals, PHYLIP
structure, plan, slabs) without a GPU, and the GPU tests have a statement to compare the device with.  Never imported by the
product."""
import re

import numpy as np

from oracle_engine_g2v import data_lines

TOK = re.compile(rb"[^ \t\n\r\x0b\x0c\x1c-\x1f]+")
PY_INT = re.compile(rb"[+-]?[0-9](_?[0-9])*")
I64 = (1 << 63) - 1


def line_table(text):
    """int64 [lines, 7] of pg_s2g_phylip_lines: {field 0 start, length, field 1 start, length, fields, flags, header count}"""
    rows = []
    for off, raw in data_lines(text):
        toks = list(TOK.finditer(raw))
        f = [(off + m.start(), m.end() - m.start()) for m in toks[:2]] + [(-1, 0)] * (2 - min(len(toks), 2))
        flags = (1 if any(b >= 0x80 for b in raw) else 0) | (2 if b"\r" in raw[:-1] else 0)
        n = 0
        if len(toks) >= 2 and all(PY_INT.fullmatch(m.group()) for m in toks[:2]):
            flags |= 4
            n = max(-I64 - 1, min(I64, int(toks[0].group())))
        rows.append([f[0][0], f[0][1], f[1][0], f[1][1], len(toks), flags, n])
    return np.array(rows, np.int64).reshape(-1, 7)


def rows_of(seqs, names, rows, members, seps):
    """the .geno rows of pg_s2g_plan's blocks"""
    out = []
    for name, R, mem, sep in zip(names, rows, members, seps):
        for x in range(R):
            out.append(name + b"\t" + str(x + 1).encode() + b"\t" +
                       b"".join(seqs[m][x:x + 1] + sep[j:j + 1] for j, m in enumerate(mem)))
    return b"".join(out)


class S2gOracleEngine:
    def __init__(self, device=0):
        self.seqs = []

    def __enter__(self):
        return self

    def __exit__(self, *a):
        pass

    def last_timings(self):
        return {}

    def s2g_fasta_load(self, text):
        self.text = text
        return np.array([i for i, b in enumerate(text) if b == ord(">")], np.int64)

    def s2g_fasta_index(self, lo, hi):
        self.seqs = [self.text[a:b].replace(b"\n", b"").replace(b"\r", b"").replace(b" ", b"") for a, b in zip(lo, hi)]
        return np.array([len(s) for s in self.seqs], np.int64)

    def s2g_phylip_load(self, text):
        self.text = text
        return line_table(text)

    def s2g_phylip_pack(self, seq_len, spans):
        buf = bytearray(int(np.sum(seq_len)))
        for src, dst, n in np.asarray(spans, np.int64).reshape(-1, 3):
            buf[dst:dst + n] = self.text[src:src + n]
        ends = np.cumsum(seq_len)
        self.seqs = [bytes(buf[e - n:e]) for e, n in zip(ends, seq_len)]

    def s2g_plan(self, names, rows, members, seps):
        for R, mem in zip(rows, members):
            assert all(len(self.seqs[m]) >= R for m in mem)
        self.out = rows_of(self.seqs, names, rows, members, seps)
        return len(self.out)

    def s2g_emit(self, at, buf, cap):
        piece = self.out[at:at + cap]
        buf[:len(piece)] = np.frombuffer(piece, np.uint8)
        return len(piece)
