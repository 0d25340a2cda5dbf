"""TEST INFRASTRUCTURE — the genoToSeq methods of the Engine (pg_seq_*) restated in plain Python (str.split() of every data
line, one string per output row), so that the CPU tests run the command line's host logic (flags, names, windows, files,
slabs) without a GPU, and the GPU tests have a statement to compare the device with.  Never imported by the product."""
import re

import numpy as np

POS = re.compile(rb"[+-]?[0-9]+")


def data_lines(text):
    """(offset, line) of every data line as the device's line index takes them: not '#', not blank"""
    out, at = [], 0
    for raw in text.split(b"\n"):
        if raw.strip() and not raw.startswith(b"#"):
            out.append((at, raw))
        at += len(raw) + 1
    return out


def line_error(raw, n_cols, col_slot, slot_width, exact):
    """(genotype column, code) of the first error of one data line as pg_seq_index orders them, or None"""
    errs = []
    if any(b >= 0x80 for b in raw):
        errs.append((0, 7))
    if b"\r" in raw[:-1]:                   # a '\r' not right before the '\n' that ends the line
        errs.append((0, 8))
    toks = raw.decode("latin-1").split()
    if len(toks) < 2:
        errs.append((0, 2))
        return min(errs)
    t = toks[1].encode("latin-1")
    if not POS.fullmatch(t):
        errs.append((0, 1))
    elif not -(1 << 31) <= int(t) <= (1 << 31) - 1:
        errs.append((0, 3))
    g = toks[2:]
    found = 0
    for c, tok in enumerate(g[:n_cols]):
        s = col_slot[c]
        if s < 0:
            continue
        if len(tok) != slot_width[s]:
            errs.append((c + 1, 4))
        else:
            found += 1
    if exact and len(g) != n_cols:
        errs.append((len(g) + 1, 6))
    elif found != len(slot_width) and not (exact and len(g) == n_cols):
        errs.append((len(g) + 1, 5))
    return min(errs) if errs else None


class SeqOracleEngine:
    def __init__(self, device=0):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        pass

    def last_timings(self):
        return {}

    def seq_index(self, col_slot, slot_width, exact, data=None, path=None, body_offset=0):
        text = data if path is None else open(path, "rb").read()[body_offset:]
        self.col_slot = [int(v) for v in col_slot]
        self.slot_col = {s: c for c, s in enumerate(self.col_slot) if s >= 0}
        self.lines = data_lines(text)
        err = (0, 0, 0)
        for n, (_, raw) in enumerate(self.lines):
            e = line_error(raw, len(self.col_slot), self.col_slot, [int(w) for w in slot_width], exact)
            if e is not None:
                err = (e[1], n + 1, e[0])
                break
        self.toks = [raw.decode("latin-1").split() for _, raw in self.lines]
        return len(self.lines), err

    def seq_meta(self, S):
        pos = np.array([int(t[1]) if len(t) > 1 and POS.fullmatch(t[1].encode()) else 0 for t in self.toks], np.int32)
        sc = [t[0] for t in self.toks]
        newsc = np.array([1 if i == 0 or sc[i] != sc[i - 1] else 0 for i in range(len(sc))], np.int8)
        off = np.array([o for o, _ in self.lines], np.int64)
        return pos, newsc, off

    def seq_plan(self, fmt, nto_gap, names, seq_slot, seq_byte, seq_width, lo, hi):
        """every row as bytes: per window the PHYLIP header, then ">name\\nseq\\n" or "name   seq\\n" (genomics.py:2232-2251)"""
        self.rows, self.parts = [], []
        wb = []
        maxw = max(int(w) for w in seq_width)
        for a, b in zip(lo, hi):
            n0 = len(self.rows)
            if fmt == "phylip":
                self.rows.append(b" %d %d" % (len(names), (b - a) * maxw))
                self.parts.append([])
            for k, name in enumerate(names):
                c, o, w = self.slot_col[int(seq_slot[k])], int(seq_byte[k]), int(seq_width[k])
                sites = [self.toks[s][2 + c][o:o + w] for s in range(a, b)]
                if nto_gap:
                    sites = [x.replace("N", "-").replace("n", "-") for x in sites]
                pre = (">" + name + "\n") if fmt == "fasta" else (name + "   ")
                self.rows.append(pre.encode())
                self.parts.append([x.encode("latin-1") for x in sites])
            wb.append(sum(len(p) + sum(len(x) for x in s) + 1 for p, s in zip(self.rows[n0:], self.parts[n0:])))
        return len(self.rows), np.array(wb, np.int64)

    def _bytes(self, r, x0=-1, x1=None):
        """cells [x0, x1) of row r: -1 the prefix, 0..n-1 the sites, n the final '\\n'"""
        n = len(self.parts[r])
        x1 = n + 1 if x1 is None else x1
        out = b""
        for x in range(max(x0, -1), x1):
            out += self.rows[r] if x == -1 else (self.parts[r][x] if x < n else b"\n")
        return out

    def seq_emit(self, row0, part0, buf, cap):
        """whole rows while they fit, else row0 alone cut after as many sites as fit (pg_seq_emit)"""
        out = self._bytes(row0, part0)
        r = row0 + 1
        if len(out) > cap:
            n = len(self.parts[row0])
            x1 = part0
            while x1 < n and len(self._bytes(row0, part0, x1 + 1)) <= cap:
                x1 += 1
            assert x1 > part0 and x1 >= 0, "buffer too small"
            out = self._bytes(row0, part0, x1)
            buf[:len(out)] = np.frombuffer(out, np.uint8)
            return row0, x1, len(out)
        while r < len(self.rows) and len(out) + len(self._bytes(r)) <= cap:
            out += self._bytes(r)
            r += 1
        buf[:len(out)] = np.frombuffer(out, np.uint8)
        return r, -1, len(out)
