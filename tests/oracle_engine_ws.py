"""TEST INFRASTRUCTURE — the windowStats methods of the Engine (pg_ws_*) restated in plain Python (str.split() of every data
line, float() of every token, numpy's summation and selection written out), so that the CPU tests run the command line's
host logic (flags, refusals, windows, messages, rows) without a GPU, and the GPU tests have a statement to compare the device
with.  Never imported by the product."""
import math
import struct

import numpy as np

from oracle_engine_g2v import data_lines
from oracle_engine_g2v import POS

NAN = float("nan")


def pairwise(x):
    """numpy's pairwise_sum of the list x: sequential from -0.0 below 8 values, eight accumulators up to 128, else split at
    n2 = n // 2 - (n // 2) % 8"""
    n = len(x)
    if n < 8:
        res = -0.0
        for v in x:
            res += v
        return res
    if n <= 128:
        r = list(x[:8])
        i = 8
        while i < n - n % 8:
            for j in range(8):
                r[j] += x[i + j]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for v in x[i:]:
            res += v
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return pairwise(x[:n2]) + pairwise(x[n2:])


def key(v):
    """order-preserving unsigned key of a float64 (-0.0 before +0.0)"""
    u = struct.unpack("<Q", struct.pack("<d", v))[0]
    return (~u & 0xFFFFFFFFFFFFFFFF) if u >> 63 else u | (1 << 63)


def stat(x, code, q):
    """one statistic of the non-NaN values x (file order); min / max / sort take -0.0 below +0.0.  Quantiles lerp as numpy
    does, b - (b - a)(1 - g) for g >= 0.5, else a + (b - a) g; equal infinite neighbours give nan, as in numpy."""
    n = len(x)
    if code == 5:
        return 0.0 + pairwise(x)
    if code == 0:
        return (0.0 + pairwise(x)) / n if n else NAN
    if code == 4:
        if not n:
            return NAN
        m = (0.0 + pairwise(x)) / n
        v = math.sqrt((0.0 + pairwise([(a - m) * (a - m) for a in x])) / n)
        return float(np.rint(v * 1e6) / 1e6)
    if not n:
        return NAN
    if code == 2:
        return min(x, key=key)
    if code == 3:
        return max(x, key=key)
    s = sorted(x, key=key)
    if code == 1:
        k = n // 2
        return 0.0 + (-0.0 + s[k]) if n % 2 else (0.0 + ((-0.0 + s[k - 1]) + s[k])) / 2
    v = (n - 1) * q
    fl = math.floor(v)
    g = v - fl
    if fl >= n - 1:                                 # at or past the last value: both neighbours are the last value
        A = B = s[n - 1]
        return B - (B - A) * (1 - g)
    A, B = s[fl], s[fl + 1]
    return B - (B - A) * (1 - g) if g >= 0.5 else A + (B - A) * g


class WsOracleEngine:
    def __init__(self, device=0):
        self.vals, self.pos = [], []

    def __enter__(self):
        return self

    def __exit__(self, *a):
        pass

    def last_timings(self):
        return {}

    def ws_spec(self, col_slot, n_slots, n_fields):
        self.col_slot, self.n_slots, self.n_fields = list(col_slot), n_slots, n_fields
        self.slot_col = [self.col_slot.index(k) for k in range(n_slots)]
        self.vals, self.pos = [], []

    def ws_chunk(self, text):
        lines = data_lines(text)
        S = len(lines)
        errs, first, flagged = [], [], []
        for i, (off, raw) in enumerate(lines):
            if any(b >= 0x80 for b in raw):
                errs.append((i, 0, 5))
            if b"\r" in raw[:-1]:
                errs.append((i, 0, 6))
            toks = raw.decode("latin-1").split()
            first.append(toks[0] if toks else None)
            if len(toks) < 2:
                errs.append((i, 0, 2))
            elif not POS.fullmatch(toks[1].encode("latin-1")):
                errs.append((i, 0, 1))
            elif not -(1 << 63) <= int(toks[1]) < (1 << 63):
                errs.append((i, 0, 3))
            pos = int(toks[1]) if len(toks) >= 2 and POS.fullmatch(toks[1].encode("latin-1")) else 0
            self.pos.append(pos if -(1 << 63) <= pos < (1 << 63) else 0)
            nv = max(len(toks) - 2, 0)
            if self.n_fields >= 0 and len(toks) >= 2 and nv != self.n_fields:
                errs.append((i, 0, 4))
            row = [NAN] * self.n_slots
            starts = [m for m in range(len(raw)) if raw[m:m + 1].strip() and (m == 0 or not raw[m - 1:m].strip())]
            for k, c in enumerate(self.slot_col):
                if c >= nv:
                    if self.n_fields < 0:
                        errs.append((i, k, 7))
                    continue
                t = toks[2 + c]
                try:
                    v = float(t)
                    st = 2 if len(t) > 20 else 0        # long tokens take the host path, as many do on the device
                except ValueError:
                    v, st = NAN, 1
                row[k] = v if st == 0 else NAN
                if st:
                    flagged.append((k * S + i, ((off + starts[2 + c]) << 32) | (len(t) << 2) | st))
            self.vals.append(row)
        run_line = [i for i in range(S) if i == 0 or first[i] != first[i - 1]]
        err = (0, 0, 0)
        if errs:
            i, k, code = min(errs)
            err = (code, i, k)
        flagged.sort()
        return (S, np.array(run_line, np.int64), np.array([lines[i][0] for i in run_line], np.int64),
                np.array([f[0] for f in flagged], np.int64), np.array([f[1] for f in flagged], np.uint64), err)

    def ws_set_values(self, line, slot, v):
        for a, b, x in zip(line, slot, v):
            self.vals[a][b] = x

    def ws_meta(self):
        return np.array(self.pos, np.int64)

    def ws_stats(self, lo, hi, codes, qs, n_slots, sort_budget=1 << 30):
        out = np.zeros((len(lo), n_slots, len(codes)))
        n = np.zeros((len(lo), n_slots), np.int64)
        for w, (a, b) in enumerate(zip(lo, hi)):
            for c in range(n_slots):
                x = [r[c] for r in self.vals[a:b] if not math.isnan(r[c])]
                n[w, c] = len(x)
                for k, (code, q) in enumerate(zip(codes, qs)):
                    out[w, c, k] = stat(x, code, q)
        return out, n
