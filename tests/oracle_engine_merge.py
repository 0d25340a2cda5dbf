"""TEST INFRASTRUCTURE — the mergeGeno methods of the Engine (pg_merge_*) restated in plain Python (str.split() of every body
line, one bytes object per output row), so that the CPU tests run the command line's host logic (flags, .fai, headers,
chunks, rounds, slabs, refusals) without a GPU, and the GPU tests have a statement to compare the device with.  Never imported
by the product."""
import numpy as np


class MergeOracleEngine:
    def __init__(self, device=0):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        pass

    def last_timings(self):
        return {}

    def merge_setup(self, names, lengths, out, n_dummy, sep, missing, method, union_min, must_include_first):
        self.scaf, self.walk0, self.names = {}, [], []
        total = 0
        for name, n in zip(names, lengths):
            self.scaf[name] = (total, int(n))
            if n > 0:
                self.walk0.append(total)
                self.names.append(name)
                total += int(n)
        self.total = total
        self.out, self.n_dummy = [bool(v) for v in out], [max(int(v), 0) for v in n_dummy]
        self.sep, self.missing, self.method = sep, missing, method
        self.nF = len(out)
        self.need_first = min(max(must_include_first, 0), self.nF)
        self.union_min = max(union_min, must_include_first)
        self.dense = (method == 2 or (method == 1 and self.union_min <= 0)) and self.need_first == 0
        self.wait = [[] for _ in range(self.nF)]         # per file: [(key, tokens)] not merged yet
        self.carry = [-1] * self.nF
        self.prev = -1
        return self.dense

    def key(self, toks):
        if len(toks) < 2 or toks[0].encode() not in self.scaf:
            return -1
        off, n = self.scaf[toks[0].encode()]
        p = toks[1]
        if not (p.isascii() and p.isdigit() and p[0] != "0" and len(p) < 20) or int(p) > n:
            return -1
        return off + int(p) - 1

    def merge_load(self, x, text):
        assert not self.wait[x]
        lines = text.split(b"\n")
        if text.endswith(b"\n"):
            lines.pop()
        prev = self.carry[x]
        for i, raw in enumerate(lines):
            bad = any(b >= 0x80 for b in raw) or b"\r" in raw[:-1]
            if bad:
                return len(lines), i, 2, prev
            toks = raw.decode("ascii").split()
            k = self.key(toks)
            if k < 0 or k <= prev:
                self.carry[x] = prev
                return len(lines), i, 1, prev
            self.wait[x].append((k, toks[2:]))
            prev = k
        self.carry[x] = prev
        return len(lines), len(lines), 0, prev

    def row(self, key, hit):
        at = np.searchsorted(self.walk0, key, side="right") - 1
        el = [self.names[at], str(key - self.walk0[at] + 1).encode()]
        for x in range(self.nF):
            if self.out[x]:
                el += [t.encode() for t in hit[x]] if x in hit else [self.missing] * self.n_dummy[x]
        return self.sep.join(el) + b"\n"

    def merge_rows(self, hi):
        assert self.prev < hi < self.total
        got = {}
        for x in range(self.nF):
            while self.wait[x] and self.wait[x][0][0] <= hi:
                k, toks = self.wait[x].pop(0)
                got.setdefault(k, {})[x] = toks
        keys = range(self.prev + 1, hi + 1) if self.dense else sorted(got)
        rows = []
        for k in keys:
            hit = got.get(k, {})
            ok = all(x in hit for x in range(self.need_first))
            if self.method == 0:
                ok = ok and len(hit) == self.nF
            elif self.method == 1:
                ok = ok and len(hit) >= self.union_min
            if ok:
                rows.append(self.row(k, hit))
        self.prev = hi
        self.text = b"".join(rows)
        return len(rows), len(self.text)

    def merge_emit(self, at, buf, cap):
        piece = self.text[at:at + cap]
        buf[:len(piece)] = np.frombuffer(piece, np.uint8)
        return len(piece)
