"""TEST INFRASTRUCTURE — the filterGenotypes methods of the Engine, backed by oracle/filter_oracle.py, so that the CPU tests
run the command line's host logic (flags, samples, populations, chunks, contig lists) without a GPU.  Never imported by the
product."""
import numpy as np

from oracle import filter_oracle as fo
from oracle_engine import OracleEngine

FMT_NAME = {0: "phased", 1: "diplo", 2: "alleles"}


class FilterOracleEngine(OracleEngine):
    def set_strict_ingest(self, on=True):
        self.strict = on

    def ingest_text(self, data, fmt, col_hap, col_ploidy, H, offset=0):
        assert getattr(self, "strict", False)
        self.fmt = FMT_NAME[fmt]
        self.col_hap = np.asarray(col_hap)
        self.lines, self.off = [], []
        o = offset
        for raw in data[offset:].split(b"\n"):
            if raw.strip() and not raw.startswith(b"#"):
                self.lines.append(raw.decode())
                self.off.append(o - offset)
            o += len(raw) + 1
        for n, line in enumerate(self.lines):
            toks = line.split()[2:]
            for c, h in enumerate(col_hap):
                if h < 0:
                    continue
                t, pl = toks[c], int(col_ploidy[c])
                want = 2 * pl - 1 if self.fmt == "phased" else (1 if self.fmt == "diplo" else pl)
                if len(t) != want or (self.fmt == "diplo" and pl != 2):
                    raise RuntimeError("data line %d, genotype column %d: the token's allele count does not match" % (n + 1, c + 1))
                chars = t if self.fmt != "phased" else t[::2]
                if any(ch not in (fo.DIPLO if self.fmt == "diplo" else "ACGTN") for ch in chars):
                    raise RuntimeError("data line %d, genotype column %d: a character other than A, C, G, T or N" % (n + 1, c + 1))
        self.S = len(self.lines)
        return self.S

    def ingest_meta(self, S, release=True):
        scaf = [ln.split(None, 1)[0] for ln in self.lines]
        newsc = np.array([i == 0 or scaf[i] != scaf[i - 1] for i in range(S)], dtype=np.int8)
        pos = np.array([int(ln.split()[1]) for ln in self.lines], dtype=np.int32)
        return pos, newsc, np.array(self.off, dtype=np.int64)

    def filter(self, spec, contig_mask=None, scaf_id=None):
        col_of = {int(h): c for c, h in enumerate(self.col_hap) if h >= 0}
        cols = [col_of[int(h)] for h in spec["samp_hap0"]]
        pops = [list(m) for m in (spec.get("pops") or [])]
        sp = dict(spec)
        self.p2m = bool(spec.get("partial_to_missing"))
        self.sites = [[fo.genotype(ln.split()[2 + c], self.fmt, self.p2m) for c in cols] for ln in self.lines]
        pod = int(spec.get("pod_size") or 10000)
        thin = int(spec.get("thin_dist") or 0)
        self.rows, flags = [], 0
        last_scaf = last_pos = None
        for s, gts in enumerate(self.sites):
            if s % pod == 0:
                last_scaf = None
            if contig_mask is not None and not contig_mask[s]:
                continue
            good = True
            pos = int(self.lines[s].split()[1])
            if thin:
                if last_scaf != scaf_id[s]:
                    last_pos, last_scaf, good = pos, scaf_id[s], False
                elif pos - last_pos < thin:
                    good = False
            if good and not spec.get("no_test"):
                good = fo.site_test(gts, pops, sp)
            if good:
                self.rows.append(s)
                c = fo.counts(gts)
                flags |= (1 if fo.is_tied(c) else 0) | (4 if c.sum() == 0 else 0)
                flags |= 2 if any(fo.is_missing(al) and not all(a == "N" for a in al) for al, _ in gts) else 0
                if thin:
                    last_pos = pos
        return len(self.rows), flags

    def filter_emit(self, fmt, freq_order, row0, buf, cap):
        out, n = b"", 0
        for s in self.rows[row0:]:
            obj = self.lines[s].split()
            row = ("\t".join(obj[:2] + fo.as_list(self.sites[s], fmt, "freq" if freq_order else None)) + "\n").encode()
            if len(out) + len(row) > cap:
                break
            out += row
            n += 1
        assert n > 0 or row0 == len(self.rows)
        buf[:len(out)] = np.frombuffer(out, dtype=np.uint8)
        return n, len(out)


class HostArray:
    """stands in for the engine's pinned buffer"""

    def __init__(self, shape, dtype):
        self.array = np.zeros(shape, dtype=dtype)

    def close(self):
        pass
