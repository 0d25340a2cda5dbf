"""TEST INFRASTRUCTURE — the parseVCF methods of the Engine (pg_vcf_*) restated in Python, so that the CPU tests run the
command line's host logic (header, flags, chunks, contig lists, the host's int() / float() settling, error reports, slabs)
without a GPU.  Its number parser leaves every token that is not a plain decimal unresolved, so the host's settling runs
often.  Never imported by the product."""
import re

import numpy as np

from genomics_general_b200 import _lib as L

TOK = re.compile(rb"[^ \t\n\r\x0b\x0c\x1c-\x1f]+")
PLAIN = re.compile(rb"[+-]?(\d+\.?\d*|\.\d+)")
V_FAIL, V_UNRESOLVED, V_PLOIDY, V_PHASED, V_ABSENT, V_PHASE_FIELD = 1, 2, 4, 8, 16, 32


def number(t):
    """(state, value): 0 resolved, 1 certainly not a float, 2 unresolved"""
    if t in (b"", b"."):
        return 1, None
    if PLAIN.fullmatch(t):
        return 0, float(t)
    return 2, None


class VcfOracleEngine:
    def __init__(self, device=0):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        pass

    def last_timings(self):
        return {}

    def vcf_set_spec(self, spec):
        self.sp = spec
        self.keys = [k.encode() for k in spec["keys"]]

    def vcf_load(self, text, prev=None):
        sp = self.sp
        self.text = text
        recs, self.fields, self.masks = [], [], []
        a = 0
        spans = []
        for m in re.finditer(rb"\r\n|\r|\n", text):
            spans.append((a, m.start()))
            a = m.end()
        if a < len(text):
            spans.append((a, len(text)))
        last = prev
        for a, e in spans:
            ln = text[a:e]
            toks = [(m.start(), m.end()) for m in TOK.finditer(ln)]
            if not toks or ln[toks[0][0]:toks[0][0] + 1] == b"#":
                continue
            r = np.zeros(1, dtype=L.VCF_LINE)[0]
            r["start"], r["end"], r["n_fields"] = a, e, len(toks)
            for k, name in ((0, "chrom"), (1, "pos"), (3, "ref"), (4, "alt"), (5, "qual"), (8, "fmt")):
                if k < len(toks):
                    r[name + "_off"], r[name + "_len"] = toks[k][0], toks[k][1] - toks[k][0]
            f = [ln[x:y] for x, y in toks]
            fl = L.VCF_NONASCII if not ln.isascii() else 0
            if len(f) >= 2 and re.fullmatch(rb"[+-]?\d{1,18}", f[1]):
                r["pos"] = int(f[1])
            else:
                fl |= L.VCF_POS_UNRESOLVED
            alts = f[4].split(b",") if len(f) >= 5 and f[4] != b"." else []
            r["n_alt"] = len(alts)
            if all(len(x) == len(f[3]) for x in alts):
                fl |= L.VCF_SAME_LEN
            if sp.get("min_qual") is not None and len(f) >= 6:
                st, q = number(f[5])
                if st == 2:
                    fl |= L.VCF_QUAL_UNRESOLVED
                elif st == 0 and q < sp["min_qual"]:
                    fl |= L.VCF_QUAL_DROP
            mask = [0] * len(self.keys)
            if len(f) >= 9:
                for j, k in enumerate(f[8].split(b":")):
                    for i, key in enumerate(self.keys):
                        if k == key:
                            if j >= 64:
                                fl |= L.VCF_FORMAT_WIDE
                            else:
                                mask[i] |= 1 << j
            if len(f) >= 2:
                if last is not None and (f[0], f[1]) == tuple(last):
                    fl |= L.VCF_DUPLICATE
                last = (f[0], f[1])
            else:
                last = None
            r["flags"] = fl
            recs.append(r)
            self.fields.append(f)
            self.masks.append(mask)
        self.recs = np.array(recs, dtype=L.VCF_LINE)
        return len(recs)

    def vcf_lines(self, line0=0, n=None):
        return self.recs[line0:None if n is None else line0 + n].copy()

    def _value(self, f, s, k):
        sp = self.sp
        c = sp["samp_col"][s]
        while c >= len(f):
            c = sp["col_prev"][c]
        vals = f[c].split(b":")
        m = self.masks[self._line][k]
        if len(vals) < 64:
            m &= (1 << len(vals)) - 1
        return vals[m.bit_length() - 1] if m else None

    def vcf_genotypes(self, rows, pos):
        sp = self.sp
        self.rows, self.pos = list(rows), list(pos)
        ns = len(sp["samp_col"])
        self.v = np.zeros((len(rows), ns), dtype=np.uint8)
        self.gt = {}
        err = None
        for r, line in enumerate(rows):
            self._line = line
            f = self.fields[line]
            rec = self.recs[line]
            site = 1 if rec["n_alt"] == 0 else (2 if rec["flags"] & L.VCF_SAME_LEN else 4)
            for s in range(ns):
                gt = self._value(f, s, 0)
                v = 0
                if gt is not None and b"|" in gt:
                    v |= V_PHASED
                if sp["field_key"] >= 0:
                    if sp["field_phase"] and gt is not None:
                        v |= V_PHASE_FIELD
                    else:
                        val = self._value(f, s, sp["field_key"])
                        if val is None:
                            v |= V_ABSENT
                        self.gt[r, s] = val
                    self.v[r, s] = v
                    continue
                if gt is None:
                    err = min(err or (1 << 64), ((line + 1) << 24) | (s << 3) | 1)
                    self.v[r, s] = V_FAIL
                    continue
                al = re.split(rb"[/|]", gt)
                gtb = 1 if len(set(al)) > 1 else (2 if al[0] == b"0" else (4 if al[0] == b"." else 8))
                for flt in sp["filters"]:
                    if not (flt["site"] & site) or not (flt["gt"] & gtb) or not flt["samples"][s]:
                        continue
                    val = self._value(f, s, flt["key"]) if flt["key"] >= 0 else None
                    ok = val is not None
                    for t in (val.split(b",") if ok else []):
                        st, x = number(t)
                        if st == 2:
                            v |= V_UNRESOLVED
                            break
                        if st == 1 or not (flt["min"] <= x <= flt["max"]):
                            ok = False
                            break
                    if v & V_UNRESOLVED:
                        break
                    if not ok:
                        v |= V_FAIL
                        break
                if len(al) != sp["samp_ploidy"][s]:
                    if sp["p2m"]:
                        v |= V_PLOIDY
                    else:
                        err = min(err or (1 << 64), ((line + 1) << 24) | (s << 3) | 2)
                self.v[r, s] = v
                self.gt[r, s] = gt
        nu = int(np.count_nonzero(self.v & V_UNRESOLVED)) if sp["field_key"] < 0 and sp["filters"] else 0
        return nu, err or 0

    def vcf_verdicts(self, n_rows, n_samp, put=None):
        if put is not None:
            self.v = np.array(put, dtype=np.uint8).reshape(n_rows, n_samp)
            return put
        return self.v.copy()

    def _geno(self, r, s, f, rec):
        sp = self.sp
        v = self.v[r, s]
        ph = b"|" if v & V_PHASED else b"/"
        m = sp["missing"]
        if sp["field_key"] >= 0:
            return m if v & V_ABSENT else (ph if v & V_PHASE_FIELD else self.gt[r, s])
        pl = sp["samp_ploidy"][s]
        alleles = [f[3]] + (f[4].split(b",") if rec["n_alt"] else [])
        if not v & (V_FAIL | V_PLOIDY):
            keys = re.split(rb"[/|]", self.gt[r, s])
            if all(re.fullmatch(rb"0|[1-9]\d{0,8}", k) and int(k) < len(alleles) for k in keys):
                got = [alleles[int(k)] if not sp["skip_indels"] or len(alleles[int(k)]) == len(f[3]) else m for k in keys]
                if sp["keep_partial"] or m not in got:
                    return ph.join(got)
        return ph.join([m] * max(pl, 0))

    def vcf_emit(self, row0, buf, cap):
        sp = self.sp
        out, n = b"", 0
        for r in range(row0, len(self.rows)):
            f, rec = self.fields[self.rows[r]], self.recs[self.rows[r]]
            cols = [f[0], str(self.pos[r]).encode()] + ([f[3]] if sp["add_ref"] else [])
            cols += [self._geno(r, s, f, rec) for s in range(len(sp["samp_col"]))]
            row = sp["sep"].join(cols) + b"\n"
            if len(out) + len(row) > cap:
                break
            out += row
            n += 1
        if n == 0 and row0 < len(self.rows):
            raise RuntimeError("pg_vcf_emit: row %d needs more than the %d bytes of the buffer" % (row0, cap))
        buf[:len(out)] = np.frombuffer(out, dtype=np.uint8)
        return n, len(out)
