#!/usr/bin/env python
"""Drop-in for the reference's VCF_processing/parseVCF.py (flags 257-289, 327) on the GPU: the VCF body is read in chunks
cut at line ends (_stream.py), each chunk is indexed and tokenised on the device (k_vcf_records), the genotypes are
evaluated there (k_vcf_genotypes) and the .geno rows are formatted there and written slab by slab (k_vcf_emit).  The host
parses the header, applies the contig lists, settles the few tokens the device's number parser leaves unresolved with
Python's own int() / float(), and checks every line with a byte >= 0x80 against str.split().

Refused up front: --simplifyALT and --expandMulti (INFO CIGAR parsing; the reference raises a KeyError on any record
without CIGAR), --field alleles (the reference joins a tuple and raises a TypeError), --devices N, a #CHROM line that does
not start with the nine fixed VCF columns, and a sample named like one of them.  Refused at the data line (and sample)
where the reference would crash: a line without one of the header's sample names or without FORMAT, a POS that int()
rejects or that is outside int64, a selected sample without GT or (without --ploidyMismatchToMissing) with another
ploidy, a line whose fields a non-ASCII whitespace character would split, and text that is not UTF-8."""
from __future__ import annotations

import argparse
import math
import re
import sys

import numpy as np

from .. import _lib as L
from ..engine import Engine, PinnedArray
from . import _common as C
from ._stream import SlabWriter, body_chunks, env_int, open_input, open_output

FIXED = ["#CHROM", "POS", "ID", "REF", "ALT", "QUAL", "FILTER", "INFO", "FORMAT"]
ASCII_WS = re.compile(rb"[ \t\n\r\x0b\x0c\x1c-\x1f]+")
SITE_BITS = {"MONO": 1, "SNP": 2, "INDEL": 4}
GT_BITS = {"Het": 1, "HomRef": 2, "Missing": 4, "HomAlt": 8}
V_FAIL, V_UNRESOLVED = 1, 2
MAX_KEYS = 40


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument("-o", "--outFile", help="Output file (.gz allowed; default stdout)")
    p.add_argument("-s", "--samples", help="sample names (separated by commas)")
    p.add_argument("--include", help="include contigs (separated by commas)")
    p.add_argument("--includeFile", help="File of contigs (one per line)")
    p.add_argument("--exclude", help="exclude contigs (separated by commas)")
    p.add_argument("--excludeFile", help="File of contigs (one per line)")
    p.add_argument("--minQual", help="Minimum QUAL for a site", type=int)
    p.add_argument("--gtf", help="Genotype filter. Syntax: flag=X min=X max=X siteTypes=X,X.. gtTypes=X,X.. samples=X,X..",
                   action="append", nargs="+")
    p.add_argument("--skipIndels", action="store_true")
    p.add_argument("--excludeDuplicates", action="store_true")
    p.add_argument("--simplifyALT", help="Refused: needs INFO CIGAR parsing", action="store_true")
    p.add_argument("--expandMulti", help="Refused: needs INFO CIGAR parsing", action="store_true")
    p.add_argument("--maxREFlen", type=int)
    p.add_argument("--ploidy", type=int, default=2)
    p.add_argument("--ploidyFile")
    p.add_argument("--ploidyMismatchToMissing", action="store_true")
    p.add_argument("--keepPartial", action="store_true")
    p.add_argument("--addRefTrack", action="store_true")
    p.add_argument("--noHeader", action="store_true")
    p.add_argument("--field", help="Optional - format field to extract")
    p.add_argument("--missing", help="Value to use for missing data")
    p.add_argument("--outSep", default="\t")
    p.add_argument("-i", "--inFile", help="Input VCF file (.gz allowed; default stdin)")
    p.add_argument("--device", help="CUDA device index", type=int, default=0)
    p.add_argument("--devices", help="Refused: the conversion runs on one GPU", type=int, default=None)
    p.add_argument("--timing", help="Write a JSON file with the wall time of each phase and the device time of each kernel",
                   metavar="FILE")
    return p


def _fail(msg):
    raise SystemExit("parseVCF: " + msg)


def _gt_filter(words):
    """parseVCF.py:244-254"""
    d = {}
    for w in words:
        kv = w.split("=")
        if len(kv) != 2 or kv[0] not in ("flag", "min", "max", "siteTypes", "gtTypes", "samples"):
            _fail("Bad genotype filter specification: %s" % " ".join(words))
        d[kv[0]] = kv[1]
    try:
        for k in ("siteTypes", "gtTypes", "samples"):
            if k in d:
                d[k] = d[k].split(",")
        d["min"] = float(d["min"]) if "min" in d else -math.inf
        d["max"] = float(d["max"]) if "max" in d else math.inf
    except ValueError:
        _fail("Bad genotype filter specification: %s" % " ".join(words))
    return d


def _contigs(args):
    """parseVCF.py:291-314"""
    inc, exc = [], []
    if args.include:
        inc += args.include.split(",")
    if args.exclude:
        exc += args.exclude.split(",")
    for path, lst in ((args.includeFile, inc), (args.excludeFile, exc)):
        if path:
            with open(path, "rt") as f:
                lst += [c.strip() for c in f.read().split("\n")]
    return set(inc), set(exc)


def _ploidies(args):
    """parseVCF.py:359-361"""
    d = {}
    if args.ploidyFile:
        with open(args.ploidyFile, "rt") as f:
            for ln in f:
                s = ln.split()
                try:
                    d[s[0]] = int(s[1])
                except (IndexError, ValueError):
                    _fail("--ploidyFile line %r is not 'sample ploidy' (the reference fails on it)" % ln)
    return d


def qual_threshold(m):
    """the smallest double >= the integer m: float(QUAL) < m (an exact comparison in Python) is float(QUAL) < this"""
    try:
        t = float(m)
    except OverflowError:
        return math.inf if m > 0 else -sys.float_info.max
    return math.nextafter(t, math.inf) if t < m else t


def read_header(src):
    """(header lines before #CHROM, the #CHROM line, body bytes read so far) — universal newlines, as the reference's text
    mode reads them (parseVCF.py:193-213)"""
    buf = b""
    at = 0
    pre = []
    while True:
        m = re.compile(rb"\r\n|\r|\n").search(buf, at)
        if m is None or (m.group() == b"\r" and m.end() == len(buf)):
            blk = src.read(1 << 20)
            if blk:
                buf += blk
                continue
            if m is None and at >= len(buf):
                _fail("no #CHROM header line")
        end, nxt = (m.start(), m.end()) if m is not None else (len(buf), len(buf))
        try:
            ln = buf[at:end].decode("utf-8")
        except UnicodeDecodeError:
            _fail("header line %d is not UTF-8" % (len(pre) + 1))
        if ln.startswith("#CHROM"):
            return pre, ln, buf[nxt:]
        pre.append(ln)
        at = nxt
        if nxt >= len(buf) and m is None:
            _fail("no #CHROM header line")


def _check_contig_line(ln):
    parts = re.split("<|>", ln)
    try:
        kv = dict([x.split("=", maxsplit=1) for x in parts[1].split(",")])
        kv["ID"]
    except (IndexError, ValueError, KeyError):
        _fail("malformed ##contig header line (the reference fails on it): %r" % ln)


def plan(args, head_line):
    """The run's tables (pg_vcf_spec) from the #CHROM line and the flags (parseVCF.py:331-368)."""
    headers = head_line.split()
    if headers[:9] != FIXED:
        _fail("the #CHROM line must start with the nine fixed columns %s" % " ".join(FIXED))
    names = headers[9:]
    for n in names:
        if n in FIXED:
            _fail("sample name %s is also the name of a fixed VCF column" % n)
    samples = args.samples.split(",") if args.samples else list(names)
    for s in samples:
        if s not in names:
            _fail("Sample %s not in VCF header" % s)
    n_cols = len(headers)
    col_prev = [-1] * n_cols
    last, first = {}, {}
    for c in range(9, n_cols):
        col_prev[c] = last.get(headers[c], -1)
        last[headers[c]] = c
        first.setdefault(headers[c], c)
    # a line must hold every name of the header (the reference reads each one, parseVCF.py:87-94)
    min_fields = max([9] + [c + 1 for c in first.values()])
    wanted = set(samples)
    col_slot = [-1] * n_cols
    k = 0
    for c in range(9, n_cols):
        if headers[c] in wanted:
            col_slot[c] = k
            k += 1
    field = args.field
    keys = ["GT"]
    if field is not None and field not in keys:
        keys.append(field)
    gtf = [_gt_filter(g) for g in (args.gtf or [])]
    for f in gtf:
        fl = f.get("flag")
        if fl is not None and fl not in ("alleles", "phase") and fl not in keys:
            keys.append(fl)
    if len(keys) > MAX_KEYS:
        _fail("%d FORMAT keys to look up (at most %d)" % (len(keys), MAX_KEYS))
    pdict = _ploidies(args)
    filters = []
    for f in gtf:
        fl = f.get("flag")
        filters.append(dict(key=keys.index(fl) if fl is not None and fl not in ("alleles", "phase") else -1,
                            min=f["min"], max=f["max"], flag=fl,
                            site=sum(b for n, b in SITE_BITS.items() if n in f["siteTypes"]) if "siteTypes" in f else 7,
                            gt=sum(b for n, b in GT_BITS.items() if n in f["gtTypes"]) if "gtTypes" in f else 15,
                            samples=[1 if ("samples" not in f or s in f["samples"]) else 0 for s in samples], spec=f))
    missing = args.missing if args.missing is not None else ("." if field is not None else "N")
    spec = dict(col_slot=col_slot, col_prev=col_prev, keys=keys, samp_col=[last[s] for s in samples],
                samp_ploidy=[pdict.get(s, args.ploidy) for s in samples],
                field_key=keys.index(field) if field is not None else -1,
                field_phase=field == "phase", filters=filters,
                min_qual=qual_threshold(args.minQual) if args.minQual else None, missing=missing.encode(),
                sep=args.outSep.encode(), skip_indels=args.skipIndels, keep_partial=args.keepPartial,
                p2m=args.ploidyMismatchToMissing, add_ref=args.addRefTrack)
    return dict(headers=headers, samples=samples, min_fields=min_fields, spec=spec)


def _gt_type(alleles):
    s = set(alleles)
    return "Het" if len(s) > 1 else ("HomRef" if "0" in s else ("Missing" if "." in s else "HomAlt"))


def settle(pl, chunk, rec, s):
    """The genotype filters of one genotype whose values the device left unresolved, with Python's float() (numpy's
    float conversion of the reference, parseVCF.py:125-128): True when every applicable filter passes."""
    f = [t.decode() for t in ASCII_WS.split(chunk[rec["start"]:rec["end"]]) if t]
    sp = pl["spec"]
    c = sp["samp_col"][s]
    while c >= len(f):
        c = sp["col_prev"][c]
    sub = dict(zip(f[8].split(":"), f[c].split(":")))
    gal = re.split("[/|]", sub["GT"])
    site = "MONO" if rec["n_alt"] == 0 else ("SNP" if rec["flags"] & L.VCF_SAME_LEN else "INDEL")
    for flt in sp["filters"]:
        g = flt["spec"]
        if ("siteTypes" in g and site not in g["siteTypes"]) or ("gtTypes" in g and _gt_type(gal) not in g["gtTypes"]) or \
                not flt["samples"][s]:
            continue
        v = sub.get(flt["flag"]) if flt["key"] >= 0 else None
        if v is None:
            return False
        try:
            x = np.array(v.split(","), dtype=float)
        except ValueError:
            return False
        if not (np.all(flt["min"] <= x) and np.all(x <= flt["max"])):
            return False
    return True


def site_pass(args, pl, chunk, recs, inc, exc, line0):
    """The site-level steps of parseVCF.py:230-237, 370-373 over one chunk's data lines: (rows kept before the first
    offending line, their POS, (first offending line, message) or None)"""
    n = len(recs)
    nf, fl = recs["n_fields"], recs["flags"]
    pos = recs["pos"].copy()
    bad = np.full(n, False)
    why = {}

    def fail(i, msg):
        if i not in why:
            why[i] = msg
        bad[i] = True
    if not chunk.isascii():
        try:
            chunk.decode("utf-8")
        except UnicodeDecodeError as e:
            i = max(int(np.searchsorted(recs["start"], e.start, side="right")) - 1, 0)
            fail(i, "the text is not UTF-8 (byte %d of data line %d)" % (e.start - int(recs["start"][i]), line0 + i + 1))
        for i in np.flatnonzero(fl & L.VCF_NONASCII):
            ln = chunk[recs["start"][i]:recs["end"][i]]
            try:
                same = ln.decode("utf-8").split() == [t.decode("utf-8") for t in ASCII_WS.split(ln) if t]
            except UnicodeDecodeError:
                same = False
            if not same:
                fail(i, "data line %d: a non-ASCII whitespace character (or text that is not UTF-8) splits its fields"
                     % (line0 + i + 1))
    short = nf < 2
    for i in np.flatnonzero(short):
        fail(i, "data line %d: fewer fields than the header" % (line0 + i + 1))
    cand = ~short
    if args.excludeDuplicates:
        cand &= (fl & L.VCF_DUPLICATE) == 0
    for i in np.flatnonzero(cand & ((fl & L.VCF_POS_UNRESOLVED) != 0)):
        r = recs[i]
        t = chunk[r["start"] + r["pos_off"]:r["start"] + r["pos_off"] + r["pos_len"]]
        try:
            pos[i] = int(t.decode("utf-8"))
        except (ValueError, UnicodeDecodeError, OverflowError):
            fail(i, "data line %d: POS %r is not an integer in the int64 range" % (line0 + i + 1, t))
    for i in np.flatnonzero(cand & (nf < pl["min_fields"])):
        fail(i, "data line %d: %d fields, fewer than the header's columns (%d) need" % (line0 + i + 1, nf[i], pl["min_fields"]))
    for i in np.flatnonzero(cand & ((fl & L.VCF_FORMAT_WIDE) != 0)):
        fail(i, "data line %d: a FORMAT key looked up past the 64th" % (line0 + i + 1))
    keep = cand & ~bad
    if inc or exc:
        for i in np.flatnonzero(keep):
            r = recs[i]
            ch = chunk[r["start"] + r["chrom_off"]:r["start"] + r["chrom_off"] + r["chrom_len"]].decode("utf-8")
            if (exc and ch in exc) or (inc and ch not in inc):
                keep[i] = False
    if args.minQual:
        keep &= (fl & L.VCF_QUAL_DROP) == 0
        for i in np.flatnonzero(keep & ((fl & L.VCF_QUAL_UNRESOLVED) != 0)):
            r = recs[i]
            try:
                q = float(chunk[r["start"] + r["qual_off"]:r["start"] + r["qual_off"] + r["qual_len"]].decode("utf-8"))
            except ValueError:
                continue
            if q < args.minQual:
                keep[i] = False
    if args.maxREFlen:
        keep &= recs["ref_len"] <= args.maxREFlen
    first = min(why) if why else None
    rows = np.flatnonzero(keep if first is None else keep & (np.arange(n) < first))
    return rows, pos[rows], (None if first is None else (first, why[first]))


def main(argv=None):
    args = build_parser().parse_args(argv)
    if args.simplifyALT or args.expandMulti:
        _fail("--simplifyALT and --expandMulti are not supported (they need INFO CIGAR parsing and write several rows per "
              "record; the reference raises a KeyError on any record without CIGAR)")
    if args.field == "alleles":
        _fail("--field alleles is not supported: the reference joins a tuple there and raises a TypeError")
    if args.devices not in (None, 1):
        _fail("--devices is not supported; the conversion runs on one GPU")
    src = open_input(args.inFile)
    pre, head_line, body0 = read_header(src)
    for ln in pre:
        if ln.startswith("##contig"):
            _check_contig_line(ln)
    pl = plan(args, head_line)
    inc, exc = _contigs(args)
    samples = pl["samples"]
    tm = C.Timing(args.timing)
    target = env_int("PG_VCF_CHUNK_BYTES", 256 << 20)
    slab = env_int("PG_VCF_SLAB_BYTES", 64 << 20)
    n_lines = n_rows = 0
    prev = None
    with (open_output(args.outFile) as out, Engine(args.device) as eng,
          SlabWriter(out.write, slab, PinnedArray) as w):
        if not args.noHeader:
            out.write((args.outSep.join(["#CHROM", "POS"] + (["REF"] if args.addRefTrack else []) + samples) + "\n").encode())
        eng.vcf_set_spec(pl["spec"])
        for chunk in body_chunks(body0, src, target):
            tm.mark("read")
            S = eng.vcf_load(chunk, prev)
            if S == 0:
                continue
            recs = eng.vcf_lines()
            tm.mark("records", eng)
            rows, pos, err = site_pass(args, pl, chunk, recs, inc, exc, n_lines)
            nu, gerr = eng.vcf_genotypes(rows, pos)
            tm.mark("genotypes", eng)
            if gerr:
                gl, gs, code = (gerr >> 24) - 1, (gerr >> 3) & ((1 << 21) - 1), gerr & 7
                if err is None or gl < err[0]:
                    r = recs[gl]
                    what = "no GT" if code == 1 else "a genotype whose ploidy is not %d (use --ploidyMismatchToMissing)" % \
                        pl["spec"]["samp_ploidy"][gs]
                    err = (gl, "data line %d (%s:%s), sample %s: %s" % (
                        n_lines + gl + 1, chunk[r["start"] + r["chrom_off"]:r["start"] + r["chrom_off"] + r["chrom_len"]].decode(),
                        int(pos[np.searchsorted(rows, gl)]), samples[gs], what))
            if err is not None:
                _fail(err[1])
            if nu:
                v = eng.vcf_verdicts(len(rows), len(samples))
                for r, s in zip(*np.nonzero(v & V_UNRESOLVED)):
                    v[r, s] &= ~np.uint8(V_UNRESOLVED | V_FAIL)
                    if not settle(pl, chunk, recs[rows[r]], s):
                        v[r, s] |= V_FAIL
                eng.vcf_verdicts(len(rows), len(samples), put=v)
                tm.mark("settle")
            row = 0
            while row < len(rows):
                k, nb = eng.vcf_emit(row, w.slab(), w.cap)
                w.write(nb)
                row += k
            tm.mark("emit", eng)
            last = recs[-1]
            if last["n_fields"] >= 2:
                s0 = int(last["start"])
                prev = (chunk[s0 + last["chrom_off"]:s0 + last["chrom_off"] + last["chrom_len"]],
                        chunk[s0 + last["pos_off"]:s0 + last["pos_off"] + last["pos_len"]])
            n_lines += S
            n_rows += len(rows)
    tm.write(lines=n_lines, rows=n_rows)


if __name__ == "__main__":
    main()
