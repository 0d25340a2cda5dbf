"""CHECKER ONLY — parseVCF.py's VCF -> .geno conversion stated in plain Python, written from the behaviour of the reference
command line (VCF_processing/parseVCF.py) and never imported by the product.

    run(data: bytes, argv: list[str]) -> bytes        the output file's bytes, or raises Refusal

Semantics (the issue that added parseVCF.py on the GPU states them at length):
  * the input is UTF-8 text read with universal newlines (\\r\\n, \\r and \\n end a line);
  * header = lines up to the first one starting with "#CHROM"; its tokens 9.. are the sample names;
  * a data line is split with str.split(); blank lines and lines whose first field starts with '#' are skipped;
  * site filters in order: --excludeDuplicates (CHROM and POS text of the previous data line), contigs, --minQual,
    --maxREFlen; then one genotype per selected sample (filters, ploidy, allele lookup, --skipIndels, --keepPartial) or
    one raw FORMAT subfield (--field).
The refusals the GPU command line makes are raised as Refusal, with the data line (1-based, counting the data lines after
the header, duplicates included) where one applies."""
from __future__ import annotations

import argparse
import math
import re

FIXED = ["#CHROM", "POS", "ID", "REF", "ALT", "QUAL", "FILTER", "INFO", "FORMAT"]
ASCII_WS = re.compile(rb"[ \t\n\r\x0b\x0c\x1c-\x1f]+")
INT64 = (-(1 << 63), (1 << 63) - 1)


class Refusal(Exception):
    def __init__(self, msg, line=None):
        super().__init__(msg)
        self.line = line


def parser():
    p = argparse.ArgumentParser()
    p.add_argument("-i", "--inFile")
    p.add_argument("-o", "--outFile")
    p.add_argument("-s", "--samples")
    p.add_argument("--include")
    p.add_argument("--includeFile")
    p.add_argument("--exclude")
    p.add_argument("--excludeFile")
    p.add_argument("--minQual", type=int)
    p.add_argument("--gtf", action="append", nargs="+")
    p.add_argument("--skipIndels", action="store_true")
    p.add_argument("--excludeDuplicates", action="store_true")
    p.add_argument("--simplifyALT", action="store_true")
    p.add_argument("--expandMulti", action="store_true")
    p.add_argument("--maxREFlen", type=int)
    p.add_argument("--ploidy", type=int, default=2)
    p.add_argument("--ploidyFile")
    p.add_argument("--ploidyMismatchToMissing", action="store_true")
    p.add_argument("--keepPartial", action="store_true")
    p.add_argument("--addRefTrack", action="store_true")
    p.add_argument("--noHeader", action="store_true")
    p.add_argument("--field")
    p.add_argument("--missing")
    p.add_argument("--outSep", default="\t")
    return p


def gt_filter(words):
    """flag= min= max= siteTypes= gtTypes= samples=  ->  dict, or Refusal"""
    d = {}
    for w in words:
        kv = w.split("=")
        if len(kv) != 2 or kv[0] not in ("flag", "min", "max", "siteTypes", "gtTypes", "samples"):
            raise Refusal("Bad genotype filter specification: %s" % " ".join(words))
        d[kv[0]] = kv[1]
    try:
        for k in ("siteTypes", "gtTypes", "samples"):
            if k in d:
                d[k] = d[k].split(",")
        d["min"] = float(d["min"]) if "min" in d else -math.inf
        d["max"] = float(d["max"]) if "max" in d else math.inf
    except ValueError:
        raise Refusal("Bad genotype filter specification: %s" % " ".join(words))
    return d


def contig_lists(a):
    inc, exc = [], []
    if a.include:
        inc += a.include.split(",")
    if a.exclude:
        exc += a.exclude.split(",")
    for path, lst in ((a.includeFile, inc), (a.excludeFile, exc)):
        if path:
            with open(path, "rt") as f:
                lst += [c.strip() for c in f.read().split("\n")]
    return set(inc), set(exc)


def ploidy_table(a):
    d = {}
    if a.ploidyFile:
        with open(a.ploidyFile, "rt") as f:
            for ln in f:
                s = ln.split()
                try:
                    d[s[0]] = int(s[1])
                except (IndexError, ValueError):
                    raise Refusal("--ploidyFile: line %r is not 'sample ploidy'" % ln)
    return d


def gt_type(alleles):
    s = set(alleles)
    if len(s) > 1:
        return "Het"
    if "0" in s:
        return "HomRef"
    if "." in s:
        return "Missing"
    return "HomAlt"


def to_float(t):
    try:
        return float(t), True
    except ValueError:
        return None, False


def check_contig_line(line):
    """a ##contig header line must hold <key=value,...> with an ID (the reference parses every such line)"""
    parts = re.split("<|>", line)
    try:
        kv = dict([x.split("=", maxsplit=1) for x in parts[1].split(",")])
        kv["ID"]
    except (IndexError, ValueError, KeyError):
        raise Refusal("malformed ##contig header line: %r" % line.rstrip())


def split_lines(text):
    return re.split(r"\r\n|\r|\n", text)


def run(data: bytes, argv):
    a = parser().parse_args(argv)
    if a.simplifyALT or a.expandMulti:
        raise Refusal("--simplifyALT / --expandMulti are not supported")
    if a.field == "alleles":
        raise Refusal("--field alleles is not supported")
    try:
        text = data.decode("utf-8")
    except UnicodeDecodeError:
        raise Refusal("the input is not UTF-8")
    lines = split_lines(text)
    raw = re.split(rb"\r\n|\r|\n", data)
    inc, exc = contig_lists(a)
    filters = [gt_filter(g) for g in (a.gtf or [])]
    pdict = ploidy_table(a)
    headers = None
    k = 0
    for k, ln in enumerate(lines):
        if ln.startswith("##contig"):
            check_contig_line(ln)
        if ln.startswith("#CHROM"):
            headers = ln.split()
            break
    if headers is None:
        raise Refusal("no #CHROM header line")
    if headers[:9] != FIXED:
        raise Refusal("the #CHROM line does not name the nine fixed VCF columns")
    names = headers[9:]
    for n in names:
        if n in FIXED:
            raise Refusal("sample name %s repeats a fixed column name" % n)
    samples = a.samples.split(",") if a.samples else list(names)
    for s in samples:
        if s not in names:
            raise Refusal("Sample %s not in VCF header" % s)
    missing = a.missing
    out = []
    if not a.noHeader:
        out.append(a.outSep.join(["#CHROM", "POS"] + (["REF"] if a.addRefTrack else []) + samples) + "\n")
    last = None
    dline = 0
    for ln, rb in zip(lines[k + 1:], raw[k + 1:]):
        dev = [t for t in ASCII_WS.split(rb) if t]
        if not dev or dev[0].startswith(b"#"):
            continue
        dline += 1
        el = ln.split()
        if el != [t.decode() for t in dev]:
            raise Refusal("data line %d: a non-ASCII whitespace character splits its fields" % dline, dline)
        if a.excludeDuplicates:
            if len(el) < 2:
                raise Refusal("data line %d: fewer fields than the header" % dline, dline)
            if last == (el[0], el[1]):
                continue
            last = (el[0], el[1])
        d = dict(zip(headers, el))
        if len(el) < 2:
            raise Refusal("data line %d: fewer fields than the header" % dline, dline)
        try:
            pos = int(d["POS"])
        except ValueError:
            raise Refusal("data line %d: POS is not an integer" % dline, dline)
        if not INT64[0] <= pos <= INT64[1]:
            raise Refusal("data line %d: POS outside int64" % dline, dline)
        if any(f not in d for f in FIXED if f != "INFO") or any(n not in d for n in names):
            raise Refusal("data line %d: fewer fields than the header" % dline, dline)
        chrom, ref, alt = d["#CHROM"], d["REF"], d["ALT"]
        if (exc and chrom in exc) or (inc and chrom not in inc):
            continue
        if a.minQual:
            q, ok = to_float(d["QUAL"])
            if ok and q < a.minQual:
                continue
        if a.maxREFlen and len(ref) > a.maxREFlen:
            continue
        alts = alt.split(",") if alt != "." else []
        alleles = [ref] + alts
        keys = d["FORMAT"].split(":")
        site_type = "MONO" if not alts else ("SNP" if all(len(x) == len(ref) for x in alts) else "INDEL")
        row = [chrom, str(pos)] + ([ref] if a.addRefTrack else [])
        for s in samples:
            sub = dict(zip(keys, d[s].split(":")))
            gt = sub.get("GT")
            if gt is not None:
                sub["alleles"] = tuple(re.split("[/|]", gt))
                sub["phase"] = "|" if "|" in gt else "/"
            if a.field is not None:
                v = sub.get(a.field)
                row.append((missing if missing is not None else ".") if v is None else v)
                continue
            if gt is None:
                raise Refusal("data line %d, sample %s: no GT" % (dline, s), dline)
            gal = sub["alleles"]
            m = missing if missing is not None else "N"
            passed = True
            for f in filters:
                if "siteTypes" in f and site_type not in f["siteTypes"]:
                    continue
                if "gtTypes" in f and gt_type(gal) not in f["gtTypes"]:
                    continue
                if "samples" in f and s not in f["samples"]:
                    continue
                v = sub.get(f.get("flag")) if f.get("flag") not in ("alleles", "phase") else None
                ok = isinstance(v, str)
                if ok:
                    for t in v.split(","):
                        x, good = to_float(t)
                        if not (good and f["min"] <= x <= f["max"]):
                            ok = False
                            break
                passed = ok
                if not passed:
                    break
            pl = pdict.get(s, a.ploidy)
            if pl != len(gal):
                if not a.ploidyMismatchToMissing:
                    raise Refusal("data line %d, sample %s: genotype %s does not match ploidy %d" % (dline, s, gt, pl), dline)
                passed = False
            if passed:
                lookup = {str(i): x for i, x in enumerate(alleles)}
                if all(x in lookup for x in gal):
                    got = [lookup[x] if (not a.skipIndels or len(lookup[x]) == len(ref)) else m for x in gal]
                    if not a.keepPartial and m in got:
                        got = [m] * pl
                else:
                    got = [m] * pl
            else:
                got = [m] * pl
            row.append(sub["phase"].join(got))
        out.append(a.outSep.join(row) + "\n")
    return "".join(out).encode("utf-8")
