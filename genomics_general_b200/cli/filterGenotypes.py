#!/usr/bin/env python
"""Drop-in for the reference's filterGenotypes.py (flags 124-183), on the GPU: every chunk of the input is tokenised on the
device (strict tokens), the contig lists, --thinDist and genomics.siteTest run as site passes over the resident matrix, and
the kept rows are formatted on the device (GenomeSite.asList) and written slab by slab (_stream.py).

Refused up front: -of randomAllele (unseeded random.sample, genomics.py:376), --HWE (inHWE calls an undefined `unique`,
genomics.py:729), --samples that leave out a population member (siteTest raises a KeyError), -of diplo with a non-diploid
sample (genomics.py:359), --forcePloidy where it would change a genotype, --hostParse and --devices N.  --cache,
--parseThreads, -t and --noPrecomp are accepted and ignored.  Tokens whose width differs from the sample's
ploidy and characters outside A C G T N are reported with their data line."""
from __future__ import annotations

import argparse
import io
import string
import sys

import numpy as np

from ..engine import Engine, PinnedArray
from . import _common as C
from ._stream import Chain, SlabWriter, env_int, open_input, open_output

FMT_CODE = {"phased": 0, "diplo": 1, "alleles": 2}


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument("-i", "--infile", help="Input geno file (.gz allowed; default stdin)")
    p.add_argument("-o", "--outfile", help="Output geno file (.gz allowed; default stdout)")
    p.add_argument("-t", "--threads", help="Accepted and ignored: the work runs on the GPU", type=int, default=1)
    p.add_argument("--verbose", action="store_true")
    p.add_argument("-if", "--inputGenoFormat", choices=["phased", "diplo", "alleles"], default="phased")
    p.add_argument("-of", "--outputGenoFormat", default="phased",
                   choices=("phased", "diplo", "bases", "alleles", "randomAllele", "coded", "count"))
    p.add_argument("--alleleOrder", default=None, choices=("freq",))
    p.add_argument("-s", "--samples")
    p.add_argument("--excludeSamples")
    p.add_argument("-p", "--pop", action="append", nargs="+", metavar=("popName", "[samples]"))
    p.add_argument("--popsFile")
    p.add_argument("--keepAllSamples", action="store_true")
    p.add_argument("--ploidy", type=int, nargs="+")
    p.add_argument("--ploidyFile")
    p.add_argument("--forcePloidy", action="store_true")
    p.add_argument("--partialToMissing", action="store_true")
    p.add_argument("--include", nargs="+")
    p.add_argument("--includeFile")
    p.add_argument("--exclude", nargs="+")
    p.add_argument("--excludeFile")
    p.add_argument("--minCalls", type=int, default=1)
    p.add_argument("--minAlleles", type=int, default=1)
    p.add_argument("--maxAlleles", type=float, default="inf")
    p.add_argument("--minVarCount", type=int, default=None)
    p.add_argument("--maxHet", type=float, default=None)
    p.add_argument("--minFreq", type=float, default=None)
    p.add_argument("--maxFreq", type=float, default=None)
    p.add_argument("--HWE", nargs=2, metavar=("P-value", "'top'/'bottom'/'both'"))
    p.add_argument("--minPopCalls", nargs="+", type=int)
    p.add_argument("--minPopAlleles", nargs="+", type=int)
    p.add_argument("--maxPopAlleles", nargs="+", type=int)
    p.add_argument("--fixedDiffs", action="store_true")
    p.add_argument("--nearlyFixedDiff", type=float)
    p.add_argument("--thinDist", type=int)
    p.add_argument("--podSize", type=int, default=10000)
    p.add_argument("--noPrecomp", help="Accepted and ignored", action="store_true")
    p.add_argument("--noTest", action="store_true")
    C.add_engine_args(p)
    return p


def _per_pop(values, popNames):
    """filterGenotypes.py:245-263: one value for every population, or one per population"""
    if len(values) == 1:
        values = values * len(popNames)
    assert len(values) == len(popNames)
    return list(values)


def plan(args, headers, first_line):
    """The reference's set-up (filterGenotypes.py:191-331) and the refusals.  Returns a dict with the samples, their
    columns and ploidies, the populations, the filter settings and the header row."""
    if args.outputGenoFormat == "randomAllele":
        raise SystemExit("filterGenotypes: -of randomAllele is not supported: the reference draws the allele with an unseeded "
                         "random.sample (genomics.py:376), so its output is not a function of the input")
    if args.HWE:
        raise SystemExit("filterGenotypes: --HWE is not supported: the reference's inHWE calls an undefined `unique` "
                         "(genomics.py:729) whenever the test runs")
    if args.hostParse:
        raise SystemExit("filterGenotypes: --hostParse is not supported: the kept rows are formatted from the device copy "
                         "of the text")
    if args.devices not in (None, 1):
        raise SystemExit("filterGenotypes: --devices is not supported; the filter runs on one GPU")
    include = list(args.include or [])
    exclude = list(args.exclude or [])
    if args.includeFile:
        with open(args.includeFile) as f:
            include += f.read().split()
    if args.excludeFile:
        with open(args.excludeFile) as f:
            exclude += f.read().split()
    include = set(include) if include else None
    exclude = set(exclude) if exclude else None
    popDict, popNames = {}, []
    mpc = mpa = xpa = None
    if args.pop:
        for pop in args.pop:
            popNames.append(pop[0])
            popDict[pop[0]] = [] if len(pop) == 1 else pop[1].split(",")
        if args.popsFile:
            with open(args.popsFile) as pf:
                for line in pf:
                    ind, pop = line.split()
                    if pop in popDict and ind not in popDict[pop]:
                        popDict[pop].append(ind)
        if args.minPopCalls:
            mpc = _per_pop(args.minPopCalls, popNames)
        if args.minPopAlleles:
            mpa = _per_pop(args.minPopAlleles, popNames)
            if args.maxPopAlleles is None:
                xpa = [4] * len(popNames)
        if args.maxPopAlleles:
            xpa = _per_pop(args.maxPopAlleles, popNames)
            if args.minPopAlleles is None:
                mpa = [0] * len(popNames)
    allSamples = headers[2:]
    samples = args.samples.split(",") if args.samples else None
    exSamples = args.excludeSamples.split(",") if args.excludeSamples else []
    if samples is not None:
        for sample in samples:
            assert sample in allSamples, "Sample name not in header: " + sample
    elif args.pop and not args.keepAllSamples:
        samples = [i for j in popDict.values() for i in j]
        assert len(set(samples)) == len(samples), "Populations cannot share the same sample"
    else:
        samples = allSamples
    samples = [s for s in samples if s not in exSamples]
    if args.minCalls:
        assert args.minCalls <= len(samples), "Minimum calls is greater than number of specified samples."
    for popName in popNames:
        popDict[popName] = [s for s in popDict[popName] if s not in exSamples]
        for sample in popDict[popName]:
            assert sample in allSamples, "Sample name not in header: " + sample
    idx = {s: k for k, s in enumerate(samples)}
    for popName in popNames:
        for s in popDict[popName]:
            if s not in idx:
                raise SystemExit("filterGenotypes: population %s member %s is not among the selected samples (the reference "
                                 "fails with a KeyError in siteTest)" % (popName, s))
    if len(set(samples)) != len(samples):
        raise SystemExit("filterGenotypes: a sample is selected twice")
    if args.ploidy is not None:
        ploidy = args.ploidy if len(args.ploidy) != 1 else args.ploidy * len(samples)
        assert len(ploidy) == len(samples), "Incorrect number of ploidy values supplied."
        ploidyDict = dict(zip(samples, ploidy))
    elif args.ploidyFile is not None:
        with open(args.ploidyFile) as pf:
            ploidyDict = dict([[s[0], int(s[1])] for s in [l.split() for l in pf]])
    else:
        ploidyDict = dict(zip(samples, [None] * len(samples)))
    if args.outputGenoFormat == "bases":
        assert args.ploidy is not None or args.ploidyFile, "Ploidy must be specified."
    # ploidy of every sample: given, or the width of its token on the first data line (later lines must match)
    toks = first_line.split()[2:]
    col = {}
    for i, n in enumerate(allSamples):
        col.setdefault(n, i)
    cols = [col[s] for s in samples]
    pl = []
    for s, c in zip(samples, cols):
        v = ploidyDict.get(s)
        if v is None:
            t = toks[c] if c < len(toks) else ""
            v = 2 if args.inputGenoFormat == "diplo" else ((len(t) + 1) // 2 if args.inputGenoFormat == "phased" else len(t))
        pl.append(int(v))
    for s, v in zip(samples, pl):
        if not 1 <= v <= 8:
            raise SystemExit("filterGenotypes: ploidy %d of sample %s is not supported (1 to 8)" % (v, s))
        if args.inputGenoFormat == "diplo" and v != 2:
            raise SystemExit("filterGenotypes: sample %s has ploidy %d; a diplo genotype holds two alleles%s" %
                             (s, v, " and --forcePloidy would change it" if args.forcePloidy else ""))
        if args.outputGenoFormat == "diplo" and v != 2:
            raise SystemExit("filterGenotypes: -of diplo needs diploid samples (genomics.py:359); %s has ploidy %d" % (s, v))
    if args.outputGenoFormat != "bases":
        head = headers[0:2] + samples
    else:
        head = headers[0:2] + [s + "_" + l for s, v in zip(samples, pl) for l in string.ascii_uppercase[:v]]
    hap0 = np.concatenate([[0], np.cumsum(pl)[:-1]]).astype(np.int32) if pl else np.zeros(0, np.int32)
    n_cols = max(len(allSamples), 1)
    col_hap = np.full(n_cols, -1, dtype=np.int32)
    col_pl = np.ones(n_cols, dtype=np.int8)
    for k, c in enumerate(cols):
        col_hap[c] = hap0[k]
        col_pl[c] = pl[k]
    pops = [[idx[s] for s in popDict[popName]] for popName in popNames]
    spec = dict(samp_hap0=hap0, samp_ploidy=np.array(pl, np.int8), pops=pops, min_calls=args.minCalls, min_alleles=args.minAlleles, max_alleles=args.maxAlleles,
                min_var_count=args.minVarCount, max_het=args.maxHet, min_freq=args.minFreq, max_freq=args.maxFreq,
                min_pop_calls=mpc, min_pop_alleles=mpa, max_pop_alleles=xpa, fixed_diffs=args.fixedDiffs,
                nearly_fixed_diff=args.nearlyFixedDiff, partial_to_missing=args.partialToMissing, no_test=args.noTest,
                thin_dist=args.thinDist or 0, pod_size=args.podSize)
    return dict(samples=samples, cols=cols, ploidy=pl, popNames=popNames, popDict=popDict, include=include, exclude=exclude,
                head=head, col_hap=col_hap, col_pl=col_pl, H=int(sum(pl)), spec=spec)


def chunks(stream, target, pod_lines):
    """Complete data lines in chunks of about `target` bytes (cut at line starts).  With pod_lines, every chunk but the
    last holds a whole number of pods, so that each chunk starts a pod."""
    rest = b""
    eof = False
    while not eof or rest:
        buf = rest
        while len(buf) < target and not eof:
            blk = stream.read(max(target - len(buf), 1 << 16))
            if not blk:
                eof = True
                break
            buf += blk
        if not buf:
            return
        cut = len(buf) if eof else buf.rfind(b"\n") + 1
        if pod_lines and not eof:
            nl = np.flatnonzero(np.frombuffer(buf, dtype=np.uint8) == 10)
            whole = (len(nl) // pod_lines) * pod_lines
            if whole == 0:                  # not one whole pod yet: read on
                rest = buf
                blk = stream.read(target)
                if not blk:
                    eof = True
                rest += blk
                continue
            cut = int(nl[whole - 1]) + 1
        elif cut == 0:                      # one line longer than the target: read on
            blk = stream.read(target)
            if not blk:
                eof = True
            rest = buf + blk
            continue
        yield buf[:cut]
        rest = buf[cut:]


def _scaffolds(data, newsc, off):
    """scaffold name of every run of equal scaffolds, and each site's run"""
    runs = np.flatnonzero(newsc)
    names = [data[int(off[r]):int(off[r]) + 4096].split(None, 1)[0].decode() for r in runs]
    run_of = np.cumsum(newsc.astype(np.int64)) - 1
    return names, run_of


def _first_data_line(src):
    """(bytes read from src so far, the first complete data line): reads on until a line that is not blank and not a '#'
    comment has ended, however long it is"""
    body = b""
    start = 0                                   # first byte of the line not yet looked at
    while True:
        nl = body.find(b"\n", start)
        if nl < 0:
            blk = src.read(1 << 20)
            if blk:
                body += blk
                continue
            nl = len(body)                      # last line without a newline
        ln = body[start:nl]
        if ln.strip() and not ln.startswith(b"#"):
            return body, ln
        if nl >= len(body):
            return body, b""
        start = nl + 1


def main(argv=None):
    args = build_parser().parse_args(argv)
    src = open_input(args.infile)
    head_line = src.readline()
    headers = head_line.decode().split()
    body0, first = _first_data_line(src)
    pl = plan(args, headers, first.decode())
    stream = io.BufferedReader(Chain(body0, src), buffer_size=1 << 20)
    spec = pl["spec"]
    fmt = args.outputGenoFormat
    freq_order = args.alleleOrder == "freq"
    tm = C.Timing(args.timing)
    target = env_int("PG_FILTER_CHUNK_BYTES", 1 << 30)
    slab = env_int("PG_FILTER_SLAB_BYTES", 64 << 20)
    pod_lines = args.podSize if args.thinDist else 0
    n_sites = n_kept = n_lines = 0
    with (open_output(args.outfile) as out, Engine(args.device) as eng,
          SlabWriter(out.write, slab, PinnedArray) as w):
        out.write(("\t".join(pl["head"]) + "\n").encode())
        eng.set_strict_ingest(True)
        for chunk in chunks(stream, target, pod_lines):
            S = eng.ingest_text(chunk, FMT_CODE[args.inputGenoFormat], pl["col_hap"], pl["col_pl"], pl["H"])
            tm.mark("ingest", eng)
            if args.thinDist:
                lines = chunk.count(b"\n") + (0 if chunk.endswith(b"\n") else 1)
                if lines != S:
                    raise SystemExit("filterGenotypes: --thinDist on a file with comment or blank lines after the header: "
                                     "the reference counts them as sites and fails on them (data lines %d-%d)" %
                                     (n_lines + 1, n_lines + lines))
                n_lines += lines
            n_sites += S
            if S == 0:
                continue
            pos, newsc, off = eng.ingest_meta(S, release=False)
            names, run_of = _scaffolds(chunk, newsc, off)
            cmask = None
            if pl["include"] is not None or pl["exclude"] is not None:
                ok = np.array([(pl["include"] is None or n in pl["include"]) and (pl["exclude"] is None or n not in pl["exclude"])
                               for n in names], dtype=np.uint8)
                cmask = ok[run_of]
            ids = {}
            run_id = np.array([ids.setdefault(n, len(ids)) for n in names], dtype=np.int32)
            nk, flags = eng.filter(spec, contig_mask=cmask, scaf_id=run_id[run_of])
            tm.mark("filter", eng)
            if fmt == "diplo" and flags & 2 and not args.partialToMissing:
                raise SystemExit("filterGenotypes: -of diplo on a kept site with a partly missing genotype: the reference "
                                 "fails there (genomics.py:360, no diplotype for such a pair); use --partialToMissing")
            if fmt == "count" and flags & 4:
                raise SystemExit("filterGenotypes: -of count on a kept site with no called allele: the reference fails "
                                 "there (genomics.py:495, no allele to count)")
            if flags & 1 and (fmt in ("coded", "count") or freq_order) and args.verbose:
                sys.stderr.write("filterGenotypes: kept sites with tied allele counts: their frequency order is the one a "
                                 "stable sort gives (numpy may break such ties otherwise)\n")
            row = 0
            while row < nk:
                rows, nb = eng.filter_emit(fmt, freq_order, row, w.slab(), w.cap)
                w.write(nb)
                row += rows
            n_kept += nk
            tm.mark("emit", eng)
            if args.verbose:
                sys.stderr.write("%d lines read, %d written\n" % (n_sites, n_kept))
    tm.write(sites=n_sites, kept=n_kept)


if __name__ == "__main__":
    main()
