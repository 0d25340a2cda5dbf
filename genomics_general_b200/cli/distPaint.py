#!/usr/bin/env python
"""Drop-in for the reference's distPaint.py (flags 157-188, populations 239-255, worker 49-92), on the GPU.

Every sample is one haploid sequence (-f haplo, ploidy 1).  For every window and sample the nearest reference population
by p-distance is chosen and confirmed by rank-sum tests (default) or by the margin of --delta_threshold; pg_distpaint does
the distances, the means and both rules on the device.  Where the reference's behaviour is kept on purpose:
  - the reference population members are HEADER positions of the samples, used as rows of the alignment the reference
    sorts by sample name (genomics.py:1122), and output column k (labelled with the k-th header name) holds the result of
    the k-th sample in name order;
  - populations follow distPaint.py:239-255, not popgenWindows': -p takes one comma-separated list (further words are
    ignored), a repeated -p resets the list and adds a second column, --popsFile lines must have exactly two fields, and
    unknown names in that file are skipped.
Where it differs: a genotype character other than A C G T N or an IUPAC letter (e.g. '-') is missing here; the reference's
worker dies on it (KeyError in genomics.py:1118).  --include / --exclude read their files as the other command lines do
(the reference opens them with mode "rU", which Python 3.11 removed).  --minData, --samples, -T and --verbose are accepted
and ignored, as by the reference.  Refused before any work: --header (the reference always takes the sample names from
the file's first line), --delta_threshold with one population (the reference's worker raises IndexError and the script
never ends) and --devices N > 1."""
from __future__ import annotations

import argparse
import re
import sys

import numpy as np

from .. import geno_io
from ..engine import Engine
from . import _common as C


def build_parser():
    p = argparse.ArgumentParser()
    C.add_window_args(p, overlap_short=True)
    p.add_argument("--minData", type=float, metavar="prop", default=0.01)
    p.add_argument("--p_threshold", type=float, default=0.05)
    p.add_argument("--delta_threshold", type=float, default=None)
    p.add_argument("-p", "--population", action="append", nargs="+", metavar=("popName", "[samples]"))
    p.add_argument("--popsFile")
    p.add_argument("--samples", metavar="sample names")
    p.add_argument("--noresult", type=int, default=-1)
    p.add_argument("-g", "--genoFile", required=True)
    p.add_argument("-o", "--outFile")
    p.add_argument("--exclude")
    p.add_argument("--include")
    p.add_argument("--header")
    p.add_argument("-T", "--threads", type=int, default=1, metavar="threads")
    p.add_argument("--verbose", action="store_true")
    p.add_argument("--addWindowID", action="store_true")
    p.add_argument("--writeFailedWindows", action="store_true")
    C.add_engine_args(p)
    return p


def reference_populations(pop_args, pops_file, allInds):
    """distPaint.py:239-255: popNames (a repeated -p appears twice) and each name's ordered member list of header
    indices (duplicates kept)."""
    popNames, members = [], {}
    for p in pop_args:
        popNames.append(p[0])
        members[p[0]] = []
        if len(p) > 1:
            for ind in p[1].split(","):
                members[p[0]].append(allInds.index(ind))
    if pops_file:
        with open(pops_file, "rt") as pf:
            popDict = dict([ln.split() for ln in pf])
        for ind in popDict.keys():
            if popDict[ind] in members and ind in allInds:
                members[popDict[ind]].append(allInds.index(ind))
    for name in popNames:
        assert len(members[name]) >= 1, f"Reference population {name} appears to have no individuals."
    return popNames, members


def check_haplo_tokens(path):
    """The width test of the device ingest (pg_ingest_set_strict level 2) for the host tokenizer: a genotype token wider
    than one character fails the reference's ploidy assertion (genomics.py:1111)."""
    wide = re.compile(rb"\S\S")
    line = 0
    for ln in geno_io.read_bytes(path).split(b"\n")[1:]:
        if not ln.strip() or ln.startswith(b"#"):
            continue
        line += 1
        f = ln.split(None, 2)
        m = wide.search(f[2]) if len(f) > 2 else None
        if m:
            raise geno_io.PgError("data line %d, genotype column %d: the token's allele count does not match the sample's "
                                  "ploidy (genomics.py:1111 asserts the same)" % (line, len(f[2][:m.start()].split()) + 1))


def main(argv=None):
    args = build_parser().parse_args(argv)
    args.genoFormat = "haplo"                    # distPaint.py:257-259, 65
    if args.header:
        raise SystemExit("distPaint: --header is not supported: the reference always reads the sample names from the "
                         "genotype file's first line")
    if args.devices not in (None, 1):
        raise SystemExit("distPaint: --devices is not supported; the assignment runs on one GPU")
    minSites, coords = C.check_window_args(args)
    assert args.population, "At least one reference population (-p) is required."
    allInds = C.header_names(args.genoFile)
    popNames, members = reference_populations(args.population, args.popsFile, allInds)
    if args.delta_threshold is not None and len(popNames) < 2:
        raise SystemExit("distPaint: --delta_threshold compares the two nearest populations and needs at least two "
                         "(with one the reference never finishes)")
    ploidyDict = dict(zip(allInds, [1] * len(allInds)))
    tm = C.Timing(args.timing)
    eng = Engine(args.device)
    with eng:
        eng.set_strict_ingest(2)
        gd = C.load_geno(args, allInds, ploidyDict, engine=eng)
        if gd.geno is not None:
            check_haplo_tokens(args.genoFile)
        tm.mark("ingest", eng)
        ws = C.make_windows(args, gd, minSites, coords, C.read_scaffold_list(args.include), C.read_scaffold_list(args.exclude))
        lo, hi = ws.ranges()
        # genoToAlignment sorts the rows by name; header indices are then used as row indices (distPaint.py:73-74, 247)
        order = np.argsort(allInds)
        hap_of_row = np.asarray(gd.hap_off, dtype=np.int64)[order]
        ref_off = np.cumsum([0] + [len(members[n]) for n in popNames]).astype(np.int32)
        ref_hap = np.array([hap_of_row[j] for n in popNames for j in members[n]], dtype=np.int32)
        tm.mark("windows")
        C.ensure_resident(eng, gd)
        eng.set_windows(lo, hi)
        delta = args.delta_threshold is not None
        r = eng.distpaint(hap_of_row, ref_off, ref_hap, minSites, delta=delta,
                          threshold=args.delta_threshold if delta else args.p_threshold, noresult=args.noresult)
        tm.mark("assignment", eng)
    csum = np.concatenate([[0], np.cumsum(np.asarray(gd.pos, dtype=np.int64))])
    out = C.open_out(args.outFile)
    out.write("\t".join(["scaffold", "start", "end", "mid", "sites"] if not args.addWindowID else
                        ["windowID", "scaffold", "start", "end", "mid", "sites"]) + "\t")
    out.write("\t".join(allInds) + "\n")
    nan_cols = ["nan"] * len(allInds)
    for k in range(len(ws)):
        sites = int(hi[k] - lo[k])
        good = sites >= minSites
        if not (good or args.writeFailedWindows):
            continue
        row = [] if not args.addWindowID else [ws.ID[k]]
        row += C.window_prefix(args, ws, k, gd, sites, csum[hi[k]] - csum[lo[k]])
        out.write("\t".join([str(x) for x in row] + ([str(int(v)) for v in r["assign"][k]] if good else nan_cols)) + "\n")
    if out is not sys.stdout:
        out.close()
    tm.mark("rows")
    tm.write(sites=int(gd.n_sites), samples=len(allInds), populations=len(popNames), windows=len(ws))


if __name__ == "__main__":
    main()
