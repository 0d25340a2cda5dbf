#!/usr/bin/env python
"""Drop-in for the reference's popgenWindows.py (same flags, header and rows), computed on the GPU.

Reference: genomics_general/popgenWindows.py — argparse 170-213, sample/pop parsing 253-307, header 319-354,
worker stats_wrapper 28-75.  The process pipeline (producer / -T workers / sorter / writer) is replaced by:
parse the whole file once -> dense int8 matrix -> all windows in one engine call -> rows.
All six --analysis modes run on the GPU.  The reference caches one haplotype distance matrix per window and its
analyses modify it in place (groupDistStats masks pairs with n_ij < minSites and the diagonal, genomics.py:959-963;
indPairDists masks the diagonal, 940), so later analyses of the same window see the masked matrix — the engine calls
below take that state as arguments (min_sites / diag_nan).
"""
from __future__ import annotations

import argparse
import itertools
import os
import sys

import numpy as np

from .. import genomics, geno_io, mgpu, multigpu
from ..engine import Engine
from . import _common as C


def build_parser():
    p = argparse.ArgumentParser()
    C.add_window_args(p, overlap_short=True)
    p.add_argument("--minData", help="Minumum proportion of individuals (or pairs) with >=minSites data", type=float,
                   metavar="prop", default=0.01)
    p.add_argument("-p", "--population", help="Pop name and optionally sample names (separated by commas)",
                   action="append", nargs="+", metavar=("popName", "[samples]"))
    p.add_argument("--popsFile", help="Optional file of sample names and populations")
    p.add_argument("--samples", help="Samples to include for individual analysis", metavar="sample names")
    p.add_argument("--ploidy", help="Ploidy for each sample", type=int, nargs="+")
    p.add_argument("--ploidyFile", help="File with samples names and ploidy as columns")
    p.add_argument("--haploid", help="Alternatively just name samples that are haploid (comma separated)",
                   metavar="sample names")
    p.add_argument("--inferPloidy", help="Ploidy will be inferred in each window (NOT RECOMMENED)", action="store_true")
    p.add_argument("--analysis", help="Type of statistics to get", nargs="+",
                   choices=("popFreq", "popDist", "popPairDist", "indPairDist", "indHet", "hapStats"),
                   default=("popDist", "popPairDist",))
    p.add_argument("--hapDist", type=float, default=0)
    p.add_argument("--roundTo", help="Round stats to X decimal places", type=int, default=4)
    p.add_argument("-g", "--genoFile", help="Input genotypes file")
    p.add_argument("-o", "--outFile", help="Results file")
    p.add_argument("--exclude", help="File of scaffolds to exclude")
    p.add_argument("--include", help="File of scaffolds to analyse")
    p.add_argument("-f", "--genoFormat", help="Format of genotypes in genotypes file",
                   choices=("phased", "pairs", "haplo", "diplo"), required=True)
    p.add_argument("--header", help="Header text if no header in input")
    p.add_argument("-T", "--threads", help="accepted for compatibility (the GPU engine replaces the workers)", type=int,
                   default=1, metavar="threads")
    p.add_argument("--verbose", action="store_true")
    p.add_argument("--addWindowID", help="Add window name or number as first column", action="store_true")
    p.add_argument("--writeFailedWindows", help="Write output even for windows with too few sites.", action="store_true")
    C.add_engine_args(p)
    return p


def main(argv=None):
    args = build_parser().parse_args(argv)
    minSites, coords = C.check_window_args(args)

    popNames, popInds, allInds = [], [], []
    if args.population is not None:
        popNames, popInds = C.parse_pop_args(args.population, args.popsFile)
        allInds += sorted(set(i for p in popInds for i in p))
    if args.samples is not None:
        allInds = sorted(set(allInds + args.samples.split(",")))
    if len(allInds) == 0:
        allInds = C.header_names(args.genoFile) if args.header is None else args.header.split()[2:]
    if len(popNames) == 0 and ("popFreq" in args.analysis or "popDist" in args.analysis or "popPairDist" in args.analysis
                               or "hapStats" in args.analysis):
        popNames.append("all")
        popInds.append(allInds)
    ploidyDict = C.ploidy_dict(args, allInds, args.haploid.split(",") if args.haploid else None)
    sampleData = genomics.SampleData(indNames=allInds, popNames=popNames, popInds=popInds, ploidyDict=ploidyDict)

    # --devices N: this process becomes rank 0 of N (ranks 1.. are re-launched copies of this command line)
    rdv = mgpu.init("genomics_general_b200.cli.popgenWindows", argv, args.devices)
    out = C.open_out(args.outFile) if (rdv is None or rdv.rank == 0) else open(os.devnull, "wt")
    out.write("scaffold,start,end,mid,sites," if not args.addWindowID else "windowID,scaffold,start,end,mid,sites,")
    stats = []
    if "popFreq" in args.analysis:
        for key in ("l_", "S_", "thetaPi_", "thetaW_", "TajD_"):
            stats += [key + n for n in popNames]
    if "popDist" in args.analysis:
        stats += ["pi_" + n for n in popNames]
    if "popPairDist" in args.analysis:
        stats += ["dxy_" + x + "_" + y for x, y in itertools.combinations(popNames, 2)]
        stats += ["Fst_" + x + "_" + y for x, y in itertools.combinations(popNames, 2)]
    ind_sorted = sorted(allInds)
    if "indPairDist" in args.analysis:
        stats += ["_".join(["d", i, j]) for i, j in itertools.combinations_with_replacement(ind_sorted, 2)]
    if "indHet" in args.analysis:      # the reference's column order here is that of list(set(...)) (popgenWindows.py:277)
        stats += ["het_" + n for n in allInds]
    if "hapStats" in args.analysis:
        for key in ("H1_", "H12_", "H2_"):
            stats += [key + n for n in popNames]
    out.write(",".join(stats) + "\n")

    eng = Engine(args.device if rdv is None else mgpu.device_for(rdv, args.device))
    tm = C.Timing(args.timing if (rdv is None or rdv.rank == 0) else None)

    # columns in the reference's haplotype order (sorted sequence names): H12's greedy clustering breaks ties by row
    col_order = C.alignment_order(sampleData.indNames, ploidyDict, args.genoFormat)
    if rdv is None:
        gd = C.load_geno(args, col_order, ploidyDict, header=args.header, engine=eng)
    else:
        gd, starts, off_all = mgpu.sharded_ingest(eng, rdv, args.genoFile, args.genoFormat, col_order, ploidyDict, args.header)
    tm.mark("ingest", eng)
    ws = C.make_windows(args, gd, minSites, coords, C.read_scaffold_list(args.include), C.read_scaffold_list(args.exclude))
    tm.mark("windows")
    sys.stderr.write("\n%d sites x %d haplotypes, %d windows\n" % (gd.n_sites, gd.n_haps, len(ws)))
    lo, hi = ws.ranges()
    written = 0
    with eng:
        P = len(popNames)
        if rdv is None:
            C.ensure_resident(eng, gd)
            eng.set_windows(lo, hi)
            eng.set_pops(C.hap_pop_vector(gd, popNames, popInds), max(P, 1))
            eng.set_freqstats("popFreq" in args.analysis)
            r = eng.popgen(minSites, args.minData)
        else:
            # this rank's windows (those that start in its share of the file) + the sites they need from the next share
            idx, llo, lhi, halo = mgpu.assign_windows(lo, hi, starts, rdv.rank)
            mgpu.fetch_halo(eng, args.genoFile, gd, starts, off_all, rdv.rank, halo, args.genoFormat, ploidyDict)
            eng.set_windows(llo, lhi)
            eng.set_pops(C.hap_pop_vector(gd, popNames, popInds), max(P, 1))
            eng.set_freqstats("popFreq" in args.analysis)          # the popFreq counters travel in the same records
            all_idx = [mgpu.assign_windows(lo, hi, starts, q)[0] for q in range(rdv.world)]
            w_max, row_of = mgpu.gathered_order(all_idx)
            mgpu.nccl_connect(eng, rdv)
            table = np.zeros((rdv.world * w_max, eng.popgen_record_width()), dtype=np.float64)
            eng.popgen_allgather(w_max, table, minSites, args.minData)          # ONE ncclAllGather of the records
            eng.nccl_finalize()
            rows = np.array([row_of[w] for w in range(len(ws))], dtype=np.int64)
            r = multigpu.unpack_device_records(table[rows] if len(rows) else table[:0], P)
        fq = None
        if "popFreq" in args.analysis:
            hp_all = C.hap_pop_vector(gd, popNames, popInds)
            if np.any(hp_all < 0):
                raise NotImplementedError("popFreq with samples outside every population (--samples) is not supported")
            if rdv is None:
                fq = eng.popgen_freqstats()
            else:                          # [l, S[P], thetaPi[P], thetaW[P], TajD[P]] behind the distance statistics of a record
                pf = r["popfreq"]
                fq = dict(l=pf[:, 0], S=pf[:, 1:1 + P], thetaPi=pf[:, 1 + P:1 + 2 * P], thetaW=pf[:, 1 + 2 * P:1 + 3 * P],
                          TajD=pf[:, 1 + 3 * P:1 + 4 * P])
        npairs = P * (P - 1) // 2
        # state of the reference's cached distance matrix when the later analyses run (popgenWindows.py:50-64)
        masked = minSites if ("popDist" in args.analysis or "popPairDist" in args.analysis) else 0
        dmat = het = hst = None
        # (on several devices these run on the rank's own windows; a rank without windows has nothing to compute)
        idle = rdv is not None and len(idx) == 0
        if "indPairDist" in args.analysis:
            inv = {gd.names.index(n): k for k, n in enumerate(ind_sorted)}
            hap_ind = np.repeat(np.array([inv[i] for i in range(len(gd.names))], dtype=np.int32), gd.ploidy.astype(np.int64))
            dmat = np.zeros((0, len(ind_sorted), len(ind_sorted))) if idle else \
                eng.pairdist(hap_ind, len(ind_sorted), False, min_sites=masked)["dist"]
        if "indHet" in args.analysis:
            inv = {gd.names.index(n): k for k, n in enumerate(allInds)}
            hap_ind = np.repeat(np.array([inv[i] for i in range(len(gd.names))], dtype=np.int32), gd.ploidy.astype(np.int64))
            het = np.zeros((0, len(allInds))) if idle else eng.ind_het(hap_ind, len(allInds), min_sites=masked)
        if "hapStats" in args.analysis:
            hst = np.zeros((0, max(P, 1), 3)) if idle else \
                eng.hapstats(args.hapDist, min_sites=masked, diag_nan=bool(masked) or "popDist" in args.analysis
                             or "popPairDist" in args.analysis or "indPairDist" in args.analysis)
        if rdv is not None:
            # The pairwise analyses have no collective: a rank publishes the arrays of its windows through the exchange
            # directory (they are on the host already), rank 0 puts them in window order.
            extras = dict(dmat=dmat, het=het, hst=hst)
            for name, arr in extras.items():
                if arr is not None:
                    rdv.put("x_" + name, np.asarray(arr, dtype=np.float64))
            if rdv.rank != 0:
                rdv.finish()
                return
            for name, arr in extras.items():
                if arr is not None:
                    full = np.full((len(ws),) + tuple(np.shape(arr)[1:]), np.nan)
                    for q in range(rdv.world):
                        if len(all_idx[q]):
                            full[all_idx[q]] = rdv.get("x_" + name, q)
                    extras[name] = full
            dmat, het, hst = extras["dmat"], extras["het"], extras["hst"]
        tm.mark("statistics", eng)
        iu = np.triu_indices(len(ind_sorted)) if dmat is not None else None
        simple = fq is None and dmat is None and het is None and hst is None
        if simple and len(ws):
            # popDist / popPairDist only: the statistics of ALL windows are rounded and printed at once by the native row
            # printer (numpy's float -> str, i.e. what str(round(np.float64(v), n)) gives; popgenWindows.py:66-74); only the
            # five prefix fields are assembled per window.  20 000 windows: 0.3 s instead of 3 s of Python.
            sites_all = np.asarray(r["sites"])
            goodv = sites_all >= minSites
            cols = []
            if "popDist" in args.analysis:
                cols.append(r["pi"])
            if "popPairDist" in args.analysis:
                cols += [r["dxy"], r["fst"]]
            M = np.concatenate(cols, axis=1) if cols else np.zeros((len(ws), 0))
            M = np.where(goodv[:, None], np.round(M.astype(np.float64), args.roundTo), np.nan)
            keep = np.flatnonzero(goodv | bool(args.writeFailedWindows))
            prefixes = []
            for k in keep:
                pre = C.window_prefix(args, ws, int(k), gd, r["sites"][k], r["pos_sum"][k])
                prefixes.append(",".join(str(x) for x in (([ws.ID[k]] if args.addWindowID else []) + pre))
                                + ("," if M.shape[1] else ""))
            if M.shape[1]:
                out.write(geno_io.format_matrix_rows(M[keep], sep=",", prefixes=prefixes))
            else:
                out.write("".join(p + "\n" for p in prefixes))
            written = len(keep)
        for k in (range(len(ws)) if not simple else ()):
            pre = C.window_prefix(args, ws, k, gd, r["sites"][k], r["pos_sum"][k])
            good = pre[4] >= minSites
            vals = []
            if good:
                if fq is not None:
                    # l is a Python int, S a numpy integer in the reference: both print without a decimal point
                    vals += [int(fq["l"][k])] * P
                    vals += [np.nan if np.isnan(v) else int(v) for v in fq["S"][k]]
                    vals += list(fq["thetaPi"][k]) + list(fq["thetaW"][k]) + list(fq["TajD"][k])
                if "popDist" in args.analysis:
                    vals += list(r["pi"][k])
                if "popPairDist" in args.analysis:
                    vals += list(r["dxy"][k]) + list(r["fst"][k])
                if dmat is not None:
                    vals += list(dmat[k][iu])
                if het is not None:
                    vals += list(het[k])
                if hst is not None:
                    vals += list(hst[k][:, 0]) + list(hst[k][:, 1]) + list(hst[k][:, 2])
                vals = [v if isinstance(v, int) else round(np.float64(v), args.roundTo) for v in vals]
            else:
                vals = [np.nan] * len(stats)
            if good or args.writeFailedWindows:
                row = ([] if not args.addWindowID else [ws.ID[k]]) + pre + vals
                out.write(",".join(str(x) for x in row) + "\n")
                written += 1
    if out is not sys.stdout:
        out.close()
    tm.mark("rows")
    tm.write(sites=int(gd.n_sites), haplotypes=int(gd.n_haps), windows=len(ws), devices=(1 if rdv is None else rdv.world))
    if rdv is not None:
        rdv.finish()
    sys.stderr.write(str(len(ws)) + " windows were tested.\n")
    sys.stderr.write(str(written) + " results were written.\n")
    sys.stderr.write("\nDone.\n")


if __name__ == "__main__":
    main()
