#!/usr/bin/env python
"""Drop-in for the reference's sfs.py (flags sfs.py:158-236): site frequency spectra of each population and, on request,
the joint spectra of pairs / trios / quartets, computed on the GPU — from genotypes (`--inputType genotypes`: per-site
counts -> target allele -> dense histograms, `pg_sfs`) or from tables of counts (`baseCounts`: the rows freq.py writes;
`targetCounts`, the script's default: e.g. freq.py --target derived --asCounts; `pg_sfs_tables`) — and written in the
reference's sparse format and order.
A request whose spectra add up to more cells than the dense histograms allow (engine.SFS_MAX_CELLS: e.g. 4-D spectra
of 129+ haplotypes per population, --doQuartets on many populations, count tables with large counts) takes the sparse
path instead (`pg_sfs_sparse` / `pg_sfs_tables_sparse`: only the non-empty cells, with their counts and first sites);
the choice is made once per request, and every other request keeps the dense path.

`--regions` / `--regionsFile` (sfs.py:266-276, 430-435): one count column per interval — the spectra of the intervals
are computed one after the other on the device (the interval is a site mask) and merged into the reference's rows.
`--subsample N` (sfs.py:23-24, 42-53, 380-403, 468-471): the reference down-samples the base counts of every population
at every site with numpy's GLOBAL Mersenne-Twister stream (`np.random.seed(--seed)`, one `np.random.choice` per
population and site, in file order).  The draw is defined by that stream, so it is made here with the same generator
(`np.random.RandomState(seed)`) on the per-site counts the device wrote, in the same order; the target allele and the
histograms of the down-sampled counts are then computed on the device (`pg_sfs_tables`).
Not covered: `--subsampleIndividuals` (the reference draws individuals with Python's *unseeded* `random.sample`, and on
Python >= 3.11 that call rejects the numpy array it is given, so every site is dropped, sfs.py:44-49).  Where the
reference's choice of the minor allele depends on numpy's unstable sort (two alleles with exactly equal counts,
sfs.py:90) the lower allele is used.  A region without coordinates ("chr1") means the whole scaffold; the reference
builds its upper limit as `np.array([np.inf], dtype=int)` (genomics.py:2367), which numpy >= 2 refuses.
"""
from __future__ import annotations

import argparse
import itertools
import sys

import numpy as np

from .. import genomics, mgpu
from ..engine import SFS_MAX_CELLS, Engine, sfs_shapes, sfs_table_dims
from . import _common as C


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument("-i", "--inputFile")
    p.add_argument("--inputType", choices=("genotypes", "baseCounts", "targetCounts"), default="targetCounts")
    p.add_argument("--scafCol", type=int, default=0)
    p.add_argument("--posCol", type=int, default=1)
    p.add_argument("--firstSampleCol", type=int, default=2)
    p.add_argument("--header")
    p.add_argument("--genoFormat", choices=("phased", "diplo", "alleles"), default="phased")
    p.add_argument("-p", "--pop", action="append", nargs="+", metavar=("popName", "[samples]"))
    p.add_argument("--popsFile")
    p.add_argument("--ploidy", type=int, nargs="+")
    p.add_argument("--ploidyFile")
    p.add_argument("--FSpops", action="append", type=str, nargs="+")
    p.add_argument("--doPairs", action="store_true")
    p.add_argument("--doTrios", action="store_true")
    p.add_argument("--doQuartets", action="store_true")
    p.add_argument("--subsample", nargs="+", type=int)
    p.add_argument("--subsampleIndividuals", action="store_true")
    p.add_argument("--pref", default="")
    p.add_argument("--suff", default=".sfs")
    p.add_argument("--pipe", action="store_true")
    p.add_argument("--polarized", action="store_true")
    p.add_argument("--outgroup")
    p.add_argument("--include", nargs="+")
    p.add_argument("--includeFile")
    p.add_argument("--exclude", nargs="+")
    p.add_argument("--excludeFile")
    p.add_argument("--regions", nargs="+")
    p.add_argument("--regionsFile")
    p.add_argument("-R", "--report", default=100000)
    p.add_argument("--verbose", action="store_true")
    p.add_argument("--seed", type=int, default=42)
    C.add_engine_args(p)
    return p


def dense_entries(hist, first):
    """Dense spectrum + first-site array -> its non-empty cells: (coords int64 [nnz, d], [count [nnz]], first [nnz]).
    `hist` / `first` may be lists (one spectrum per --regions interval): a cell is then non-empty in ANY interval, there is
    one count array per interval, and `first` is the cell's first site over the intervals that hold it."""
    hs = list(hist) if isinstance(hist, (list, tuple)) else [hist]
    fs = list(first) if isinstance(first, (list, tuple)) else [first]
    big = np.iinfo(np.int64).max
    tot = hs[0].copy()
    fmin = np.where(hs[0] > 0, fs[0], big)
    for h, f1 in zip(hs[1:], fs[1:]):
        tot = tot + h
        fmin = np.minimum(fmin, np.where(h > 0, f1, big))
    nz = np.argwhere(tot > 0)
    return nz, [h[tuple(nz.T)] for h in hs], fmin[tuple(nz.T)]


def order_entries(coords, counts, first):
    """Non-empty cells (coords [nnz, d], one count array per interval, first site [nnz]; any order) -> rows
    [k1, .., kd, count, ..] in the order the reference writes its nested SparseFS dictionaries (sfs.py:116-122): at every
    nesting level, keys in order of first appearance.  A site hits one cell of a spectrum, so the first sites are
    distinct and the order is total."""
    if len(coords) == 0:
        return []
    big = np.iinfo(np.int64).max
    f = np.asarray(first, dtype=np.int64)
    keys = []
    for lev in range(coords.shape[1]):
        _, inv = np.unique(coords[:, :lev + 1], axis=0, return_inverse=True)
        inv = np.asarray(inv).reshape(-1)
        m = np.full(inv.max() + 1, big, dtype=np.int64)
        np.minimum.at(m, inv, f)
        keys.append(m[inv])
    order = np.lexsort(tuple(reversed(keys)))
    return [list(map(int, coords[i])) + [int(c[i]) for c in counts] for i in order]


def ordered_chains(hist, first):
    """Dense spectrum + first-site array (or one of each per --regions interval) -> rows in the reference's order: a row
    carries one count per interval, and a key appears when its first site in ANY interval does (sfs.py:492-494 adds the
    whole boolean vector at once)."""
    return order_entries(*dense_entries(hist, first))


def merge_sparse(parts):
    """[(coords, count, first)] of one spectrum (one per interval or per rank) -> the union of their cells: (coords,
    [count per part, 0 where the part lacks the cell], first site over the parts that hold it)"""
    big = np.iinfo(np.int64).max
    d = parts[0][0].shape[1]
    allc = np.concatenate([np.asarray(p[0], dtype=np.int64).reshape(-1, d) for p in parts])
    if len(allc) == 0:
        return allc, [np.zeros(0, dtype=np.int64) for _ in parts], np.zeros(0, dtype=np.int64)
    coords, inv = np.unique(allc, axis=0, return_inverse=True)
    inv = np.asarray(inv).reshape(-1)
    counts, fmin, o = [], np.full(len(coords), big, dtype=np.int64), 0
    for c, n, f in parts:
        k = inv[o:o + len(c)]
        cnt = np.zeros(len(coords), dtype=np.int64)
        cnt[k] = n
        counts.append(cnt)
        np.minimum.at(fmin, k, np.asarray(f, dtype=np.int64))
        o += len(c)
    return coords, counts, fmin


def sparse_rows(per, n_spectra):
    """[(per spectrum (coords, count, first), n) per interval] -> the rows of every spectrum (cells merged over the
    intervals as merge_intervals + ordered_chains do for dense spectra)"""
    return [order_entries(*merge_sparse([p[0][k] for p in per])) for k in range(n_spectra)]


def write_rows(args, FSpops, rows):
    """one file per spectrum (<pref><pops joined by _><suff>, sfs.py:495-497) or everything to stdout (--pipe, 491-493)"""
    for i, grp in enumerate(FSpops):
        text = "\n".join("\t".join(str(x) for x in row) for row in rows[i]) + "\n"
        if args.pipe:
            sys.stdout.write(text)
        else:
            with open(args.pref + "_".join(grp) + args.suff, "w") as out:
                out.write(text)


def write_spectra(args, FSpops, hists, firsts):
    """dense spectra (one per FSpops entry, or one list per entry over the --regions intervals) -> write_rows"""
    write_rows(args, FSpops, [ordered_chains(hists[i], firsts[i]) for i in range(len(FSpops))])


def use_sparse(groups, dims):
    """the sparse path exactly where the dense spectra would exceed their limit (engine.SFS_MAX_CELLS in all); decided once
    per request, so every interval and every rank takes the same path"""
    return sum(sfs_shapes(groups, dims)[1]) > SFS_MAX_CELLS


def parse_region_text(text):
    """genomics.parseRegionText (genomics.py:2323-2336): chrom | chrom:pos | chrom:from-to (a reversed pair is swapped)."""
    parts = text.split(":")
    if len(parts) >= 3 and parts[2] != "" and parts[2] not in "+-":
        raise ValueError("Incorrect region specification")
    try:
        ft = [int(x) for x in parts[1].split("-")]
        if len(ft) == 1:
            ft.append(None)
        if ft[1] is not None and ft[0] > ft[1]:
            ft = ft[::-1]
        return (parts[0], ft[0], ft[1])
    except Exception:
        return (parts[0], None, None)


def read_intervals(args):
    """--regions / --regionsFile -> [(chrom, start, end)], both ends inclusive, end None = open (genomics.Intervals,
    genomics.py:2361-2367: no start = 0; no end = the start, i.e. one position; neither = the whole scaffold)."""
    if args.regions:
        tuples = [parse_region_text(r) for r in args.regions]
    elif args.regionsFile:
        with open(args.regionsFile, "rt") as f:
            tuples = [tuple(line.split()) for line in f if line.strip()]
    else:
        return None
    out = []
    for t in tuples:
        has_start = len(t) > 1 and t[1] is not None
        start = int(t[1]) if has_start else 0
        end = int(t[2]) if len(t) > 2 and t[2] is not None else (start if has_start else None)
        out.append((str(t[0]), start, end))
    sys.stderr.write("Recording SFS for {} intervals\n".format(len(out)))
    return out


def interval_masks(intervals, scaffold_of_site, pos, base_mask):
    """Intervals.containsPoint (genomics.py:2377-2378) for every site: one uint8 mask per interval, ANDed with the
    --include / --exclude mask.  Without intervals: [base_mask]."""
    if intervals is None:
        return [base_mask]
    pos = np.asarray(pos, dtype=np.int64)
    out = []
    for chrom, start, end in intervals:
        m = (scaffold_of_site == chrom) & (pos >= start)
        if end is not None:
            m &= pos <= end
        if base_mask is not None:
            m &= base_mask.astype(bool)
        out.append(m.astype(np.uint8))
    return out


def considered_sites(masks, n):
    """sites that get as far as the draw: inside --include / --exclude and inside at least one interval (sfs.py:427-435)"""
    if masks[0] is None:
        return np.ones(n, dtype=bool)
    return np.logical_or.reduce([np.asarray(m, dtype=bool) for m in masks])


def subsample_sizes(args, inPopNames):
    """sfs.py:380-385"""
    if args.subsampleIndividuals:
        raise NotImplementedError("--subsampleIndividuals: the reference draws with Python's unseeded random.sample (and drops "
                                  "every site on Python >= 3.11, sfs.py:44-49); not supported")
    if args.subsample is None:
        return None
    sub = list(args.subsample)
    if len(sub) == 1:
        sub = sub * len(inPopNames)
    assert len(sub) == len(inPopNames), \
        "subsample list ({}) must match number of ingroup populations ({}).".format(len(sub), len(inPopNames))
    return sub


def downsample_counts(counts, sizes, seed, considered):
    """downSampleBaseCounts at every considered site (sfs.py:23-24, 51, 470): for site after site and in-group population
    after population, N alleles are drawn without replacement from the population's base counts with the legacy global
    stream numpy seeds with --seed; a population with fewer than N alleles raises inside the reference's list
    comprehension, the site is dropped and the populations after it draw nothing.  counts: [n, >= len(sizes), 4];
    returns (down-sampled copy, uint8 mask of the sites that went through)."""
    rs = np.random.RandomState(seed)
    out = np.array(counts, dtype=np.int64, copy=True)
    ok = np.zeros(len(out), dtype=np.uint8)
    npop = len(sizes)
    tot = out[:, :npop].sum(axis=2)
    cum = np.cumsum(out[:, :npop], axis=2)
    # np.random.choice(pool, N, replace=False) is `permutation(len(pool))[:N]` applied to the pool (numpy's legacy generator):
    # the same permutation is drawn here and mapped to alleles through the cumulative counts, without building the pool
    for s in np.flatnonzero(considered):
        good = True
        for i, N in enumerate(sizes):
            n = tot[s, i]
            if N > n or (n == 0 and N != 0):
                good = False
                break
            out[s, i] = np.bincount(np.searchsorted(cum[s, i], rs.permutation(n)[:N], side="right"), minlength=4)
        ok[s] = good
    return out, ok


def merge_intervals(per, n_spectra):
    """[(hists, firsts, n) per interval] -> (per spectrum: list of the intervals' hists, list of their firsts).  Tables
    size their histograms by the largest count they hold, so the shapes are the same for every interval."""
    if len(per) == 1:
        return per[0][0], per[0][1]
    return ([[p[0][k] for p in per] for k in range(n_spectra)], [[p[1][k] for p in per] for k in range(n_spectra)])


def main_tables(args, include, exclude):
    """--inputType baseCounts | targetCounts (sfs.py:330-365, 456-474): one column per population."""
    import gzip
    import io
    import pandas as pd
    opener = gzip.open if args.inputFile and args.inputFile.endswith(".gz") else open
    with (opener(args.inputFile, "rt") if args.inputFile else sys.stdin) as f:
        header = args.header if args.header else f.readline()
        body = "".join(line for line in f if line[:1] != "#")
    names = header.split()[2:]
    popNames = []
    if args.pop or args.FSpops:
        for pop in args.pop or []:
            popNames.append(pop[0])
        for pop in [p for pops in (args.FSpops or []) for p in pops]:
            if pop not in popNames:
                popNames.append(pop)
    else:
        popNames = list(names)
    sys.stderr.write("\nPopulations:\n" + " ".join(popNames) + "\n")
    outgroup = None
    inPopNames = list(popNames)
    if args.inputType == "baseCounts" and (args.polarized or args.outgroup):
        outgroup = args.outgroup if args.outgroup else popNames[-1]
        inPopNames = [pn for pn in popNames if pn != outgroup]
        sys.stderr.write("\nFrequencies will be polarized assuming outgroup is {}\n".format(outgroup))
    if args.FSpops:
        FSpops = [list(g) for g in args.FSpops]
    else:
        FSpops = [[pn] for pn in inPopNames]
        if args.doPairs:
            FSpops += [list(c) for c in itertools.combinations(inPopNames, 2)]
        if args.doTrios:
            FSpops += [list(c) for c in itertools.combinations(inPopNames, 3)]
        if args.doQuartets:
            FSpops += [list(c) for c in itertools.combinations(inPopNames, 4)]
    df = pd.read_csv(io.StringIO(body), sep=r"\s+", header=None, names=["scaffold", "position"] + names, dtype=str)
    order = inPopNames + ([outgroup] if outgroup else [])
    mask = None
    sc = df["scaffold"].to_numpy().astype(str) if len(df) else np.zeros(0, dtype=str)
    if include or exclude:
        mask = np.array([(not include or x in include) and (x not in exclude) for x in sc], dtype=np.uint8)
    intervals = read_intervals(args)
    masks = interval_masks(intervals, sc, df["position"].to_numpy(dtype=np.int64) if intervals else None, mask)
    sub = subsample_sizes(args, inPopNames)
    if args.inputType == "baseCounts":
        cols = []
        for pn in order:
            parts = df[pn].str.split(",", expand=True).to_numpy(dtype=np.float64)      # "a,c,g,t" (floats allowed, 459)
            cols.append(parts.astype(np.int64))
        table = np.stack(cols, axis=1) if len(df) else np.zeros((0, len(order), 4), dtype=np.int64)
        assert table.max(initial=0) <= 65535, "counts above 65535 are not supported"
        kind = "base"
        if sub is not None:                                              # sfs.py:468-471
            table, went = downsample_counts(table, sub, args.seed, considered_sites(masks, len(table)))
            masks = [went if m is None else (m & went) for m in masks]
    else:
        table = df[order].to_numpy(dtype=np.int64) if len(df) else np.zeros((0, len(order)), dtype=np.int64)
        kind = "target"
    groups = [tuple(inPopNames.index(pn) for pn in grp) for grp in FSpops]
    og = len(inPopNames) if outgroup else -1
    with Engine(args.device) as eng:
        if use_sparse(groups, sfs_table_dims(kind, table)[1]):
            per = [eng.sfs_tables_sparse(kind, table, len(inPopNames), groups, outgroup=og, site_mask=m) for m in masks]
            return write_rows(args, FSpops, sparse_rows(per, len(FSpops)))
        per = [eng.sfs_tables(kind, table, len(inPopNames), groups, outgroup=og, site_mask=m) for m in masks]
    write_spectra(args, FSpops, *merge_intervals(per, len(FSpops)))


def main(argv=None):
    args = build_parser().parse_args(argv)
    assert (args.scafCol, args.posCol, args.firstSampleCol) == (0, 1, 2), "non-default column layout is not supported"
    if not args.polarized and args.outgroup is None and args.inputType != "targetCounts":
        sys.stderr.write("\nNo outgroup provided. Minor allele frequency will be used.\n")
    include = set(args.include or [])
    exclude = set(args.exclude or [])
    if args.includeFile:
        include |= set(open(args.includeFile, "rt").read().split())
    if args.excludeFile:
        exclude |= set(open(args.excludeFile, "rt").read().split())
    if args.inputType != "genotypes":
        return main_tables(args, include, exclude)

    headerInds = C.header_names(args.inputFile) if args.header is None else args.header.split()[2:]
    popNames, popDict = [], {}
    if args.pop or args.FSpops:                                         # sfs.py:291-309
        for pop in args.pop or []:
            popNames.append(pop[0])
            popDict[pop[0]] = [] if len(pop) == 1 else pop[1].split(",")
        for pop in [p for pops in (args.FSpops or []) for p in pops]:
            if pop not in popNames:
                popNames.append(pop)
                popDict[pop] = []
        if args.popsFile:
            with open(args.popsFile, "rt") as pf:
                for line in pf:
                    if not line.strip():
                        continue
                    ind, pop = line.split()
                    if pop in popDict and ind not in popDict[pop]:
                        popDict[pop].append(ind)
    else:
        popNames, popDict = ["all"], {"all": list(headerInds)}
    for pn in popNames:
        assert len(popDict[pn]) >= 1, "Population {} has no samples".format(pn)
    allSamples = [s for pn in popNames for s in popDict[pn]]
    if args.ploidy is not None:
        ploidy = args.ploidy if len(args.ploidy) != 1 else args.ploidy * len(allSamples)
        assert len(ploidy) == len(allSamples), "Incorrect number of ploidy values supplied."
        ploidyDict = dict(zip(allSamples, ploidy))
    elif args.ploidyFile is not None:
        with open(args.ploidyFile, "rt") as pf:
            ploidyDict = dict([[s[0], int(s[1])] for s in [l.split() for l in pf if l.strip()]])
    else:
        ploidyDict = dict(zip(allSamples, [2] * len(allSamples)))
    sys.stderr.write("\nPopulations:\n" + " ".join(popNames) + "\n")
    outgroup = None
    inPopNames = list(popNames)
    if args.polarized or args.outgroup:                                  # sfs.py:369-373
        outgroup = args.outgroup if args.outgroup else popNames[-1]
        inPopNames = [pn for pn in popNames if pn != outgroup]
        sys.stderr.write("\nFrequencies will be polarized assuming outgroup is {}\n".format(outgroup))
    if args.FSpops:
        FSpops = [list(g) for g in args.FSpops]
    else:
        FSpops = [[pn] for pn in inPopNames]
        if args.doPairs:
            FSpops += [list(c) for c in itertools.combinations(inPopNames, 2)]
        if args.doTrios:
            FSpops += [list(c) for c in itertools.combinations(inPopNames, 3)]
        if args.doQuartets:
            FSpops += [list(c) for c in itertools.combinations(inPopNames, 4)]

    # engine populations: the in-group first, the outgroup last
    enginePops = inPopNames + ([outgroup] if outgroup else [])
    sampleData = genomics.SampleData(indNames=list(allSamples), popNames=enginePops,
                                     popInds=[popDict[pn] for pn in enginePops], ploidyDict=ploidyDict)
    args.genoFile, args.hostParse = args.inputFile, getattr(args, "hostParse", False)
    # --devices N (genotype input): spectra add up over the sites, so every rank tokenises its share of the file and counts it;
    # the dense histograms and the first site of every cell (its index in the whole file: local index + the sites of the
    # ranks before) go to rank 0 through the exchange directory — no collective.
    rdv = mgpu.init("genomics_general_b200.cli.sfs", argv, args.devices)
    if rdv is not None and (args.subsample or args.subsampleIndividuals):
        raise NotImplementedError("--subsample draws from ONE random stream over the sites in file order; use one device")
    eng = Engine(args.device if rdv is None else mgpu.device_for(rdv, args.device))
    if rdv is None:
        gd = C.load_geno(args, sampleData.indNames, ploidyDict, header=args.header, engine=eng)
    else:
        gd = mgpu.local_ingest(eng, rdv, args.inputFile, args.genoFormat, sampleData.indNames, ploidyDict, args.header)
    mask = None
    if include or exclude:
        ok = np.array([(not include or n in include) and (n not in exclude) for n in gd.scaf_names], dtype=np.uint8)
        mask = ok[gd.scaf_ids]
    intervals = read_intervals(args)
    masks = interval_masks(intervals, np.asarray(gd.scaf_names, dtype=str)[gd.scaf_ids] if intervals else None, gd.pos, mask)
    with eng:
        C.ensure_resident(eng, gd)
        hp = C.hap_pop_vector(gd, enginePops, [popDict[pn] for pn in enginePops])
        eng.set_pops(hp, len(enginePops))
        sizes = [int((hp == x).sum()) for x in range(len(enginePops))]
        groups = [tuple(inPopNames.index(pn) for pn in grp) for grp in FSpops]
        og = len(inPopNames) if outgroup else -1
        sub = subsample_sizes(args, inPopNames)
        if sub is None:
            sparse = use_sparse(groups, [n + 1 for n in sizes])
            per = [(eng.sfs_sparse if sparse else eng.sfs)(len(inPopNames), groups, sizes, outgroup=og, site_mask=m)
                   for m in masks]
        else:
            for pn, n in zip(inPopNames, sub):                            # sfs.py:391-392
                have = sizes[enginePops.index(pn)]
                assert have >= n, "Population {} has fewer than {} haplotypes ({}).".format(pn, n, have)
            # per-site counts from the device, the reference's random draw on them, target allele + histograms on the device;
            # after a draw every in-group population holds exactly N alleles, which is the completeness test of sfs.py:453
            counts = eng.site_counts()
            table, went = downsample_counts(counts, sub, args.seed, considered_sites(masks, len(counts)))
            assert table.max(initial=0) <= 65535
            sparse = use_sparse(groups, sfs_table_dims("base", table)[1])
            per = [(eng.sfs_tables_sparse if sparse else eng.sfs_tables)("base", table, len(inPopNames), groups, outgroup=og,
                                                                          site_mask=went if m is None else (m & went))
                   for m in masks]
    if rdv is not None and sparse:
        # the ranks' non-empty cells, first sites made file-wide; rank 0 takes the union (counts summed, first site the
        # smallest)
        n_before = int(sum(int(x) for x in rdv.allgather("sfs_sites", np.array(gd.n_sites, dtype=np.int64))[:rdv.rank]))
        for i, (entries, _) in enumerate(per):
            for k, (coords, count, first) in enumerate(entries):
                rdv.put("sfs_c_%d_%d" % (i, k), coords)
                rdv.put("sfs_n_%d_%d" % (i, k), count)
                rdv.put("sfs_f_%d_%d" % (i, k), first + n_before)
        if rdv.rank != 0:
            rdv.finish()
            return
        merged = []
        for i in range(len(per)):
            entries = []
            for k in range(len(FSpops)):
                parts = [tuple(rdv.get("sfs_%s_%d_%d" % (x, i, k), q) for x in "cnf") for q in range(rdv.world)]
                coords, counts, first = merge_sparse(parts)
                entries.append((coords, np.sum(counts, axis=0), first))
            merged.append((entries, 0))
        per = merged
        rdv.finish()
    elif rdv is not None:
        n_before = int(sum(int(x) for x in rdv.allgather("sfs_sites", np.array(gd.n_sites, dtype=np.int64))[:rdv.rank]))
        for i, (hists, firsts, _) in enumerate(per):
            for k in range(len(FSpops)):
                rdv.put("sfs_h_%d_%d" % (i, k), hists[k])
                rdv.put("sfs_f_%d_%d" % (i, k), np.where(hists[k] > 0, firsts[k] + n_before, 0))
        if rdv.rank != 0:
            rdv.finish()
            return
        big = np.iinfo(np.int64).max
        merged = []
        for i in range(len(per)):
            H, F = [], []
            for k in range(len(FSpops)):
                hs = [rdv.get("sfs_h_%d_%d" % (i, k), q) for q in range(rdv.world)]
                fs = [rdv.get("sfs_f_%d_%d" % (i, k), q) for q in range(rdv.world)]
                H.append(np.sum(hs, axis=0))
                F.append(np.min([np.where(h > 0, f, big) for h, f in zip(hs, fs)], axis=0))
            merged.append((H, F, 0))
        per = merged
        rdv.finish()
    if sparse:
        write_rows(args, FSpops, sparse_rows(per, len(FSpops)))
    else:
        write_spectra(args, FSpops, *merge_intervals(per, len(FSpops)))


if __name__ == "__main__":
    main()
