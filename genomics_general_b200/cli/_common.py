"""Shared pieces of the four drop-in command lines (flag handling that the reference repeats in every
script: windows, populations, ploidy, files).  Citations are genomics_general/<file>:<line>."""
from __future__ import annotations

import gzip
import re
import sys

import numpy as np

from .. import geno_io, windows as W


def add_window_args(p, overlap_short=True, cat=False):
    """popgenWindows.py:172-178 / ABBABABAwindows.py:111-117 / distMat.py:118-128"""
    choices = ("sites", "coordinate", "predefined") + (("cat",) if cat else ())
    p.add_argument("--windType", help="Type of windows to make", choices=choices, default="coordinate")
    p.add_argument("-w", "--windSize", help="Window size in bases", type=int, metavar="sites")
    p.add_argument("-s", "--stepSize", help="Step size for sliding window", type=int, metavar="sites")
    p.add_argument("-m", "--minSites", help="Minumum good sites per window", type=int, metavar="sites", default=1)
    if overlap_short:
        p.add_argument("-O", "--overlap", help="Overlap for sites sliding window", type=int, metavar="sites")
    else:
        p.add_argument("--overlap", help="Overlap for sites sliding window", type=int, metavar="sites")
    p.add_argument("-D", "--maxDist", help="Maximum span distance for sites window", type=int)
    p.add_argument("--windCoords", help="Window coordinates file (scaffold start end)")


def add_engine_args(p):
    p.add_argument("--device", help="CUDA device index", type=int, default=0)
    p.add_argument("--parseThreads", help="Host threads for the .geno tokenizer", type=int, default=None)
    p.add_argument("--hostParse", help="Tokenise the .geno text on the host instead of on the GPU", action="store_true")
    p.add_argument("--cache", help="Keep a binary cache <genoFile>.gbin of the ingested matrix and load it on later runs "
                                   "(same file, format, samples and ploidy)", action="store_true")
    p.add_argument("--timing", help="Write a JSON file with the wall time of each phase and the device time of each kernel",
                   metavar="FILE")
    p.add_argument("--devices", help="Number of GPUs: every GPU tokenises its share of the file and computes the windows that "
                                     "start there (one process per GPU, one NCCL all-gather of the rows)", type=int, default=None)


def check_window_args(args, with_id=False):
    """The reference's assertions (popgenWindows.py:218-244). Returns (minSites, windCoords)."""
    coords = None
    if args.windType == "coordinate":
        assert args.windSize, "Window size must be provided."
        assert not args.overlap, "Overlap does not apply to coordinate windows. Use --stepSize instead."
        assert not args.maxDist, "Maximum distance only applies to sites windows."
    elif args.windType == "sites":
        assert args.windSize, "Window size (number of sites) must be provided."
        assert not args.stepSize, "Step size only applies to coordinate windows. Use --overlap instead."
    elif args.windType == "predefined":
        assert args.windCoords, "Please provide a file of window coordinates."
        assert not args.overlap, "Overlap does not apply for predefined windows."
        assert not args.maxDist, "Maximum does not apply for predefined windows."
        assert not args.stepSize, "Step size does not apply for predefined windows."
        assert not args.include, "You cannot only include specific scaffolds if using predefined windows."
        assert not args.exclude, "You cannot exclude specific scaffolds if using predefined windows."
        coords = []
        with open(args.windCoords, "rt") as wc:
            for line in wc:
                f = line.split()
                if not f:
                    continue
                c = (f[0], int(f[1]), int(f[2]))
                if with_id and len(f) > 3:
                    c += (f[3],)
                coords.append(c)
    minSites = args.minSites
    if not minSites:
        minSites = args.windSize
    return minSites, coords


def read_scaffold_list(path):
    if not path:
        return None
    with open(path, "rt") as f:
        return [line.rstrip() for line in f.readlines()]


def parse_pop_args(pop_args, pops_file):
    """-p name [a,b,c] ... + --popsFile  (popgenWindows.py:259-277)."""
    popNames, popInds = [], []
    for p in pop_args:
        popNames.append(p[0])
        popInds.append(p[1].split(",") if len(p) > 1 else [])
    if pops_file:
        with open(pops_file, "rt") as pf:
            popDict = dict([ln.split() for ln in pf if ln.strip()])
        for ind in popDict.keys():
            if popDict[ind] in popNames:
                popInds[popNames.index(popDict[ind])].append(ind)
    for p in popInds:
        assert len(p) >= 1, "All populations must be represented by at least one sample."
    return popNames, popInds


def ploidy_dict(args, allInds, haploid_list):
    """popgenWindows.py:293-305."""
    if getattr(args, "ploidy", None) is not None:
        ploidy = args.ploidy if len(args.ploidy) != 1 else args.ploidy * len(allInds)
        assert len(ploidy) == len(allInds), "Incorrect number of ploidy values supplied."
        return dict(zip(allInds, ploidy))
    if getattr(args, "ploidyFile", None) is not None:
        with open(args.ploidyFile, "rt") as pf:
            return dict([[s[0], int(s[1])] for s in [l.split() for l in pf if l.strip()]])
    if getattr(args, "inferPloidy", False):
        return infer_ploidy(args, allInds)
    base = 1 if args.genoFormat == "haplo" else 2
    d = dict(zip(allInds, [base] * len(allInds)))
    for s in haploid_list or []:
        d[s] = 1
    return d


def first_data_line(args):
    """First genotype line of the input (the line after the header; '#' and blank lines skipped)."""
    path = getattr(args, "genoFile", None)
    has_header = not getattr(args, "header", None)
    if path is None:
        lines = iter(stdin_bytes().split(b"\n", 64))
    else:
        lines = gzip.open(path, "rb") if path.endswith(".gz") else open(path, "rb")
    try:
        for ln in lines:
            if has_header:
                has_header = False
                continue
            if ln.strip() and not ln.startswith(b"#"):
                return ln.decode()
    finally:
        if path is not None:
            lines.close()
    return ""


def infer_ploidy(args, allInds):
    """--inferPloidy (popgenWindows.py:299-300): the reference leaves every ploidy None and genoToAlignment takes the number
    of sequences splitSeq makes of the window's genotype tokens (genomics.py:1109-1110, 390-396: characters 0,2,.. of a
    phased token, every character of a pairs / alleles / haplo token, two for a diplo letter).  The dense engine holds one
    matrix for the whole file, so the token widths of the first genotype line fix the ploidies; a later line whose tokens
    have another width is reported by the tokenizer with its line number (the reference would give that window a
    different number of haplotypes)."""
    names = header_names(getattr(args, "genoFile", None)) if not getattr(args, "header", None) else args.header.split()[2:]
    toks = first_data_line(args).split()[2:]
    fmt = args.genoFormat
    width = {}
    for n, t in zip(names, toks):
        width.setdefault(n, 2 if fmt == "diplo" else (len(t) + 1) // 2 if fmt == "phased" else len(t))
    base = 1 if fmt == "haplo" else 2
    return dict((s, width.get(s, base)) for s in allInds)


_STDIN = {}        # the piped input is read once: the header comes from its first line, load_geno gets the same bytes


def stdin_bytes():
    if "data" not in _STDIN:
        _STDIN["data"] = geno_io.read_bytes(sys.stdin.buffer)
    return _STDIN["data"]


def alignment_order(indNames, ploidyDict, genoFormat="phased"):
    """Samples in the order their haplotypes take in the reference's Alignment: genoToAlignment sorts the sequence names
    (`ind_A`, `ind_B`, ...; the plain name for haploids) with np.argsort (genomics.py:1111-1121), e.g. s10 before s1
    ('0' < '_').  The order only matters where ties are broken by position (H12's greedy clustering, 1239-1261)."""
    base = 1 if genoFormat == "haplo" else 2
    keys = [n if int((ploidyDict or {}).get(n, base) or base) == 1 else n + "_A" for n in indNames]
    return [indNames[i] for i in np.argsort(keys)] if keys else list(indNames)


def header_names(path):
    """Sample names of the header line; with no path the genotypes are piped in (freq.py:228-233, sfs.py:282-287)."""
    if path is None:
        data = stdin_bytes()
        return data[:data.find(b"\n") if b"\n" in data else len(data)].decode().split()[2:]
    with (gzip.open(path, "rt") if path.endswith(".gz") else open(path, "rt")) as gf:
        return gf.readline().split()[2:]


def open_out(path):
    if path:
        return gzip.open(path, "wt") if path.endswith(".gz") else open(path, "wt")
    return sys.stdout


def load_geno(args, samples, ploidyDict, header=None, engine=None):
    """The whole file as a dense matrix.  With an engine the text is tokenised on the GPU and the matrix stays there
    (GenoData.geno is None); files too large for device memory, and --hostParse, go through the host tokenizer."""
    src = args.genoFile if args.genoFile else stdin_bytes()
    cache = None
    if engine is not None and getattr(args, "cache", False) and isinstance(src, str) and not src.endswith(".gz"):
        cache = src + ".gbin"
        gd = geno_io.load_gbin(cache, engine, src, args.genoFormat, samples=samples, ploidy=ploidyDict, header=header)
        if gd is not None:
            return gd
    gd = _load_geno_uncached(args, src, samples, ploidyDict, header, engine)
    if cache is not None:
        geno_io.save_gbin(cache, gd, src, args.genoFormat, eng=engine)
    return gd


def _load_geno_uncached(args, src, samples, ploidyDict, header, engine):
    if engine is not None and not getattr(args, "hostParse", False):
        if not isinstance(src, str) or src.endswith(".gz"):
            src = geno_io.read_bytes(src)          # stdin / gzip: decompressed in host memory
        try:
            return geno_io.ingest_geno(engine, src, geno_format=args.genoFormat, samples=samples, ploidy=ploidyDict,
                                       header=header)
        except geno_io.PgError as e:
            if "do not fit in device memory" not in str(e):
                raise
    return geno_io.parse_geno(src, geno_format=args.genoFormat, samples=samples, ploidy=ploidyDict, header=header,
                              threads=getattr(args, "parseThreads", None))


class Timing:
    """--timing FILE (SURVEY.md section 5: the reference only prints progress counters): wall seconds of each phase of the
    command line and the device milliseconds of every kernel of the statistics calls, as one JSON object."""

    def __init__(self, path):
        import time
        self.path, self.t0, self.last = path, time.perf_counter(), time.perf_counter()
        self.phases, self.kernels = {}, {}

    def mark(self, name, eng=None):
        import time
        now = time.perf_counter()
        self.phases[name] = self.phases.get(name, 0.0) + (now - self.last)
        self.last = now
        if eng is not None:
            try:
                for k, v in eng.last_timings().items():
                    self.kernels[k] = self.kernels.get(k, 0.0) + v["ms"]
            except Exception:
                pass

    def write(self, **extra):
        import json
        import time
        if not self.path:
            return
        with open(self.path, "wt") as f:
            json.dump(dict(phases_s=self.phases, kernels_ms=self.kernels, total_s=time.perf_counter() - self.t0, **extra), f,
                      indent=1)


def ensure_resident(eng, gd):
    """Upload the host matrix unless the device-side tokenizer already built it in place."""
    if gd.geno is not None:
        eng.upload(gd.geno, gd.pos)


def make_windows(args, gd, minSites, coords, include=None, exclude=None):
    if args.windType == "coordinate":
        return W.sliding_coord_windows(gd.scaf_ids, gd.scaf_names, gd.pos, args.windSize, args.stepSize or args.windSize,
                                       include, exclude)
    if args.windType == "sites":
        return W.sliding_sites_windows(gd.scaf_ids, gd.scaf_names, gd.pos, args.windSize, args.overlap or 0,
                                       args.maxDist if args.maxDist else None, minSites, include, exclude)
    if args.windType == "predefined":
        return W.predefined_coord_windows(gd.scaf_ids, gd.scaf_names, gd.pos, coords)
    raise ValueError(args.windType)


def window_prefix(args, ws, k, gd, sites, pos_sum):
    """scaffold,start,end,mid,sites of one window (popgenWindows.py:37-39)."""
    n = int(sites)
    mid = W.mid_pos(int(pos_sum), n)
    if args.windType in ("coordinate", "predefined"):
        start, end = ws.start[k], ws.end[k]
    else:
        start, end = int(gd.pos[ws.lo[k]]), int(gd.pos[ws.hi[k] - 1])      # firstPos / lastPos
    return [ws.scaffold[k], start, end, mid, n]


def hap_pop_vector(gd, popNames, popInds):
    """population index of every haplotype column (-1: in no population). A sample listed in several
    populations is not representable by the reference either (Alignment.groups becomes a tuple)."""
    samp_pop = {}
    for k, inds in enumerate(popInds):
        for i in inds:
            if i in samp_pop and samp_pop[i] != k:
                raise ValueError("sample %s is in more than one population" % i)
            samp_pop[i] = k
    per_sample = np.array([samp_pop.get(n, -1) for n in gd.names], dtype=np.int32)
    return np.repeat(per_sample, gd.ploidy.astype(np.int64))


FASTA_TOK = re.compile(rb"[^ \t\n\r\x0b\x0c\x1c-\x1f]+")
FASTA_NEWLINE = re.compile(rb"[\r\n]")


def fasta_records(data, starts, fail):
    """genomics.parseFasta's pieces (the text between '>' bytes at `starts`) after universal newlines: (names, [first
    newline, end) of every piece's sequence).  fail(message) is called where parseFasta raises: every piece's name is taken
    before any piece's newline, as parseFasta does."""
    ends = list(starts[1:]) + [len(data)]
    names = []
    for a, b in zip(starts, ends):
        m = FASTA_TOK.search(data, a + 1, b)
        if m is None:
            fail("the record at byte %d has no name (the reference fails with an IndexError)" % a)
        names.append(m.group().decode())
    lo = []
    for a, b in zip(starts, ends):
        m = FASTA_NEWLINE.search(data, a + 1, b)
        if m is None:
            fail("record %s has no newline (the reference fails with a ValueError)" % names[len(lo)])
        lo.append(m.start())
    return names, np.array(lo, np.int64), np.array(ends, np.int64)
