#!/usr/bin/env python
"""Drop-in for the reference's genoToSeq.py (flags 8-30), on the GPU: the .geno body goes to the device, every data line's
token starts are indexed there, and the alignments (FASTA or PHYLIP, for the whole file, per window or per contig) are
transposed out of the device copy of the text slab by slab (_stream.py).

Refused before any work, where the reference crashes: --seqNameFormat other than `sample` (a KeyError), -S with -M windows or
contigs (the generators iterate the string's characters), --windType sites without --maxDist or --overlap, --separateFiles
with -M cat or without -s, --splitPhased ploidies the reference cannot pair with the names, no samples, and --devices N.
After the index, before any output: a coordinate window with no site (firstPos() of an empty window), a second coordinate
window on a scaffold without --stepSize, and positions that decrease inside a scaffold in -M windows / contigs.
Narrowed (DESIGN.md section 8): every token of a column is as wide as on the first data line, with --splitPhased each
sample's ceil(width / 2) equals its ploidy, and the text is ASCII with '\\n' or '\\r\\n' line ends."""
from __future__ import annotations

import argparse
import contextlib
import mmap
import re
import string

import numpy as np

from .. import windows as W
from ..engine import Engine, PgError, PinnedArray
from . import _common as C
from ._stream import SlabWriter, env_int, open_input, open_output

TOK = re.compile(rb"[^ \t\n\r\x0b\x0c\x1c-\x1f]+")
CONTIG_WINDOW = 10 ** 7          # -M contigs: coordinate windows of 1e7 bp, step 1e7 (genoToSeq.py:74-79)
ERRORS = {1: "the position is not an integer", 2: "the line has no position field", 3: "the position is outside the int32 range",
          4: "the token of sample %s is not as wide as that column's token on the first data line (the reference would write "
             "sequences of unequal length)",
          5: "sample %s has no genotype column on this line (the reference fails with a KeyError)",
          6: "%s genotype columns, the header names %d (the reference fails on an assertion)",
          7: "a byte outside ASCII (the reference reads characters, which this engine does not)",
          8: "a '\\r' ends a line by itself (the reference reads it as a line end, this engine does not)"}


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument("-g", "--genoFile", help="Input geno file (.gz allowed; default stdin)")
    p.add_argument("-s", "--seqFile", help="Output sequence file (default stdout)")
    p.add_argument("-f", "--format", choices=("phylip", "fasta"), default="fasta")
    p.add_argument("-M", "--mode", choices=("cat", "windows", "contigs"), default="cat")
    p.add_argument("-S", "--samples", help="Name of sample(s)")
    p.add_argument("--NtoGap", help="Convert 'N' or 'n' to '-'", action="store_true")
    p.add_argument("--seqNameFormat", default="sample",
                   choices=("sample", "contig", "sample_contig", "contig_position", "sample_contig_position"))
    p.add_argument("--splitPhased", action="store_true")
    p.add_argument("--ploidy", nargs="+", type=int, default=[2])
    p.add_argument("--separateFiles", action="store_true")
    p.add_argument("--gzip", action="store_true")
    p.add_argument("--windType", choices=("sites", "coordinate"), default="sites")
    p.add_argument("--windSize", type=int)
    p.add_argument("--minSites", type=int)
    p.add_argument("--stepSize", type=int)
    p.add_argument("--overlap", type=int)
    p.add_argument("--maxDist", type=int)
    p.add_argument("--device", help="CUDA device index", type=int, default=0)
    p.add_argument("--devices", help="Not supported: the transpose runs on one GPU", type=int, default=None)
    p.add_argument("--timing", help="Write a JSON file with the wall time of each phase and the device time of each kernel",
                   metavar="FILE")
    return p


def haploid_names(names, ploidy):
    """makeHaploidNames (genomics.py:448-453): (names, ploidy of every name); raises KeyError where the reference does"""
    ploidy = list(ploidy)
    if len(ploidy) == 1:
        ploidy = ploidy * len(names)
    if all(p == 1 for p in ploidy):
        return list(names), {n: 1 for n in names}
    pd = dict(zip(names, ploidy))
    return [n + "_" + letter for n in names for letter in string.ascii_uppercase[:pd[n]]], pd


def check_args(args):
    """the refusals that need no input"""
    def no(msg):
        raise SystemExit("genoToSeq: " + msg)
    if args.devices not in (None, 1):
        no("--devices is not supported; the transpose runs on one GPU")
    if args.seqNameFormat != "sample":
        no("--seqNameFormat %s is not supported: the reference fails with a KeyError on it (genoToSeq.py:104-116 looks the "
           "renamed sequences up by their new names)" % args.seqNameFormat)
    if args.samples and args.mode != "cat":
        no("-S with -M %s is not supported: the reference's window generators get the raw string and iterate its characters "
           "(genoToSeq.py:81-84)" % args.mode)
    if args.separateFiles and args.mode == "cat":
        no("--separateFiles with -M cat is not supported: the reference never opens an output file on that path "
           "(genoToSeq.py:44, 61)")
    if args.separateFiles and not args.seqFile:
        no("--separateFiles needs -s: the reference names the files after it (genoToSeq.py:94)")
    if args.mode == "windows":
        if not args.windSize:
            no("-M windows needs --windSize")
        if args.windType == "sites" and args.maxDist is None:
            no("--windType sites needs --maxDist: the reference compares the span against None (genomics.py:2052)")
        if args.windType == "sites" and args.overlap is None:
            no("--windType sites needs --overlap: the reference's GenoWindow.trim asserts on it after the first window "
               "(genomics.py:1780)")
        if args.windType == "coordinate" and args.stepSize is not None and args.stepSize < 1:
            no("--stepSize must be at least 1")
        if args.windType == "sites" and args.overlap is not None and args.overlap >= args.windSize:
            no("--overlap must be smaller than --windSize: the reference's sites windows would not advance")
    if args.splitPhased and any(p < 1 for p in args.ploidy):
        no("--ploidy values must be at least 1")


def plan(args, all_names, first_tokens):
    """The sequences (name, column, first byte, width) and the index spec: the reference's set-up (genoToSeq.py:53-61,
    GenoFileReader, parseGenoFile, GenoWindow.seqDict) with the refusals.  first_tokens: genotype tokens of the first data
    line (None: no data line)."""
    def no(msg):
        raise SystemExit("genoToSeq: " + msg)
    n_cols = len(all_names)
    samples = args.samples.split(",") if args.samples else None
    if args.splitPhased:
        try:
            reader_names, reader_pd = haploid_names(all_names, args.ploidy)
        except KeyError as e:
            no("--ploidy gives %d values for the %d header samples: the reference fails with a KeyError on %s" %
               (len(args.ploidy), n_cols, e))
        col_pl = [reader_pd[n] for n in all_names]
        flat = [(c, a) for c in range(n_cols) for a in range(col_pl[c])]       # the split alleles of a line, in order
    if samples is None:
        out_names = reader_names if args.splitPhased else list(all_names)
        if args.splitPhased:
            src = [flat[out_names.index(n)] for n in out_names]                # seqDict: names.index (genomics.py:1792)
        else:
            src = [(out_names.index(n), 0) for n in out_names]
    else:
        if args.splitPhased:
            try:
                out_names, _ = haploid_names(samples, args.ploidy)
            except KeyError as e:
                no("--ploidy gives %d values for the %d samples of -S: the reference fails with a KeyError on %s" %
                   (len(args.ploidy), len(samples), e))
            last = {n: i for i, n in enumerate(reader_names)}                  # dict(zip(names, GTs)): the last one wins
            for n in out_names:
                if n not in last:
                    no("sequence %s is not among the header's split names: the reference fails with a KeyError" % n)
            src = [flat[last[n]] for n in out_names]
        else:
            last = {n: i for i, n in enumerate(all_names)}
            for n in samples:
                if n not in last:
                    no("sample %s is not in the header: the reference fails with a KeyError" % n)
            out_names = list(samples)
            src = [(last[n], 0) for n in out_names]
    if not out_names:
        no("no samples: the reference fails on max() of no sequences (genomics.py:2240)")
    # slots: the columns whose tokens are read or, with --splitPhased, checked (the split is positional over every column)
    slot_cols = list(range(n_cols)) if args.splitPhased else sorted(set(c for c, _ in src))
    col_slot = np.full(max(n_cols, 1), -1, np.int32)
    for s, c in enumerate(slot_cols):
        col_slot[c] = s
    if first_tokens is not None:
        for c in slot_cols:
            if c >= len(first_tokens):
                no("data line 1: sample %s has no genotype column" % all_names[c])
        widths = [len(first_tokens[c]) for c in slot_cols]
        if args.splitPhased:
            for c, w in zip(slot_cols, widths):
                if (w + 1) // 2 != col_pl[c]:
                    no("data line 1: the token of sample %s holds %d alleles, its ploidy is %d (the reference asserts on the "
                       "total, or shifts alleles between samples when the totals agree)" % (all_names[c], (w + 1) // 2,
                                                                                            col_pl[c]))
        for c, w in zip(slot_cols, widths):
            if w > 1024:
                no("data line 1: the token of sample %s is %d characters wide (at most 1024)" % (all_names[c], w))
    else:
        widths = [1] * len(slot_cols)
    width_of = dict(zip(slot_cols, widths))
    seq_slot = [int(col_slot[c]) for c, _ in src]
    seq_byte = [2 * a for _, a in src] if args.splitPhased else [0] * len(src)
    seq_width = [1] * len(src) if args.splitPhased else [width_of[c] for c, _ in src]
    return dict(names=out_names, col_slot=col_slot[:n_cols], slot_width=np.array(widths, np.int32), exact=samples is None,
                seq_slot=seq_slot, seq_byte=seq_byte, seq_width=seq_width)


def _first_data_line(data):
    """the first line of the body that the line index takes as a data line (not '#', not blank)"""
    at = 0
    while at < len(data):
        nl = data.find(b"\n", at)
        end = len(data) if nl < 0 else nl
        ln = data[at:end]
        if ln.strip() and not ln.startswith(b"#"):
            return ln
        at = end + 1
    return None


def windows_for(args, S, pos, newsc, scaf_name):
    """(scaffold, lo, hi) of every alignment: the whole file, or the reference's window generators over the data lines"""
    if args.mode == "cat":
        return [None], np.array([0], np.int64), np.array([S], np.int64)
    if S == 0:
        if args.mode == "windows" and args.windType == "sites":
            raise SystemExit("genoToSeq: sites windows on a file with no data line: the reference fails adding the missing "
                             "first site (genomics.py:2052-2055)")
        return [], np.zeros(0, np.int64), np.zeros(0, np.int64)
    ids = np.cumsum(newsc.astype(np.int64)) - 1
    runs = np.flatnonzero(newsc)
    names = [scaf_name(int(r)) for r in runs]
    down = np.flatnonzero((np.diff(pos.astype(np.int64)) < 0) & (newsc[1:] == 0))
    if len(down):
        raise SystemExit("genoToSeq: data line %d: the position decreases inside scaffold %s; windows need sorted positions" %
                         (int(down[0]) + 2, names[ids[down[0] + 1]]))
    coord = args.mode == "contigs" or args.windType == "coordinate"
    if coord:
        size = CONTIG_WINDOW if args.mode == "contigs" else args.windSize
        step = CONTIG_WINDOW if args.mode == "contigs" else args.stepSize
        ws = W.sliding_coord_windows(ids, names, pos, size, step or size)
        if not step:
            for k in range(len(ws)):
                if ws.start[k] != 1:
                    raise SystemExit("genoToSeq: scaffold %s needs a second coordinate window and no --stepSize is given: the "
                                     "reference asserts in GenoWindow.slide (genomics.py:1769)" % ws.scaffold[k])
        for k in range(len(ws)):
            if ws.hi[k] == ws.lo[k]:
                raise SystemExit("genoToSeq: scaffold %s, window %d-%d holds no site: the reference fails in firstPos() "
                                 "(genomics.py:1763)" % (ws.scaffold[k], ws.start[k], ws.end[k]))
    else:
        ws = W.sliding_sites_windows(ids, names, pos, args.windSize, args.overlap, args.maxDist, args.minSites)
        run_end = {int(b) for b in np.concatenate([runs[1:], [S]])}
        for k in range(len(ws)):
            if ws.hi[k] not in run_end and ws.hi[k] - ws.lo[k] < args.overlap:
                raise SystemExit("genoToSeq: scaffold %s: a window of %d sites (cut by --maxDist) is followed by one that keeps "
                                 "--overlap %d of them; the reference's trim keeps a different count there" %
                                 (ws.scaffold[k], ws.hi[k] - ws.lo[k], args.overlap))
    lo, hi = ws.ranges()
    return list(ws.scaffold), lo, hi


class _Writer:
    """the output files: one stream, or with --separateFiles one file per alignment, opened as its first byte arrives"""

    def __init__(self, args, scaffolds, lo, hi, pos, win_bytes):
        self.args = args
        self.cum = np.concatenate([[0], np.cumsum(win_bytes)]).astype(np.int64)
        self.scaffolds, self.lo, self.hi, self.pos = scaffolds, lo, hi, pos
        self.at, self.cur, self.f = 0, -1, None
        self.files = contextlib.ExitStack()
        if not args.separateFiles:
            name = args.seqFile
            if name and args.gzip and not name.endswith(".gz"):
                name += ".gz"
            self.f = self.files.enter_context(open_output(name))

    def _name(self, w):
        """seqFile.scaffold[_first_last].fa|.phy[.gz] (genoToSeq.py:91-100)"""
        name = self.args.seqFile + "." + self.scaffolds[w]
        if self.args.mode == "windows":
            name += "_%d_%d" % (int(self.pos[self.lo[w]]), int(self.pos[self.hi[w] - 1]))
        name += ".fa" if self.args.format == "fasta" else ".phy"
        return name + (".gz" if self.args.gzip else "")

    def write(self, view):
        g0, self.at = self.at, self.at + len(view)
        if not self.args.separateFiles:
            self.f.write(view)
            return
        at = 0
        w = int(np.searchsorted(self.cum, g0, side="right")) - 1
        while at < len(view):
            if w != self.cur:
                self.files.close()
                self.f = self.files.enter_context(open_output(self._name(w)))
                self.cur = w
            n = min(len(view) - at, int(self.cum[w + 1]) - (g0 + at))
            self.f.write(view[at:at + n])
            at += n
            if g0 + at == self.cum[w + 1]:
                w += 1

    def close(self):
        self.files.close()


def main(argv=None):
    args = build_parser().parse_args(argv)
    check_args(args)
    tm = C.Timing(args.timing)
    path, data = None, None
    if args.genoFile and not args.genoFile.endswith(".gz"):
        path = args.genoFile
        with open(path, "rb") as f:
            head = f.readline()
            body_offset = len(head)
            first = None
            for ln in f:
                ln = ln.rstrip(b"\n")
                if ln.strip() and not ln.startswith(b"#"):
                    first = ln
                    break
    else:
        raw = open_input(args.genoFile).read()
        nl = raw.find(b"\n")
        head = raw if nl < 0 else raw[:nl + 1]
        body_offset = len(head)
        data = raw[body_offset:]
        first = _first_data_line(data)
    all_names = head.decode().split()[2:]
    first_tokens = [t.decode("latin-1") for t in TOK.findall(first)[2:]] if first is not None else None
    pl = plan(args, all_names, first_tokens)
    tm.mark("plan")
    slab = env_int("PG_SEQ_SLAB_BYTES", 64 << 20)
    with Engine(args.device) as eng:
        try:
            S, err = eng.seq_index(pl["col_slot"], pl["slot_width"], pl["exact"], data=data, path=path, body_offset=body_offset)
        except PgError as e:
            if "do not fit in device memory" in str(e):
                raise SystemExit("genoToSeq: the body of the input does not fit in device memory with 1 GiB to spare; there is "
                                 "no chunked path (%s)" % e)
            raise
        tm.mark("index", eng)
        if err[0]:
            msg = ERRORS.get(err[0], "error %d" % err[0])
            if err[0] in (4, 5):
                msg = msg % all_names[err[2] - 1]
            elif err[0] == 6:
                msg = msg % (err[2] - 1, len(all_names))
            raise SystemExit("genoToSeq: data line %d: %s" % (err[1], msg))
        pos, newsc, off = eng.seq_meta(S)
        if path is not None and S:
            fh = open(path, "rb")
            mm = mmap.mmap(fh.fileno(), 0, access=mmap.ACCESS_READ)
            text, base = mm, body_offset
        else:
            fh = mm = None
            text, base = data, 0

        def scaf_name(i):
            a = base + int(off[i])
            return TOK.search(text, a).group().decode()
        scaffolds, lo, hi = windows_for(args, S, pos, newsc, scaf_name)
        if mm is not None:
            mm.close()
            fh.close()
        tm.mark("windows")
        R, win_bytes = eng.seq_plan(args.format, args.NtoGap, pl["names"], pl["seq_slot"], pl["seq_byte"], pl["seq_width"],
                                    lo, hi)
        tm.mark("plan_rows", eng)
        out = _Writer(args, scaffolds, lo, hi, pos, win_bytes)
        with SlabWriter(out.write, slab, PinnedArray) as w:
            row, part = 0, -1
            while row < R:
                row, part, nb = eng.seq_emit(row, part, w.slab(), w.cap)
                tm.mark("emit", eng)
                w.write(nb)
        out.close()
        tm.mark("write")
    tm.write(sites=S, alignments=len(lo), bytes=out.at)


if __name__ == "__main__":
    main()
