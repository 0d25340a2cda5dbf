#!/usr/bin/env python
"""Drop-in for the reference's mergeGeno.py on the GPU: several .geno files joined into one table keyed by position, in the
order of the .fai's walk (every site 1..length of every scaffold), by --method intersect, union or all.

The host reads the .fai, the headers and the flags; each body is read in chunks of complete lines, cut at '\\n' only
(_stream.py), and the device indexes each chunk's lines, finds where the file stalls (the first line that the reference's
walk would never consume: fewer than two fields, a scaffold not in the .fai, a site that is not str(n) for 1 <= n <=
length, or a position not after the line before), merges the files' positions up to a bound and writes the rows into
slabs.  The bound of each round is the smallest last loaded position over the files still reading, so only the file(s)
that set it read their next chunk and the device holds about one chunk per file: inputs larger than device memory stream
through.

Refused before any output, where the reference crashes: an input that cannot be opened or read, a .fai line with fewer than
2 fields or a length int() rejects, an --outputOnly index outside the files.  Narrowed (DESIGN.md section 8): a .fai that
names a scaffold twice, a .fai whose lengths sum to 2^62 or more, and a byte >= 0x80 or a '\\r' that ends a line by itself in
a body line the walk reaches (up to and including the line where the file stalls; lines after it are never read).  Such a
line found after rows were written removes the -o file.  --verbose reports each round, not each site."""
from __future__ import annotations

import argparse
import os
import sys

from ..engine import Engine, PinnedArray
from . import _common as C
from ._stream import SlabWriter, body_chunks, env_int, first_line, open_input, open_output

METHODS = {"intersect": 0, "union": 1, "all": 2}
WALK_LIMIT = 1 << 62


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument("-i", "--inputFile", help="Input file", action="append", required=True)
    p.add_argument("-f", "--fai", help="Reference fasta index file", action="store", required=True)
    p.add_argument("-o", "--outputFile", help="Output file", action="store")
    p.add_argument("--method", help="How to merge", action="store", choices=tuple(METHODS), default="intersect")
    p.add_argument("--unionMin", help="Minimum files represented for menthod union", action="store", type=int, default=1)
    p.add_argument("--mustIncludeFirst", help="The first n files MUST be present", action="store", type=int, default=0)
    p.add_argument("--outSep", help="Output file separator", action="store", default="\t")
    p.add_argument("--missing", help="Missing genotype for method union or all", action="store", default="N")
    p.add_argument("--outputOnly", help="Which output files to include in output (1 based)", action="store", type=int,
                   nargs="+")
    p.add_argument("--verbose", help="Report each merge round", action="store_true")
    C.add_engine_args(p)
    return p


def _fail(msg):
    raise SystemExit("mergeGeno: " + msg)


def read_fai(path):
    """[(name, length)] of the .fai in file order (mergeGeno.py:33), refused where the reference fails, where a name comes
    twice and where the walk reaches 2^62 positions"""
    scafs = []
    try:
        with open(path, "rt") as fai:
            for k, ln in enumerate(fai):
                f = ln.split()[:2]
                if len(f) < 2:
                    _fail("%s line %d has fewer than 2 fields (the reference fails with a ValueError)" % (path, k + 1))
                try:
                    scafs.append((f[0], int(f[1])))
                except ValueError:
                    _fail("%s line %d: the length %r is not an integer (the reference fails with a ValueError)"
                          % (path, k + 1, f[1]))
    except (OSError, UnicodeDecodeError) as e:
        _fail("cannot read the .fai %s: %s" % (path, e))
    seen = set()
    for name, _ in scafs:
        if name in seen:
            _fail("%s names scaffold %s twice (the reference walks it twice with its last length; this engine refuses "
                  "it)" % (path, name))
        seen.add(name)
    if sum(max(n, 0) for _, n in scafs) >= WALK_LIMIT:
        _fail("%s: the scaffold lengths sum to 2^62 or more" % path)
    return scafs


def _open(path):
    try:
        return open_input(path)
    except OSError as e:
        _fail("cannot open input %s: %s" % (path, e))


def main(argv=None):
    args = build_parser().parse_args(argv)
    if args.devices not in (None, 1):
        _fail("--devices is not supported; the merge runs on one GPU")
    if args.hostParse or args.cache:
        _fail("--hostParse and --cache do not apply: the merge streams the text through the GPU")
    tm = C.Timing(args.timing)
    srcs = [_open(p) for p in args.inputFile]
    nF = len(srcs)
    scafs = read_fai(args.fai)
    heads, bodies = [], []
    for path, src in zip(args.inputFile, srcs):
        try:
            h, rest = first_line(src) or (b"", b"")
            heads.append(h.decode().split())
        except (OSError, EOFError, UnicodeDecodeError) as e:
            _fail("cannot read the header of %s: %s" % (path, e))
        bodies.append(rest)
    out_idx = [i - 1 for i in args.outputOnly] if args.outputOnly else list(range(nF))
    for i in out_idx:
        if not -nF <= i < nF:
            _fail("--outputOnly %d: there are %d input files (the reference fails with an IndexError)" % (i + 1, nF))
    sep = args.outSep
    header = sep.join([sep.join(heads[0][0:2]), sep.join([sep.join(heads[x][2:]) for x in out_idx])]) + "\n"
    target = env_int("PG_MERGE_CHUNK_BYTES", 64 << 20)
    slab = env_int("PG_MERGE_SLAB_BYTES", 64 << 20)
    dense_rows = env_int("PG_MERGE_DENSE_ROWS", 1 << 22)
    total = sum(max(n, 0) for _, n in scafs)
    tm.mark("setup")
    with Engine(args.device) as eng:
        dense = eng.merge_setup([n.encode() for n, _ in scafs], [n for _, n in scafs],
                                [1 if x in out_idx else 0 for x in range(nF)], [max(len(h) - 2, 0) for h in heads],
                                sep.encode(), args.missing.encode(), METHODS[args.method], args.unionMin,
                                args.mustIncludeFirst)
        gens = [body_chunks(b, s, target, cut_at_cr=False) for b, s in zip(bodies, srcs)]
        last = [-1] * nF                        # walk index of each file's last loaded line
        done = [False] * nF                     # stalled or at its end: sets no bound
        lines_before = [0] * nF
        out = w = None

        def load(x):
            chunk = next(gens[x], None)
            tm.mark("read")
            if chunk is None:
                done[x] = True
                return
            n, stall, state, key = eng.merge_load(x, chunk)
            tm.mark("lines", eng)
            if state == 2:
                _refuse(args, out, w, "%s line %d: a byte outside ASCII or a '\\r' that ends a line by itself (the reference "
                        "reads characters and universal newlines, which this engine does not)"
                        % (args.inputFile[x], lines_before[x] + stall + 2))
            lines_before[x] += n
            last[x] = key
            if state == 1:
                done[x] = True
                gens[x].close()
                if args.verbose:
                    sys.stderr.write("{} stops at line {}.\n".format(args.inputFile[x], lines_before[x] - n + stall + 2))

        for x in range(nF):
            load(x)
        with open_output(args.outputFile) as out, SlabWriter(out.write, slab, PinnedArray) as w:
            out.write(header.encode())
            sys.stderr.write("Merging...\n")
            n_rows = 0
            prev = -1
            while total > 0:
                live = [last[x] for x in range(nF) if not done[x]]
                bound = min(live) if live else total - 1
                while prev < bound:
                    hi = min(bound, prev + dense_rows) if dense else bound
                    rows, nbytes = eng.merge_rows(hi)
                    tm.mark("rows", eng)
                    at = 0
                    while at < nbytes:
                        nb = eng.merge_emit(at, w.slab(), w.cap)
                        tm.mark("emit", eng)
                        w.write(nb)
                        at += nb
                    n_rows += rows
                    prev = hi
                if args.verbose:
                    sys.stderr.write("Merged to walk position {}: {} lines written.\n".format(prev + 1, n_rows))
                if not live:
                    break
                for x in range(nF):
                    if not done[x] and last[x] == bound:
                        load(x)
        tm.mark("write")
        for g in gens:
            g.close()
    sys.stderr.write("{} lines written to output.\n".format(n_rows))
    tm.write(files=nF, rows=n_rows, walk=total)


def _refuse(args, out, w, msg):
    """refuse the run: every submitted write finishes, and an output file already begun is removed"""
    if w is not None:
        w.wait()
    if out is not None and args.outputFile:
        out.close()
        os.remove(args.outputFile)
    _fail(msg)


if __name__ == "__main__":
    main()
