#!/usr/bin/env python
"""Drop-in for the reference's seqToGeno.py (flags 9-18) on the GPU: FASTA / PHYLIP alignments become .geno rows, one row
per site and one column per sequence (-M samples), one row per site of every sequence (-M contigs), or one contig per
alignment of a multi-PHYLIP file.  The text goes to the device once: a FASTA through the loader genoToVCF uses for its
reference, a PHYLIP file through a warp-per-line pass whose line table the host turns into the sequences' field-1 spans.
The transpose of the resident sequences into rows runs on the device, slab by slab (_stream.py).

Refused before any output, where the reference crashes: a single -P value > 1 (a list multiplied by a float), -P values
below 1 where a ploidy > 1 groups the sequences, a -P list that does not sum to the number of sequences (an assertion),
--randomPhase with a ploidy > 1 (len() of a zip), multi-PHYLIP with a ploidy > 1 (a TypeError), a -S name missing from the
input or from any multi-PHYLIP alignment (a ValueError), multi-PHYLIP alignments with different sequence counts (an
assertion), PHYLIP with no header (a ValueError), a header whose count is below 1 or that has fewer sequence lines than its
count, a used sequence line with one field (an IndexError), a FASTA piece with no newline (a ValueError) or no name (an
IndexError), -M samples with no sequences and an output column shorter than the first (of its alignment): the reference
writes the rows before it and then fails with an IndexError; and --devices N.
Narrowed (DESIGN.md section 8): a byte >= 0x80 (the reference counts characters), a '\\r' in a FASTA read from stdin (the
reference reads stdin without universal newlines and keeps it as a character), for PHYLIP a '\\r' that ends a line by itself
and a line that starts with '#', and an input that does not fit in device memory with 1 GiB to spare (there is no chunked
path, as the reference reads the whole file)."""
from __future__ import annotations

import argparse
import re

import numpy as np

from ..engine import Engine, PgError, PinnedArray
from . import _common as C
from ._stream import SlabWriter, env_int, open_input, open_output

LF_HI, LF_CR, LF_HEAD = 1, 2, 4       # flags of the PHYLIP line table (include/pgwin.h pg_s2g_phylip_lines)


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument("-s", "--seqFile", help="Input sequence file (.gz allowed; default stdin)")
    p.add_argument("-g", "--genoFile", help="Output geno file (.gz allowed; default stdout)")
    p.add_argument("-f", "--format", help="Sequence file format", choices=("phylip", "fasta"), default="fasta")
    p.add_argument("-M", "--mode", help="Output mode for separate sequences", choices=("samples", "contigs"),
                   default="samples")
    p.add_argument("-C", "--chrom", help="Name for chromosome or contig if sequences are samples", default="contig0")
    p.add_argument("-N", "--name", help="Name for sample if sequences are contigs", default="sample0")
    p.add_argument("-S", "--sequences", help="Sequences to output", nargs="+", type=str)
    p.add_argument("--merge", help="For multi-phylip input, do not increment scaffold numbers", action="store_true")
    p.add_argument("-P", "--ploidy", help="Ploidy for joining sequences", nargs="+", type=int, default=[1])
    p.add_argument("--randomPhase", help="Randomize phase for fused sequences", action="store_true")
    p.add_argument("--device", help="CUDA device index", type=int, default=0)
    p.add_argument("--devices", help="Not supported: the transpose runs on one GPU", type=int, default=None)
    p.add_argument("--timing", help="Write a JSON file with the wall time of each phase and the device time of each kernel",
                   metavar="FILE")
    return p


def _fail(msg):
    raise SystemExit("seqToGeno: " + msg)


def check_args(args):
    """the refusals that need no input"""
    if args.devices not in (None, 1):
        _fail("--devices is not supported; the transpose runs on one GPU")
    if max(args.ploidy) > 1:
        if len(args.ploidy) == 1:
            _fail("a single -P value above 1 is not supported: the reference multiplies a list by a float "
                  "(genomics.py:426) and fails with a TypeError")
        if min(args.ploidy) < 1:
            _fail("-P values must be at least 1 (the reference cannot group sequences by %s)" % args.ploidy)
        if args.randomPhase:
            _fail("--randomPhase with a ploidy above 1 is not supported: the reference takes len() of a zip "
                  "(genomics.py:437) and fails with a TypeError")


def _line_of(data, at):
    """the 1-based line (universal newlines) of byte `at`"""
    head = data[:at]
    return head.count(b"\n") + head.count(b"\r") - head.count(b"\r\n") + 1


def first_index(names):
    """name -> its first index (list.index)"""
    out = {}
    for i, n in enumerate(names):
        out.setdefault(n, i)
    return out


def load_fasta(eng, data, from_stdin):
    """the FASTA's records on the device: (names, lengths)"""
    if from_stdin and b"\r" in data:
        _fail("line %d: a '\\r' in a FASTA read from stdin (the reference reads stdin without universal newlines and keeps it "
              "as a character; this engine does not)" % _line_of(data, data.index(b"\r")))
    starts = eng.s2g_fasta_load(data)
    names, lo, hi = C.fasta_records(data, starts, _fail)
    return names, eng.s2g_fasta_index(lo, hi)


def load_phylip(eng, data):
    """genomics.parsePhylip on the device's line table: a list of alignments (names, sequence indices) and the lengths of the
    sequences, which the device packs into the resident layout"""
    hash_at = 0 if data.startswith(b"#") else data.find(b"\n#") + 1
    if data.startswith(b"#") or hash_at > 0:
        _fail("line %d starts with '#' (this engine's line index skips such lines, the reference reads them)" %
              _line_of(data, hash_at))
    lines = eng.s2g_phylip_load(data)
    lines = lines[lines[:, 4] > 0]                      # parsePhylip drops the lines without a field
    cr = np.flatnonzero(lines[:, 5] & LF_CR)
    if len(cr):
        _fail("line %d: a '\\r' ends a line by itself (the reference reads it as a line end, this engine does not)" %
              _line_of(data, int(lines[cr[0], 0])))
    heads = np.flatnonzero(lines[:, 5] & LF_HEAD)
    if not len(heads):
        _fail("the PHYLIP input has no header line (two integer fields); the reference fails with a ValueError")
    bounds = np.append(heads, len(lines))
    aligns, seq_id, seq_base = [], np.full(len(lines), -1, np.int64), 0
    for k in range(len(heads)):
        h, end = int(bounds[k]), int(bounds[k + 1])
        n = int(lines[h, 6])
        if n < 1:
            _fail("line %d: the header counts %d sequences (the reference writes no sequence for it)" %
                  (_line_of(data, int(lines[h, 0])), n))
        if end - h - 1 < n:
            _fail("line %d: the header counts %d sequences, %d lines follow it (the reference reads past them)" %
                  (_line_of(data, int(lines[h, 0])), n, end - h - 1))
        one = np.flatnonzero(lines[h + 1:end, 4] == 1)
        if len(one):
            _fail("line %d: a sequence line with one field (the reference fails with an IndexError)" %
                  _line_of(data, int(lines[h + 1 + one[0], 0])))
        names = [data[int(a):int(a) + int(b)].decode() for a, b in lines[h + 1:h + 1 + n, :2]]
        seq_id[h + 1:end] = seq_base + np.arange(end - h - 1) % n
        aligns.append((names, list(range(seq_base, seq_base + n))))
        seq_base += n
    used = np.flatnonzero(seq_id >= 0)
    order = used[np.argsort(seq_id[used], kind="stable")]      # sequence by sequence, its lines in order
    f1_len = lines[order, 3]
    dst = np.concatenate([[0], np.cumsum(f1_len)[:-1]]).astype(np.int64) if len(order) else np.zeros(0, np.int64)
    seq_len = np.bincount(seq_id[used], weights=lines[used, 3], minlength=seq_base).astype(np.int64)
    eng.s2g_phylip_pack(seq_len, np.stack([lines[order, 2], dst, f1_len], axis=1) if len(order) else np.zeros((0, 3)))
    return aligns, seq_len


def plan(args, aligns, lens):
    """the header line and the blocks of the output (name, rows, members, separators), with the reference's rules and
    refusals (seqToGeno.py:56-98, genomics.haploToPhased)"""
    ploidy = args.ploidy if max(args.ploidy) > 1 else None
    blocks = []

    def columns(seqs, names, groups):
        """[(name, [members])] of the ploidy groups (zip-truncated together)"""
        if groups is None:
            return [(n, [s]) for n, s in zip(names, seqs)]
        if sum(groups) != len(seqs):
            _fail("-P %s sums to %d, the input gives %d sequences (the reference fails on an assertion)" %
                  (" ".join(map(str, groups)), sum(groups), len(seqs)))
        out, at = [], 0
        for p in groups:
            out.append(("_".join(names[at:at + p]), seqs[at:at + p]))
            at += p
        return out

    def add_rows(name, cols, where):
        """one block of rows over the columns: as many as the first column's, a shorter later column refused"""
        rows = min(int(lens[m]) for m in cols[0][1])
        for cname, mem in cols[1:]:
            n = min(int(lens[m]) for m in mem)
            if n < rows:
                _fail("%scolumn %s holds %d sites, the first holds %d (the reference writes the rows before it and then "
                      "fails with an IndexError)" % (where, cname, n, rows))
        add_block(name, rows, cols)

    def add_block(name, rows, cols):
        mem, sep = [], []
        for c, (_, m) in enumerate(cols):
            mem += m
            sep += [b"|"] * (len(m) - 1) + [b"\n" if c == len(cols) - 1 else b"\t"]
        blocks.append((name.encode(), rows, mem, b"".join(sep)))

    if len(aligns) == 1:
        names, seqs = aligns[0]
        if args.sequences is not None:
            idx = first_index(names)
            for x in args.sequences:
                if x not in idx:
                    _fail("sequence %s is not in the input (the reference fails with a ValueError)" % x)
            seqs = [seqs[idx[x]] for x in args.sequences]
            names = list(args.sequences)
        cols = columns(seqs, names, ploidy)
        if args.mode == "samples":
            if not cols:
                _fail("-M samples with no sequences: the reference writes the header and fails with an IndexError")
            add_rows(args.chrom, cols, "")
            head = "#CHROM\tPOS\t" + "\t".join(n for n, _ in cols) + "\n"
        else:
            for n, mem in cols:
                add_block(n, min(int(lens[m]) for m in mem), [(n, mem)])
            head = "#CHROM\tPOS\t" + args.name + "\n"
        return head.encode(), blocks
    if ploidy is not None:
        _fail("multi-PHYLIP input with a ploidy above 1 is not supported: the reference fails with a TypeError "
              "(makePhasedNames has no randomPhase argument)")
    counts = {len(n) for n, _ in aligns}
    if len(counts) != 1:
        _fail("the alignments of a multi-PHYLIP input hold different numbers of sequences (%s); the reference fails on an "
              "assertion" % ", ".join(str(len(n)) for n, _ in aligns))
    out_names = list(args.sequences) if args.sequences else list(aligns[0][0])
    for i, (names, seqs) in enumerate(aligns):
        idx = first_index(names)
        for x in out_names:
            if x not in idx:
                _fail("sequence %s is not in alignment %d (the reference fails with a ValueError)" % (x, i + 1))
        cols = [(x, [seqs[idx[x]]]) for x in out_names]
        add_rows(args.chrom if args.merge else args.chrom + str(i), cols, "alignment %d: " % (i + 1))
    return ("#CHROM\tPOS\t" + "\t".join(out_names) + "\n").encode(), blocks


def main(argv=None):
    args = build_parser().parse_args(argv)
    check_args(args)
    tm = C.Timing(args.timing)
    data = open_input(args.seqFile).read()
    tm.mark("read")
    if not data.isascii():
        _fail("a byte outside ASCII at line %d (the reference reads characters, which this engine does not)" %
              _line_of(data, re.search(rb"[\x80-\xff]", data).start()))
    slab = env_int("PG_S2G_SLAB_BYTES", 64 << 20)
    with Engine(args.device) as eng:
        try:
            if args.format == "fasta":
                names, lens = load_fasta(eng, data, not args.seqFile)
                aligns = [(names, list(range(len(names))))]
            else:
                aligns, lens = load_phylip(eng, data)
        except PgError as e:
            if "do not fit in device memory" in str(e):
                _fail("the input does not fit in device memory with 1 GiB to spare; there is no chunked path (%s)" % e)
            raise
        tm.mark("load", eng)
        del data
        head, blocks = plan(args, aligns, lens)
        total = eng.s2g_plan([b[0] for b in blocks], [b[1] for b in blocks], [b[2] for b in blocks],
                             [b[3] for b in blocks])
        tm.mark("plan", eng)
        with open_output(args.genoFile) as out, SlabWriter(out.write, slab, PinnedArray) as w:
            out.write(head)
            at = 0
            while at < total:
                nb = eng.s2g_emit(at, w.slab(), w.cap)
                tm.mark("emit", eng)
                w.write(nb)
                at += nb
        tm.mark("write")
    tm.write(sequences=int(len(lens)), rows=int(sum(b[1] for b in blocks)), bytes=int(total))


if __name__ == "__main__":
    main()
