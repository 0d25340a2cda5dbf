#!/usr/bin/env python
"""Drop-in for the reference's VCF_processing/genoToVCF.py (flags 29-33) on the GPU: .geno genotypes become VCF GT records,
with REF from a reference FASTA.  The body is read in chunks cut at line ends and the rows are written slab by slab
(_stream.py); the device indexes each chunk's lines and tokens, counts every site's alleles, orders them, looks up the
reference base and writes the VCF rows into the slabs.  The FASTA is loaded once: its sequences are compacted on the device
and stay there.

Refused before any output, where the reference crashes or writes something else: no -f, a -s name that is not in the
header, no selected samples, --devices N, --hostParse and --cache, a .fai line with fewer than 2 fields, a FASTA piece with
no newline or no name token, a FASTA with a byte >= 0x80, an empty input.  Refused at the data line (and sample), after the
rows before it are written as the reference writes them: a missing selected column, a bad diplo token, a scaffold that is
not in the FASTA, a position outside its contig.  Narrowed (DESIGN.md section 8): lines with a byte >= 0x80, a '\\r' that
ends a line by itself, POS forms other than [+-]?[0-9]+, POS outside int64, and a line of only two fields (the reference
would read its position as the first sample's genotype).  Blank lines are skipped."""
from __future__ import annotations

import argparse
import gzip
import re
import sys

import numpy as np

from ..engine import Engine, PinnedArray
from . import _common as C
from ._stream import SlabWriter, body_chunks, env_int, first_line, open_input, open_output

FORMATS = {"phased": 0, "diplo": 1, "pairs": 2}
TOK = re.compile(rb"[^ \t\n\r\x0b\x0c\x1c-\x1f]+")
# error codes of pg_g2v_sites (include/pgwin.h); %s takes the sample name where the code names one
ERRORS = {1: "the position is not an integer of the form [+-]digits (the reference's int() fails on it, or accepts a form "
             "such as 1_000 that this engine does not)",
          2: "the line has no position field (the reference fails with an IndexError)",
          3: "the position is outside the int64 range",
          4: "the line has only two fields (the reference would read its position as the first sample's genotype)",
          5: "a byte outside ASCII (the reference reads characters, which this engine does not)",
          6: "a '\\r' ends a line by itself (the reference reads it as a line end, this engine does not)",
          7: "sample %s has no genotype column on this line (the reference fails with a KeyError)",
          8: "the genotype of sample %s is not one of the diplo codes ACGKMNSRTWY (the reference fails with a KeyError)",
          9: "scaffold %s is not a record of the reference FASTA (the reference fails with a KeyError)",
          10: "position %s is outside its reference contig (the reference fails with an IndexError)"}


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument("-g", "--genoFile", help="Input geno file (.gz allowed; default stdin)")
    p.add_argument("-f", "--genoFormat", help="Genotype format", choices=tuple(FORMATS))
    p.add_argument("-o", "--outFile", help="Output vcf file (.gz allowed; default stdout)")
    p.add_argument("-r", "--reference", help="Reference fasta (.gz allowed)")
    p.add_argument("-s", "--samples", help="Samples to include (separated by commas)")
    C.add_engine_args(p)
    return p


def _fail(msg):
    raise SystemExit("genoToVCF: " + msg)


def read_fai(reference):
    """[first two fields] of every line of <reference>.fai, or None when it cannot be read (the reference only warns)"""
    try:
        with open(reference + ".fai", "rt") as fai:
            return [line.split()[:2] for line in fai]
    except Exception:
        sys.stderr.write("WARNING: Could not parse fai file, vcf header will not contain contig entries...\n")
        return None


def fasta_records(data, starts):
    """genomics.parseFasta's pieces of the reference (_common.fasta_records), refused where parseFasta raises"""
    return C.fasta_records(data, starts, lambda msg: _fail("reference FASTA: " + msg))


def plan(args, names):
    """the selected samples and the spec tables: col_slot / col_prev over the header's genotype columns, sel_col the column
    of every selected sample (dict(zip(names, GTs)) keeps the last column of a name, genomics.py:1896)"""
    samples = args.samples.split(",") if args.samples else list(names)
    last, col_prev = {}, []
    for c, n in enumerate(names):
        col_prev.append(last.get(n, -1))
        last[n] = c
    for s in samples:
        if s not in last:
            _fail("sample %s is not in the header (the reference fails with a KeyError)" % s)
    if not samples:
        _fail("no samples: the header names none (the reference fails on its first data line)")
    wanted = set(samples)
    col_slot, k = [], 0
    for n in names:
        col_slot.append(k if n in wanted else -1)
        k += n in wanted
    return samples, dict(col_slot=col_slot, col_prev=col_prev, sel_col=[last[s] for s in samples])


def header_text(args, samples, fai, has_records):
    out = ["##fileformat=VCFv4.2\n"]
    if has_records:
        out.append("##reference=file:{}\n".format(args.reference.split("/")[-1]))
        for f in fai or []:
            out.append("##contig=<ID={},length={}>\n".format(f[0], f[1]))
    out.append('##FORMAT=<ID=GT,Number=1,Type=String,Description="Genotype">\n')
    out.append("#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\t" + "\t".join(samples) + "\n")
    return "".join(out).encode()


def main(argv=None):
    args = build_parser().parse_args(argv)
    if args.devices not in (None, 1):
        _fail("--devices is not supported; the conversion runs on one GPU")
    if args.hostParse or args.cache:
        _fail("--hostParse and --cache do not apply: the conversion streams the text through the GPU")
    if args.genoFormat is None:
        _fail("-f/--genoFormat is required (the reference fails on the first data line without it)")
    tm = C.Timing(args.timing)
    fa = fai = None
    if args.reference:
        sys.stderr.write("Parsing reference...\n")
        fai = read_fai(args.reference)
        with (gzip.open(args.reference, "rb") if args.reference.endswith(".gz") else open(args.reference, "rb")) as f:
            fa = f.read()
        if not fa.isascii():
            _fail("reference FASTA: a byte outside ASCII (this engine reads ASCII sequences only)")
    src = open_input(args.genoFile)
    first = first_line(src)
    if first is None:
        _fail("the input is empty: it has no header line (the reference fails with a StopIteration)")
    head, body0 = first
    names = head.decode().split()[2:]
    samples, spec = plan(args, names)
    target = env_int("PG_G2V_CHUNK_BYTES", 256 << 20)
    slab = env_int("PG_G2V_SLAB_BYTES", 64 << 20)
    with Engine(args.device) as eng:
        rec = {}
        if fa is not None:
            starts = eng.g2v_ref_load(fa)
            tm.mark("reference_load", eng)
            if len(starts):
                rec_names, lo, hi = fasta_records(fa, starts)
                eng.g2v_ref_index(lo, hi)
                rec = {n: k for k, n in enumerate(rec_names)}          # dict(zip(names, seqs)): the last one wins
            if rec and fai is not None:
                for k, f in enumerate(fai):
                    if len(f) < 2:
                        _fail("%s.fai line %d has fewer than 2 fields (the reference fails with an IndexError while "
                              "writing the header)" % (args.reference, k + 1))
            del fa
            tm.mark("reference", eng)
        eng.g2v_spec(FORMATS[args.genoFormat], spec["col_slot"], spec["col_prev"], spec["sel_col"], bool(rec))
        with open_output(args.outFile) as out, SlabWriter(out.write, slab, PinnedArray) as w:
            out.write(header_text(args, samples, fai, bool(rec)))
            sys.stderr.write("Converting...\n")
            n_lines, n_rows, lines_before = 0, 0, 1
            for chunk in body_chunks(body0, src, target):
                tm.mark("read")
                S, run_line, run_off = eng.g2v_chunk(chunk)
                tm.mark("tokens", eng)
                run_rec = np.array([rec.get(TOK.search(chunk, int(o)).group().decode(), -1) for o in run_off]
                                   if rec else [], np.int32)
                rows, nbytes, err = eng.g2v_sites(run_rec)
                tm.mark("sites", eng)
                at = 0
                while at < nbytes:
                    nb = eng.g2v_emit(at, w.slab(), w.cap)
                    tm.mark("emit", eng)
                    w.write(nb)
                    at += nb
                if err[0]:
                    w.wait()
                    _fail(_message(err, chunk, samples, lines_before))
                n_lines += S
                n_rows += rows
                lines_before += chunk.count(b"\n")
                sys.stderr.write("{} lines converted...\n".format(n_lines))
        tm.mark("write")
    tm.write(lines=n_lines, rows=n_rows)


def _message(err, chunk, samples, lines_before):
    """'line N: ...' in the file's numbering (the header is line 1) for the error (code, data line of the chunk, column,
    byte offset of the line in the chunk)"""
    code, line, col, off = err
    toks = TOK.findall(chunk, off, chunk.find(b"\n", off) if chunk.find(b"\n", off) >= 0 else len(chunk))
    msg = ERRORS.get(code, "error %d" % code)
    if code in (7, 8):
        msg = msg % samples[col - 1]
    elif code == 9:
        msg = msg % toks[0].decode()
    elif code == 10:
        msg = msg % toks[1].decode()
    return "line %d: %s" % (lines_before + chunk.count(b"\n", 0, off) + 1, msg)


if __name__ == "__main__":
    main()
