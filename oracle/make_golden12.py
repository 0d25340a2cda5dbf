#!/usr/bin/env python
"""TEST INFRASTRUCTURE — fixtures for seqToGeno.py from the UNMODIFIED reference script.

    python oracle/make_golden12.py [/path/to/genomics_general]

Writes seeded FASTA and PHYLIP inputs under tests/golden/s2g12/, runs the reference seqToGeno.py on every case of CASES in a
scratch directory and commits what it writes (the output file or its stdout), gzip-compressed, next to them, with
tests/golden/cases12.json listing the cases.  Cases where the reference fails record the exception it raised and the output
it had written before it failed.

The FASTA inputs hold lines wrapped at mixed widths, CRLF and lone '\\r' line ends, blank lines, text before the first '>', a
'>' in the middle of a line, header descriptions, a blank header line, lowercase, IUPAC and '-' characters, a tab inside a
sequence line, a duplicated name and later sequences longer than the first.  The PHYLIP inputs hold sequential and
interleaved alignments (continuation lines of two fields, of which the reference reads field 1), the header forms '+3 4',
'3 1_0' and '3 4 extra', lines before the first header, blank and CRLF lines, and multi-PHYLIP files whose alignments order
their sequences differently."""
import gzip
import json
import os
import random
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "..", "tests", "golden")
DIR = os.path.join(GOLD, "s2g12")
CHARS = "ACGTACGTACGTacgtNnRYKM-"


def seq(rng, n):
    return "".join(rng.choice(CHARS) for _ in range(n))


def wrap(rng, s, crlf=False, lone_cr=False):
    out, at = [], 0
    while at < len(s):
        w = rng.choice((7, 10, 13, 60))
        out.append(s[at:at + w])
        at += w
    ends = ["\r\n" if crlf and k % 2 else "\r" if lone_cr and k % 3 == 2 else "\n" for k in range(len(out))]
    return "".join(a + b for a, b in zip(out, ends))


def write(name, text):
    with open(os.path.join(DIR, name), "wb") as f:
        f.write(text.encode() if isinstance(text, str) else text)


def write_inputs():
    rng = random.Random(12)
    s = {k: seq(rng, n) for k, n in [("s0", 50), ("s1", 50), ("s2", 57), ("s3", 64), ("s4", 52), ("dup", 51),
                                    ("dup2", 55), ("s6", 70)]}
    main = "notes before the first record\n\n"
    main += ">s0 first record description\n" + wrap(rng, s["s0"])
    main += ">s1\n" + wrap(rng, s["s1"], crlf=True) + "\n\n"
    main += ">s2 desc\twith tab\n" + wrap(rng, s["s2"][:20]) + s["s2"][20:24] + "\t" + s["s2"][24:] + "\n"
    main += ">s3\n" + wrap(rng, s["s3"], lone_cr=True)
    main += ">dup\n" + wrap(rng, s["dup"]) + s["s4"][:5] + " " + s["s4"][5:9] + ">s4 mid-line record\n" + wrap(rng, s["s4"])
    main += ">\n" + wrap(rng, "blankhead" + s["dup2"])
    main += ">dup second of the name\n" + wrap(rng, s["s6"])
    write("main.fa", main)
    with gzip.GzipFile(os.path.join(DIR, "main.fa.gz"), "wb", mtime=0) as g:
        g.write(main.encode())
    write("lf.fa", "".join(">%s\n%s" % (k, wrap(rng, s[k])) for k in ("s0", "s1", "s2")))
    write("empty.fa", "")
    write("short.fa", ">a\n%s\n>b\n%s\n>c\n%s\n" % (seq(rng, 30), seq(rng, 30), seq(rng, 20)))
    write("nonewline.fa", ">a\nACGT\n>b ACGT")
    write("noname.fa", ">a\nACGT\n> \n>b\nAC\n")
    a = {k: seq(rng, 24).upper() for k in "abcd"}
    write("seq.phy", "leading text line\nmore leading text\n 4 24\n" + "".join("%s  %s\n" % (k, a[k]) for k in "abcd"))
    il = "+3 16 extra fields\r\n"
    il += "".join("%s %s\r\n" % (k, a[k][:8]) for k in "abc") + "\n"
    il += "".join("%s %s\n" % (a[k][8:12], a[k][12:16]) for k in "abc")
    il += "".join("x%s %s\n" % (k, a[k][16:20]) for k in "abc")
    write("interleaved.phy", il)
    write("forms.phy", "3 1_0\n" + "".join("%s %s\n" % (k, a[k][:10]) for k in "abc"))
    m = ""
    for i, order in enumerate(["abc", "cab", "bca"]):
        m += ("3 %d\n" if i != 1 else "+3 %d\n") % (6 + i) + "".join("%s %s\n" % (k, seq(rng, 6 + i).upper()) for k in order)
        m += "\n"
    write("multi.phy", m)
    write("multi_uneven.phy", "2 4\na ACGT\nb CCGT\n3 4\na ACGT\nb GGGG\nc TTTT\n")
    write("multi_short.phy", "2 4\na ACGT\nb CCGT\n2 4\nb ACG\na TTTT\n")
    write("nohead.phy", "a ACGT\nb CCGT\n")
    write("zero.phy", "0 4\na ACGT\n")
    write("fewlines.phy", "3 4\na ACGT\nb CCGT\n")
    write("onefield.phy", "2 4\na ACGT\nb\n")


CASES = [
    # name, input ("-" = stdin from lf.fa), args, dest
    ("fa_default", "main.fa", [], "stdout"),
    ("fa_gz_in_out", "main.fa.gz", [], "out.geno.gz"),
    ("fa_stdin", "-", [], "stdout"),
    ("fa_file_out", "lf.fa", ["-C", "chr9"], "out.geno"),
    ("fa_S_reorder_dup", "main.fa", ["-S", "s0", "s2", "dup", "s0"], "stdout"),
    ("fa_C", "main.fa", ["-C", "scaffold_7"], "stdout"),
    ("fa_contigs", "main.fa", ["-M", "contigs", "-N", "indiv1"], "stdout"),
    ("fa_contigs_groups", "main.fa", ["-M", "contigs", "-P", "2", "1", "3", "2"], "stdout"),
    ("fa_contigs_empty", "empty.fa", ["-M", "contigs"], "stdout"),
    ("fa_P22", "main.fa", ["-S", "s0", "s3", "s1", "s2", "-P", "2", "2"], "stdout"),
    ("fa_P13", "main.fa", ["-S", "s0", "s1", "s2", "s3", "-P", "1", "3"], "stdout"),
    ("fa_P1111_on_2", "main.fa", ["-S", "s0", "s1", "-P", "1", "1", "1", "1"], "stdout"),
    ("fa_P_zip_truncation", "main.fa", ["-S", "s2", "s0", "s3", "s1", "-P", "2", "2"], "stdout"),
    ("fa_randomphase_p1", "main.fa", ["--randomPhase"], "stdout"),
    ("phy_sequential", "seq.phy", ["-f", "phylip"], "stdout"),
    ("phy_interleaved", "interleaved.phy", ["-f", "phylip", "-C", "chrI"], "stdout"),
    ("phy_forms_contigs", "forms.phy", ["-f", "phylip", "-M", "contigs"], "stdout"),
    ("phy_sequential_P", "seq.phy", ["-f", "phylip", "-P", "2", "2"], "stdout"),
    ("multi", "multi.phy", ["-f", "phylip"], "stdout"),
    ("multi_merge", "multi.phy", ["-f", "phylip", "--merge", "-C", "chrM", "-M", "contigs"], "stdout"),
    ("multi_S", "multi.phy", ["-f", "phylip", "-S", "c", "a"], "out.geno.gz"),
    # the reference fails on these
    ("fail_single_ploidy", "main.fa", ["-P", "2"], "stdout"),
    ("fail_ploidy_sum", "main.fa", ["-P", "2", "3"], "stdout"),
    ("fail_randomphase_ploidy", "main.fa", ["-S", "s0", "s1", "s2", "-P", "1", "2", "--randomPhase"], "stdout"),
    ("fail_multi_ploidy", "multi.phy", ["-f", "phylip", "-P", "1", "2"], "stdout"),
    ("fail_S_missing", "main.fa", ["-S", "s0", "zz"], "stdout"),
    ("fail_multi_S_missing", "multi.phy", ["-f", "phylip", "-S", "a", "zz"], "stdout"),
    ("fail_multi_counts", "multi_uneven.phy", ["-f", "phylip"], "stdout"),
    ("fail_phylip_no_header", "nohead.phy", ["-f", "phylip"], "stdout"),
    ("fail_header_count_zero", "zero.phy", ["-f", "phylip"], "stdout"),
    ("fail_header_few_lines", "fewlines.phy", ["-f", "phylip"], "stdout"),
    ("fail_one_field_line", "onefield.phy", ["-f", "phylip"], "stdout"),
    ("fail_fasta_no_newline", "nonewline.fa", [], "stdout"),
    ("fail_fasta_no_name", "noname.fa", [], "stdout"),
    ("fail_samples_empty", "empty.fa", [], "stdout"),
    ("fail_shorter_later", "short.fa", [], "stdout"),
    ("fail_multi_shorter_later", "multi_short.phy", ["-f", "phylip"], "stdout"),
]


def run_case(ref, case):
    name, inp, args, dest = case
    work = tempfile.mkdtemp()
    try:
        cmd = [sys.executable, os.path.join(ref, "seqToGeno.py")] + list(args)
        if inp != "-":
            cmd += ["-s", os.path.join(DIR, inp)]
        if dest != "stdout":
            cmd += ["-g", os.path.join(work, dest)]
        stdin = open(os.path.join(DIR, "lf.fa"), "rb") if inp == "-" else subprocess.DEVNULL
        r = subprocess.run(cmd, cwd=work, stdin=stdin, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                           env=dict(os.environ, PYTHONPATH=ref))
        entry = dict(name=name, input=inp, args=list(args), dest=dest)
        if r.returncode != 0:
            entry["fails"] = r.stderr.decode().strip().splitlines()[-1]
        if dest == "stdout":
            data = r.stdout
        else:
            data = open(os.path.join(work, dest), "rb").read()
            data = gzip.decompress(data) if dest.endswith(".gz") else data
        fix = name + ".geno.gz"
        with gzip.GzipFile(os.path.join(DIR, fix), "wb", mtime=0) as g:
            g.write(data)
        entry["output"] = fix
        return entry
    finally:
        shutil.rmtree(work)


def main(ref):
    if os.path.isdir(DIR):
        shutil.rmtree(DIR)
    os.makedirs(DIR)
    write_inputs()
    cases = [run_case(ref, c) for c in CASES]
    with open(os.path.join(GOLD, "cases12.json"), "w") as f:
        json.dump(cases, f, indent=1)
    for c in cases:
        print(c["name"], "FAILS " + c["fails"] if "fails" in c else "ok")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
