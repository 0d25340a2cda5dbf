#!/usr/bin/env python
"""TEST INFRASTRUCTURE — fixtures for genoToVCF.py from the UNMODIFIED reference script.

    python oracle/make_golden11.py [/path/to/genomics_general]

Writes seeded .geno and FASTA inputs under tests/golden/g2v11/, runs the reference VCF_processing/genoToVCF.py on every case
of CASES in a scratch directory and commits what it writes (the output file or its stdout), gzip-compressed, next to them,
with tests/golden/cases11.json listing the cases.  Cases where the reference fails record the exception it raised and the
output it had written before it failed.

The inputs cover every tie pattern of up to four counted bases (counts 0-3 of A, C, G, T), all-missing sites, lowercase,
'-' and IUPAC characters, phased tokens of widths 1-5 with mixed phase characters and a ploidy that changes from line to
line, pairs tokens holding '/', every diplo code, a comment line between data lines, CRLF line ends, the POS forms 007, +4,
0 and negative, and a FASTA with text before its first '>', description text, spaces inside sequence lines, CRLF, lowercase
and N bases, a '>' inside a sequence line and a duplicated name (plain and .gz, with and without a .fai).

The reference orders a site's alleles with np.argsort(counts)[::-1] (genomics.py:556).  numpy's vectorised argsort (AVX2 /
AVX-512 dispatch) breaks ties between equal counts in an order that depends on the CPU; its portable sort is stable and gives
ties to the later letter of ACGT.  The reference runs here with the vectorised paths disabled (NPY_DISABLE_CPU_FEATURES), so
that the fixtures hold that stable order on every machine."""
import gzip
import itertools
import json
import os
import random
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "..", "tests", "golden")
DIR = os.path.join(GOLD, "g2v11")

LENGTHS = {"chrA": 200, "chrB": 150, "chrC": 60}
SEQ_CHARS = "ACGTACGTACGTacgtNn"
TOKEN_CHARS = "ACGTACGTACGTACGTNNNacgt-RK"
DIPLO = "ACGKMNSRTWY"
NO_SIMD_SORT = "AVX512F AVX512CD AVX512_SKX AVX512_CLX AVX512_CNL AVX512_ICL AVX512_SPR AVX2 FMA3 F16C"


def _write(name, text, gz=False):
    data = text.encode() if isinstance(text, str) else text
    if gz:
        with gzip.GzipFile(os.path.join(DIR, name), "wb", mtime=0) as f:
            f.write(data)
    else:
        with open(os.path.join(DIR, name), "wb") as f:
            f.write(data)


def _fasta(rng):
    """text before the first '>', descriptions, spaces inside sequence lines, CRLF on one record, a '>' inside a sequence
    line (it starts a record named by the token after it), and chrA twice (the later record wins)"""
    def seq(n):
        return "".join(rng.choice(SEQ_CHARS) for _ in range(n))

    def lines(s, width, eol="\n"):
        out = []
        for k in range(0, len(s), width):
            piece = s[k:k + width]
            if k // width == 1:
                piece = piece[:5] + " " + piece[5:] + "  "          # spaces inside a sequence line are dropped
            out.append(piece + eol)
        return "".join(out)
    parts = ["this text comes before the first record\n"]
    parts.append(">chrA first copy, replaced below\n" + lines(seq(90), 40))
    parts.append(">chrB some description\r\n" + lines(seq(LENGTHS["chrB"]), 50, "\r\n"))
    c = seq(LENGTHS["chrC"])
    parts.append(">chrC\n" + lines(c, 30) + "GGTT>inner piece\nACGTNNacgt\n")
    parts.append(">chrA\tsecond copy\n" + lines(seq(LENGTHS["chrA"]), 60))
    return "".join(parts)


def _fai(fasta_name):
    return "".join("%s\t%d\t%d\t60\t61\n" % (n, LENGTHS[n], 10 * k) for k, n in enumerate(("chrA", "chrB", "chrC"))) + \
        "inner\t10\t999\t10\t11\n"


def _phased_token(rng, width, chars=TOKEN_CHARS):
    al = [rng.choice(chars) for _ in range((width + 1) // 2)]
    out = al[0]
    for a in al[1:]:
        out += rng.choice("||/") + a
    if width % 2 == 0:
        out += rng.choice(chars)
    return out


def write_inputs():
    rng = random.Random(1111)
    names = ["s%d" % i for i in range(8)]
    head = "#CHROM\tPOS\t" + "\t".join(names)
    body = []
    scafs = ["chrA"] * 3 + ["chrB"] * 2 + ["chrC"]

    def pos_of(sc, k):
        return 1 + (k * 7) % LENGTHS[sc]
    # every tie pattern: counts 0-3 of each of A, C, G, T among 16 alleles, the rest N
    for k, cnt in enumerate(itertools.product(range(4), repeat=4)):
        al = [b for b, n in zip("ACGT", cnt) for _ in range(n)] + ["N"] * (16 - sum(cnt))
        rng.shuffle(al)
        sc = "chrA" if k < 128 else ("chrB" if k < 200 else "chrA")        # chrA again after chrB: an unsorted file
        body.append("\t".join([sc, str(pos_of(sc, k))] + [al[2 * i] + "|" + al[2 * i + 1] for i in range(8)]))
        if k == 40:
            body.append("# a comment line between data lines")
    # all-missing sites, and sites whose only calls are lowercase, '-' or IUPAC (none of them counted)
    for k in range(6):
        body.append("\t".join(["chrC", str(pos_of("chrC", k))] + ["N|N"] * 8))
        body.append("\t".join(["chrC", str(pos_of("chrC", k + 9))] + [rng.choice(["a|c", "-|-", "R|K", "A|-", "n|A", "N|a"])
                                                                      for _ in range(8)]))
    # random tokens of widths 1-5 with mixed phase characters, a ploidy that changes from line to line
    for k in range(300):
        sc = scafs[k % len(scafs)]
        w = rng.choice([1, 2, 3, 3, 3, 4, 5])
        toks = [_phased_token(rng, w if rng.random() < 0.8 else rng.choice([1, 2, 3, 4, 5])) for _ in range(8)]
        body.append("\t".join([sc, str(pos_of(sc, k + 300))] + toks))
    main = head + "\n" + "\n".join(body) + "\n"
    _write("main.geno", main)
    _write("main.geno.gz", main, gz=True)
    # POS forms: leading zeros, '+', 0 (the last base with -r) and negative (from the end with -r)
    ls = [head] + ["\t".join(["chrA", p] + [_phased_token(rng, 3) for _ in range(8)])
                   for p in ("007", "+4", "0", "-3", "-0", "200", "-199", "+000012")]
    _write("pos.geno", "\n".join(ls) + "\n")
    # CRLF line ends, a comment, space-separated fields
    ls = ["#CHROM POS s0 s1 s2"]
    for k in range(40):
        if k == 10:
            ls.append("#comment")
        ls.append(" ".join(["chrB", str(1 + 3 * k)] + [_phased_token(rng, 3) for _ in range(3)]))
    _write("crlf.geno", "\r\n".join(ls) + "\r\n")
    # pairs tokens, '/' among them (an allele of its own in the pairs format)
    pn = ["p%d" % i for i in range(4)]
    ls = ["#CHROM\tPOS\t" + "\t".join(pn)]
    for k in range(120):
        toks = ["".join(rng.choice("ACGTACGTN/-a") for _ in range(rng.choice([1, 2, 2, 3, 4]))) for _ in pn]
        ls.append("\t".join(["chrC" if k < 60 else "chrA", str(1 + k % 60)] + toks))
    _write("pairs.geno", "\n".join(ls) + "\n")
    # every diplo code, in every column; a bad token in column d5 (read only when d5 is selected)
    dn = ["d%d" % i for i in range(6)]
    ls = ["#CHROM\tPOS\t" + "\t".join(dn)]
    for k in range(66):
        toks = [DIPLO[(k + i) % len(DIPLO)] for i in range(6)]
        ls.append("\t".join(["chrB", str(1 + k)] + toks))
    _write("diplo.geno", "\n".join(ls) + "\n")
    ls[30] = ls[30].rsplit("\t", 1)[0] + "\tX"
    _write("diplo_bad.geno", "\n".join(ls) + "\n")
    # header only; empty; no sample names; short line; scaffold not in the FASTA; position outside a contig; blank line
    _write("header_only.geno", head + "\n")
    _write("empty.geno", "")
    _write("nonames.geno", "#CHROM\tPOS\nchrA\t5\n")
    ls = [head] + ["\t".join(["chrA", str(k + 1)] + [_phased_token(rng, 3) for _ in range(8)]) for k in range(20)]
    short = list(ls)
    short[12] = short[12].rsplit("\t", 3)[0]
    _write("short.geno", "\n".join(short) + "\n")
    miss = list(ls)
    miss[15] = miss[15].replace("chrA", "chrZ", 1)
    _write("scafmiss.geno", "\n".join(miss) + "\n")
    rng_ = list(ls)
    rng_[9] = rng_[9].replace("chrA\t9\t", "chrA\t201\t", 1)
    _write("posrange.geno", "\n".join(rng_) + "\n")
    blank = list(ls)
    blank.insert(7, "")
    _write("blank.geno", "\n".join(blank) + "\n")
    # FASTA files
    fa = _fasta(rng)
    _write("ref.fa", fa)
    _write("ref.fa.fai", _fai("ref.fa"))
    _write("ref.fa.gz", fa, gz=True)
    _write("ref.fa.gz.fai", _fai("ref.fa.gz"))
    _write("refnofai.fa.gz", fa, gz=True)
    _write("norecords.fa", "no records here\njust text\n")
    _write("badfai.fa", fa)
    _write("badfai.fa.fai", "chrA\t200\nchrB\n")
    _write("nonewline.fa", ">chrA\nACGT\n>chrB desc")
    _write("notoken.fa", ">chrA\nACGT\n>  \t\n")


M = "main.geno"
CASES = [
    # (name, input ("-" = stdin), args, destination: "stdout" or an output file name)
    ("phased", M, ["-f", "phased"], "stdout"),
    ("phased_stdin", "-", ["-f", "phased"], "stdout"),
    ("phased_ref", M, ["-f", "phased", "-r", "ref.fa"], "out.vcf"),
    ("phased_ref_gz_in_out", "main.geno.gz", ["-f", "phased", "-r", "ref.fa.gz"], "out.vcf.gz"),
    ("phased_ref_gz_nofai", M, ["-f", "phased", "-r", "refnofai.fa.gz"], "stdout"),
    ("phased_norecords", M, ["-f", "phased", "-r", "norecords.fa"], "stdout"),
    ("samples_reorder_dup", M, ["-f", "phased", "-s", "s3,s0,s3,s7"], "out.vcf"),
    ("samples_ref", "main.geno.gz", ["-f", "phased", "-s", "s5,s1", "-r", "ref.fa"], "stdout"),
    ("pos_forms", "pos.geno", ["-f", "phased"], "stdout"),
    ("pos_forms_ref", "pos.geno", ["-f", "phased", "-r", "ref.fa"], "stdout"),
    ("crlf", "crlf.geno", ["-f", "phased", "-r", "ref.fa"], "stdout"),
    ("pairs", "pairs.geno", ["-f", "pairs"], "stdout"),
    ("pairs_ref", "pairs.geno", ["-f", "pairs", "-r", "ref.fa"], "out.vcf.gz"),
    ("diplo", "diplo.geno", ["-f", "diplo"], "stdout"),
    ("diplo_ref", "diplo.geno", ["-f", "diplo", "-r", "ref.fa"], "stdout"),
    ("diplo_unread_bad_column", "diplo_bad.geno", ["-f", "diplo", "-s", "d0,d2,d4"], "stdout"),
    ("header_only", "header_only.geno", ["-f", "phased", "-r", "ref.fa"], "stdout"),
    # the reference fails on these
    ("fail_no_format", M, [], "stdout"),
    ("fail_sample_not_in_header", M, ["-f", "phased", "-s", "s1,zz"], "stdout"),
    ("fail_missing_column", "short.geno", ["-f", "phased"], "stdout"),
    ("fail_no_names", "nonames.geno", ["-f", "phased"], "stdout"),
    ("fail_bad_diplo", "diplo_bad.geno", ["-f", "diplo"], "stdout"),
    ("fail_scaffold_not_in_fasta", "scafmiss.geno", ["-f", "phased", "-r", "ref.fa"], "stdout"),
    ("fail_position_outside_contig", "posrange.geno", ["-f", "phased", "-r", "ref.fa"], "stdout"),
    ("fail_blank_line", "blank.geno", ["-f", "phased"], "stdout"),
    ("fail_fai_short_line", M, ["-f", "phased", "-r", "badfai.fa"], "stdout"),
    ("fail_fasta_no_newline", M, ["-f", "phased", "-r", "nonewline.fa"], "stdout"),
    ("fail_fasta_no_token", M, ["-f", "phased", "-r", "notoken.fa"], "stdout"),
    ("fail_empty_input", "empty.geno", ["-f", "phased"], "stdout"),
]


def run_case(ref, case):
    name, inp, args, dest = case
    work = tempfile.mkdtemp()
    try:
        argv = [os.path.join(DIR, a) if k > 0 and args[k - 1] == "-r" else a for k, a in enumerate(args)]
        cmd = [sys.executable, os.path.join(ref, "VCF_processing", "genoToVCF.py")] + argv
        if inp != "-":
            cmd += ["-g", os.path.join(DIR, inp)]
        if dest != "stdout":
            cmd += ["-o", os.path.join(work, dest)]
        stdin = open(os.path.join(DIR, M), "rb") if inp == "-" else subprocess.DEVNULL
        r = subprocess.run(cmd, cwd=work, stdin=stdin, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                           env=dict(os.environ, PYTHONPATH=ref, NPY_DISABLE_CPU_FEATURES=NO_SIMD_SORT))
        entry = dict(name=name, input=inp, args=list(args), dest=dest)
        if r.returncode != 0:
            entry["fails"] = r.stderr.decode().strip().splitlines()[-1]
        if dest == "stdout":
            data = r.stdout
        else:
            data = open(os.path.join(work, dest), "rb").read()
            data = gzip.decompress(data) if dest.endswith(".gz") else data
        fix = name + ".vcf.gz"
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
    with open(os.path.join(GOLD, "cases11.json"), "w") as f:
        json.dump(cases, f, indent=1)
    for c in cases:
        print(c["name"], "FAILS " + c["fails"] if "fails" in c else "ok")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
