#!/usr/bin/env python
"""TEST INFRASTRUCTURE — fixtures for mergeGeno.py from the UNMODIFIED reference script.

    python oracle/make_golden14.py [/path/to/genomics_general]

Writes seeded .geno inputs and .fai files under tests/golden/merge14/, runs the reference mergeGeno.py on each case of CASES
and commits its output (gzip) next to them, with tests/golden/cases14.json listing the cases.  A case the reference fails on
records "fails" (the reference's exception) instead of an output.  The medium inputs (4 files x 20 000 lines over a
3-scaffold, 100 kb .fai) are committed gzipped; the reference reads them as .gz."""
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
DIR = os.path.join(GOLD, "merge14")
BASES = "ACGTN"


def gt(rng):
    return rng.choice(BASES) + "/" + rng.choice(BASES)


def body(rng, scafs, frac, n_samp, sep="\t"):
    out = []
    for name, n in scafs:
        for p in range(1, n + 1):
            if rng.random() < frac:
                out.append(sep.join([name, str(p)] + [gt(rng) for _ in range(n_samp)]))
    return out


def header(n_samp, tag, sep="\t"):
    return sep.join(["#CHROM", "POS"] + ["%s%d" % (tag, k) for k in range(n_samp)])


def gz_write(path, data):
    with open(path, "wb") as f:
        f.write(gzip.compress(data, mtime=0))


def write(name, lines, end="\n", final=True, gz=False):
    data = end.join(lines) + (end if final and lines else "")
    path = os.path.join(DIR, name)
    if gz:
        gz_write(path, data.encode())
    else:
        with open(path, "wb") as f:
            f.write(data.encode())


def make_inputs():
    rng = random.Random(14)
    os.makedirs(DIR, exist_ok=True)
    small = [("chr1", 60), ("chr2", 45)]
    with open(os.path.join(DIR, "main.fai"), "w") as f:      # extra columns, lengths 0 and negative, an uncovered scaffold
        f.write("chr1\t60\t6\t60\t61\nchr2\t45\t75\t45\t46\nchrZero\t0\t130\t60\t61\nchrNeg\t-5\t140\t60\t61\n"
                "chr5\t30\t150\t30\t31\n")
    with open(os.path.join(DIR, "short.fai"), "w") as f:
        f.write("chr1\t60\nchr2\n")
    with open(os.path.join(DIR, "badint.fai"), "w") as f:
        f.write("chr1\t60\nchr2\tabc\n")
    write("a.geno", [header(3, "a")] + body(rng, small, 0.6, 3))
    gz_write(os.path.join(DIR, "a.geno.gz"), open(os.path.join(DIR, "a.geno"), "rb").read())
    # b: two samples, mixed runs of spaces and tabs, lines with more or fewer genotypes than the header
    bl = []
    for ln in body(rng, small, 0.5, 2):
        t = ln.split("\t")
        k = rng.random()
        if k < 0.1:
            t = t + [gt(rng)]
        elif k < 0.2:
            t = t[:3]
        elif k < 0.25:
            t = t[:2]
        seps = [rng.choice(["\t", " ", "  ", "\t ", " \t\t"]) if rng.random() < 0.3 else "\t" for _ in t]
        bl.append("".join(x + s for x, s in zip(t, seps[:-1] + [""])) + (" " if rng.random() < 0.1 else ""))
    write("b.geno", [header(2, "b")] + bl)
    write("c.geno", ["#CHROM POS"] + [ln for ln in body(rng, small, 0.4, 0)])        # no sample columns
    write("d.geno", [header(4, "d")] + body(rng, small, 0.7, 4), final=False)       # no final newline
    write("crlf.geno", [header(2, "r")] + body(rng, small, 0.5, 2), end="\r\n")
    write("empty.geno", [])
    write("headonly.geno", [header(2, "h")])
    # one file per stall kind: the line after the first few is the stall
    base = [header(2, "s")] + body(rng, [("chr1", 20)], 0.7, 2)
    stalls = {"order": "chr1\t5\tA/A\tC/C", "dup": None, "blank": "", "hash": "#chr1\t40\tA/A\tA/A",
              "scaf_missing": "chrX\t3\tA/A\tA/A", "scaf_order": "chr5\t3\tA/A\tA/A", "beyond": "chr1\t61\tA/A\tA/A",
              "zero": "chr1\t0\tA/A\tA/A", "lead0": "chr1\t041\tA/A\tA/A", "plus": "chr1\t+41\tA/A\tA/A",
              "space_only": "  \t ", "one_field": "chr1"}
    tail = ["chr1\t50\tG/G\tT/T", "chr2\t3\tG/G\tT/T", "chr5\t10\tG/G\tT/T"]
    for k, v in stalls.items():
        mid = [base[-1]] if v is None else [v]
        write("stall_%s.geno" % k, base + mid + tail)
    write("stall_first.geno", [header(2, "s"), "chr2\t1\tA/A\tA/A", "chr1\t5\tA/A\tA/A", "chr1\t6\tA/A\tA/A"])
    write("stall_last.geno", [header(2, "s")] + body(rng, [("chr1", 20)], 0.7, 2) + ["chr1\t3\tA/A\tA/A"])
    write("scaf_order_ok.geno", [header(2, "o"), "chr1\t60\tA/A\tA/A", "chr2\t1\tC/C\tC/C", "chr5\t30\tG/G\tG/G"])
    # medium: 4 files x 20 000 lines over 3 scaffolds of 100 kb in all
    med = [("m1", 50000), ("m2", 30000), ("m3", 20000)]
    with open(os.path.join(DIR, "med.fai"), "w") as f:
        for n, l in med:
            f.write("%s\t%d\n" % (n, l))
    for x in range(4):
        write("med%d.geno.gz" % x, [header(3 + x, "m%d_" % x)] + body(rng, med, 0.2, 3 + x), gz=True)


def cases():
    c = []

    def add(name, files, fai="main.fai", extra=(), dest="stdout", fails=False):
        args = sum((["-i", f] for f in files), []) + ["-f", fai] + list(extra)
        c.append(dict(name=name, args=args, dest=dest, fails=fails))

    abc = ["a.geno", "b.geno", "c.geno"]
    for m in ("intersect", "union", "all"):
        add("method_" + m, abc, extra=["--method", m])
    for u in ("0", "1", "2", "5"):
        add("union_min_" + u, abc, extra=["--method", "union", "--unionMin", u])
    for n in range(0, 5):
        add("must_first_%d_union" % n, abc, extra=["--method", "union", "--mustIncludeFirst", str(n)])
        add("must_first_%d_all" % n, abc, extra=["--method", "all", "--mustIncludeFirst", str(n)])
        add("must_first_%d_intersect" % n, ["a.geno", "d.geno"], extra=["--mustIncludeFirst", str(n)])
    add("must_first_neg_union_min_neg", abc, extra=["--method", "union", "--unionMin", "-1", "--mustIncludeFirst", "-2"])
    add("output_only_subset", abc, extra=["--method", "union", "--outputOnly", "1", "3"])
    add("output_only_reordered", abc, extra=["--method", "union", "--outputOnly", "3", "1"])
    add("output_only_dup", abc, extra=["--method", "all", "--outputOnly", "2", "2", "1"])
    add("output_only_zero", abc, extra=["--method", "union", "--outputOnly", "0"])
    add("output_only_negative", abc, extra=["--method", "union", "--outputOnly", "-1"])
    add("sep_comma", abc, extra=["--method", "union", "--outSep", ","])
    add("sep_space", abc, extra=["--method", "union", "--outSep", " "])
    add("sep_literal_tab", abc, extra=["--method", "all", "--outSep", "\\t"])
    add("missing_empty", abc, extra=["--method", "union", "--missing", ""])
    add("missing_nn", abc, extra=["--method", "all", "--missing", "N/N"])
    for k in ("order", "dup", "blank", "hash", "scaf_missing", "scaf_order", "beyond", "zero", "lead0", "plus",
              "space_only", "one_field", "first", "last"):
        add("stall_" + k, ["a.geno", "stall_%s.geno" % k], extra=["--method", "union"])
    add("scaf_order_ok", ["scaf_order_ok.geno", "a.geno"], extra=["--method", "union"])
    add("no_final_newline", ["d.geno", "a.geno"], extra=["--method", "union"])
    add("crlf", ["crlf.geno", "a.geno"], extra=["--method", "union"])
    add("empty_file", ["empty.geno", "a.geno"], extra=["--method", "union"])
    add("empty_only", ["empty.geno"], extra=["--method", "all"])
    add("header_only", ["a.geno", "headonly.geno"], extra=["--method", "all"])
    add("same_file_twice", ["a.geno", "a.geno"])
    add("one_file_all", ["b.geno"], extra=["--method", "all"])
    add("gz_in_out", ["a.geno.gz", "b.geno"], extra=["--method", "union"], dest="out.geno.gz")
    add("file_out", ["a.geno", "b.geno"], extra=["--method", "union"], dest="out.geno")
    med = ["med%d.geno.gz" % x for x in range(4)]
    for m in ("intersect", "union", "all"):
        add("medium_" + m, med, fai="med.fai", extra=["--method", m])
    add("medium_union2_first", med, fai="med.fai", extra=["--method", "union", "--unionMin", "2", "--mustIncludeFirst", "1"])
    add("fail_fai_short_line", abc, fai="short.fai", fails=True)
    add("fail_fai_bad_length", abc, fai="badint.fai", fails=True)
    add("fail_output_only_range", ["a.geno", "b.geno"], extra=["--outputOnly", "3"], fails=True)
    add("fail_missing_input", ["a.geno", "nosuch.geno"], fails=True)
    return c


def run(ref, case):
    work = tempfile.mkdtemp()
    try:
        args = []
        for k, a in enumerate(case["args"]):
            args.append(os.path.join(DIR, a) if k > 0 and case["args"][k - 1] in ("-i", "-f") else a)
        if case["dest"] != "stdout":
            args += ["-o", case["dest"]]
        r = subprocess.run([sys.executable, os.path.join(ref, "mergeGeno.py")] + args, cwd=work, stdout=subprocess.PIPE,
                           stderr=subprocess.PIPE)
        if case["fails"]:
            assert r.returncode != 0, case["name"]
            return None, r.stderr.decode().strip().splitlines()[-1].split(":")[0]
        assert r.returncode == 0, (case["name"], r.stderr.decode())
        if case["dest"] == "stdout":
            return r.stdout, None
        data = open(os.path.join(work, case["dest"]), "rb").read()
        return (gzip.decompress(data) if case["dest"].endswith(".gz") else data), None
    finally:
        shutil.rmtree(work)


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
    make_inputs()
    out = []
    for case in cases():
        data, err = run(ref, case)
        entry = dict(name=case["name"], args=case["args"], dest=case["dest"])
        if err is not None:
            entry["fails"] = err
        else:
            entry["output"] = case["name"] + ".out.gz"
            gz_write(os.path.join(DIR, entry["output"]), data)
        out.append(entry)
    with open(os.path.join(GOLD, "cases14.json"), "w") as f:
        json.dump(out, f, indent=1)
    print("%d cases under %s" % (len(out), DIR))


if __name__ == "__main__":
    main()
