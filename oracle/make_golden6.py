#!/usr/bin/env python
"""TEST INFRASTRUCTURE — fixtures for filterGenotypes.py from the UNMODIFIED reference script.

    python oracle/make_golden6.py [/path/to/genomics_general]

Writes three seeded inputs (phased with '|' and '/' mixed, diplo, alleles; haploid, diploid and triploid samples; partly
and fully missing genotypes; multi-allelic sites; two scaffolds; positions with leading zeros) under tests/golden/filter6/,
runs the reference filterGenotypes.py on each case of CASES and commits its output next to them, with tests/golden/
cases6.json listing the cases.  The inputs hold no site with four alleles: on an exact tie of allele counts the reference's
frequency order is whatever numpy's sort gives, which for four alleles is not the stable order the engine uses
(pg_filter_stats flag 1 marks such sites).  Every reference run sleeps about 11 s at exit; the cases run in parallel."""
import gzip
import json
import os
import random
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "..", "tests", "golden")
DIR = os.path.join(GOLD, "filter6")

PLOIDY_A = [1, 2, 2, 2, 2, 3, 2, 1]


def _alleles(rng):
    """two or three alleles for a site"""
    k = 3 if rng.random() < 0.2 else 2
    return rng.sample("ACGT", k)


def _pos_field(rng, p):
    return ("00" + str(p)) if rng.random() < 0.1 else str(p)


def make_phased(rng, n=220):
    rows = []
    pos = 0
    for i in range(n):
        scaf = "scaf1" if i < 130 else "scaf2"
        pos = pos + rng.randint(1, 9) if i != 130 else rng.randint(1, 9)
        al = _alleles(rng)
        w = [0.7] + [0.3 / (len(al) - 1)] * (len(al) - 1)
        toks = []
        for pl in PLOIDY_A:
            a = rng.choices(al, w, k=pl)
            r = rng.random()
            if r < 0.06:
                a = ["N"] * pl
            elif r < 0.12 and pl > 1:
                a[rng.randrange(pl)] = "N"
            if rng.random() < 0.05:          # an invariant-looking site now and then
                a = [al[0]] * pl
            sep = "|" if rng.random() < 0.6 else "/"
            toks.append(sep.join(a))
        rows.append("\t".join([scaf, _pos_field(rng, pos)] + toks))
    return "\t".join(["#CHROM", "POS"] + ["s%d" % (k + 1) for k in range(len(PLOIDY_A))]) + "\n" + "\n".join(rows) + "\n"


def make_diplo(rng, n=120):
    pair = {"AA": "A", "CC": "C", "GG": "G", "TT": "T", "AC": "M", "AG": "R", "AT": "W", "CG": "S", "CT": "Y", "GT": "K"}
    rows = []
    for i in range(n):
        scaf = "chrA" if i < 70 else "chrB"
        al = _alleles(rng)
        toks = []
        for _ in range(6):
            if rng.random() < 0.08:
                toks.append("N")
                continue
            a = sorted(rng.choices(al, [0.6] + [0.4 / (len(al) - 1)] * (len(al) - 1), k=2))
            toks.append(pair["".join(a)])
        rows.append("\t".join([scaf, _pos_field(rng, 10 * (i + 1))] + toks))
    return "\t".join(["scaffold", "position"] + ["d%d" % (k + 1) for k in range(6)]) + "\n" + "\n".join(rows) + "\n"


def make_alleles(rng, n=120):
    ploidy = [2, 2, 3, 1, 2]
    rows = []
    for i in range(n):
        scaf = "c1" if i < 50 else "c2"
        al = _alleles(rng)
        toks = []
        for pl in ploidy:
            a = rng.choices(al, [0.65] + [0.35 / (len(al) - 1)] * (len(al) - 1), k=pl)
            if rng.random() < 0.08:
                a[0] = "N"
            toks.append("".join(a))
        rows.append("\t".join([scaf, _pos_field(rng, 3 * (i + 1))] + toks))
    return "\t".join(["scaffold", "position"] + ["a%d" % (k + 1) for k in range(len(ploidy))]) + "\n" + "\n".join(rows) + "\n"


POPS = ["-p", "P1", "s1,s2,s3", "-p", "P2", "s4,s5,s6", "-p", "P3", "s7,s8"]

CASES = [
    ("phased_default", "phased.geno", []),
    ("diplo_out", "phased.geno", ["-s", "s2,s3,s4,s5", "-of", "diplo", "--partialToMissing", "--minCalls", "2"]),
    ("coded_biallelic", "phased.geno", ["-of", "coded", "--minAlleles", "2", "--maxAlleles", "2"]),
    ("count_out", "phased.geno", ["-of", "count", "--minCalls", "3"]),
    ("bases_freq", "phased.geno", ["-of", "bases", "--ploidy"] + [str(p) for p in PLOIDY_A] + ["--alleleOrder", "freq"]),
    ("alleles_tuple_varcount_het", "phased.geno", ["-of", "alleles", "--minVarCount", "2", "--maxHet", "0.5"]),
    ("alleles_freq_minmaxfreq", "phased.geno", ["-of", "alleles", "--alleleOrder", "freq", "--minFreq", "0.1",
                                                "--maxFreq", "0.4"]),
    ("pops_calls_alleles", "phased.geno", POPS + ["--minPopCalls", "1", "2", "1", "--minPopAlleles", "1",
                                                  "--maxPopAlleles", "2"]),
    ("pops_fixed_keepall", "phased.geno", POPS + ["--fixedDiffs", "--keepAllSamples", "--minCalls", "0"]),
    ("pops_nearly_fixed_gz", "phased.geno", POPS + ["--nearlyFixedDiff", "0.5", "--excludeSamples", "s8"]),
    ("include_thin_pods", "phased.geno", ["--include", "scaf1", "scaf2", "--thinDist", "20", "--podSize", "37"]),
    ("exclude_thin_notest", "phased.geno", ["--exclude", "scaf2", "--thinDist", "15", "--podSize", "23", "--noTest"]),
    ("mincalls0_maxhet_p2m", "phased.geno", ["--minCalls", "0", "--maxHet", "0.3", "--partialToMissing"]),
    ("pops_overlap_keepall", "phased.geno", ["-p", "all", "s1,s2,s3,s4,s5,s6,s7,s8", "-p", "P1", "s1,s2", "-p", "P2",
                                             "s2,s6,s7", "--keepAllSamples", "--minPopCalls", "7", "1", "2",
                                             "--minPopAlleles", "1", "--maxPopAlleles", "2"]),
    ("diplo_in", "diplo.geno", ["-if", "diplo", "--minCalls", "2", "--excludeSamples", "d3", "-s", "d1,d2,d3,d4,d6"]),
    ("alleles_in_coded", "alleles.geno", ["-if", "alleles", "-of", "coded", "--maxHet", "0.6", "--minAlleles", "2"]),
]


def run(ref, name, infile, extra):
    out = os.path.join(DIR, name + (".out.gz" if name.endswith("_gz") else ".out"))
    cmd = [sys.executable, os.path.join(ref, "filterGenotypes.py"), "-i", os.path.join(DIR, infile), "-o", out] + extra
    subprocess.run(cmd, check=True, cwd=ref, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    if out.endswith(".gz"):
        with gzip.open(out, "rb") as f:
            data = f.read()
        os.remove(out)
        out = out[:-3]
        with open(out, "wb") as f:
            f.write(data)
    return dict(name=name, input=infile, args=extra, expected=os.path.basename(out), gz=name.endswith("_gz"))


def main(ref="/root/reference"):
    os.makedirs(DIR, exist_ok=True)
    rng = random.Random(20261016)
    for fname, text in (("phased.geno", make_phased(rng)), ("diplo.geno", make_diplo(rng)),
                        ("alleles.geno", make_alleles(rng))):
        with open(os.path.join(DIR, fname), "wt") as f:
            f.write(text)
    with ThreadPoolExecutor(8) as ex:
        cases = list(ex.map(lambda c: run(ref, *c), CASES))
    with open(os.path.join(GOLD, "cases6.json"), "wt") as f:
        json.dump(cases, f, indent=1)
    print("wrote %d filterGenotypes cases under %s" % (len(cases), DIR))


if __name__ == "__main__":
    main(*sys.argv[1:])
