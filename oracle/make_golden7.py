#!/usr/bin/env python
"""TEST INFRASTRUCTURE — fixtures for distPaint.py from the UNMODIFIED reference script.

    python oracle/make_golden7.py [/path/to/genomics_general]

Writes seeded haploid inputs under tests/golden/paint7/, runs the reference distPaint.py on each case of CASES and commits
its output next to them, with tests/golden/cases7.json listing the cases.  The data: three reference populations of seven
samples (a, b, c) whose allele frequencies differ per site, so that rank-sum tests can reach p < 0.05, and six query
samples (q) that copy one of the three or a fourth, unsampled population in stretches of about 60 sites; two scaffolds,
the second starting at position 2500 (empty coordinate windows before it); 5 % missing genotypes.  Under numpy 2 the
reference's failed-window rows need `np.NaN`, so each run goes through a shim that sets it and then runs the script as it
is.  The reference's worker processes are forked; the cases run in parallel."""
import gzip
import json
import os
import random
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "..", "tests", "golden")
DIR = os.path.join(GOLD, "paint7")

SHIM = ("import runpy, sys\nimport numpy as np\nnp.NaN = np.nan\nsys.path.insert(0, sys.argv[1])\n"
        "sys.argv = sys.argv[2:]\nrunpy.run_path(sys.argv[0], run_name='__main__')\n")

REFS = {p: ["%s%02d" % (p, k + 1) for k in range(7)] for p in "abc"}
QUERIES = ["q%02d" % (k + 1) for k in range(6)]
FREQS = (0.03, 0.3, 0.7, 0.97)


def _sites(rng, n_sites=900):
    """(scaffold, position, {sample: base}) rows; sources: 0..2 = a..c, 3 = the unsampled population"""
    rows = []
    src = {q: rng.randrange(4) for q in QUERIES}
    for s in range(n_sites):
        scaf, pos = ("chr1", 10 * s + rng.randint(1, 9)) if s < 500 else ("chr2", 2500 + 10 * (s - 500) + rng.randint(1, 9))
        if s % 60 == 0:
            src = {q: rng.randrange(4) for q in QUERIES}
        ref, alt = rng.sample("ACGT", 2)
        f = [rng.choice(FREQS) for _ in range(4)]
        calls = {}
        for p, names in REFS.items():
            for n in names:
                calls[n] = alt if rng.random() < f["abc".index(p)] else ref
        for q in QUERIES:
            calls[q] = alt if rng.random() < f[src[q]] else ref
        for n in calls:
            if rng.random() < 0.05:
                calls[n] = "N"
        rows.append((scaf, pos, calls))
    return rows


def _write(path, rows, header_names, columns, iupac=0.0, rng=None):
    lines = ["\t".join(["#CHROM", "POS"] + header_names)]
    for scaf, pos, calls in rows:
        toks = [calls[c] for c in columns]
        if iupac:
            toks = [rng.choice("KMRSWY") if rng.random() < iupac else t for t in toks]
        lines.append("\t".join([scaf, str(pos)] + toks))
    text = "\n".join(lines) + "\n"
    if path.endswith(".gz"):
        with gzip.open(path, "wt") as f:
            f.write(text)
    else:
        with open(path, "wt") as f:
            f.write(text)


def make_inputs(rng):
    rows = _sites(rng)
    names = REFS["a"] + REFS["b"] + REFS["c"] + QUERIES
    _write(os.path.join(DIR, "sorted.geno"), rows, names, names)
    _write(os.path.join(DIR, "sorted.geno.gz"), rows, names, names)
    _write(os.path.join(DIR, "iupac.geno"), rows, names, names, iupac=0.04, rng=rng)
    # the same columns under names whose sorted order is not the header order: s10 before s1, members interleaved
    perm = list(range(len(names)))
    rng.shuffle(perm)
    cols = [names[k] for k in perm]
    _write(os.path.join(DIR, "unsorted.geno"), rows, ["s%d" % (k + 1) for k in range(len(names))], cols)
    renamed = {c: "s%d" % (k + 1) for k, c in enumerate(cols)}
    # ties: every b sample's column is a copy of the matching a sample's, so populations a and b have the same means;
    # z01 is missing everywhere
    trows = []
    for scaf, pos, calls in rows:
        c = dict(calls)
        for a, b in zip(REFS["a"], REFS["b"]):
            c[b] = c[a]
        c["z01"] = "N"
        trows.append((scaf, pos, c))
    _write(os.path.join(DIR, "ties.geno"), trows, names + ["z01"], names + ["z01"])
    with open(os.path.join(DIR, "pops.txt"), "wt") as f:
        f.write("a05 A\nb02 B\nc01 C\nnobody B\nq01 X\nb07 A\n")
    with open(os.path.join(DIR, "windows.txt"), "wt") as f:
        f.write("chr1 1 1500\nchr1 1200 4000\nchr2 2600 5000\nchr2 100 900\n")
    return renamed


def _pops(renamed=None):
    args = []
    for p, names in REFS.items():
        args += ["-p", p.upper(), ",".join(renamed[n] for n in names) if renamed else ",".join(names)]
    return args


def cases(renamed):
    # unsorted header: members listed in a non-sorted, interleaved order
    inter = ["-p", "A", ",".join(renamed[n] for n in REFS["a"][::-1]), "-p", "B",
             ",".join(renamed[n] for n in (REFS["b"][1::2] + REFS["b"][0::2])), "-p", "C", ",".join(renamed[n] for n in REFS["c"])]
    return [
        ("rank_sorted", "sorted.geno", ["-w", "1000"] + _pops()),
        ("rank_unsorted", "unsorted.geno", ["-w", "1000"] + inter),
        ("delta_failed_windows", "sorted.geno", ["-w", "800", "-m", "70", "--delta_threshold", "0.02",
                                                 "--writeFailedWindows"] + _pops()),
        ("sites_overlap_id", "sorted.geno", ["--windType", "sites", "-w", "70", "-O", "20", "--addWindowID"] + _pops()),
        ("predefined", "sorted.geno", ["--windType", "predefined", "--windCoords", "windows.txt", "--addWindowID"] + _pops()),
        ("popsfile_inline", "sorted.geno", ["-w", "1000", "--popsFile", "pops.txt", "--noresult", "9",
                                            "-p", "A", "a01,a02,a03,a04,a02", "extra", "words",
                                            "-p", "B", "b01,b03,b04,b05,b06,a01",
                                            "-p", "C", "c02,c03",
                                            "-p", "C", "c04,c05,c06,c07",
                                            "-p", "X", "q02"]),
        ("ties_all_missing", "ties.geno", ["-w", "1000"] + _pops()),
        ("iupac", "iupac.geno", ["-w", "1000"] + _pops()),
        ("p_threshold", "sorted.geno", ["-w", "1000", "--p_threshold", "0.2"] + _pops()),
        ("gzip_in_out", "sorted.geno.gz", ["-w", "1000", "-m", "50"] + _pops()),
    ]


def run(ref, shim, name, infile, extra):
    gz = name.endswith("_out")
    out = os.path.join(DIR, name + (".tsv.gz" if gz else ".tsv"))
    cmd = [sys.executable, shim, ref, os.path.join(ref, "distPaint.py"), "-g", os.path.join(DIR, infile), "-o", out] + \
        [os.path.join(DIR, a) if a in ("windows.txt", "pops.txt") else a for a in extra]
    subprocess.run(cmd, check=True, cwd=ref, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL, timeout=600)
    if gz:
        with gzip.open(out, "rb") as f:
            data = f.read()
        os.remove(out)
        out = out[:-3]
        with open(out, "wb") as f:
            f.write(data)
    return dict(name=name, input=infile, args=extra, expected=os.path.basename(out), gz=gz)


def main(ref="/root/reference"):
    import tempfile
    os.makedirs(DIR, exist_ok=True)
    rng = random.Random(20261017)
    renamed = make_inputs(rng)
    with tempfile.TemporaryDirectory() as td:
        shim = os.path.join(td, "shim.py")
        with open(shim, "wt") as f:
            f.write(SHIM)
        with ThreadPoolExecutor(8) as ex:
            done = list(ex.map(lambda c: run(ref, shim, *c), cases(renamed)))
    with open(os.path.join(GOLD, "cases7.json"), "wt") as f:
        json.dump(done, f, indent=1)
    print("wrote %d distPaint cases under %s" % (len(done), DIR))


if __name__ == "__main__":
    main(*sys.argv[1:])
