#!/usr/bin/env python
"""TEST INFRASTRUCTURE — distPaint.py fixtures at large populations, from the UNMODIFIED reference script.

    python oracle/make_golden8.py [/path/to/genomics_general]

Writes a seeded haploid input under tests/golden/paint8/, runs the reference distPaint.py on each case of CASES (through
make_golden7's np.NaN shim) and commits its output next to it, with tests/golden/cases8.json listing the cases.  The data:
reference populations of 9, 130 and 300 samples (a, b, c) whose allele frequencies differ per site, and twelve query
samples (q) that copy one of the three or a fourth, unsampled population in stretches of about 40 sites; 5 % missing
genotypes; windows of about 40 sites.  So every member list runs numpy's pairwise summation past 8, 128 and its split, and
every rank-sum test counts ranks over more than one warp of members.  The reference makes one Python pairDist call per
(sample, member) pair: each case runs with -T 4 and a timeout, since the reference hangs rather than exits when a worker
dies."""
import json
import os
import random
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

from make_golden7 import SHIM, _write

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "..", "tests", "golden")
DIR = os.path.join(GOLD, "paint8")

SIZES = {"a": 9, "b": 130, "c": 300}
REFS = {p: ["%s%03d" % (p, k + 1) for k in range(n)] for p, n in SIZES.items()}
QUERIES = ["q%02d" % (k + 1) for k in range(12)]
FREQS = (0.03, 0.3, 0.7, 0.97)


def _sites(rng, n_sites=330):
    """(scaffold, position, {sample: base}) rows; sources: 0..2 = a..c, 3 = the unsampled population"""
    rows = []
    src = {}
    for s in range(n_sites):
        if s % 40 == 0:
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
        rows.append(("chr1", 10 * s + rng.randint(1, 9), calls))
    return rows


def _pops():
    args = []
    for p, names in REFS.items():
        args += ["-p", p.upper(), ",".join(names)]
    return args


CASES = [
    ("rank_large", ["-w", "400"] + _pops()),
    ("delta_large", ["-w", "400", "--delta_threshold", "0.01"] + _pops()),
    ("minsites_large", ["-w", "400", "-m", "36", "--writeFailedWindows"] + _pops()),
]


def run(ref, shim, name, extra):
    out = os.path.join(DIR, name + ".tsv")
    cmd = [sys.executable, shim, ref, os.path.join(ref, "distPaint.py"), "-g", os.path.join(DIR, "large.geno"), "-o", out,
           "-T", "4"] + extra
    subprocess.run(cmd, check=True, cwd=ref, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL, timeout=1200)
    return dict(name=name, input="large.geno", args=extra, expected=os.path.basename(out), gz=False)


def main(ref="/root/reference"):
    import tempfile
    os.makedirs(DIR, exist_ok=True)
    rng = random.Random(20261018)
    names = REFS["a"] + REFS["b"] + REFS["c"] + QUERIES
    _write(os.path.join(DIR, "large.geno"), _sites(rng), names, names)
    with tempfile.TemporaryDirectory() as td:
        shim = os.path.join(td, "shim.py")
        with open(shim, "wt") as f:
            f.write(SHIM)
        with ThreadPoolExecutor(len(CASES)) as ex:
            done = list(ex.map(lambda c: run(ref, shim, *c), CASES))
    with open(os.path.join(GOLD, "cases8.json"), "wt") as f:
        json.dump(done, f, indent=1)
    print("wrote %d distPaint cases under %s" % (len(done), DIR))


if __name__ == "__main__":
    main(*sys.argv[1:])
