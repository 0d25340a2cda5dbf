#!/usr/bin/env python
"""TEST INFRASTRUCTURE — fixtures for windowStats.py from the UNMODIFIED reference script.

    python oracle/make_golden13.py [/path/to/genomics_general]

Writes seeded per-site tables under tests/golden/ws13/, runs the reference windowStats.py on each case of CASES and commits
its output (gzip) next to them, with tests/golden/cases13.json listing the cases (the larger tables are committed gzipped and
read as .gz by the tests; the reference reads them plain); a case the reference fails on records the
output it wrote first and "fails".  Under Python 3 and numpy 2 the script needs np.NaN, open(..., "rU") and
`print >> sys.stderr`, so each run goes through a shim that restores them and then runs the script as it is.  -o and .gz
input fail in the reference whatever the shim does; the tests check those against the stdout fixtures."""
import gzip
import json
import os
import random
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "..", "tests", "golden")
DIR = os.path.join(GOLD, "ws13")

SHIM = ("import builtins, runpy, sys\nimport numpy as np\nnp.NaN = np.nan\n"
        "_open = builtins.open\n"
        "def _o(f, mode='r', *a, **k):\n    return _open(f, 'r' if mode == 'rU' else mode, *a, **k)\n"
        "builtins.open = _o\n"
        "class _E:\n    def __init__(s, e): s.e = e\n    def __rrshift__(s, o): return s\n"
        "    def __getattr__(s, n): return getattr(s.e, n)\n"
        "sys.stderr = _E(sys.stderr)\n"
        "sys.path.insert(0, sys.argv[1])\nsys.argv = sys.argv[2:]\nrunpy.run_path(sys.argv[0], run_name='__main__')\n")


def _val(rng):
    k = rng.random()
    if k < 0.08:
        return "nan"
    if k < 0.1:
        return rng.choice(["inf", "-inf", "0.0", "-0.0" if False else "0", "1"])
    if k < 0.4:
        return repr(round(rng.gauss(0, 5), rng.randint(0, 4)))
    if k < 0.7:
        return repr(rng.random() * 10 ** rng.randint(-6, 8))
    return repr(rng.uniform(-1, 1))


def main_table(rng):
    lines = ["scaffold\tposition\ta\tb\tc\td"]
    for scaf, n, step in (("chr1", 700, 7), ("chr2", 260, 13), ("chr3", 45, 40)):
        p = rng.randint(1, 5)
        for i in range(n):
            p += rng.randint(1, step)
            if rng.random() < 0.02:
                lines.append("#comment %d" % i)
            d = _val(rng) if rng.random() < 0.05 else "nan"
            lines.append("\t".join([scaf, str(p), _val(rng), _val(rng), _val(rng), d]))
    return "\n".join(lines) + "\n"


FORMS = ["1_0", ".5", "1.", "+3", "nan", "-nan", "NaN", "Infinity", "-INFINITY", "inf", "1e400", "4.9e-325",
         "2.4703282292062328e-324", "1.7976931348623157e308", "0.1000000000000000055511151231257827",
         "9007199254740993", "9007199254740992.5000000000000000001", "1.00000000000000011102230246251565404236316680908203125",
         "1.000000000000000111022302462515654042363166809082031250001", "123456789012345678901234.5", "-0.0000000000000000000001",
         "2.2250738585072011e-308", "1e1_0", "5e-1", "12345678901234567", "0.30000000000000004"]


def forms_table(rng):
    lines = ["s\tp\tx\ty"]
    for i, f in enumerate(FORMS * 3):
        lines.append("c\t%d\t%s\t%s" % (i + 1, f, repr(rng.uniform(0, 1e-3))))
    return "\n".join(lines) + "\n"


def big_table(rng):
    lines = ["s\tp\tv\tw"]
    for i in range(10500):
        lines.append("big\t%d\t%r\t%s" % (i + 1, rng.gauss(100, 30), repr(rng.expovariate(1.0)) if i % 3 else "nan"))
    return "\n".join(lines) + "\n"


def bad_table(rng):
    lines = ["s\tp\tv"]
    for i in range(60):
        lines.append("a\t%d\t%r" % (i + 1, rng.random()))
    for i in range(5):
        lines.append("b\t%d\t%s" % (i + 1, "NA" if i == 2 else repr(rng.random())))
    for i in range(40):
        lines.append("c\t%d\t%r" % (i + 1, rng.random()))
    return "\n".join(lines) + "\n"


INPUTS = {
    "main.tsv": main_table,
    "forms.tsv": forms_table,
    "big.tsv": big_table,
    "bad.tsv": bad_table,
    "head_only.tsv": lambda rng: "s\tp\tv\n",
    "nohead.tsv": lambda rng: "".join("x\t%d\t%r\t%r\n" % (i + 1, rng.random(), rng.random()) for i in range(30)),
    "short_line.tsv": lambda rng: "s\tp\ta\tb\nc\t1\t1.0\t2.0\nc\t2\t3.0\nc\t3\t4.0\t5.0\n",
    "empty_col.tsv": lambda rng: "s\tp\ta\tb\nc\t1\t1.0\tnan\nc\t2\t3.0\tnan\nc\t30\t4.0\t5.0\n",
    "coords.txt": lambda rng: "chr1 1 500\nchr1 400 900\nchr1 2000 2600\nchr2 1 1000\nchr2 900 3000\nchr9 1 10\nchr3 1 99999\n",
    "exclude.txt": lambda rng: "chr2\n",
}

GZIPPED = ("main.tsv", "big.tsv", "bad.tsv")
ALL = ["--stats"] + ["mean", "median", "min", "max", "sd", "sum", "q5", "q10", "q25", "q75", "q90", "q95"]
CASES = [
    ("coord_default", "main.tsv", ["-w", "500", "--columns", "a", "b", "c"]),
    ("coord_step", "main.tsv", ["-w", "400", "-s", "150", "-m", "8", "--columns", "a", "b", "c"] + ALL),
    ("coord_minsites", "main.tsv", ["-w", "300", "-m", "40", "--stats", "mean", "q25", "max", "--columns", "a", "b", "c"]),
    ("sites", "main.tsv", ["--windType", "sites", "-w", "50", "-m", "10", "--columns", "a", "b", "c"] + ALL),
    ("sites_overlap", "main.tsv", ["--windType", "sites", "-w", "60", "-O", "25", "-m", "10", "--columns", "a", "b", "c", "--columns", "a", "b", "c"]),
    ("sites_maxdist", "main.tsv", ["--windType", "sites", "-w", "40", "-D", "150", "-m", "5", "--stats", "median", "sd"]),
    ("predefined", "main.tsv", ["--windType", "predefined", "--windCoords", "coords.txt", "--stats", "mean", "median", "sum"]),
    ("columns_subset", "main.tsv", ["-w", "1000", "--columns", "c", "a", "--stats", "max", "min", "mean"]),
    ("columns_dup", "main.tsv", ["-w", "1000", "--columns", "b", "b", "a", "--stats", "median", "median", "q95"]),
    ("mostly_nan", "main.tsv", ["-w", "2000", "--columns", "d", "--stats", "mean", "median", "sd", "sum", "q5", "q95"]),
    ("repeat_stats", "main.tsv", ["-w", "800", "--stats", "sum", "mean", "sum", "q10", "q90"]),
    ("sites_exclude", "main.tsv", ["--windType", "sites", "-w", "100", "-m", "20", "--exclude", "exclude.txt"]),
    ("forms", "forms.tsv", ["-w", "10"] + ALL),
    ("forms_sites", "forms.tsv", ["--windType", "sites", "-w", "7", "--columns", "x", "--stats", "mean", "sum", "sd"]),
    ("big_sites_7", "big.tsv", ["--windType", "sites", "-w", "7", "--columns", "v"] + ALL),
    ("big_sites_8", "big.tsv", ["--windType", "sites", "-w", "8", "--stats", "mean", "sum", "sd", "median"]),
    ("big_sites_9", "big.tsv", ["--windType", "sites", "-w", "9", "--stats", "mean", "sum", "sd", "median"]),
    ("big_sites_127", "big.tsv", ["--windType", "sites", "-w", "127", "-O", "2"] + ALL),
    ("big_sites_128", "big.tsv", ["--windType", "sites", "-w", "128", "--stats", "mean", "sum", "sd", "q75"]),
    ("big_sites_129", "big.tsv", ["--windType", "sites", "-w", "129", "--stats", "mean", "sum", "sd", "q75"]),
    ("big_sites_255", "big.tsv", ["--windType", "sites", "-w", "255", "--stats", "mean", "sum", "sd", "median"]),
    ("big_sites_256", "big.tsv", ["--windType", "sites", "-w", "256", "--stats", "mean", "sum", "sd", "median"]),
    ("big_sites_257", "big.tsv", ["--windType", "sites", "-w", "257", "-O", "100"] + ALL),
    ("big_coord_large", "big.tsv", ["-w", "11000", "-s", "3000"] + ALL),
    ("bad_not_evaluated", "bad.tsv", ["-w", "100", "-m", "10"]),
    ("failed_windows", "main.tsv", ["-w", "100", "-m", "30", "--stats", "mean", "q5"]),
    ("no_window", "head_only.tsv", ["-w", "100"]),
    ("headers", "nohead.tsv", ["-w", "10", "--headers", "s", "p", "u", "v"]),
    ("fail_bad_token", "bad.tsv", ["-w", "100"]),
    ("fail_empty_min", "empty_col.tsv", ["-w", "20", "--stats", "mean", "min"]),
    ("fail_short_line", "short_line.tsv", ["-w", "100"]),
    ("fail_columns_missing_on_line", "short_line.tsv", ["-w", "100", "--columns", "b"]),
    ("fail_column_not_in_header", "main.tsv", ["-w", "100", "--columns", "zz"]),
]


def run(ref, case):
    name, inp, args = case
    argv = [sys.executable, "-c", SHIM, ref, os.path.join(ref, "windowStats.py"), "-i", inp] + args
    r = subprocess.run(argv, cwd=DIR, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    with open(os.path.join(DIR, name + ".csv.gz"), "wb") as f:
        f.write(gzip.compress(r.stdout, mtime=0))
    c = dict(name=name, input=inp, args=args, output=name + ".csv.gz")
    if r.returncode != 0:
        c["fails"] = r.stderr.decode().strip().split("\n")[-1]
    return c


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
    os.makedirs(DIR, exist_ok=True)
    rng = random.Random(13)
    for fn, make in INPUTS.items():
        with open(os.path.join(DIR, fn), "w") as f:
            f.write(make(rng))
    with ThreadPoolExecutor(8) as ex:
        cases = list(ex.map(lambda c: run(ref, c), CASES))
    for fn in GZIPPED:
        path = os.path.join(DIR, fn)
        with open(path, "rb") as f, open(path + ".gz", "wb") as g:
            g.write(gzip.compress(f.read(), mtime=0))
        os.remove(path)
    for c in cases:
        if c["input"] in GZIPPED:
            c["input"] += ".gz"
    with open(os.path.join(GOLD, "cases13.json"), "w") as f:
        f.write("[\n" + ",\n".join(json.dumps(c) for c in cases) + "\n]\n")
    for c in cases:
        print(c["name"], c.get("fails", "ok"))


if __name__ == "__main__":
    main()
