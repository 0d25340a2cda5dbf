#!/usr/bin/env python
"""Times windowStats.py on the GPU: a seeded table of N lines x 4 value columns (5 % nan) through the command line with
--timing (phases and per-kernel device milliseconds), and the unmodified reference (staged under oracle/_ref/ by
oracle/build_ref_ws.py) on the first REF_LINES lines of the same file.  Prints one JSON object with the card's name and power
limit; writes nothing into the tree (the table and outputs go to a temporary directory).

    python tools/ws_timing.py [N] [REF_LINES]
"""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..")
REF = os.path.join(ROOT, "oracle", "_ref")
SHIM = ("import builtins, runpy, sys\nimport numpy as np\nnp.NaN = np.nan\n"
        "sys.path.insert(0, sys.argv[1])\nsys.argv = sys.argv[2:]\nrunpy.run_path(sys.argv[0], run_name='__main__')\n")


def table(path, n, seed=3):
    rng = np.random.default_rng(seed)
    pos = np.cumsum(rng.integers(1, 20, n))
    M = rng.normal(0, 3, (n, 4))
    M[rng.random((n, 4)) < 0.05] = np.nan
    with open(path, "w") as f:
        f.write("scaffold\tposition\ta\tb\tc\td\n")
        step = 1 << 20
        for a in range(0, n, step):
            f.write("".join("chr1\t%d\t%r\t%r\t%r\t%r\n" % (p, *map(float, r)) for p, r in zip(pos[a:a + step], M[a:a + step])))


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
    ref_lines = int(sys.argv[2]) if len(sys.argv) > 2 else 200_000
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    args = ["-w", "50000", "--stats", "mean", "median", "min", "max", "sd", "sum", "q5", "q95"]
    res = dict(gpu=gpu, lines=n, args=args)
    with tempfile.TemporaryDirectory() as tmp:
        inp = os.path.join(tmp, "t.tsv")
        table(inp, n)
        res["input_bytes"] = os.path.getsize(inp)
        tj = os.path.join(tmp, "timing.json")
        cmd = [sys.executable, "-m", "genomics_general_b200.cli.windowStats", "-i", inp, "-o", os.path.join(tmp, "o.csv"),
               "--timing", tj] + args
        for _ in range(2):                                   # the first run loads the module and warms the caches
            t0 = time.perf_counter()
            subprocess.run(cmd, cwd=ROOT, check=True, stderr=subprocess.DEVNULL)
            res["wall_s"] = time.perf_counter() - t0
        res["timing"] = json.load(open(tj))
        res["lines_per_s"] = n / res["wall_s"]
        if os.path.exists(os.path.join(REF, "windowStats.py")):
            head = os.path.join(tmp, "head.tsv")
            with open(inp) as f, open(head, "w") as g:
                for k, line in enumerate(f):
                    if k > ref_lines:
                        break
                    g.write(line)
            t0 = time.perf_counter()
            r = subprocess.run([sys.executable, "-c", SHIM, REF, os.path.join(REF, "windowStats.py"), "-i", head] + args,
                               stdout=open(os.path.join(tmp, "ref.csv"), "w"), stderr=subprocess.PIPE, text=True)
            t = time.perf_counter() - t0
            res["reference"] = (dict(lines=ref_lines, wall_s=t, lines_per_s=ref_lines / t) if r.returncode == 0 else
                                dict(failed=r.stderr.strip().split("\n")[-1]))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
