#!/usr/bin/env python
"""seqToGeno.py timing on one GPU: a seeded FASTA of --seqs sequences x --sites sites (60-base lines; 100 x 10 M is about
1 GB) is written to a temporary directory, then

  * the command line converts it plain, from a .gz copy, to .gz output and with -M contigs; --timing gives the kernels'
    CUDA-event times (the FASTA's upload, '>' marks, sequence flags and select; the transpose per slab) and the wall time of
    each phase, and every kernel's bytes moved are set against the 3.35 TB/s data-sheet bound of the H100 SXM;
  * the unmodified reference (oracle/_ref/seqToGeno.py, staged by build()) converts the first --ref-sites sites of every
    sequence, and its output is compared with the command line's on the same input.

    python tools/s2g_timing.py [--seqs 100] [--sites 10000000] [--ref-sites 200000] [--out results.json]

The card's name and power limit are read in the same run and written with the numbers."""
import argparse
import gzip
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
PEAK = 3.35e12                   # H100 SXM HBM3 data-sheet bandwidth, bytes/s


def write_fasta(path, n_seq, n_sites, seed):
    rng = np.random.default_rng(seed)
    with open(path, "wb") as f:
        for k in range(n_seq):
            f.write(b">q%d\n" % k)
            for lo in range(0, n_sites, 6_000_000):
                n = min(n_sites, lo + 6_000_000) - lo
                s = np.frombuffer(b"ACGTN", np.uint8)[rng.choice(5, size=n, p=[.3, .2, .2, .27, .03])]
                full = n // 60
                lines = np.full((full, 61), ord("\n"), np.uint8)
                lines[:, :60] = s[:full * 60].reshape(-1, 60)
                f.write(lines.tobytes())
                if n % 60:
                    f.write(s[full * 60:].tobytes() + b"\n")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        return "unknown (%s)" % e


def run_cli(args, tmp):
    timing = os.path.join(tmp, "timing.json")
    t0 = time.perf_counter()
    r = subprocess.run([sys.executable, "-m", "genomics_general_b200.cli.seqToGeno"] + args + ["--timing", timing], cwd=REPO,
                       capture_output=True, text=True)
    wall = time.perf_counter() - t0
    if r.returncode != 0:
        raise SystemExit("seqToGeno failed: %s" % r.stderr[-2000:])
    return wall, json.load(open(timing))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seqs", type=int, default=100)
    ap.add_argument("--sites", type=int, default=10_000_000)
    ap.add_argument("--ref-sites", type=int, default=200_000)
    ap.add_argument("--out")
    a = ap.parse_args()
    res = dict(card=card(), seqs=a.seqs, sites=a.sites)
    with tempfile.TemporaryDirectory() as tmp:
        fa = os.path.join(tmp, "in.fa")
        write_fasta(fa, a.seqs, a.sites, 12)
        with open(fa, "rb") as f, gzip.open(fa + ".gz", "wb", compresslevel=1) as g:
            shutil.copyfileobj(f, g)
        fa_bytes = os.path.getsize(fa)
        res["input_bytes"] = fa_bytes
        res["input_gz_bytes"] = os.path.getsize(fa + ".gz")
        out = os.path.join(tmp, "out.geno")
        runs = {"plain": (["-s", fa], out), "gz_in": (["-s", fa + ".gz"], out), "gz_out": (["-s", fa], out + ".gz"),
                "contigs": (["-s", fa, "-M", "contigs"], out)}
        for name, (extra, dest) in runs.items():
            run_cli(extra + ["-g", dest], tmp)                            # warm-up: library load, page cache
            wall, t = run_cli(extra + ["-g", dest], tmp)
            out_bytes = os.path.getsize(dest)
            raw_out = t.get("bytes", out_bytes)
            k = t["kernels_ms"]
            # bytes each kernel moves: marks read the text and write a flag per byte; keep reads both and writes the flags;
            # select reads text and flags and writes the sequences; the transpose reads the sequences and writes the rows
            moved = {"s2g_fa_marks": 2 * fa_bytes, "s2g_fa_keep": 3 * fa_bytes, "s2g_fa_select": 3 * fa_bytes,
                     "s2g_tile": a.seqs * a.sites + raw_out}
            res[name] = dict(wall_s=round(wall, 3), sites_per_s=round(a.sites / wall), output_bytes=out_bytes,
                             phases_s={p: round(v, 3) for p, v in t["phases_s"].items()},
                             kernels_ms={p: round(v, 2) for p, v in k.items()},
                             kernel_fraction_of_peak={p: round(moved[p] / (k[p] * 1e-3) / PEAK, 3)
                                                      for p in moved if k.get(p)})
            print(name, json.dumps(res[name]), flush=True)
        # the unmodified reference on a prefix of every sequence, and the same input through the command line
        ref = os.path.join(REPO, "oracle", "_ref", "seqToGeno.py")
        if os.path.exists(ref) and os.path.exists(os.path.join(REPO, "oracle", "_ref", "genomics.py")):
            small = os.path.join(tmp, "small.fa")
            write_fasta(small, a.seqs, a.ref_sites, 12)
            t0 = time.perf_counter()
            r = subprocess.run([sys.executable, ref, "-s", small, "-g", os.path.join(tmp, "ref.geno")], capture_output=True,
                               text=True, env=dict(os.environ, PYTHONPATH=os.path.dirname(ref)))
            ref_wall = time.perf_counter() - t0
            wall, _ = run_cli(["-s", small, "-g", os.path.join(tmp, "ours.geno")], tmp)
            same = r.returncode == 0 and open(os.path.join(tmp, "ref.geno"), "rb").read() == \
                open(os.path.join(tmp, "ours.geno"), "rb").read()
            res["reference"] = dict(sites=a.ref_sites, wall_s=round(ref_wall, 3), sites_per_s=round(a.ref_sites / ref_wall),
                                    returncode=r.returncode, ours_wall_s=round(wall, 3), identical=same,
                                    stderr_tail=r.stderr[-300:] if r.returncode else "")
            print("reference", json.dumps(res["reference"]), flush=True)
        else:
            res["reference"] = "not measured: oracle/_ref/seqToGeno.py is not staged"
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
