#!/usr/bin/env python
"""genoToSeq.py timing on one GPU: a seeded phased .geno file (--sites x --samples diploid samples, one scaffold) is written to
a temporary directory, then

  * the command line makes a FASTA alignment of the whole file (-M cat), the same with --splitPhased, and 5,000-site windows
    (-M windows --windType sites, one output file), each from the plain file; --timing gives the kernels' CUDA-event times
    (token index, row lengths, frame and transpose) and the wall time of each phase;
  * the unmodified reference (oracle/_ref/genoToSeq.py, staged by build()) converts the first --ref-sites sites in cat mode,
    and its output is compared with the command line's on the same sample.

    python tools/seq_timing.py [--sites 1000000] [--samples 100] [--ref-sites 20000] [--out results.json]

The card's name and power limit are read in the same run and written with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def write_geno(path, n_samp, n_sites, seed):
    """fixed-width lines: 'chr1', a 10-digit position, n_samp phased diploid tokens"""
    rng = np.random.default_rng(seed)
    with open(path, "wb") as f:
        f.write(("#CHROM\tPOS\t" + "\t".join("s%d" % i for i in range(n_samp)) + "\n").encode())
        width = 5 + 10 + 1 + 4 * n_samp
        for lo in range(0, n_sites, 100000):
            n = min(n_sites, lo + 100000) - lo
            m = np.empty((n, width), np.uint8)
            m[:, :5] = np.frombuffer(b"chr1\t", np.uint8)
            pos = 1000000000 + 10 * np.arange(lo, lo + n, dtype=np.int64)
            for d in range(10):
                m[:, 5 + d] = ord("0") + (pos // 10 ** (9 - d)) % 10
            g = m[:, 16:].reshape(n, n_samp, 4)
            alle = np.frombuffer(b"ACGTN", np.uint8)[rng.choice(5, size=(n, n_samp, 2), p=[.3, .2, .2, .27, .03])]
            g[:, :, 0] = alle[:, :, 0]
            g[:, :, 1] = ord("|")
            g[:, :, 2] = alle[:, :, 1]
            g[:, :, 3] = ord("\t")
            m[:, 15] = ord("\t")
            m[:, -1] = ord("\n")
            f.write(m.tobytes())


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        return "unknown (%s)" % e


def run_cli(args, tmp):
    timing = os.path.join(tmp, "timing.json")
    t0 = time.perf_counter()
    r = subprocess.run([sys.executable, "-m", "genomics_general_b200.cli.genoToSeq"] + args + ["--timing", timing], cwd=REPO,
                       capture_output=True, text=True)
    wall = time.perf_counter() - t0
    if r.returncode != 0:
        raise SystemExit("genoToSeq failed: %s" % r.stderr[-2000:])
    return wall, json.load(open(timing))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sites", type=int, default=1000000)
    ap.add_argument("--samples", type=int, default=100)
    ap.add_argument("--ref-sites", type=int, default=20000)
    ap.add_argument("--out")
    a = ap.parse_args()
    res = dict(card=card(), sites=a.sites, samples=a.samples)
    with tempfile.TemporaryDirectory() as tmp:
        geno = os.path.join(tmp, "in.geno")
        write_geno(geno, a.samples, a.sites, 11)
        size = os.path.getsize(geno)
        res["input_bytes"] = size
        out = os.path.join(tmp, "out.fa")
        runs = {"cat": [], "cat_splitPhased": ["--splitPhased"],
                "windows_5000_sites": ["-M", "windows", "--windType", "sites", "--windSize", "5000", "--overlap", "0",
                                       "--maxDist", "2000000000"]}
        for name, extra in runs.items():
            run_cli(["-g", geno, "-s", out] + extra, tmp)                 # warm-up: library load, allocations
            wall, t = run_cli(["-g", geno, "-s", out] + extra, tmp)
            k = t["kernels_ms"]
            outb = os.path.getsize(out)
            res[name] = dict(wall_s=round(wall, 3), sites_per_s=round(a.sites / wall), output_bytes=outb, phases_s=t["phases_s"],
                             kernels_ms=k, index_bytes_read=size, index_bytes_written=a.sites * a.samples * 4,
                             emit_bytes_written=outb,
                             emit_GBps=round(outb / (1e-3 * (k.get("seq_tile", 0) + k.get("seq_frame", 0))) / 1e9, 1)
                             if k.get("seq_tile") else None)
            print(name, json.dumps(res[name]), flush=True)
        # the unmodified reference on a bounded sample, and the same sample through the command line
        ref = os.path.join(REPO, "oracle", "_ref", "genoToSeq.py")
        if os.path.exists(ref):
            sample = os.path.join(tmp, "sample.geno")
            with open(geno, "rb") as f, open(sample, "wb") as g:
                for i, line in enumerate(f):
                    if i > a.ref_sites:
                        break
                    g.write(line)
            t0 = time.perf_counter()
            r = subprocess.run([sys.executable, ref, "-g", sample, "-s", os.path.join(tmp, "ref.fa")], capture_output=True,
                               text=True, env=dict(os.environ, PYTHONPATH=os.path.dirname(ref)))
            ref_wall = time.perf_counter() - t0
            wall, _ = run_cli(["-g", sample, "-s", os.path.join(tmp, "ours.fa")], tmp)
            same = r.returncode == 0 and open(os.path.join(tmp, "ref.fa"), "rb").read() == open(os.path.join(tmp, "ours.fa"),
                                                                                                 "rb").read()
            res["reference_cat"] = dict(sites=a.ref_sites, wall_s=round(ref_wall, 3), sites_per_s=round(a.ref_sites / ref_wall),
                                        returncode=r.returncode, ours_wall_s=round(wall, 3), identical=same)
            print("reference", json.dumps(res["reference_cat"]), flush=True)
        else:
            res["reference_cat"] = "not measured: oracle/_ref/genoToSeq.py is not staged"
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
