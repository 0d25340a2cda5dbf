#!/usr/bin/env python
"""genoToVCF.py timing on one GPU: a seeded phased .geno file (--sites x --samples diploid samples over three scaffolds) and a
seeded FASTA of three 35 Mb contigs are written to a temporary directory, then

  * the command line converts the file without -r and with -r, from the plain file, from a .gz copy, and with .gz output;
    --timing gives the kernels' CUDA-event times (FASTA load: '>' marks, sequence flags and select; per chunk: text upload
    and line index, token pass, scaffold runs, site pass, scan, emit) and the wall time of each phase;
  * the unmodified reference (oracle/_ref/genoToVCF.py, staged by build()) converts the first --ref-sites sites with -r, and
    its output is compared with the command line's on the same sample.

    python tools/g2v_timing.py [--sites 1000000] [--samples 100] [--ref-sites 20000] [--out results.json]

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
CONTIG = 35_000_040                # a multiple of the 60-base lines
# the reference's np.argsort breaks count ties by the CPU's vectorised sort unless it is disabled (oracle/make_golden11.py)
NO_SIMD_SORT = "AVX512F AVX512CD AVX512_SKX AVX512_CLX AVX512_CNL AVX512_ICL AVX512_SPR AVX2 FMA3 F16C"


def write_geno(path, n_samp, n_sites, seed):
    """fixed-width lines: 'chrK', an 8-digit position inside the contig, n_samp phased diploid tokens"""
    rng = np.random.default_rng(seed)
    per = (n_sites + 2) // 3
    with open(path, "wb") as f:
        f.write(("#CHROM\tPOS\t" + "\t".join("s%d" % i for i in range(n_samp)) + "\n").encode())
        width = 5 + 8 + 1 + 4 * n_samp
        for lo in range(0, n_sites, 100000):
            n = min(n_sites, lo + 100000) - lo
            idx = np.arange(lo, lo + n, dtype=np.int64)
            m = np.empty((n, width), np.uint8)
            m[:, :3] = np.frombuffer(b"chr", np.uint8)
            m[:, 3] = ord("1") + idx // per
            m[:, 4] = ord("\t")
            pos = 10_000_000 + (CONTIG - 10_000_001) * (idx % per) // per
            for d in range(8):
                m[:, 5 + d] = ord("0") + (pos // 10 ** (7 - d)) % 10
            m[:, 13] = ord("\t")
            g = m[:, 14:].reshape(n, n_samp, 4)
            alle = np.frombuffer(b"ACGTN", np.uint8)[rng.choice(5, size=(n, n_samp, 2), p=[.3, .2, .2, .27, .03])]
            g[:, :, 0] = alle[:, :, 0]
            g[:, :, 1] = ord("|")
            g[:, :, 2] = alle[:, :, 1]
            g[:, :, 3] = ord("\t")
            m[:, -1] = ord("\n")
            f.write(m.tobytes())


def write_fasta(path, seed):
    rng = np.random.default_rng(seed)
    with open(path, "wb") as f:
        for k in range(3):
            f.write(b">chr%d description\n" % (k + 1))
            s = np.frombuffer(b"ACGTacgtN", np.uint8)[rng.choice(9, size=CONTIG, p=[.2, .2, .2, .2, .04, .04, .04, .04, .04])]
            lines = np.full((CONTIG // 60, 61), ord("\n"), np.uint8)
            lines[:, :60] = s.reshape(-1, 60)
            f.write(lines.tobytes())


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        return "unknown (%s)" % e


def run_cli(args, tmp):
    timing = os.path.join(tmp, "timing.json")
    t0 = time.perf_counter()
    r = subprocess.run([sys.executable, "-m", "genomics_general_b200.cli.genoToVCF"] + args + ["--timing", timing], cwd=REPO,
                       capture_output=True, text=True)
    wall = time.perf_counter() - t0
    if r.returncode != 0:
        raise SystemExit("genoToVCF failed: %s" % r.stderr[-2000:])
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
        geno, fa = os.path.join(tmp, "in.geno"), os.path.join(tmp, "ref.fa")
        write_geno(geno, a.samples, a.sites, 11)
        write_fasta(fa, 12)
        with open(geno, "rb") as f, gzip.open(geno + ".gz", "wb", compresslevel=1) as g:
            shutil.copyfileobj(f, g)
        res["input_bytes"] = os.path.getsize(geno)
        res["input_gz_bytes"] = os.path.getsize(geno + ".gz")
        res["fasta_bytes"] = os.path.getsize(fa)
        out = os.path.join(tmp, "out.vcf")
        runs = {"plain": (["-g", geno], out), "plain_ref": (["-g", geno, "-r", fa], out),
                "gz_in_ref": (["-g", geno + ".gz", "-r", fa], out), "gz_out_ref": (["-g", geno, "-r", fa], out + ".gz")}
        for name, (extra, dest) in runs.items():
            run_cli(["-f", "phased", "-o", dest] + extra, tmp)            # warm-up: library load, page cache
            wall, t = run_cli(["-f", "phased", "-o", dest] + extra, tmp)
            res[name] = dict(wall_s=round(wall, 3), sites_per_s=round(a.sites / wall), output_bytes=os.path.getsize(dest),
                             phases_s={k: round(v, 3) for k, v in t["phases_s"].items()},
                             kernels_ms={k: round(v, 2) for k, v in t["kernels_ms"].items()})
            print(name, json.dumps(res[name]), flush=True)
        # the unmodified reference on a bounded sample, and the same sample through the command line
        ref = os.path.join(REPO, "oracle", "_ref", "genoToVCF.py")
        if os.path.exists(ref) and os.path.exists(os.path.join(REPO, "oracle", "_ref", "genomics.py")):
            sample = os.path.join(tmp, "sample.geno")
            with open(geno, "rb") as f, open(sample, "wb") as g:
                for i, line in enumerate(f):
                    if i > a.ref_sites:
                        break
                    g.write(line)
            t0 = time.perf_counter()
            r = subprocess.run([sys.executable, ref, "-f", "phased", "-g", sample, "-r", fa, "-o", os.path.join(tmp, "ref.vcf")],
                               capture_output=True, text=True,
                               env=dict(os.environ, PYTHONPATH=os.path.dirname(ref), NPY_DISABLE_CPU_FEATURES=NO_SIMD_SORT))
            ref_wall = time.perf_counter() - t0
            wall, _ = run_cli(["-f", "phased", "-g", sample, "-r", fa, "-o", os.path.join(tmp, "ours.vcf")], tmp)
            same = r.returncode == 0 and open(os.path.join(tmp, "ref.vcf"), "rb").read() == \
                open(os.path.join(tmp, "ours.vcf"), "rb").read()
            res["reference"] = dict(sites=a.ref_sites, wall_s=round(ref_wall, 3), sites_per_s=round(a.ref_sites / ref_wall),
                                    returncode=r.returncode, ours_wall_s=round(wall, 3), identical=same,
                                    stderr_tail=r.stderr[-300:] if r.returncode else "")
            print("reference", json.dumps(res["reference"]), flush=True)
        else:
            res["reference"] = "not measured: oracle/_ref/genoToVCF.py is not staged"
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
