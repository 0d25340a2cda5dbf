#!/usr/bin/env python
"""parseVCF.py timing on one GPU: a seeded VCF with realistic FORMAT (GT:AD:DP:GQ:PL) is written to a temporary
directory, then

  * the command line converts it from a plain file and from a .gz copy (lines/s; --timing gives the kernels' CUDA-event
    times and the wall time of each phase), with the host's gzip decompression of the same file timed on its own;
  * the unmodified reference (oracle/_ref/parseVCF.py, staged by build()) converts the first --ref-lines data lines, as
    bench.py's reference arm runs it, and both outputs of that sample are compared.

    python tools/vcf_timing.py [--samples 100 1000] [--lines 200000 20000] [--out results.json]

The card's name and power limit are read in the same run and written with the numbers."""
import argparse
import gzip
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def write_vcf(path, n_samp, n_lines, seed):
    rng = np.random.default_rng(seed)
    pool = []
    for _ in range(4096):
        a, b = rng.integers(0, 2, 2)
        sep = "|" if rng.random() < 0.5 else "/"
        gt = "./." if rng.random() < 0.03 else "%d%s%d" % (a, sep, b)
        dp = int(rng.integers(0, 60))
        ad = "%d,%d" % (dp // 2, dp - dp // 2)
        pl = ",".join(str(int(x)) for x in rng.integers(0, 255, 3))
        pool.append("%s:%s:%d:%d:%s" % (gt, ad, dp, int(rng.integers(0, 99)), pl))
    pool = np.array(pool, dtype=object)
    head = "##fileformat=VCFv4.2\n##contig=<ID=chr1,length=1000000000>\n" + "\t".join(
        ["#CHROM", "POS", "ID", "REF", "ALT", "QUAL", "FILTER", "INFO", "FORMAT"] + ["s%d" % i for i in range(n_samp)]) + "\n"
    with open(path, "wt") as f:
        f.write(head)
        for lo in range(0, n_lines, 2000):
            rows = []
            for i in range(lo, min(n_lines, lo + 2000)):
                ref, alt = rng.choice(list("ACGT"), 2, replace=False)
                rows.append("chr1\t%d\t.\t%s\t%s\t%d\tPASS\tDP=%d\tGT:AD:DP:GQ:PL\t" % (10 * i + 1, ref, alt, 30 + i % 50, 300) +
                            "\t".join(pool[rng.integers(0, len(pool), n_samp)]))
            f.write("\n".join(rows) + "\n")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        return "unknown (%s)" % e


def run_cli(args):
    from genomics_general_b200.cli import parseVCF as P
    t0 = time.perf_counter()
    P.main(args)
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, nargs="+", default=[100, 1000])
    ap.add_argument("--lines", type=int, nargs="+", default=[200000, 20000])
    ap.add_argument("--ref-lines", type=int, default=2000)
    ap.add_argument("--out", help="also write every result as one JSON file")
    a = ap.parse_args()
    res = dict(card=card(), runs=[])
    ref = os.path.join(REPO, "oracle", "_ref", "parseVCF.py")
    with tempfile.TemporaryDirectory() as tmp:
        for ns, nl in zip(a.samples, a.lines):
            vcf = os.path.join(tmp, "in.vcf")
            write_vcf(vcf, ns, nl, seed=ns)
            size = os.path.getsize(vcf)
            with open(vcf, "rb") as f, gzip.open(vcf + ".gz", "wb", compresslevel=6) as g:
                g.write(f.read())
            t0 = time.perf_counter()
            with gzip.open(vcf + ".gz", "rb") as g:
                while g.read(64 << 20):
                    pass
            t_gunzip = time.perf_counter() - t0
            run_cli(["-i", vcf, "-o", os.path.join(tmp, "warm.geno"), "-s", "s0"])      # module load, first launches
            tj = os.path.join(tmp, "t.json")
            t_plain = run_cli(["-i", vcf, "-o", os.path.join(tmp, "out.geno"), "--timing", tj])
            kern = json.load(open(tj))
            t_gz = run_cli(["-i", vcf + ".gz", "-o", os.path.join(tmp, "out2.geno")])
            r = dict(samples=ns, lines=nl, bytes=size, cli_plain_s=t_plain, cli_plain_lines_per_s=nl / t_plain,
                     cli_gz_s=t_gz, cli_gz_lines_per_s=nl / t_gz, host_gunzip_s=t_gunzip, kernels_ms=kern["kernels_ms"],
                     phases_s=kern["phases_s"])
            if os.path.exists(ref):
                sub = os.path.join(tmp, "sub.vcf")
                with open(vcf, "rb") as f, open(sub, "wb") as o:
                    for k, ln in enumerate(f):
                        if k >= a.ref_lines + 3:
                            break
                        o.write(ln)
                t0 = time.perf_counter()
                subprocess.run([sys.executable, ref, "-i", sub, "-o", os.path.join(tmp, "ref.geno")], check=True,
                               stderr=subprocess.DEVNULL)
                t_ref = time.perf_counter() - t0
                run_cli(["-i", sub, "-o", os.path.join(tmp, "sub.geno")])
                same = open(os.path.join(tmp, "ref.geno"), "rb").read() == open(os.path.join(tmp, "sub.geno"), "rb").read()
                r.update(ref_lines=a.ref_lines, ref_s=t_ref, ref_lines_per_s=a.ref_lines / t_ref, ref_output_identical=same)
            res["runs"].append(r)
            print(json.dumps(r), flush=True)
            for p in (vcf, vcf + ".gz"):
                os.remove(p)
    if a.out:
        with open(a.out, "wt") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(dict(card=res["card"])))


if __name__ == "__main__":
    main()
