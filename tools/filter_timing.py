#!/usr/bin/env python
"""Sites per second of filterGenotypes on the GPU: writes a synthetic phased .geno to a temporary directory, runs the
command line on it (wall time, output to /dev/null) and, on the same text, the filter kernels alone (pg_filter on the
resident matrix, CUDA-event times of filter_sites / filter_thin, best of --reps).

    python tools/filter_timing.py --sites 2000000 --samples 100 [--reps 5]"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def write_geno(path, S, n, seed=1):
    rng = np.random.default_rng(seed)
    base = np.array(list("ACGT"))
    with open(path, "wt") as f:
        f.write("\t".join(["#CHROM", "POS"] + ["s%d" % k for k in range(n)]) + "\n")
        block = 20000
        for s0 in range(0, S, block):
            m = min(block, S - s0)
            ref = rng.integers(0, 4, m)
            alt = (ref + rng.integers(1, 4, m)) % 4
            var = rng.random(m) < 0.3
            a = np.where((rng.random((m, n, 2)) < 0.2) & var[:, None, None], alt[:, None, None], ref[:, None, None])
            g = base[a]
            g[rng.random((m, n, 2)) < 0.02] = "N"
            toks = np.char.add(np.char.add(g[:, :, 0], "|"), g[:, :, 1])
            lines = ["scaf1\t%d\t" % (10 * (s0 + i) + 1) + "\t".join(toks[i]) for i in range(m)]
            f.write("\n".join(lines) + "\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sites", type=int, default=1000000)
    ap.add_argument("--samples", type=int, default=100)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    from genomics_general_b200.cli import filterGenotypes as F
    from genomics_general_b200.engine import Engine
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "in.geno")
        write_geno(path, a.sites, a.samples)
        args = ["-i", path, "-o", os.devnull, "--minCalls", "50", "--minAlleles", "2", "--maxHet", "0.5"]
        F.main(args)                                    # warm-up (context, module loads)
        t0 = time.perf_counter()
        F.main(args)
        cli_s = time.perf_counter() - t0
        data = open(path, "rb").read()
        body = data[data.find(b"\n") + 1:]
        n = a.samples
        hap0 = np.arange(0, 2 * n, 2, dtype=np.int32)
        with Engine(0) as eng:
            eng.set_strict_ingest(True)
            S = eng.ingest_text(body, 0, hap0, np.full(n, 2, np.int8), 2 * n)
            eng.ingest_meta(S, release=False)
            spec = dict(samp_hap0=hap0, samp_ploidy=np.full(n, 2, np.int8), P=0, min_calls=50, min_alleles=2, max_het=0.5)
            best = None
            for _ in range(a.reps):
                eng.filter(spec)
                ms = sum(v["ms"] for k, v in eng.last_timings().items() if k.startswith("filter"))
                best = ms if best is None else min(best, ms)
    print(json.dumps(dict(sites=a.sites, samples=a.samples, cli_s=round(cli_s, 3), cli_sites_per_s=a.sites / cli_s,
                          kernel_ms=round(best, 3), kernel_sites_per_s=a.sites / (best / 1e3))))


if __name__ == "__main__":
    main()
