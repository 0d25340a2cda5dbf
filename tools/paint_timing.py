#!/usr/bin/env python
"""Device time of distPaint's assignment: a synthetic haploid matrix filled on the GPU (pg_synth_fill, ploidy 1), windows
of --window sites, --pops reference populations of --members samples each, every sample a query; pg_distpaint's kernels
as CUDA-event times from pg_last_timings (best of --reps, after one warm-up call), for the rank-sum and the delta rule.
Prints one JSON object with the card's name and power limit.

    python tools/paint_timing.py [--samples 1000 --sites 2000000 --window 5000 --pops 4 --members 50 --reps 3]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=1000)
    ap.add_argument("--sites", type=int, default=2000000)
    ap.add_argument("--window", type=int, default=5000)
    ap.add_argument("--pops", type=int, default=4)
    ap.add_argument("--members", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    from genomics_general_b200 import synth
    from genomics_general_b200.engine import Engine
    spec = synth.SynthSpec(a.pops, a.samples // a.pops, ploidy=1, miss=0.02, seed=5)
    H = spec.n_haps
    rng = np.random.default_rng(1)
    pops = [rng.choice(np.arange(p * spec.haps_per_pop, (p + 1) * spec.haps_per_pop), a.members, replace=False)
            for p in range(a.pops)]
    ref_off = np.cumsum([0] + [len(m) for m in pops]).astype(np.int32)
    ref_hap = np.concatenate(pops).astype(np.int32)
    lo = np.arange(0, a.sites, a.window, dtype=np.int64)
    hi = np.minimum(lo + a.window, a.sites)
    res = dict(samples=H, sites=a.sites, windows=len(lo), pops=a.pops, members=a.members)
    with Engine(0) as eng:
        eng.synth_fill(spec, a.sites)
        eng.set_windows(lo, hi)
        for rule, delta, thr in (("ranksum", False, 0.05), ("delta", True, 0.01)):
            eng.distpaint(np.arange(H), ref_off, ref_hap, 1, delta=delta, threshold=thr)
            best = None
            for _ in range(a.reps):
                r = eng.distpaint(np.arange(H), ref_off, ref_hap, 1, delta=delta, threshold=thr)
                t = {k: v["ms"] for k, v in eng.last_timings().items()}
                if best is None or sum(t.values()) < sum(best.values()):
                    best = t
            res[rule] = dict(kernels_ms=best, total_kernel_ms=sum(best.values()),
                             assigned_share=float((r["assign"] >= 0).mean()))
    try:
        res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                    capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        res["gpu"] = "unknown"
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
