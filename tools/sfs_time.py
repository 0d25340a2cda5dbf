#!/usr/bin/env python
"""Time the SFS paths on the GPU: the dense histograms (pg_sfs) against the sparse spectra (pg_sfs_sparse) on one request
below the dense limit, and the sparse path on a request above it.

    python tools/sfs_time.py [--sites 10000000] [--reps 3] [--out result.json]

For each case: the whole call (Engine.sfs / Engine.sfs_sparse return host arrays, so the call ends in a synchronise), the
kernel times from the engine's CUDA events (last_timings), the bytes copied device-to-host, and the card's name and power
limit read in the same run.  The outputs of the two paths are compared cell for cell before anything is timed."""
import argparse
import itertools
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from genomics_general_b200 import synth  # noqa: E402
from genomics_general_b200.engine import SFS_MAX_CELLS, Engine, sfs_shapes  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    return r.stdout.strip().split("\n")[0] if r.returncode == 0 else "unknown (nvidia-smi failed)"


def timed(eng, fn, reps):
    fn()                                                      # warm-up: buffers grown, modules loaded
    walls, kernels = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        walls.append(time.perf_counter() - t0)
        kernels.append({k: round(v["ms"], 3) for k, v in eng.last_timings().items()})
    i = int(np.argsort(walls)[len(walls) // 2])
    return out, dict(wall_ms=[round(1e3 * w, 2) for w in walls], median_wall_ms=round(1e3 * walls[i], 2), kernel_ms=kernels[i])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sites", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    res = dict(card=card(), sites=a.sites)
    with Engine(0) as eng:
        # ---- below the limit: one 4-D spectrum of 4 x 50 diploid samples (101^4 = 1.04e8 cells), dense vs sparse
        spec = synth.SynthSpec(4, 50, miss=0.001, seed=3)
        eng.synth_fill(spec, a.sites)
        eng.set_pops(spec.hap_pop(), 4)
        groups, sizes = [(0, 1, 2, 3)], [100] * 4
        cells = sum(sfs_shapes(groups, [101] * 4)[1])
        (h, f, n_d), td = timed(eng, lambda: eng.sfs(4, groups, sizes), a.reps)
        (sp, n_s), ts = timed(eng, lambda: eng.sfs_sparse(4, groups, sizes), a.reps)
        nz = np.flatnonzero(h[0].reshape(-1))
        assert n_d == n_s and np.array_equal(sp[0][1], h[0].reshape(-1)[nz]) and np.array_equal(sp[0][2], f[0].reshape(-1)[nz])
        assert np.array_equal(sp[0][0], np.argwhere(h[0] > 0))
        nnz = len(nz)
        td["result_d2h_bytes"] = cells * 16                  # histogram + first-site array
        ts["result_d2h_bytes"] = nnz * 24                    # cell, count, first of the non-empty cells
        res["below_limit_4d"] = dict(cells=cells, nnz=nnz, sites_counted=n_d, dense=td, sparse=ts, equal=True)
        # ---- above the limit: 6 x 36 diploid samples, singles + 15 quartets (--doQuartets): sparse only
        spec = synth.SynthSpec(6, 36, miss=0.001, seed=5)
        eng.synth_fill(spec, a.sites)
        eng.set_pops(spec.hap_pop(), 6)
        groups = [(x,) for x in range(6)] + list(itertools.combinations(range(6), 4))
        cells = sum(sfs_shapes(groups, [73] * 6)[1])
        assert cells > SFS_MAX_CELLS
        (sp, n_s), ts = timed(eng, lambda: eng.sfs_sparse(6, groups, [72] * 6), a.reps)
        nnz = int(sum(len(e[1]) for e in sp))
        ts["result_d2h_bytes"] = nnz * 24
        res["above_limit_quartets"] = dict(cells=cells, nnz=nnz, sites_counted=n_s, sparse=ts)
    txt = json.dumps(res)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "wt") as fo:
            fo.write(txt + "\n")


if __name__ == "__main__":
    main()
