"""Kernel time of genomics.fourPop per window on the C2 shape (10 M sites x 400 haplotypes, 2 % missing, 2000 windows).  Prints
one JSON line (ms of the site pass, HBM GB/s of the algorithmic bytes, a checksum)."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from genomics_general_b200 import synth  # noqa: E402
from genomics_general_b200.engine import Engine  # noqa: E402

S = int(float(os.environ.get("FP_SITES", "10000000")))
with Engine(0) as eng:
    spec = synth.SynthSpec(4, 50, miss=0.02, seed=20260925)
    eng.synth_fill(spec, S)
    eng.set_pops(spec.hap_pop(), 4)
    lo = np.arange(0, S, 5000, dtype=np.int64)
    eng.set_windows(lo, np.minimum(lo + 5000, S))
    out = {}
    for name, kw in (("default", {}), ("polarize", dict(polarize=True)), ("fixed", dict(fixed=True))):
        for _ in range(3):
            r = eng.fourpop(0, 1, 2, 3, 0.5, **kw)
        ms = eng.last_timings()["k1_fourpop"]["ms"]
        out[name] = dict(ms=round(ms, 4), GBps=round(S * 404 / ms / 1e6, 1),
                         check=float(sum(np.nansum(r[k]) for k in eng.FOURPOP_KEYS)), used=float(np.nansum(r["sitesUsed"])))
    print(json.dumps(out))
