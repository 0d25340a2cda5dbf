"""One 2%-missing popgen pass on the C2 row shape (for profiler captures of the pairwise kernels)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from genomics_general_b200 import synth
from genomics_general_b200.engine import Engine
S = int(float(os.environ.get("K2T_SITES", "2000000")))
with Engine(0) as eng:
    spec = synth.SynthSpec(4, 50, miss=0.02, seed=20260925)
    eng.synth_fill(spec, S)
    eng.set_pops(spec.hap_pop(), 4)
    lo = np.arange(0, S, 5000, dtype=np.int64); hi = np.minimum(lo + 5000, S)
    eng.set_windows(lo, hi)
    for _ in range(int(os.environ.get("K2T_REPS", "2"))):
        r = eng.popgen(100, 0.01)
    print({k: round(v["ms"], 3) for k, v in eng.last_timings().items()})
