"""Device-side timing of the BASELINE.json configs (C1..C5 shapes) on one GPU. Not the bench contract — a probe
whose output feeds DESIGN.md's tables."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from genomics_general_b200 import synth, windows
from genomics_general_b200.engine import Engine

def tm(eng): return {k: round(v["ms"], 3) for k, v in eng.last_timings().items()}

def run(name, P, spp, S, miss, what, wsites=5000, eng=None, reps=2):
    spec = synth.SynthSpec(P, spp, miss=miss, seed=20260923 + len(name))
    eng.synth_fill(spec, S)
    H = spec.n_haps
    lo = np.arange(0, S, wsites, dtype=np.int64); hi = np.minimum(lo + wsites, S)
    eng.set_windows(lo, hi)
    out = dict(config=name, P=P, H=H, S=S, miss=miss, windows=len(lo))
    for _ in range(reps):
        t = time.perf_counter()
        if what == "popgen":
            eng.set_pops(spec.hap_pop(), P); r = eng.popgen(100, 0.01)
            out["paths"] = np.bincount(r["path"], minlength=3).tolist()
        elif what == "abba":
            eng.set_pops(spec.hap_pop(), P); r = eng.abbababa(0, 1, 2, P - 1, 0.5)
        elif what == "fourpop":
            eng.set_pops(spec.hap_pop(), P); r = eng.fourpop(0, 1, 2, P - 1, 0.5)
        elif what == "distcat":
            hap_ind = np.repeat(np.arange(spec.n_samples, dtype=np.int32), 2)
            r = eng.pairdist_cat(hap_ind, spec.n_samples, False)
        elif what == "counts":
            eng.set_pops(spec.hap_pop(), P); n = min(S, 2_000_000); r = eng.site_counts(0, n); out["count_sites"] = n
        elif what == "distmat":
            hap_ind = np.repeat(np.arange(spec.n_samples, dtype=np.int32), 2)
            r = eng.pairdist(hap_ind, spec.n_samples, False)
        out["wall_ms"] = round((time.perf_counter() - t) * 1e3, 2)
        out["kernel_ms"] = tm(eng)
    k = out["kernel_ms"]
    main = {"popgen": "k1_popgen", "abba": "k1_abba", "counts": "k1_counts", "fourpop": "k1_fourpop"}.get(what)
    if main and main in k:
        n = out.get("count_sites", S)
        out["k1_GBps"] = round(n * (H + 4) / (k[main] * 1e-3) / 1e9, 1)
    out["sites_per_s_wall"] = round(out.get("count_sites", S) / (out["wall_ms"] * 1e-3))
    print(json.dumps(out), flush=True)
    return out

if __name__ == "__main__":
    scale = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0
    with Engine(0) as eng:
        run("C1 popgen 2x10 100k", 2, 10, 100_000, 0.0, "popgen", eng=eng)
        run("C1 popgen 2x10 100k miss", 2, 10, 100_000, 0.02, "popgen", eng=eng)
        run("C2 popgen 4x50 10M", 4, 50, int(10_000_000 * scale), 0.0, "popgen", eng=eng)
        run("C2 popgen 4x50 10M miss", 4, 50, int(10_000_000 * scale), 0.02, "popgen", eng=eng)
        run("C3 abba 4x50 10M", 4, 50, int(10_000_000 * scale), 0.02, "abba", eng=eng)
        run("C3 fourpop 4x50 10M", 4, 50, int(10_000_000 * scale), 0.02, "fourpop", eng=eng)
        run("C4 distmat 500 2M", 1, 500, int(2_000_000 * scale), 0.02, "distmat", eng=eng, reps=1)
        run("C4 distmat --windType cat 500 2M", 1, 500, int(2_000_000 * scale), 0.02, "distcat", eng=eng, reps=1)
        run("C5 popgen 8x100 (1/8 of 100M)", 8, 100, int(12_500_000 * scale), 0.0, "popgen", eng=eng)
        run("C5 freq counts 8x100", 8, 100, int(12_500_000 * scale), 0.02, "counts", eng=eng)
        run("C5 popgen 8x100 miss (1M sites)", 8, 100, int(1_000_000 * scale), 0.02, "popgen", eng=eng, reps=1)
