"""The popgen site pass on the one-hot bytes (PG_K1_BYTE_PASS) and on the packed companion, timed alternately in one process
at the C2 shape (4 x 50 diploid samples, H = 400, 10 M sites) and the C5 shape (8 x 100 diploid samples, H = 1600, 12.5 M
sites).  Per pass and shape: median / min / max of the k1_popgen kernel time (CUDA events) over the rounds, the bytes the
pass reads per site (row + 4-byte position), the achieved GB/s, and whether the records of the two passes are bit-identical.
Prints one JSON line with the card's name and power limit.

    python tools/packed_site_pass.py [--rounds 5] [--calls 10] [--c5-sites 12500000]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from genomics_general_b200 import synth  # noqa: E402
from genomics_general_b200.engine import Engine  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    return q.stdout.strip() if q.returncode == 0 else "unknown (nvidia-smi failed)"


def row_bytes(H):
    chunks = max(1, (H + 15) // 16)
    one_hot = (chunks + 1 if chunks % 2 == 0 else chunks) * 16
    packed = (3 * ((H + 31) // 32) * 4 + 15) // 16 * 16
    return {"byte": one_hot + 4, "packed": packed + 4}


def records(r):
    out = {}
    for k, v in r.items():
        v = np.array(v)
        out[k] = v.view(np.uint64) if v.dtype == np.float64 else v
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=10, help="timed calls per pass and round")
    ap.add_argument("--c2-sites", type=int, default=10_000_000)
    ap.add_argument("--c5-sites", type=int, default=12_500_000)
    args = ap.parse_args()
    out = {"card": card(), "shapes": {}}
    with Engine(0) as eng:
        for name, P, spp, S, w in (("C2", 4, 50, args.c2_sites, 50_000), ("C5", 8, 100, args.c5_sites, 5000)):
            spec = synth.SynthSpec(P, spp, 2, seed=11, miss=0.0)
            eng.synth_fill(spec, S)
            eng.set_pops(spec.hap_pop(), P)
            lo = np.arange(0, S, w, dtype=np.int64)
            eng.set_windows(lo, np.minimum(lo + w, S))
            H = spec.n_haps
            nbytes = row_bytes(H)
            ms = {"byte": [], "packed": []}
            rec = {}
            for rnd in range(args.rounds):
                for kind in ("byte", "packed"):
                    if kind == "byte":
                        os.environ["PG_K1_BYTE_PASS"] = "1"
                    else:
                        os.environ.pop("PG_K1_BYTE_PASS", None)
                    r = eng.popgen(1, 0.01)                  # warm-up (and re-plan after the switch)
                    rec.setdefault(kind, records(r))
                    for _ in range(args.calls):
                        eng.popgen(1, 0.01)
                        ms[kind].append(eng.last_timings()["k1_popgen"]["ms"])
            os.environ.pop("PG_K1_BYTE_PASS", None)
            res = {"H": H, "P": P, "sites": S}
            for kind in ("byte", "packed"):
                a = np.array(ms[kind])
                med = float(np.median(a))
                res[kind] = {"k1_popgen_ms_median": med, "ms_min": float(a.min()), "ms_max": float(a.max()),
                             "bytes_per_site": nbytes[kind], "GBps": S * nbytes[kind] / (med * 1e-3) / 1e9,
                             "samples": len(a)}
            res["speedup"] = res["byte"]["k1_popgen_ms_median"] / res["packed"]["k1_popgen_ms_median"]
            res["records_bit_identical"] = all(np.array_equal(rec["byte"][k], rec["packed"][k]) for k in rec["byte"])
            out["shapes"][name] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
