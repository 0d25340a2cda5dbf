"""The popgen site pass four ways, timed alternately in one process: on the one-hot bytes (PG_K1_BYTE_PASS), on every row of
the packed companion (PG_K1_NO_UNIFORM), on the packed rows of the varied sites only ("varied_rows", the default where
enough sites are uniform: complete biallelic rows as one allele bit per haplotype, the others as three planes, walked on all
the team's lanes; the uniform sites and positions come from per-site prefixes), and on that stream with every varied row in
three planes ("varied_planes", PG_K1_UNI_BITS=0), at the C2 shape (4 x 50 diploid samples, H = 400, 10 M sites) with 50,000-site windows and with the benchmark's 5,000-site
windows (C2_w5000), and the C5 shape (8 x 100 diploid samples, H = 1600, 12.5 M sites).  Per pass and shape: median / min / max of the k1_popgen kernel time (CUDA events) over the rounds, the bytes the
pass reads per site, the achieved GB/s, the time of the varied-row build (k1_uniform, once per data change), the varied-row
stream's geometry (row budget R, tile bound Tmax, ring stages and bytes, tiles, mean rows and sites per tile), and whether the
records of the four passes are bit-identical.

--sweep adds, at C2 and C5: the elided pass under PG_K1_UNI_R / PG_K1_UNI_TMAX / PG_K1_STAGES settings; at C2: and the packed pass against the elided one
(forced on) at small uniform fractions, the measurement behind the fraction from which the stream is kept.
Prints one JSON line with the card's name and power limit.

    python tools/packed_site_pass.py [--rounds 5] [--calls 10] [--c5-sites 12500000] [--sweep]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from genomics_general_b200 import synth  # noqa: E402
from genomics_general_b200.engine import Engine  # noqa: E402

PASS_ENV = {"byte": {"PG_K1_BYTE_PASS": "1"}, "packed": {"PG_K1_NO_UNIFORM": "1"}, "varied_rows": {},
            "varied_planes": {"PG_K1_UNI_BITS": "0"}}
STREAMS = ("varied_rows", "varied_planes")
KNOBS = ("PG_K1_BYTE_PASS", "PG_K1_NO_UNIFORM", "PG_K1_UNIFORM_FORCE", "PG_K1_TILE_KB", "PG_K1_STAGES", "PG_K1_UNI_BITS")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    return q.stdout.strip() if q.returncode == 0 else "unknown (nvidia-smi failed)"


def row_bytes(H):
    chunks = max(1, (H + 15) // 16)
    one_hot = (chunks + 1 if chunks % 2 == 0 else chunks) * 16
    packed = (3 * ((H + 31) // 32) * 4 + 15) // 16 * 16
    return one_hot, packed


def records(r):
    out = {}
    for k, v in r.items():
        v = np.array(v)
        out[k] = v.view(np.uint64) if v.dtype == np.float64 else v
    return out


def set_env(env):
    for k in KNOBS:
        os.environ.pop(k, None)
    os.environ.update(env)


def replan(eng):
    """the launch plan is cached per data shape; a byte-pass call in between makes the next packed call plan again"""
    env = {k: os.environ[k] for k in KNOBS if k in os.environ}
    set_env(dict(env, PG_K1_BYTE_PASS="1"))
    eng.popgen(1, 0.01)
    set_env(env)


def timed(eng, calls):
    ms = []
    for _ in range(calls):
        eng.popgen(1, 0.01)
        ms.append(eng.last_timings()["k1_popgen"]["ms"])
    return ms


def stats(ms, S, bytes_per_site):
    a = np.array(ms)
    med = float(np.median(a))
    return {"k1_popgen_ms_median": med, "ms_min": float(a.min()), "ms_max": float(a.max()),
            "bytes_per_site": bytes_per_site, "GBps": S * bytes_per_site / (med * 1e-3) / 1e9, "samples": len(a)}


def load(eng, P, spp, S, w, p_variable=0.30, miss=0.0):
    spec = synth.SynthSpec(P, spp, 2, seed=11, miss=miss, p_variable=p_variable)
    eng.synth_fill(spec, S)
    eng.set_pops(spec.hap_pop(), P)
    lo = np.arange(0, S, w, dtype=np.int64)
    eng.set_windows(lo, np.minimum(lo + w, S))
    return spec.n_haps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=10, help="timed calls per pass and round")
    ap.add_argument("--c2-sites", type=int, default=10_000_000)
    ap.add_argument("--c5-sites", type=int, default=12_500_000)
    ap.add_argument("--sweep", action="store_true")
    args = ap.parse_args()
    out = {"card": card(), "shapes": {}}
    with Engine(0) as eng:
        for name, P, spp, S, w in (("C2", 4, 50, args.c2_sites, 50_000), ("C2_w5000", 4, 50, args.c2_sites, 5000),
                                   ("C5", 8, 100, args.c5_sites, 5000)):
            H = load(eng, P, spp, S, w)
            one_hot, packed = row_bytes(H)
            ms = {k: [] for k in PASS_ENV}
            build_ms, rec, varied = {k: [] for k in STREAMS}, {}, None
            wd = (H + 31) // 32
            one_plane = 0
            for rnd in range(args.rounds):
                for kind, env in PASS_ENV.items():
                    if kind in STREAMS and rnd % 2:
                        env = dict(env, PG_K1_UNIFORM_FORCE="1")   # a different key: the next call rebuilds the stream
                    set_env(env)
                    r = eng.popgen(1, 0.01)                      # warm-up (and re-plan / rebuild after the switch)
                    if kind in STREAMS:
                        t = eng.last_timings()
                        if "k1_uniform" in t:       # at 8 populations both streams are three-plane: the same stream
                            build_ms[kind].append(t["k1_uniform"]["ms"])
                        used, varied = eng.uniform_stream()
                        assert used
                        if kind == "varied_rows":
                            one_plane = eng.uniform_rows()[0]     # none at 8 populations
                        R, stages, stage_bytes = eng.uniform_ring()
                        _, Tmax, site_lo, row0 = eng.uniform_tiles()
                        geometry = {"R": R, "Tmax": Tmax, "stages": stages, "stage_bytes": stage_bytes,
                                    "tiles": len(site_lo) - 1, "rows_per_tile_mean": float(np.diff(row0).mean()),
                                    "sites_per_tile_mean": float(np.diff(site_lo).mean())}
                    rec.setdefault(kind, records(r))
                    ms[kind].extend(timed(eng, args.calls))
            set_env({})
            res = {"H": H, "P": P, "sites": S, "varied_sites": varied, "uniform_fraction": 1 - varied / S}
            res["byte"] = stats(ms["byte"], S, one_hot + 4)
            res["packed"] = stats(ms["packed"], S, packed + 4)
            # per varied site its row and its slot: one plane of wd words for a complete biallelic site
            res["one_plane_rows"] = one_plane
            res["varied_rows"] = stats(ms["varied_rows"], S, (one_plane * (4 * wd + 2) + (varied - one_plane) * (packed + 2)) / S)
            res["varied_planes"] = stats(ms["varied_planes"], S, varied / S * (packed + 2))
            for k in STREAMS:
                res[k]["k1_uniform_build_ms_median"] = float(np.median(build_ms[k])) if build_ms[k] else None
            res["varied_rows"]["geometry"] = geometry
            res["speedup_varied_rows_vs_packed"] = (res["packed"]["k1_popgen_ms_median"] /
                                                    res["varied_rows"]["k1_popgen_ms_median"])
            res["speedup_varied_rows_vs_planes"] = (res["varied_planes"]["k1_popgen_ms_median"] /
                                                    res["varied_rows"]["k1_popgen_ms_median"])
            res["records_bit_identical"] = all(np.array_equal(rec["byte"][k], rec[o][k])
                                               for k in rec["byte"] for o in ("packed",) + STREAMS)
            out["shapes"][name] = res
        if args.sweep:
            for name, P, spp, S, w in (("C2", 4, 50, args.c2_sites, 50_000), ("C5", 8, 100, args.c5_sites, 5000)):
                load(eng, P, spp, S, w)
                geo = {}
                for r, tm, st in ((0, 0, 0), (32, 0, 0), (64, 0, 0), (128, 0, 0), (256, 0, 0), (0, 256, 0), (0, 2048, 0),
                                  (0, 0, 4)):
                    env = {k: str(v) for k, v in (("PG_K1_UNI_R", r), ("PG_K1_UNI_TMAX", tm), ("PG_K1_STAGES", st)) if v}
                    set_env(env)
                    eng.popgen(1, 0.01)
                    a = np.array(timed(eng, args.calls * 2))
                    geo[" ".join("%s=%s" % kv for kv in env.items()) or "default"] = {
                        "ms_median": float(np.median(a)), "ring": eng.uniform_ring()}
                    for k in ("PG_K1_UNI_R", "PG_K1_UNI_TMAX"):
                        os.environ.pop(k, None)
                set_env({})
                out[name.lower() + "_budget_sweep"] = geo
            S = args.c2_sites
            H = load(eng, 4, 50, S, 50_000)
            geo = {}
            for tk, st in ((16, 0), (32, 0), (64, 0), (96, 0), (64, 2), (32, 4)):
                env = {"PG_K1_TILE_KB": str(tk)}
                if st:
                    env["PG_K1_STAGES"] = str(st)
                set_env(env)
                replan(eng)
                eng.popgen(1, 0.01)
                a = np.array(timed(eng, args.calls * 2))
                geo["tile_kb=%d stages=%s" % (tk, st or "auto")] = {"ms_median": float(np.median(a)), "ms_min": float(a.min()),
                                                                     "ms_max": float(a.max())}
            set_env({})
            replan(eng)
            out["c2_geometry_varied_rows"] = geo
            cross = {}
            for pv in (0.80, 0.90, 0.95, 0.99):
                load(eng, 4, 50, S, 50_000, p_variable=pv)
                row = {}
                for kind, env in (("packed", {"PG_K1_NO_UNIFORM": "1"}), ("varied_rows", {"PG_K1_UNIFORM_FORCE": "1"})):
                    set_env(env)
                    eng.popgen(1, 0.01)
                    if kind == "varied_rows":
                        row["k1_uniform_build_ms"] = eng.last_timings()["k1_uniform"]["ms"]
                        row["uniform_fraction"] = 1 - eng.uniform_stream()[1] / S
                    row[kind + "_ms_median"] = float(np.median(timed(eng, args.calls * 2)))
                cross["p_variable=%.2f" % pv] = row
            set_env({})
            out["c2_crossover"] = cross
    print(json.dumps(out))


if __name__ == "__main__":
    main()
