#!/usr/bin/env python
"""mergeGeno.py timing on one GPU: --files seeded .geno files of --lines lines x --samples samples each (every file holds a
random two thirds of the positions of a 2-scaffold genome of 1.5 * lines sites) are written to a temporary directory, plain
and gzipped, then for --method intersect, union and all, from the plain and from the .gz inputs:

  * the command line merges them with --timing (the kernels' CUDA-event times and the wall time of each host phase);
  * the unmodified reference (oracle/_ref/mergeGeno.py, staged by build()) merges the same inputs, and the two outputs are
    compared by sha256.

    python tools/merge_timing.py [--files 4] [--lines 1000000] [--samples 50] [--no-ref] [--out results.json]

The card's name and power limit are read in the same run and written with the numbers."""
import argparse
import gzip
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(REPO, "oracle", "_ref", "mergeGeno.py")


def make_inputs(tmp, files, lines, samples, seed=14):
    rng = np.random.default_rng(seed)
    genome = int(lines * 1.5)
    fai = [("chr1", genome * 3 // 5), ("chr2", genome - genome * 3 // 5)]
    with open(os.path.join(tmp, "g.fai"), "w") as f:
        for n, l in fai:
            f.write("%s\t%d\n" % (n, l))
    bases = np.array(list("ACGTN"))
    paths = []
    for x in range(files):
        keys = np.sort(rng.choice(genome, size=lines, replace=False))
        pool = ["\t".join(a + "/" + b for a, b in zip(rng.choice(bases, samples), rng.choice(bases, samples)))
                for _ in range(997)]
        pick = rng.integers(0, len(pool), lines)
        scaf = (keys >= fai[0][1]).astype(np.int64)
        site = keys - scaf * fai[0][1] + 1
        head = "\t".join(["#CHROM", "POS"] + ["f%d_s%d" % (x, k) for k in range(samples)]) + "\n"
        text = (head + "".join("%s\t%d\t%s\n" % (fai[s][0], p, pool[k])
                               for s, p, k in zip(scaf.tolist(), site.tolist(), pick.tolist()))).encode()
        p = os.path.join(tmp, "in%d.geno" % x)
        with open(p, "wb") as f:
            f.write(text)
        with gzip.open(p + ".gz", "wb", compresslevel=6) as f:
            f.write(text)
        paths.append(p)
    return os.path.join(tmp, "g.fai"), paths


def sha(path):
    h = hashlib.sha256()
    with (gzip.open(path, "rb") if path.endswith(".gz") else open(path, "rb")) as f:
        for blk in iter(lambda: f.read(1 << 24), b""):
            h.update(blk)
    return h.hexdigest()


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                           text=True, timeout=60)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=4)
    ap.add_argument("--lines", type=int, default=1000000)
    ap.add_argument("--samples", type=int, default=50)
    ap.add_argument("--no-ref", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    res = dict(card=card(), files=a.files, lines=a.lines, samples=a.samples, runs=[])
    tmp = tempfile.mkdtemp()
    try:
        t0 = time.perf_counter()
        fai, paths = make_inputs(tmp, a.files, a.lines, a.samples)
        res["input_bytes"] = sum(os.path.getsize(p) for p in paths)
        res["generate_s"] = round(time.perf_counter() - t0, 2)
        env = dict(os.environ, PYTHONPATH=REPO)
        for gz in (False, True):
            ins = [p + ".gz" if gz else p for p in paths]
            for method in ("intersect", "union", "all"):
                argv = sum((["-i", p] for p in ins), []) + ["-f", fai, "--method", method]
                ours = os.path.join(tmp, "ours.geno")
                tj = os.path.join(tmp, "t.json")
                t0 = time.perf_counter()
                subprocess.run([sys.executable, "-m", "genomics_general_b200.cli.mergeGeno"] + argv +
                               ["-o", ours, "--timing", tj], check=True, env=env, stderr=subprocess.DEVNULL)
                run = dict(method=method, gz=gz, cli_s=round(time.perf_counter() - t0, 3), out_bytes=os.path.getsize(ours),
                           timing=json.load(open(tj)))
                if not a.no_ref and os.path.exists(REF):
                    theirs = os.path.join(tmp, "ref.geno")
                    t0 = time.perf_counter()
                    subprocess.run([sys.executable, REF] + argv + ["-o", theirs], check=True, stderr=subprocess.DEVNULL)
                    run["ref_s"] = round(time.perf_counter() - t0, 3)
                    run["identical"] = sha(ours) == sha(theirs)
                    os.remove(theirs)
                os.remove(ours)
                res["runs"].append(run)
                print(json.dumps(run), flush=True)
    finally:
        shutil.rmtree(tmp)
    res["card_after"] = card()
    print(json.dumps(dict((k, v) for k, v in res.items() if k != "runs")))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
