#!/usr/bin/env python
"""Drop-in for the reference's windowStats.py on the GPU: per-window mean, median, min, max, sd, sum and quantiles of the
numeric columns of a per-site table (scaffold, position, value columns), in sliding coordinate, sliding sites or predefined
windows.  The text is read in chunks cut at line ends (_stream.py); the device parses every value to float64, keeps them
column-major with the positions, and reduces every (window, column) pair in one warp with numpy's own summation order.  The
windows come from windows.py, the rows are printed by the native row formatter.

Where the reference crashes under Python 3 the command line does what the script evidently means (DESIGN.md section 8): -o
writes the file (gzip for .gz), .gz input is read as text, --include / --exclude read one scaffold per line, and failed
windows and quantiles of an empty column are written as nan.  Refused before any output: a value float() rejects inside an
evaluated window, min or max of an evaluated window whose column has no value, a line whose field count differs from the
header (without --columns) or that lacks a named column (with --columns), a --columns name not in the header, an empty
input without --headers.  Narrowed:
ASCII only, a lone '\\r' line end, positions other than [+-]?[0-9]+ within int64, and coordinate or predefined windows over
positions that decrease within a scaffold run.  Blank lines are skipped.  --verbose and --writeFailedWindows have no effect,
as in the reference."""
from __future__ import annotations

import argparse
import re

import numpy as np

from .. import geno_io
from .. import windows as W
from ..engine import Engine
from . import _common as C
from ._stream import body_chunks, env_int, first_line, open_input, open_output

STATS = ("mean", "median", "min", "max", "sd", "sum", "q5", "q10", "q25", "q75", "q90", "q95")
CODES = {"mean": (0, 0.0), "median": (1, 0.0), "min": (2, 0.0), "max": (3, 0.0), "sd": (4, 0.0), "sum": (5, 0.0),
         "q5": (6, 0.05), "q10": (6, 0.1), "q25": (6, 0.25), "q75": (6, 0.75), "q90": (6, 0.9), "q95": (6, 0.95)}
TOK = re.compile(rb"[^ \t\n\r\x0b\x0c\x1c-\x1f]+")
# error codes of pg_ws_chunk (include/pgwin.h); %s takes the column name where the code names one
ERRORS = {1: "the position is not an integer of the form [+-]digits (the reference's int() fails on it, or accepts a form "
             "such as 1_000 that this engine does not)",
          2: "the line has no position field (the reference fails with an IndexError)",
          3: "the position is outside the int64 range",
          4: "the line's field count differs from the header's (the reference fails with an AssertionError)",
          5: "a byte outside ASCII (the reference reads characters, which this engine does not)",
          6: "a '\\r' ends a line by itself (the reference reads it as a line end, this engine does not)",
          7: "the line has no column %s (the reference fails with a KeyError)"}


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--windType", help="Type of windows to make", choices=("sites", "coordinate", "predefined"),
                   default="coordinate")
    p.add_argument("-w", "--windSize", help="Window size in bases", type=int, metavar="sites")
    p.add_argument("-s", "--stepSize", help="Step size for sliding window", type=int, metavar="sites")
    p.add_argument("-m", "--minSites", help="Minumum good sites per window", type=int, metavar="sites", default=1)
    p.add_argument("-O", "--overlap", help="Overlap for sites sliding window", type=int, metavar="sites")
    p.add_argument("-D", "--maxDist", help="Maximum span distance for sites window", type=int)
    p.add_argument("--windCoords", help="Window coordinates file (scaffold start end)")
    p.add_argument("--stats", help="Which statistics to compute", nargs="+", choices=STATS,
                   default=("mean", "median", "min", "max", "sd", "sum"))
    p.add_argument("-i", "--inFile", help="Input file (.gz allowed; default stdin)")
    p.add_argument("-o", "--outFile", help="Results file (.gz allowed; default stdout)")
    p.add_argument("--headers", help="Headers text (separated by spaces) if no header in input", nargs="+")
    p.add_argument("--columns", help="Columns to analyse, separated by spaces", nargs="+")
    p.add_argument("--exclude", help="File of scaffolds to exclude")
    p.add_argument("--include", help="File of scaffolds to analyse")
    p.add_argument("--verbose", help="Verbose output (no effect, as in the reference)", action="store_true")
    p.add_argument("--writeFailedWindows", help="No effect, as in the reference", action="store_true")
    p.add_argument("--device", help="CUDA device index", type=int, default=0)
    p.add_argument("--devices", help="Number of GPUs (only 1)", type=int, default=None)
    p.add_argument("--timing", help="Write a JSON file with the wall time of each phase and the device time of each kernel",
                   metavar="FILE")
    return p


def _fail(msg):
    raise SystemExit("windowStats: " + msg)


def check_args(args):
    """the reference's assertions (windowStats.py:56-82); returns (minSites, windCoords)"""
    coords = None
    if args.windType == "coordinate":
        tests = [(args.windSize, "Window size must be provided."),
                 (not args.overlap, "Overlap does not apply to coordinate windows. Use --stepSize instead."),
                 (not args.maxDist, "Maximum distance only applies to sites windows.")]
    elif args.windType == "sites":
        tests = [(args.windSize, "Window size (number of sites) must be provided."),
                 (not args.stepSize, "Step size only applies to coordinate windows. Use --overlap instead.")]
    else:
        tests = [(args.windCoords, "Please provide a file of window coordinates."),
                 (not args.overlap, "Overlap does not apply for predefined windows."),
                 (not args.maxDist, "Maximum does not apply for predefined windows."),
                 (not args.stepSize, "Step size does not apply for predefined windows."),
                 (not args.include, "You cannot only include specific scaffolds if using predefined windows."),
                 (not args.exclude, "You cannot exclude specific scaffolds if using predefined windows.")]
    for ok, msg in tests:
        if not ok:
            _fail(msg)
    if args.windType == "predefined":
        with open(args.windCoords, "r") as wc:
            coords = tuple([(x, int(y), int(z)) for x, y, z in [line.split()[:3] for line in wc]])
    min_sites = args.minSites
    if not min_sites:
        min_sites = args.windSize
    return min_sites, coords


def read_scafs(path):
    if not path:
        return None
    with open(path, "r") as f:
        return [line.rstrip() for line in f]


def plan(names, columns):
    """output names, the value column every output column reads, the distinct columns (slots) and the slot of every output
    column.  Without --columns, a name read more than once takes its first column (GenoWindow.seqDict's names.index); with
    --columns, its last (dict(zip(names, GTs)) in parseGenoLine)."""
    if columns:
        last = {n: c for c, n in enumerate(names)}
        for n in columns:
            if n not in last:
                _fail("column %s is not in the header (the reference fails with a KeyError)" % n)
        out_names, read = list(columns), [last[n] for n in columns]
    else:
        out_names, read = list(names), [names.index(n) for n in names]
    cols = sorted(set(read))
    slot_of = {c: k for k, c in enumerate(cols)}
    col_slot = [slot_of.get(c, -1) for c in range(len(names))]
    return out_names, col_slot, len(cols), [slot_of[c] for c in read]


def main(argv=None):
    args = build_parser().parse_args(argv)
    if args.devices not in (None, 1):
        _fail("--devices is not supported; the statistics run on one GPU")
    min_sites, coords = check_args(args)
    include, exclude = read_scafs(args.include), read_scafs(args.exclude)
    codes = [CODES[s][0] for s in args.stats]
    qs = [CODES[s][1] for s in args.stats]
    tm = C.Timing(args.timing)
    src = open_input(args.inFile)
    if args.headers:
        head, body0 = " ".join(args.headers).encode(), b""
    else:
        first = first_line(src)
        if first is None:
            _fail("the input is empty: it has no header line (the reference fails with a StopIteration)")
        head, body0 = first
    try:
        names = head.decode("ascii").split()[2:]
    except UnicodeDecodeError:
        _fail("the header has a byte outside ASCII (this engine reads ASCII text only)")
    out_names, col_slot, n_slots, out_slot = plan(names, args.columns)
    target = env_int("PG_WS_CHUNK_BYTES", 256 << 20)
    budget = env_int("PG_WS_SORT_BYTES", 1 << 30)
    with Engine(args.device) as eng:
        eng.ws_spec(col_slot, n_slots, -1 if args.columns else len(names))
        run_names, run_start = [], []       # scaffold runs over all data lines
        rejected = []                       # (data line, slot, file line) of tokens float() rejects
        n_lines, lines_before, n_host = 0, 1 if not args.headers else 0, 0
        for chunk in body_chunks(body0, src, target):
            tm.mark("read")
            S, run_line, run_off, fidx, ftok, err = eng.ws_chunk(chunk)
            tm.mark("parse", eng)
            if err[0]:
                _fail(_message(err, chunk, lines_before, [out_names[out_slot.index(k)] if k in out_slot else "?"
                                                          for k in range(n_slots)]))
            for ln, o in zip(run_line, run_off):
                nm = TOK.search(chunk, int(o)).group().decode()
                if not run_names or run_names[-1] != nm:
                    run_names.append(nm)
                    run_start.append(n_lines + int(ln))
            if len(fidx):
                slot, line = np.divmod(fidx, S)
                off = (ftok >> np.uint64(32)).astype(np.int64)
                ln_ = ((ftok >> np.uint64(2)) & np.uint64((1 << 30) - 1)).astype(np.int64)
                st = (ftok & np.uint64(3)).astype(np.int64)
                fix = ([], [], [])
                for k in range(len(fidx)):
                    tok = chunk[off[k]:off[k] + ln_[k]]
                    v = None
                    if st[k] == 2:
                        n_host += 1
                        try:
                            v = float(tok.decode())
                        except ValueError:
                            v = None
                    if v is None:
                        rejected.append((n_lines + int(line[k]), int(slot[k]),
                                         lines_before + chunk.count(b"\n", 0, int(off[k])) + 1, tok.decode()))
                    else:
                        fix[0].append(n_lines + int(line[k]))
                        fix[1].append(int(slot[k]))
                        fix[2].append(v)
                eng.ws_set_values(*fix)
            n_lines += S
            lines_before += chunk.count(b"\n")
            tm.mark("host_tokens")
        pos = eng.ws_meta()
        scaf_ids = np.zeros(n_lines, np.int64)
        uniq = {}
        ids = [uniq.setdefault(n, len(uniq)) for n in run_names]
        bounds = run_start + [n_lines]
        for r in range(len(run_start)):
            scaf_ids[bounds[r]:bounds[r + 1]] = ids[r]
        scaf_names = list(uniq)
        if args.windType != "sites" and n_lines > 1:
            same = scaf_ids[1:] == scaf_ids[:-1]
            down = np.flatnonzero(same & (pos[1:] < pos[:-1]))
            if len(down):
                _fail("data line %d: position %d is below the one before it on scaffold %s (coordinate and predefined "
                      "windows need positions that do not decrease within a scaffold)" % (
                          down[0] + 2, pos[down[0] + 1], scaf_names[scaf_ids[down[0] + 1]]))
        if args.windType == "coordinate":
            ws = W.sliding_coord_windows(scaf_ids, scaf_names, pos, args.windSize, args.stepSize or args.windSize,
                                         include, exclude)
        elif args.windType == "sites":
            ws = W.sliding_sites_windows(scaf_ids, scaf_names, pos, args.windSize, args.overlap or 0,
                                         args.maxDist if args.maxDist else None, min_sites, include, exclude)
        else:
            ws = W.predefined_coord_windows(scaf_ids, scaf_names, pos, coords)
        tm.mark("windows")
        lo, hi = ws.ranges()
        sites = hi - lo
        ev = np.flatnonzero(sites >= min_sites)
        if rejected and len(ev):
            rl = np.array([r[0] for r in rejected], np.int64)
            order = np.argsort(rl, kind="stable")
            for w in ev:
                a, b = np.searchsorted(rl[order], [lo[w], hi[w]])
                if b > a:
                    r = rejected[order[a]]
                    _fail("line %d: float() rejects the value %r of column %s, inside window %d (%s:%s-%s) (the reference "
                          "fails with a ValueError)" % (r[2], r[3], _slot_name(r[1], out_names, out_slot), w + 1,
                                                        ws.scaffold[w], _lim(ws, w, pos, 0), _lim(ws, w, pos, 1)))
        vals, cnt = eng.ws_stats(lo[ev], hi[ev], codes, qs, n_slots, budget)
        tm.mark("stats", eng)
    if any(c in (2, 3) for c in codes) and len(ev):
        empty = np.argwhere(cnt[:, out_slot] == 0)
        if len(empty):
            w, j = ev[empty[0][0]], empty[0][1]
            _fail("window %d (%s:%s-%s) has no value in column %s: its min and max are undefined (the reference fails with a "
                  "ValueError)" % (w + 1, ws.scaffold[w], _lim(ws, w, pos, 0), _lim(ws, w, pos, 1), out_names[j]))
    K = len(codes)
    M = np.full((len(ws), len(out_names) * K), np.nan)
    if len(ev):
        M[ev] = vals[:, out_slot, :].reshape(len(ev), -1)
    prefixes = []
    for w in range(len(ws)):
        n = int(sites[w])
        p = pos[lo[w]:hi[w]]
        if args.windType == "sites":
            start, end = (int(p.min()), int(p.max())) if n else (None, None)
        else:
            start, end = ws.start[w], ws.end[w]
        mid = W.mid_pos(int(p.sum()), n)
        prefixes.append("%s,%s,%s,%s,%d," % (ws.scaffold[w], start, end, mid, n))
    with open_output(args.outFile) as out:
        out.write(b"scaffold,start,end,mid,sites")
        if len(ws):
            out.write("".join("," + ",".join(n + "_" + s for s in args.stats) for n in out_names).encode() + b"\n")
            if M.shape[1]:
                out.write(geno_io.format_matrix_rows(M, sep=",", prefixes=prefixes).encode())
            else:
                out.write("".join(p + "\n" for p in prefixes).encode())
    tm.mark("write")
    tm.write(lines=n_lines, windows=len(ws), host_tokens=n_host)


def _lim(ws, w, pos, k):
    if ws.start[w] is None:
        p = pos[ws.lo[w]:ws.hi[w]]
        return int(p.min() if k == 0 else p.max())
    return ws.start[w] if k == 0 else ws.end[w]


def _slot_name(slot, out_names, out_slot):
    return out_names[out_slot.index(slot)]


def _message(err, chunk, lines_before, slot_names):
    """'line N: ...' in the file's numbering for the error (code, data line of the chunk, slot)"""
    code, line, slot = err
    starts = [m.start() for m in re.finditer(rb"(?m)^(?!#)[ \t\r\x0b\x0c]*[^ \t\r\x0b\x0c\n]", chunk)]
    off = starts[line] if line < len(starts) else 0
    msg = ERRORS.get(code, "error %d" % code)
    if code == 7:
        msg = msg % slot_names[slot]
    return "line %d: %s" % (lines_before + chunk.count(b"\n", 0, off) + 1, msg)


if __name__ == "__main__":
    main()
