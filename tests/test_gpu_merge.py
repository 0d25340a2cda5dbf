"""mergeGeno.py on the device: every fixture of the unmodified reference (tests/golden/merge14) with default and tiny chunks and
slabs, and the device against a vectorised numpy statement of the merge (per-file valid prefix, np.unique of the keys, the
write rule) at its edges: 1, 2 and 33 files, stalls at chunk boundaries and on the first and last line, positions where the
decimal width changes, a 3 x 10^7 walk written whole by --method all, and 8 files x 2 M lines."""

import numpy as np
import pytest

from test_merge_cpu import OK, TINY, case_argv, expected, run_cli

pytestmark = pytest.mark.gpu
METHOD = {"intersect": 0, "union": 1, "all": 2}


@pytest.mark.parametrize("env", [None, TINY], ids=["default", "tiny"])
@pytest.mark.parametrize("case", OK, ids=[c["name"] for c in OK])
def test_device_matches_reference(case, env, tmp_path, monkeypatch):
    if env is not None and case["name"].startswith("medium"):
        env = dict(env, PG_MERGE_CHUNK_BYTES="4096")
    assert run_cli(case_argv(case), case["dest"], tmp_path, monkeypatch, None, env) == expected(case)


def expect(fai, keys, toks, n_dummy, method, union_min=1, must_first=0, sep="\t", missing="N"):
    """the rows for files whose merged lines are keys[x] (sorted walk indices; the valid prefix) and whose every line carries
    the genotypes toks[x]"""
    names = [n for n, l in fai if l > 0]
    off = np.cumsum([0] + [l for n, l in fai if l > 0])
    total = int(off[-1])
    nF = len(keys)
    allk = np.concatenate([np.asarray(k, np.int64) for k in keys]) if nF else np.zeros(0, np.int64)
    uk, cnt = np.unique(allk, return_counts=True)
    mask = np.zeros(len(uk), np.int64)
    for x, k in enumerate(keys):
        mask[np.searchsorted(uk, k)] |= 1 << x
    need = min(max(must_first, 0), nF)
    umin = max(union_min, must_first)
    dense = (method == 2 or (method == 1 and umin <= 0)) and need == 0
    if dense:
        rows = np.arange(total, dtype=np.int64)
        m = np.zeros(total, np.int64)
        m[uk] = mask
    else:
        ok = (mask & ((1 << need) - 1)) == (1 << need) - 1
        if method == 0:
            ok &= cnt == nF
        elif method == 1:
            ok &= cnt >= umin
        rows, m = uk[ok], mask[ok]
    tails = {}
    out = []
    scaf = np.searchsorted(off, rows, side="right") - 1
    site = rows - off[scaf] + 1
    for s, p, mm in zip(scaf.tolist(), site.tolist(), m.tolist()):
        t = tails.get(mm)
        if t is None:
            t = tails[mm] = "".join(((sep + sep.join(toks[x])) if toks[x] else "") if (mm >> x) & 1
                                    else (sep + missing) * n_dummy[x] for x in range(nF))
        out.append("%s%s%d%s\n" % (names[s], sep, p, t))
    return "".join(out).encode()


def write_inputs(tmp_path, fai, keys, toks, stall_lines=None):
    names = [n for n, l in fai if l > 0]
    off = np.cumsum([0] + [l for n, l in fai if l > 0])
    f = tmp_path / "x.fai"
    f.write_text("".join("%s\t%d\n" % (n, l) for n, l in fai))
    paths = []
    for x, k in enumerate(keys):
        k = np.asarray(k, np.int64)
        scaf = np.searchsorted(off, k, side="right") - 1
        site = k - off[scaf] + 1
        tail = ("\t" + "\t".join(toks[x])) if toks[x] else ""
        head = "\t".join(["#CHROM", "POS"] + ["f%d_%d" % (x, j) for j in range(len(toks[x]))])
        body = "".join("%s\t%d%s\n" % (names[s], p, tail) for s, p in zip(scaf.tolist(), site.tolist()))
        if stall_lines and stall_lines[x]:
            body += stall_lines[x]
        p = tmp_path / ("in%d.geno" % x)
        p.write_bytes((head + "\n" + body).encode())
        paths.append(str(p))
    return str(f), paths


def run(tmp_path, monkeypatch, fai, keys, toks, method, env=None, union_min=1, must_first=0, stall_lines=None, sep="\t"):
    f, paths = write_inputs(tmp_path, fai, keys, toks, stall_lines)
    argv = sum((["-i", p] for p in paths), []) + ["-f", f, "--method", method, "--unionMin", str(union_min),
                                                   "--mustIncludeFirst", str(must_first), "--outSep", sep]
    got = run_cli(argv, "stdout", tmp_path, monkeypatch, None, env)
    head = sep.join(["#CHROM" + sep + "POS", sep.join(sep.join("f%d_%d" % (x, j) for j in range(len(toks[x])))
                                                     for x in range(len(keys)))])
    want = head.encode() + b"\n" + expect(fai, keys, toks, [len(t) for t in toks], METHOD[method], union_min, must_first,
                                          sep)
    return got, want


def random_keys(rng, total, n, frac):
    return [np.sort(rng.choice(total, size=int(total * frac), replace=False)) for _ in range(n)]


@pytest.mark.parametrize("nF", [1, 2, 33])
@pytest.mark.parametrize("method,union_min,must_first", [("intersect", 1, 0), ("union", 1, 0), ("union", 0, 0),
                                                         ("union", 2, 1), ("all", 1, 0), ("all", 1, 2)])
def test_file_counts_and_rules(nF, method, union_min, must_first, tmp_path, monkeypatch):
    rng = np.random.default_rng(nF * 7 + union_min)
    fai = [("s1", 300), ("s0", 0), ("s2", 200)]
    keys = random_keys(rng, 500, nF, 0.9 if method == "intersect" else 0.3)
    toks = [["A/C"] * (x % 4) for x in range(nF)]
    for env in (None, {"PG_MERGE_CHUNK_BYTES": "100", "PG_MERGE_SLAB_BYTES": "64", "PG_MERGE_DENSE_ROWS": "33"}):
        got, want = run(tmp_path, monkeypatch, fai, keys, toks, method, env, union_min, must_first)
        assert got == want


@pytest.mark.parametrize("where", ["first", "last", "boundary"])
def test_stalls_on_first_last_line_and_chunk_boundaries(where, tmp_path, monkeypatch):
    rng = np.random.default_rng(3)
    fai = [("s1", 2000)]
    keys = random_keys(rng, 1990, 3, 0.4)
    toks = [["G/T"], ["A/A", "C/C"], []]
    after = "s1\t1999\tA\ns1\t2000\tA\n"         # valid lines the stall hides
    for chunk in (160, 161, 200, 241, 4096):
        ks = list(keys)
        stall = [None, None, None]
        if where == "first":
            ks[0] = keys[0][:0]
            stall[0] = "s1\t0\tA\n" + after
        elif where == "last":
            stall[1] = "s1\t1\tA/A\tC/C\n"
        else:                                    # lines of 8-10 bytes: the stall falls at or near a chunk's first line
            k = chunk // 9
            ks[2] = keys[2][:k]
            stall[2] = "s1\t%d\n" % (keys[2][k - 1] + 1) + after
        env = {"PG_MERGE_CHUNK_BYTES": str(chunk), "PG_MERGE_SLAB_BYTES": "50"}
        f, paths = write_inputs(tmp_path, fai, ks, toks, stall)
        argv = sum((["-i", p] for p in paths), []) + ["-f", f, "--method", "union"]
        got = run_cli(argv, "stdout", tmp_path, monkeypatch, None, env)
        assert got.split(b"\n", 1)[1] == expect(fai, ks, toks, [len(t) for t in toks], 1), chunk


def test_positions_where_the_decimal_width_changes(tmp_path, monkeypatch):
    fai = [("a", 10 ** 6 + 3), ("b", 10 ** 5), ("c", 12)]
    off = [0, 10 ** 6 + 3, 10 ** 6 + 3 + 10 ** 5]
    sites = [(0, p) for p in (1, 9, 10, 11, 99, 100, 101, 999, 1000, 9999, 10000, 99999, 100000, 999999, 10 ** 6,
                               10 ** 6 + 3)] + [(1, p) for p in (1, 9, 10, 99999, 100000)] + [(2, p) for p in (9, 10, 12)]
    k = np.array([off[s] + p - 1 for s, p in sites], np.int64)
    keys = [k, k[::2], k[1::3]]
    toks = [["A/T"], [], ["C/G", "N/N"]]
    for env in (None, {"PG_MERGE_CHUNK_BYTES": "64", "PG_MERGE_SLAB_BYTES": "40"}):
        for method in ("intersect", "union"):
            got, want = run(tmp_path, monkeypatch, fai, keys, toks, method, env)
            assert got == want
        got, want = run(tmp_path, monkeypatch, fai, keys, toks, "union", env, sep=" :: ")
        assert got == want


def test_all_over_a_3e7_walk_with_small_slabs(tmp_path, monkeypatch):
    fai = [("chrA", 10 ** 7), ("chrB", 10 ** 7), ("chrC", 10 ** 7)]
    rng = np.random.default_rng(30)
    keys = random_keys(rng, 3 * 10 ** 7, 1, 0.002)
    f, paths = write_inputs(tmp_path, fai, keys, [["A/A"]])
    got = run_cli(["-i", paths[0], "-f", f, "--method", "all"], "stdout", tmp_path, monkeypatch, None,
                  {"PG_MERGE_SLAB_BYTES": str(1 << 16), "PG_MERGE_CHUNK_BYTES": str(1 << 14)})
    body = memoryview(got)[got.index(b"\n") + 1:]
    # the expected text, scaffold by scaffold in pieces of 10^6 sites
    hit = np.zeros(3 * 10 ** 7, bool)
    hit[keys[0]] = True
    at = 0
    for s, (name, n) in enumerate(fai):
        for p0 in range(0, n, 10 ** 6):
            h = hit[s * 10 ** 7 + p0:s * 10 ** 7 + p0 + 10 ** 6]
            piece = "".join("%s\t%d\t%s\n" % (name, p0 + i + 1, "A/A" if h[i] else "N") for i in range(len(h))).encode()
            assert body[at:at + len(piece)] == piece, (name, p0)
            at += len(piece)
    assert at == len(body)


def test_eight_files_of_two_million_lines(tmp_path, monkeypatch):
    fai = [("chrA", 10 ** 7), ("chrB", 10 ** 7), ("chrC", 10 ** 7)]
    rng = np.random.default_rng(8)
    keys = [np.sort(rng.choice(3 * 10 ** 7, size=2 * 10 ** 6, replace=False)) for _ in range(8)]
    toks = [["A/C", "G/T"][: 1 + x % 2] for x in range(8)]
    got, want = run(tmp_path, monkeypatch, fai, keys, toks, "union", {"PG_MERGE_CHUNK_BYTES": str(8 << 20)})
    assert got == want
    got, want = run(tmp_path, monkeypatch, fai, keys, toks, "union", None, union_min=3, must_first=1)
    assert got == want
