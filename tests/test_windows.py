"""CPU tests of the host window logic (genomics_general_b200/windows.py) against
 (a) the reference generators' output (tests/golden/generator_cases.json) and
 (b) the oracle's literal state-machine restatement on random inputs."""
import json
import math
import os

import numpy as np
import pytest

from genomics_general_b200 import windows as W
from oracle import dense_oracle as do
from helpers import GOLDEN

GEN = json.load(open(os.path.join(GOLDEN, "generator_cases.json")))


def _ids(scaf):
    names = []
    ids = []
    for s in scaf:
        if not names or names[-1] != s:
            if s in names:
                names.append(s)         # a scaffold that re-appears later is a new run; same name
            else:
                names.append(s)
        ids.append(len(names) - 1)
    return np.array(ids, dtype=np.int32), names


def _run(kind, p, scaf, pos):
    ids, names = _ids(scaf)
    if kind == "coordinate":
        return W.sliding_coord_windows(ids, names, pos, p["windSize"], p["stepSize"], exclude=p.get("exclude"))
    if kind == "sites":
        return W.sliding_sites_windows(ids, names, pos, p["windSites"], p["overlap"], p["maxDist"], p["minSites"],
                                       exclude=p.get("exclude"))
    return W.predefined_coord_windows(ids, names, pos, [tuple(c) for c in p["windCoords"]])


@pytest.mark.parametrize("idx", range(len(GEN["cases"])))
def test_against_reference_generators(idx):
    case = GEN["cases"][idx]
    scaf, pos = GEN["scaffolds"], GEN["positions"]
    ws = _run(case["kind"], case["params"], scaf, pos)
    assert len(ws) == len(case["windows"])
    for k, r in enumerate(case["windows"]):
        assert ws.scaffold[k] == r["scaffold"]
        assert [pos[i] for i in range(ws.lo[k], ws.hi[k])] == r["positions"], (k, ws.lo[k], ws.hi[k])
        if case["kind"] != "sites":
            assert [ws.start[k], ws.end[k]] == r["limits"]
        assert ws.ID[k] == r["ID"], (k, ws.ID[k], r["ID"])       # windowID column of --addWindowID


def _random_layout(rng):
    scaf, pos = [], []
    for k in range(int(rng.integers(1, 5))):
        n = int(rng.integers(1, 120))
        span = int(rng.integers(n, 40 * n + 2))
        p = np.sort(rng.choice(np.arange(1, span + 1), size=n, replace=False))
        scaf += ["sc%d" % k] * n
        pos += [int(x) for x in p]
    return scaf, pos


@pytest.mark.parametrize("seed", range(25))
def test_coordinate_against_oracle_state_machine(seed):
    rng = np.random.default_rng(seed)
    scaf, pos = _random_layout(rng)
    wsz = int(rng.integers(5, 400))
    step = [None, int(rng.integers(1, 500))][int(rng.integers(0, 2))]
    ws = _run("coordinate", dict(windSize=wsz, stepSize=step), scaf, pos)
    ref = do.sliding_coord_windows(scaf, pos, wsz, step)
    assert len(ws) == len(ref)
    for k, r in enumerate(ref):
        assert (ws.scaffold[k], ws.start[k], ws.end[k]) == (r["scaffold"], r["start"], r["end"])
        assert list(range(ws.lo[k], ws.hi[k])) == r["sites"]


@pytest.mark.parametrize("seed", range(40))
def test_sites_against_oracle_state_machine(seed):
    rng = np.random.default_rng(100 + seed)
    scaf, pos = _random_layout(rng)
    wsz = int(rng.integers(2, 40))
    ov = int(rng.integers(0, wsz))
    ms = [None, int(rng.integers(1, wsz + 1))][int(rng.integers(0, 2))]
    md = [None, int(rng.integers(5, 300))][int(rng.integers(0, 2))]
    try:
        ref = do.sliding_sites_windows(scaf, pos, wsz, ov, md if md else math.inf, ms)
    except AssertionError:
        with pytest.raises(RuntimeError):
            _run("sites", dict(windSites=wsz, overlap=ov, maxDist=md, minSites=ms), scaf, pos)
        return
    ws = _run("sites", dict(windSites=wsz, overlap=ov, maxDist=md, minSites=ms), scaf, pos)
    assert len(ws) == len(ref)
    for k, r in enumerate(ref):
        assert ws.scaffold[k] == r["scaffold"]
        assert list(range(ws.lo[k], ws.hi[k])) == r["sites"]


@pytest.mark.parametrize("seed", range(25))
def test_predefined_against_oracle_state_machine(seed):
    rng = np.random.default_rng(500 + seed)
    scaf, pos = _random_layout(rng)
    names = sorted(set(scaf), key=scaf.index)
    coords = []
    for sc in names:
        if rng.random() < 0.25:
            continue
        mx = max(p for s, p in zip(scaf, pos) if s == sc)
        start = 1
        for _ in range(int(rng.integers(1, 6))):
            start = start + int(rng.integers(0, max(2, mx // 3)))
            end = start + int(rng.integers(0, max(2, mx // 2)))
            coords.append((sc, start, end))
    if not coords:
        coords = [(names[0], 1, 10)]
    ws = _run("predefined", dict(windCoords=coords), scaf, pos)
    ref = do.predefined_coord_windows(scaf, pos, coords)
    assert len(ws) == len(ref)
    for k, r in enumerate(ref):
        assert (ws.scaffold[k], ws.start[k], ws.end[k]) == (r["scaffold"], r["start"], r["end"])
        assert list(range(ws.lo[k], ws.hi[k])) == r["sites"], (k, coords)


def test_mid_pos_matches_python_round():
    assert W.mid_pos(5, 2) == 2          # 2.5 -> 2 (banker's)
    assert W.mid_pos(7, 2) == 4          # 3.5 -> 4
    assert math.isnan(W.mid_pos(0, 0))


def test_geno_window_mutators_follow_the_reference_container():
    """GenoWindow.addSite / addBlock / slide / trim (genomics.py:1745-1788) on the dense-backed mirror: positions, token
    rows and the int8 matrix stay aligned; the expected states are the reference container's (the same calls on
    genomics_general/genomics.GenoWindow give these lists — the `[:-0]` slice of trim included; the reference's own
    addBlock cannot run: its chained comparison of a list / array of positions raises, genomics.py:1749)."""
    from genomics_general_b200 import genomics as G
    w = G.GenoWindow(scaffold="chr1", limits=[1, 100], names=["a", "b"], ploidy=[2, 2])
    w.addSite(["A/T", "N/N"], 5)
    w.addSite(["C/C", "G/T"], 17)
    w.addBlock([["A/A", "A/A"], ["T/T", "N/G"], ["G/G", "C/C"]], [30, 42, 88])
    assert w.seqLen() == 5 and w.firstPos() == 5 and w.lastPos() == 88 and w.midPos() == 36
    assert w.geno.tolist() == [[0, 3, -1, -1], [1, 1, 2, 3], [0, 0, 0, 0], [3, 3, -1, 2], [2, 2, 1, 1]]
    assert w.seqDict()["b"] == ["N/N", "G/T", "A/A", "N/G", "C/C"]
    with pytest.raises(AssertionError):
        w.addSite(["A/A", "A/A"], 101)
    with pytest.raises(AssertionError):
        w.addSite(["A/A"], 50)
    w.addSite(["T/T", "T/T"], ignorePosition=True)
    assert np.isnan(w.positions[-1]) and w.seqLen() == 6
    w.trim(right=True, remove=1)
    w.slide(step=15)                                    # limits 16..115: the site at 5 leaves
    assert w.limits == [16, 115] and w.positions == [17, 30, 42, 88]
    assert w.geno.tolist() == [[1, 1, 2, 3], [0, 0, 0, 0], [3, 3, -1, 2], [2, 2, 1, 1]]
    w.slide(newLimits=[31, 60])
    assert w.positions == [42, 88]                      # only the left edge drops sites (1773-1777)
    w.trim(leave=1)
    assert w.positions == [88] and w.sites == [["G/G", "C/C"]] and w.geno.tolist() == [[2, 2, 1, 1]]
    c = w.copy()
    c.trim(right=True, leave=1)                         # nothing to remove -> the reference's slice [:-0] empties the window
    assert c.positions == [] and c.seqLen() == 0 and c.geno.shape == (0, 4)
    assert w.positions == [88]
    with pytest.raises(TypeError):
        w.trim(right=True, remove=0)                    # seqLen() - None, as in the reference


def test_line_readers_follow_the_reference():
    """parseGenoLine / GenoFileReader / makeHaploidNames of the drop-in API (genomics.py:1884-1945, 448-453) against what
    the reference returns for the same text (tests/golden/reader_cases.json, written by running the reference's own
    classes): dict and list rows, '#' lines skipped, phased genotypes split into alleles, the parsed-line cache counter,
    the end-of-file record, integer / float tables."""
    import io
    from genomics_general_b200 import genomics as G
    c = json.load(open(os.path.join(GOLDEN, "reader_cases.json")))
    for name in ("plain", "split2", "split212"):
        e = c[name]
        kw = e["kw"]
        assert G.GenoFileReader(io.StringIO(c["text"]), **kw).names == e["names"]
        assert list(G.GenoFileReader(io.StringIO(c["text"]), **kw).siteBySite(asDict=True)) == e["dict_rows"]
        assert list(G.GenoFileReader(io.StringIO(c["text"]), **kw).siteBySite(asDict=False)) == e["list_rows"]
        r = G.GenoFileReader(io.StringIO(c["text"]), **kw)
        assert [r.nextSite() for _ in range(5)] == e["next5"]
        assert r.precompDict["__counter__"] == e["counter"]
    assert list(G.GenoFileReader(io.StringIO(c["counts_text"]), type=int).siteBySite()) == c["counts_rows"]
    assert G.parseGenoLine("x 1.5 2", ["u"], posCol=-1, firstSampleCol=1, type=float, asDict=False) == c["float_line"]
    assert G.parseGenoLine("", ["u"]) == c["empty_line"]
    assert [G.makeHaploidNames(["a", "b"], 1), G.makeHaploidNames(["a", "b"], [3, 1])] == c["haploid_names"]
