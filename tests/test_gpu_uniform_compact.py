"""The varied-row stream's two passes per tile (csrc/k1.cu k1_site_pass_packed<..., UNI = true>): pass V walks a tile's varied
rows, packed onto the team's lanes, Gv lanes per row (the plan's per site; PG_K1_UNI_GV forces 1 .. 32), and pass U adds every
slot's position and the sums of the uniform sites without a walk, on the warps that walked no row when there are enough of
them.  Every record field, popFreq columns included, must be bit-identical to the packed pass that streams every row
(PG_K1_NO_UNIFORM) and to the byte pass (PG_K1_BYTE_PASS).  The data are laid out on the stream's own tiles
(Engine.uniform_tile), and the cases cover tiles with no varied row, with exactly as many rows as the team has lanes at each
Gv, and with more rows than lanes; segment boundaries inside a warp's rows, 1-site and overlapping windows; forced flushes;
uniform-missing sites at tile edges; forced geometries; H from 1 to 1600 with 1 to 9 populations."""
import numpy as np
import pytest

from test_gpu_uniform_sites import genotypes, layout, three_passes

pytestmark = pytest.mark.gpu

GVS = [None, 1, 2, 4, 8, 32]


@pytest.fixture(scope="module")
def eng():
    from genomics_general_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(autouse=True)
def _no_gv(monkeypatch):
    monkeypatch.delenv("PG_K1_UNI_GV", raising=False)


def gv_knobs(gv, **more):
    knobs = {k: str(v) for k, v in more.items()}
    if gv is not None:
        knobs["PG_K1_UNI_GV"] = str(gv)
    return knobs


def tiled(rng, S, H, T, counts):
    """tile t (T sites) has counts[t % len(counts)] varied sites at random slots; the other sites are uniform, a tenth of
    them missing in every haplotype, and so are the first and last slot of every third tile"""
    g, _ = genotypes(rng, S, H, 0.0)
    ref = rng.integers(0, 4, S)
    varied = np.zeros(S, bool)
    for t, s0 in enumerate(range(0, S, T)):
        n = min(counts[t % len(counts)], min(T, S - s0))
        varied[s0 + rng.choice(min(T, S - s0), n, replace=False)] = True
    uni = ~varied
    g[uni] = ref[uni, None]
    g[uni & (rng.random(S) < 0.1)] = -1
    for s0 in range(0, S, 3 * T):
        for s in (s0, min(s0 + T, S) - 1):
            g[s] = -1
    g[-1] = -1
    return g, varied


def dense_windows(rng, S, varied):
    """random windows, 1-site windows over the first tiles, windows that start or end at varied sites (segment boundaries
    between the rows of one warp), and overlapping windows sliding by 7 sites"""
    lo = [rng.integers(0, S, 40)]
    hi = [np.minimum(lo[0] + rng.integers(1, 900, 40), S)]
    one = np.arange(0, min(S, 2000))
    lo.append(one)
    hi.append(one + 1)
    vs = np.flatnonzero(varied)
    pick = vs[rng.permutation(len(vs))[:300]] if len(vs) else np.zeros(0, np.int64)
    lo.append(pick)
    hi.append(np.minimum(pick + rng.integers(1, 40, len(pick)), S))
    lo.append(np.maximum(pick - rng.integers(1, 40, len(pick)), 0))
    hi.append(pick + 1)
    slide = np.arange(0, S - 50, 7)
    lo.append(slide)
    hi.append(slide + 50)
    return np.concatenate(lo).astype(np.int64), np.concatenate(hi).astype(np.int64)


def stream_tile(eng, monkeypatch, S, H, P):
    """(sites per tile, lanes per team) of the varied-row stream at this shape and under the knobs set now, from a popgen call
    on placeholder data of the shape"""
    g, _ = genotypes(np.random.default_rng(0), S, H, 0.7)
    eng.upload(g, np.arange(1, S + 1, dtype=np.int32))
    eng.set_pops(layout(np.random.default_rng(1), H, P), P)
    eng.set_windows(np.array([0], np.int64), np.array([S], np.int64))
    monkeypatch.setenv("PG_K1_UNIFORM_FORCE", "1")
    eng.popgen(1, 0.01)
    monkeypatch.delenv("PG_K1_UNIFORM_FORCE")
    T, wpt = eng.uniform_tile()
    assert T > 0 and wpt > 0
    return T, 32 * wpt


def counts_for(T, lanes):
    """per-tile varied rows: none, exactly the team's lanes at Gv = 1, 2, 4, 8, 32, one row, and more rows than lanes (up to
    every site of the tile)"""
    c = [0, lanes, lanes // 2, lanes // 4, lanes // 8, lanes // 32, 1, lanes + 1, (lanes + T) // 2, T, 0, lanes // 2 + 1,
         lanes - 1]
    return [min(max(x, 0), T) for x in c]


def load(eng, rng, g, P, varied):
    S, H = g.shape
    eng.upload(g, np.cumsum(rng.integers(1, 50, S)).astype(np.int32))
    eng.set_pops(layout(rng, H, P), P)
    lo, hi = dense_windows(rng, S, varied)
    eng.set_windows(lo, hi)


@pytest.mark.parametrize("gv", GVS, ids=str)
def test_varied_rows_per_tile(eng, gv, monkeypatch):
    rng = np.random.default_rng(100 + (gv or 0))
    T, lanes = stream_tile(eng, monkeypatch, 12000, 400, 4)
    g, varied = tiled(rng, T * 26 + 77, 400, T, counts_for(T, lanes))
    load(eng, rng, g, 4, varied)
    three_passes(eng, monkeypatch, gv_knobs(gv))


@pytest.mark.parametrize("gv", [None, 1, 4, 32], ids=str)
def test_every_site_varied(eng, gv, monkeypatch):
    """the stream forced on at 0 % uniform sites: every tile has more rows than the team has lanes"""
    rng = np.random.default_rng(200 + (gv or 0))
    g, _ = genotypes(rng, 5003, 400, 0.0)
    load(eng, rng, g, 4, np.ones(len(g), bool))
    three_passes(eng, monkeypatch, gv_knobs(gv))


@pytest.mark.parametrize("gv", [None, 2, 32], ids=str)
@pytest.mark.parametrize("limit", [1, 2])
def test_forced_flushes(eng, gv, limit, monkeypatch):
    rng = np.random.default_rng(300 + limit + (gv or 0))
    T, lanes = stream_tile(eng, monkeypatch, 4000, 400, 4)
    g, varied = tiled(rng, T * 9 + 5, 400, T, counts_for(T, lanes))
    load(eng, rng, g, 4, varied)
    three_passes(eng, monkeypatch, gv_knobs(gv, PG_K1_ACC_LIMIT=limit))


@pytest.mark.parametrize("knobs", [{"PG_K1_G": 8, "PG_K1_WPT": 2}, {"PG_K1_NW": 8}, {"PG_K1_I": 1},
                                   {"PG_K1_STAGES": 2, "PG_K1_WPT": 1}, {"PG_K1_TILE_KB": 4}], ids=str)
@pytest.mark.parametrize("gv", [None, 8], ids=str)
def test_geometries(eng, knobs, gv, monkeypatch):
    rng = np.random.default_rng(len(str(knobs)) + (gv or 0))
    knobs = gv_knobs(gv, **knobs)
    for k, v in knobs.items():
        monkeypatch.setenv(k, v)
    T, lanes = stream_tile(eng, monkeypatch, 6007, 400, 4)
    g, varied = tiled(rng, 6007, 400, T, counts_for(T, lanes))
    load(eng, rng, g, 4, varied)
    three_passes(eng, monkeypatch, knobs)


SHAPES = [(H, P) for H in (1, 33, 400, 1600) for P in (1, 4, 8, 9) if P <= H]


@pytest.mark.parametrize("H,P", SHAPES, ids=str)
def test_shapes_and_populations(eng, H, P, monkeypatch):
    rng = np.random.default_rng(H * 10 + P)
    T, lanes = stream_tile(eng, monkeypatch, 4003, H, P)
    g, varied = tiled(rng, 4003, H, T, counts_for(T, lanes))
    if H == 1:                                       # one haplotype: every site is uniform
        varied[:] = False
    load(eng, rng, g, P, varied)
    three_passes(eng, monkeypatch)
    three_passes(eng, monkeypatch, gv_knobs(2))
