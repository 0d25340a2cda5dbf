"""Tiles of the varied-row stream cut by a budget of varied rows (csrc/k1.cu uniform_prepare): group k runs from the site of
varied rank k R to the next group's, a group of more than Tmax sites is split into pieces of Tmax, and the CTAs own ranges of
these tiles with slot tables of their own (uniform_slots).  Every record field, popFreq columns included, must be
bit-identical to the packed pass that streams every row (PG_K1_NO_UNIFORM) and to the byte pass (PG_K1_BYTE_PASS), and the
tile table (Engine.uniform_tiles) must cover [0, S) in order with at most R varied rows and at most Tmax sites per tile,
cut at every varied row whose rank is a multiple of R.  PG_K1_UNI_R / PG_K1_UNI_TMAX set R and Tmax."""
import numpy as np
import pytest

from test_gpu_uniform_sites import genotypes, layout, run, three_passes

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from genomics_general_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(autouse=True)
def _clean(monkeypatch):
    for k in ("PG_K1_UNI_GV", "PG_K1_UNI_R", "PG_K1_UNI_TMAX"):
        monkeypatch.delenv(k, raising=False)


def varied_of(g):
    return np.any(g != g[:, :1], axis=1)


def check_tiles(eng, monkeypatch, g, knobs):
    """the stream's tile table against the rule, from a forced-stream call under knobs"""
    _, used = run(eng, monkeypatch, dict(knobs, PG_K1_UNIFORM_FORCE="1"))
    assert used
    R, Tmax, site_lo, row0 = eng.uniform_tiles()
    S = len(g)
    if "PG_K1_UNI_R" in knobs:
        assert R == int(knobs["PG_K1_UNI_R"])
    rank = np.concatenate([[0], np.cumsum(varied_of(g))])
    assert site_lo[0] == 0 and site_lo[-1] == S
    sites = np.diff(site_lo)
    assert sites.min() >= 1 and sites.max() <= Tmax
    assert np.array_equal(row0, rank[site_lo])
    assert np.diff(row0).max() <= R
    cuts = np.flatnonzero(varied_of(g))[R::R]          # the sites of ranks R, 2R, ... start tiles
    assert np.isin(cuts, site_lo).all()
    return R, Tmax, site_lo


def patterned(rng, S, H, uniform=0.7, runs=()):
    """genotypes with a `uniform` share of uniform sites, and uniform runs [a, b) (every haplotype one allele, or every one
    missing when the run's flag is set)"""
    g, _ = genotypes(rng, S, H, uniform)
    for a, b, missing in runs:
        g[a:b] = -1 if missing else rng.integers(0, 4, (b - a))[:, None]
    return g


def load(eng, rng, g, P, windows=None):
    S, H = g.shape
    eng.upload(g, np.cumsum(rng.integers(1, 50, S)).astype(np.int32))
    eng.set_pops(layout(rng, H, P), P)
    if windows is None:
        lo = rng.integers(0, S, 60)
        windows = (lo, np.minimum(lo + rng.integers(1, 700, 60), S))
    eng.set_windows(np.asarray(windows[0], np.int64), np.asarray(windows[1], np.int64))


def both(eng, monkeypatch, g, knobs):
    out = check_tiles(eng, monkeypatch, g, knobs)
    three_passes(eng, monkeypatch, knobs)
    return out


@pytest.mark.parametrize("R", [31, 32, 33, 128])
def test_row_budget(eng, R, monkeypatch):
    """tiles of R - 1, R and R + 1 rows against one lane count"""
    rng = np.random.default_rng(R)
    g = patterned(rng, 9000, 400)
    load(eng, rng, g, 4)
    both(eng, monkeypatch, g, {"PG_K1_UNI_R": str(R)})


@pytest.mark.parametrize("tmax", [8, 16, 40, 512])
def test_long_groups(eng, tmax, monkeypatch):
    """groups longer than Tmax, long uniform and uniform-missing runs (pieces with no row), tiles starting anywhere"""
    rng = np.random.default_rng(tmax)
    g = patterned(rng, 7001, 400, 0.8, runs=[(100, 1300, False), (1301, 2700, True), (4000, 4003, True), (6990, 7001, False)])
    load(eng, rng, g, 4)
    _, Tm, site_lo = both(eng, monkeypatch, g, {"PG_K1_UNI_R": "64", "PG_K1_UNI_TMAX": str(tmax)})
    assert Tm == tmax and np.any(site_lo % 8 != 0)


def test_windows_on_tile_edges(eng, monkeypatch):
    """windows that start and end on every tile boundary (so on every CTA boundary) and one site off them, set after the
    stream was built: the slot tables follow the windows"""
    rng = np.random.default_rng(3)
    knobs = {"PG_K1_UNI_R": "24", "PG_K1_UNI_TMAX": "64"}
    g = patterned(rng, 20000, 400)
    load(eng, rng, g, 4)
    _, _, site_lo = both(eng, monkeypatch, g, knobs)
    S = len(g)
    for shift in (0, 1, -1):
        lo = np.clip(site_lo[:-1] + shift, 0, S - 1)
        hi = np.clip(np.concatenate([site_lo[2:], [S]]) + shift, 1, S)
        eng.set_windows(lo.astype(np.int64), np.maximum(hi, lo + 1).astype(np.int64))
        three_passes(eng, monkeypatch, knobs)


@pytest.mark.parametrize("S", [1, 5, 100])
def test_fewer_sites_than_a_tile(eng, S, monkeypatch):
    rng = np.random.default_rng(S)
    g = patterned(rng, S, 400)
    load(eng, rng, g, 4, ([0, 0], [S, max(1, S // 2)]))
    both(eng, monkeypatch, g, {})


def test_reupload_same_shape(eng, monkeypatch):
    """a same-shape upload with another uniform pattern and the same populations and windows: the next call rebuilds the
    tiles and their slot tables"""
    rng = np.random.default_rng(4)
    knobs = {"PG_K1_UNI_R": "40"}
    S = 12000
    lo = rng.integers(0, S, 80)
    win = (lo, np.minimum(lo + rng.integers(1, 900, 80), S))
    pos = np.cumsum(rng.integers(1, 50, S)).astype(np.int32)
    g1 = patterned(rng, S, 400, 0.9)
    g2 = patterned(rng, S, 400, 0.4, runs=[(0, 3000, False)])
    eng.upload(g1, pos)
    eng.set_pops(layout(rng, 400, 4), 4)
    eng.set_windows(*win)
    t1 = both(eng, monkeypatch, g1, knobs)[2]
    for g in (g2, g1):
        eng.upload(g, pos)                               # Engine.upload drops the windows: the same ones again
        eng.set_windows(*win)
        t = both(eng, monkeypatch, g, knobs)[2]
    assert np.array_equal(t, t1)


@pytest.mark.parametrize("knobs", [{"PG_K1_UNI_GV": "1"}, {"PG_K1_UNI_GV": "4", "PG_K1_UNI_R": "50"},
                                   {"PG_K1_UNI_GV": "32"}, {"PG_K1_ACC_LIMIT": "1"}, {"PG_K1_ACC_LIMIT": "2"},
                                   {"PG_K1_STAGES": "2"}, {"PG_K1_NW": "8"}, {"PG_K1_WPT": "1", "PG_K1_STAGES": "3"},
                                   {"PG_K1_G": "8", "PG_K1_WPT": "2"}, {"PG_K1_TILE_KB": "4"}], ids=str)
def test_knobs(eng, knobs, monkeypatch):
    rng = np.random.default_rng(len(str(knobs)))
    for k, v in knobs.items():
        monkeypatch.setenv(k, v)
    g = patterned(rng, 6007, 400, 0.7, runs=[(2000, 2600, False)])
    load(eng, rng, g, 4)
    both(eng, monkeypatch, g, knobs)


SHAPES = [(H, P) for H in (1, 33, 400, 1600) for P in (1, 4, 8, 9) if P <= H]


@pytest.mark.parametrize("H,P", SHAPES, ids=str)
def test_shapes_and_populations(eng, H, P, monkeypatch):
    rng = np.random.default_rng(H * 10 + P)
    g = patterned(rng, 4003, H, 0.7, runs=[(500, 1400, True)])
    load(eng, rng, g, P)
    both(eng, monkeypatch, g, {})
    both(eng, monkeypatch, g, {"PG_K1_UNI_R": "16", "PG_K1_UNI_TMAX": "24"})
