"""The varied-row stream's word-major tiles and its segment lookups (csrc/k1.cu k1_uni_codes, k1_site_pass_packed<..., UNI =
true>): word x of a tile's varied row j is stored at word x * nvar + j of the tile, so a layout index off by a row or a tile
moves words between rows; and both passes find a site's segment by galloping from the segment after their current one, so
a wrong bracket shows on jumps over many segments and at the last segment.  Every record field, popFreq columns included,
must be bit-identical to the packed pass that streams every row (PG_K1_NO_UNIFORM) and to the byte pass (PG_K1_BYTE_PASS)."""
import numpy as np
import pytest

from test_gpu_uniform_sites import genotypes, layout, run, three_passes

pytestmark = pytest.mark.gpu

R, TMAX = 128, 256


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


def with_varied(rng, H, varied):
    """genotypes whose varied sites are exactly `varied`: the others carry one allele, a tenth of them missing everywhere"""
    S = len(varied)
    g, _ = genotypes(rng, S, H, 0.0)
    ref = rng.integers(0, 4, S)
    uni = ~varied
    g[uni] = ref[uni, None]
    g[uni & (rng.random(S) < 0.1)] = -1
    return g


def counted_tiles(rng, S):
    """varied sites such that, with R = 128 and Tmax = 256, the first tiles hold 1, 31, 33, 0 and 63 varied rows (one group
    of R rows cut into pieces of Tmax sites), then a tile of exactly R rows in R consecutive sites and a piece with none;
    the rest random"""
    varied = np.zeros(S, bool)
    for piece, n in enumerate([1, 31, 33, 0, 63]):
        varied[piece * TMAX + rng.choice(TMAX, n, replace=False)] = True
    varied[5 * TMAX:5 * TMAX + R] = True
    varied[1600:] = rng.random(S - 1600) < 0.3
    varied[1600] = True
    return varied


def load(eng, rng, g, P, lo, hi):
    S, H = g.shape
    eng.upload(g, np.cumsum(rng.integers(1, 50, S)).astype(np.int32))
    eng.set_pops(layout(rng, H, P), P)
    eng.set_windows(np.asarray(lo, np.int64), np.asarray(hi, np.int64))


@pytest.mark.parametrize("H,P,gv", [(400, 4, None), (400, 4, 2), (400, 4, 32), (1600, 8, None), (1600, 8, 4), (33, 2, None)],
                         ids=str)
def test_tiles_of_1_31_33_and_R_rows(eng, H, P, gv, monkeypatch):
    rng = np.random.default_rng(H + P)
    S = 9000
    g = with_varied(rng, H, counted_tiles(rng, S))
    lo = rng.integers(0, S, 50)
    load(eng, rng, g, P, lo, np.minimum(lo + rng.integers(1, 700, 50), S))
    knobs = {"PG_K1_UNI_R": str(R), "PG_K1_UNI_TMAX": str(TMAX)}
    if gv is not None:
        knobs["PG_K1_UNI_GV"] = str(gv)
    _, used = run(eng, monkeypatch, dict(knobs, PG_K1_UNIFORM_FORCE="1"))
    assert used
    r, tmax, site_lo, row0 = eng.uniform_tiles()
    assert (r, tmax) == (R, TMAX)
    nvar = np.diff(row0)
    assert list(nvar[:7]) == [1, 31, 33, 0, 63, R, 0]
    assert list(site_lo[:8]) == [0, 256, 512, 768, 1024, 1280, 1536, 1600]
    three_passes(eng, monkeypatch, knobs)


def gapped_windows(S, a, b, first_gap):
    """1-site windows on every site of [a, b), then from b on 1-site windows with gaps of 1, 2, 3, ... sites between them,
    and a window over the last sites"""
    lo = list(range(a, b))
    s, gap = b, first_gap
    while s < S - 40:
        lo.append(s)
        s += 1 + gap
        gap = gap % 7 + 1
    hi = [x + 1 for x in lo]
    return lo + [S - 30], hi + [S]


@pytest.mark.parametrize("H,P", [(400, 4), (1600, 8)], ids=str)
@pytest.mark.parametrize("gv", [None, 2], ids=str)
def test_jumps_over_hundreds_of_segments(eng, H, P, gv, monkeypatch):
    """varied rows before and after 800 uniform sites that each have a 1-site window, so the lane after the run moves
    hundreds of segments on, as does pass U when it passes from one warp's 32 sites to the next; windows with gaps between
    them after that; and sites in the last segment"""
    rng = np.random.default_rng(H * 3 + (gv or 0))
    S = 6000
    varied = rng.random(S) < 0.5
    varied[100:900] = False
    varied[S - 5:] = True
    g = with_varied(rng, H, varied)
    lo, hi = gapped_windows(S, 100, 900, 1)
    load(eng, rng, g, P, lo, hi)
    knobs = {} if gv is None else {"PG_K1_UNI_GV": str(gv)}
    three_passes(eng, monkeypatch, knobs)
    three_passes(eng, monkeypatch, dict(knobs, PG_K1_UNI_R="32", PG_K1_UNI_TMAX="64"))


@pytest.mark.parametrize("end", [6000, 5000])
def test_last_segment(eng, end, monkeypatch):
    """one window over the last varied sites, with the data ending at it or going on 1000 sites past it: a lane's first
    segment can be the last one, and the search must not look past it"""
    rng = np.random.default_rng(end)
    S = 6000
    g = with_varied(rng, 400, rng.random(S) < 0.4)
    load(eng, rng, g, 4, [0, 10, end - 700], [5, 20, end])
    three_passes(eng, monkeypatch)
    three_passes(eng, monkeypatch, {"PG_K1_UNI_R": "32", "PG_K1_UNI_TMAX": "64"})
