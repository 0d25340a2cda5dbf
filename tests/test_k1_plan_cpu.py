"""CPU tests of the site pass's launch plan (ctx.cu pg_make_k1_plan, through pg_debug_k1_plan_ex): every row length up to
the documented limit gets a plan the kernels accept, and every longer row is refused (no device needed)."""
import pytest

from genomics_general_b200 import engine

SMEM_CAP = 227 * 1024 - 2048          # dynamic shared memory the site pass allows itself, before the mask tables


def pitch_for(H):
    c = max(1, (H + 15) // 16)
    return (c + 1 if c % 2 == 0 else c) * 16


def tile_bytes(T, pitch):
    return (T * pitch + T * 4 + 127) // 128 * 128


def fits(H, lanes, table_bytes):
    """DESIGN.md §4 (K1): a row runs iff two stages of the smallest tile fit next to the mask tables.  The smallest tile is 4
    sites (a 4-row piece of positions); with G = 4 lanes per site (4 populations, one lane each) it is 8 sites."""
    t_min = 8 if lanes == 4 else 4
    return 2 * tile_bytes(t_min, pitch_for(H)) <= SMEM_CAP - table_bytes


@pytest.fixture(autouse=True)
def _no_knobs(monkeypatch):
    for k in ("PG_K1_G", "PG_K1_WPT", "PG_K1_I", "PG_K1_STAGES", "PG_K1_TILE_KB"):
        monkeypatch.delenv(k, raising=False)


@pytest.mark.parametrize("nw", [8, 12])
@pytest.mark.parametrize("lanes", [0, 4, 8])
def test_k1_plan_sweep_accepts_exactly_the_rows_that_fit(nw, lanes):
    tb = 4096
    refused = []
    for H in range(1, 30001):
        p = engine.k1_plan(10 ** 6, H, nw=nw, lanes=lanes, table_bytes=tb)
        want = fits(H, lanes, tb)
        assert p["ok"] == want, (H, p, want)
        if lanes:
            assert p["lanes_per_site"] == lanes
        if not want:
            refused.append(H)
            continue
        assert p["tile_sites"] % 4 == 0 and nw % p["warps_per_tile"] == 0, (H, p)
        assert 2 <= p["stages"] <= 8 and p["smem_bytes"] <= 227 * 1024, (H, p)
        assert p["smem_bytes"] == p["stages"] * tile_bytes(p["tile_sites"], p["pitch"]) + 256 + tb, (H, p)
    # one boundary: everything below it runs, everything above it is refused
    assert refused and refused == list(range(refused[0], 30001))
    last_ok = refused[0] - 1
    if lanes == 4:
        assert 14000 < last_ok < 16368
    else:
        assert last_ok == 28272        # the general plan with 4 KiB of mask tables


def test_k1_plan_limit_moves_with_the_mask_tables():
    # with the smallest mask tables (a few contiguous populations) rows of up to 28,688 haplotypes run
    assert engine.k1_plan(10 ** 6, 28688, table_bytes=600)["ok"]
    assert not engine.k1_plan(10 ** 6, 28689, table_bytes=600)["ok"]
    assert not engine.k1_plan(10 ** 6, 28688, table_bytes=4096)["ok"]


def test_k1_plan_overrides_are_reported(monkeypatch):
    monkeypatch.setenv("PG_K1_STAGES", "2")
    monkeypatch.setenv("PG_K1_WPT", "1")
    p = engine.k1_plan(10 ** 6, 1000, nw=12)
    assert p["stages"] == 2 and p["warps_per_tile"] == 1 and p["ok"]
    monkeypatch.setenv("PG_K1_WPT", "8")                   # does not divide 12 consumer warps
    assert not engine.k1_plan(10 ** 6, 1000, nw=12)["ok"]
