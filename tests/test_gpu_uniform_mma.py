"""The varied-row stream's one-plane rows counted on the tensor cores (csrc/k1.cu varied_mma): a warp takes its complete
biallelic rows in blocks of 32, one row per lane, as two m16 tiles of an mma.m16n8k256 .and.popc over K-blocks of 8 words
(256 haplotypes), with the populations' member bits as the B operand (build_word_tables' bit_frag).  Every record field, the
popFreq columns included, must be bit-identical to the stream with every varied row in three planes (PG_K1_UNI_BITS=0), to
the packed pass over every row (PG_K1_NO_UNIFORM) and to the byte pass (PG_K1_BYTE_PASS), at the routine's edges: haplotype
counts at word and K-block edges, 1 to 4 populations, tiles whose one-plane row count is at and around a multiple of 32,
tiles that end at the word budget, bits past H left over from a wider matrix, lanes per three-plane row, forced flushes and
window sizes."""
import numpy as np
import pytest

from test_gpu_uniform_bits import KNOBS, four_passes, layout, load, mixed, sites, windows

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from genomics_general_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(autouse=True)
def _no_knobs(monkeypatch):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)


def biallelic(rng, S, H, third=0.0, uniform=0.0):
    """complete biallelic sites, with shares of third-allele (three-plane) and uniform sites"""
    kinds = rng.choice(["b", "t", "u"], S, p=[1.0 - third - uniform, third, uniform])
    return sites(rng, kinds, H)


# words per plane wd = ceil(H / 32): every wd % 8 (K-block of 8 words) is met, and H at and around 32, 256 and 512
H_EDGES = [1, 31, 32, 33, 70, 100, 180, 255, 256, 257, 288, 400, 511, 512, 513, 2000]


@pytest.mark.parametrize("H", H_EDGES)
@pytest.mark.parametrize("P", [1, 2, 3, 4])
def test_haplotype_edges(eng, H, P, monkeypatch):
    """contiguous populations at odd P, interleaved ones with unused haplotypes at even P; the rows keep a wider matrix's
    bytes past H"""
    if P > H:
        pytest.skip("fewer haplotypes than populations")
    rng = np.random.default_rng(H * 8 + P)
    S = 3000
    g = mixed(rng, S, H, (0.3, 0.02, 0.6, 0.04, 0.04)) if H > 1 else sites(rng, rng.choice(["u", "m", "b"], S), 1)
    hp = layout(rng, H, P, P % 2 == 0) if H > 1 else np.zeros(1, np.int32)
    lo, hi = windows(rng, S, 400)
    load(eng, g, hp, P, lo, hi, rng=rng, stale=True)
    four_passes(eng, monkeypatch)


@pytest.mark.parametrize("R", [32, 33, 47, 48, 49, 63, 95, 129])
def test_block_tails(eng, R, monkeypatch):
    """tiles of exactly R one-plane rows (a budget of R varied rows, every varied site complete biallelic): n1 = 0, 1, 15, 16,
    17 and 31 mod 32; then the same budget with a few three-plane rows behind each tile's one-plane rows"""
    rng = np.random.default_rng(R)
    S, H, P = 4000, 100, 4
    lo, hi = windows(rng, S, 300)
    load(eng, biallelic(rng, S, H), layout(rng, H, P, True), P, lo, hi, rng=rng)
    four_passes(eng, monkeypatch, {"PG_K1_UNI_R": str(R)})
    load(eng, biallelic(rng, S, H, third=0.05, uniform=0.3), layout(rng, H, P, False), P, lo, hi, rng=rng)
    four_passes(eng, monkeypatch, {"PG_K1_UNI_R": str(R), "PG_K1_UNI_TMAX": "256"})


@pytest.mark.parametrize("H,P", [(33, 2), (100, 4), (400, 4), (513, 3)])
def test_word_budget(eng, H, P, monkeypatch):
    """every site complete biallelic: the tiles are cut by the word budget alone and end exactly at it"""
    rng = np.random.default_rng(H + P)
    S = 20000
    lo, hi = windows(rng, S, 5000)
    load(eng, biallelic(rng, S, H), layout(rng, H, P, False), P, lo, hi, rng=rng, stale=True)
    four_passes(eng, monkeypatch)


@pytest.mark.parametrize("knobs", [{"PG_K1_UNI_GV": "2"}, {"PG_K1_UNI_GV": "4"}, {"PG_K1_UNI_GV": "32"},
                                   {"PG_K1_ACC_LIMIT": "1"}, {"PG_K1_ACC_LIMIT": "3"},
                                   {"PG_K1_ACC_LIMIT": "2", "PG_K1_UNI_R": "40"}], ids=str)
def test_knobs(eng, knobs, monkeypatch):
    """the three-plane rows' lanes per row (the one-plane rows keep a row per lane), and flushes forced inside a block"""
    rng = np.random.default_rng(len(str(knobs)))
    S, H, P = 5000, 200, 3
    g = mixed(rng, S, H, (0.4, 0.02, 0.5, 0.04, 0.04))
    lo, hi = windows(rng, S, 700)
    load(eng, g, layout(rng, H, P, True), P, lo, hi, rng=rng)
    four_passes(eng, monkeypatch, knobs)


@pytest.mark.parametrize("w,P", [(5000, 4), (50000, 2)])
def test_window_sizes(eng, w, P, monkeypatch):
    rng = np.random.default_rng(w + P)
    S, H = 150_000, 200
    g = mixed(rng, S, H, (0.69, 0.0, 0.3, 0.01, 0.0))      # no missing genotype: the windows take the site pass
    lo = np.arange(0, S, w, dtype=np.int64)
    load(eng, g, layout(rng, H, P, False), P, lo, np.minimum(lo + w, S), rng=rng)
    r = four_passes(eng, monkeypatch)
    assert np.all(r["path"] == 1)
