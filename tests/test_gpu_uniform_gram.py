"""The varied-row stream's one-plane rows summed as a Gram (csrc/k1.cu k1_site_pass_packed<..., UNI, GRAM>, gram_counts,
imma_u8): where every population has at most 255 haplotypes, a warp counts a block of 32 complete biallelic rows with
populations as the M of an mma.m16n8k256 .and.popc, packs the counts as bytes, accumulates the Gram of its rows' counts (with a
column of ones for the count sums and the row count) in an s32 IMMA, and folds it into its slot once per segment, or before
an entry could overflow.  Above 255 haplotypes the rows keep varied_mma and the per-row sums.  Every record field, the popFreq
columns included, must be bit-identical to the stream with every varied row in three planes (PG_K1_UNI_BITS=0), the packed
pass over every row and the byte pass, and agree with oracle/dense_oracle.py, at the Gram's edges: blocks that straddle one
or many segment boundaries, overlapping windows, blocks of fewer than 32 rows, forced folds, populations of 255 and 256
haplotypes, 1 to 4 populations with haplotypes in none, and H off the word and K-block multiples."""
import numpy as np
import pytest

from test_gpu_site_pass_bounds import check_popgen
from test_gpu_uniform_bits import KNOBS, four_passes, layout, load, set_knobs, sites

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


def complete(rng, S, H, uniform=0.3, third=0.03):
    """complete sites only (every window takes the site pass): uniform, biallelic (one plane) and third-allele (three planes)"""
    return sites(rng, rng.choice(["u", "b", "t"], S, p=[uniform, 1.0 - uniform - third, third]), H)


def oracle(eng, g, hp, P, lo, hi, pos, what, n=40):
    """the stream's records of n windows spread over the list, against the dense oracle"""
    wins = np.unique(np.linspace(0, len(lo) - 1, min(n, len(lo))).astype(int))
    check_popgen(eng, g, hp, P, lo, hi, pos, wins, what)


def run_both(eng, monkeypatch, g, hp, P, lo, hi, rng, what, knobs=None):
    pos = load(eng, g, hp, P, lo, hi, rng=rng)
    four_passes(eng, monkeypatch, knobs)
    set_knobs(monkeypatch, dict(knobs or {}, PG_K1_UNIFORM_FORCE="1"))
    oracle(eng, g, hp, P, lo, hi, pos, what)


@pytest.mark.parametrize("w,step", [(1, 1), (7, 7), (31, 31), (33, 33), (500, 500), (33, 10), (300, 7)])
def test_segment_boundaries(eng, w, step, monkeypatch):
    """windows of 1 to 33 sites put one or many segment boundaries inside a 32-row block; step < w overlaps them"""
    rng = np.random.default_rng(w * 100 + step)
    S, H, P = 3000, 100, 4
    g = complete(rng, S, H)
    lo = np.arange(0, S, step, dtype=np.int64)
    run_both(eng, monkeypatch, g, layout(rng, H, P, True), P, lo, np.minimum(lo + w, S), rng, "w%d s%d" % (w, step))


@pytest.mark.parametrize("R", [1, 5, 31, 33, 70])
def test_short_blocks(eng, R, monkeypatch):
    """tiles of at most R varied rows: n1 below 32 and off its multiples, so blocks end early"""
    rng = np.random.default_rng(R + 7)
    S, H, P = 2500, 70, 3
    g = complete(rng, S, H)
    lo = np.arange(0, S, 90, dtype=np.int64)
    run_both(eng, monkeypatch, g, layout(rng, H, P, False), P, lo, np.minimum(lo + 90, S), rng, "R%d" % R,
             {"PG_K1_UNI_R": str(R)})


@pytest.mark.parametrize("limit", ["1", "64", "65", "100", "333"])
def test_forced_folds(eng, limit, monkeypatch):
    """the Gram folds every max(acc_limit / 2, 32) rows inside a segment, as well as at its end"""
    rng = np.random.default_rng(int(limit))
    S, H, P = 6000, 200, 4
    g = complete(rng, S, H, uniform=0.1)
    lo = np.arange(0, S, 2500, dtype=np.int64)
    run_both(eng, monkeypatch, g, layout(rng, H, P, True), P, lo, np.minimum(lo + 2500, S), rng, "limit " + limit,
             {"PG_K1_ACC_LIMIT": limit})


@pytest.mark.parametrize("N", [254, 255, 256])
def test_byte_limit(eng, N, monkeypatch):
    """a population of 255 haplotypes takes the Gram, one of 256 the per-row sums; unassigned haplotypes around them"""
    rng = np.random.default_rng(N)
    H, P, S = N + 40, 2, 2000
    hp = np.full(H, -1, np.int32)
    hp[rng.permutation(H)[:N]] = 0
    free = np.flatnonzero(hp < 0)
    hp[free[:25]] = 1
    g = complete(rng, S, H)
    lo = np.arange(0, S, 150, dtype=np.int64)
    run_both(eng, monkeypatch, g, hp, P, lo, np.minimum(lo + 150, S), rng, "N%d" % N)


@pytest.mark.parametrize("H", [37, 100, 300, 513])
@pytest.mark.parametrize("P", [1, 2, 3, 4])
def test_populations(eng, H, P, monkeypatch):
    """1 to 4 populations (padded to 2 or 4, the padding's counts zero), haplotypes in no population at even P"""
    rng = np.random.default_rng(H * 4 + P)
    S = 2000
    g = complete(rng, S, H)
    lo = np.arange(0, S, 250, dtype=np.int64)
    hp = layout(rng, H, P, True) if P % 2 == 0 else (np.arange(H) * P // H).astype(np.int32)     # contiguous, even sizes
    run_both(eng, monkeypatch, g, hp, P, lo, np.minimum(lo + 250, S), rng, "H%d P%d" % (H, P))
