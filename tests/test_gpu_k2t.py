"""The tensor-core pairwise path (csrc/k2t.cu: wgmma u8 Gram kernels over bit-packed planes) against plain numpy
and against the round-1 POPC kernels, through the C-ABI: integer pair matrices bit-exact on every tile geometry (one group,
several 128-row tiles, a separate A region beyond 256 haplotypes, 1600 haplotypes), multi-allelic sites, window edges inside a
64-site chunk, per-sample and per-haplotype missingness, many windows per persistent CTA, and the smallest ring configurations
(PG_K2T_NRAW / PG_K2T_NSTAGES) that stress the mbarrier hand-overs."""
import os

import numpy as np
import pytest

from genomics_general_b200 import synth
from helpers import ref_counts

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from genomics_general_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


SHAPES = [  # (pops, samples per pop, sites, missing, p_third, windows)
    (2, 10, 3000, 0.05, 0.01, [(0, 3000), (100, 164), (5, 70), (64, 128), (1000, 1001)]),
    (2, 10, 3000, 0.0, 0.01, [(0, 3000), (17, 2100)]),
    (3, 22, 2500, 0.10, 0.20, [(0, 2500), (63, 1999)]),
    (4, 50, 6000, 0.02, 0.01, [(0, 5000), (5000, 6000), (123, 4567)]),
    (1, 300, 1500, 0.03, 0.01, [(0, 1500), (200, 900)]),
    (1, 500, 1200, 0.02, 0.05, [(0, 1200)]),
    (8, 100, 700, 0.02, 0.01, [(0, 700), (65, 640)]),
]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "H%d_miss%g" % (s[0] * s[1] * 2, s[3]))
def test_pair_counts_bit_exact_vs_numpy_and_popc(eng, shape, monkeypatch):
    P, spp, S, miss, p3, wins = shape
    spec = synth.SynthSpec(P, spp, miss=miss, seed=1234 + P * 7 + spp, p_third=p3)
    eng.synth_fill(spec, S)
    g, _ = eng.download(0, S)
    eng.set_windows(np.array([w[0] for w in wins], dtype=np.int64), np.array([w[1] for w in wins], dtype=np.int64))
    for w, (lo, hi) in enumerate(wins):
        rd, rn = ref_counts(g[lo:hi])
        monkeypatch.delenv("PG_K2_POPC", raising=False)
        for ch in ("2", "1"):                      # 128-site and 64-site stages of the co-valid Gram kernel
            monkeypatch.setenv("PG_K2T_CH", ch)
            d, n = eng.pair_counts(w)
            assert np.array_equal(n, rn) and np.array_equal(d, rd), (w, lo, hi, ch)
        monkeypatch.delenv("PG_K2T_CH")
        if P * spp * 2 <= 600:
            monkeypatch.setenv("PG_K2_POPC", "1")
            d2, n2 = eng.pair_counts(w)
            assert np.array_equal(d2, d) and np.array_equal(n2, n)
    monkeypatch.delenv("PG_K2_POPC", raising=False)


def test_allele_level_missingness_uses_one_mask_row_per_haplotype(eng):
    """haplotypes of a sample with different missingness: the per-sample compaction of the valid plane must be refused"""
    rng = np.random.default_rng(3)
    S, H = 900, 24
    g = rng.integers(0, 4, (S, H)).astype(np.int8)
    g[rng.random((S, H)) < 0.1] = -1                      # per allele, not per genotype
    eng.upload(g, np.arange(1, S + 1, dtype=np.int32))
    eng.set_windows([0, 100], [S, 777])
    for w, (lo, hi) in enumerate(((0, S), (100, 777))):
        rd, rn = ref_counts(g[lo:hi])
        d, n = eng.pair_counts(w)
        assert np.array_equal(n, rn) and np.array_equal(d, rd)


@pytest.mark.parametrize("env", [{}, {"PG_K2T_NRAW": "1"}, {"PG_K2T_NRAW": "1", "PG_K2T_NSTAGES": "1"}, {"PG_K2T_NSTAGES": "2"},
                                 {"PG_K2T_NO_PAIRS": "1"}, {"PG_K2T_CH": "2"}, {"PG_K2T_CH": "2", "PG_K2T_NRAW": "1"},
                                 {"PG_K2T_CH": "1"}], ids=lambda e: "_".join("%s%s" % (k[7:], v) for k, v in e.items()) or "default")
def test_many_windows_per_cta_equal_the_popc_kernels(eng, env, monkeypatch):
    """600 windows over one persistent CTA per SM, every ring geometry: statistics identical to the POPC path, run after run"""
    S = 3_000_000
    spec = synth.SynthSpec(4, 50, miss=0.02, seed=20260925)
    eng.synth_fill(spec, S)
    eng.set_pops(spec.hap_pop(), 4)
    lo = np.arange(0, S, 5000, dtype=np.int64)
    eng.set_windows(lo, np.minimum(lo + 5000, S))
    monkeypatch.setenv("PG_K2_POPC", "1")
    ref = eng.popgen(100, 0.01)
    monkeypatch.delenv("PG_K2_POPC")
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    for rep in range(2):
        r = eng.popgen(100, 0.01)
        assert np.all(r["path"] == 2)
        for key in ("sites", "pos_sum"):
            assert np.array_equal(r[key], ref[key]), (key, rep, env)
        for key in ("pi", "dxy", "fst"):
            # integer matrices are identical; the sample-pair epilogue divides once per four haplotype pairs, the
            # POPC path's epilogue once per pair: the block sums differ by rounding only
            assert np.array_equal(np.isnan(r[key]), np.isnan(ref[key])), (key, rep, env)
            assert np.allclose(r[key], ref[key], rtol=1e-12, atol=1e-12, equal_nan=True), (key, rep, env)
        if rep == 0:
            first = r
        else:
            for key in ("pi", "dxy", "fst"):
                assert np.array_equal(r[key], first[key], equal_nan=True), (key, env)      # run after run: bit-identical


def _direct_popgen(g, hap_pop, P, lo, hi, min_sites, min_data):
    """pi / dxy of one window straight from the definition (genomics.py:931-993): mean over haplotype pairs of diff / n"""
    d, n = ref_counts(g[lo:hi])
    with np.errstate(divide="ignore", invalid="ignore"):
        dist = np.where((n > 0) & (n >= min_sites), d / n.astype(np.float64), np.nan)
    idx = [np.flatnonzero(hap_pop == X) for X in range(P)]
    pi = np.full(P, np.nan)
    for X in range(P):
        blk = dist[np.ix_(idx[X], idx[X])].copy()
        np.fill_diagonal(blk, np.nan)
        if blk.size and 1.0 - np.isnan(blk).sum() / blk.size >= min_data and (~np.isnan(blk)).any():
            pi[X] = np.nanmean(blk)
    dxy = []
    for X in range(P):
        for Y in range(X + 1, P):
            blk = dist[np.ix_(idx[X], idx[Y])]
            ok = blk.size and 1.0 - np.isnan(blk).sum() / blk.size >= min_data and (~np.isnan(blk)).any()
            dxy.append(np.nanmean(blk) if ok else np.nan)
    return pi, np.array(dxy)


@pytest.mark.parametrize("sizes,nwin", [((5, 7, 9), 3), ((1, 2, 3, 4, 5, 6, 7, 8), 2), ((50, 50, 50, 50), 7), ((101,), 1),
                                        ((3, 3), 400)], ids=["odd3", "tiny8", "c2x7", "single101", "many_small"])
def test_sample_pair_epilogue_every_layout(eng, sizes, nwin, monkeypatch):
    """the sample-pair epilogue (one division per four haplotype pairs, folded diagonal blocks, blocks of a window dealt over
    several CTAs when windows are few) against the definition and against the per-pair epilogue of the POPC path: odd and even
    population sizes, one population, many populations with few windows, many windows"""
    P = len(sizes)
    rng = np.random.default_rng(11 + sum(sizes) + nwin)
    S = 600 * nwin
    nS = sum(sizes)
    hap_pop = np.repeat(np.arange(P), [2 * s for s in sizes]).astype(np.int32)
    g = rng.integers(0, 2, size=(S, 2 * nS)).astype(np.int8)
    g[rng.random((S, 2 * nS)) < 0.02] = 2                                   # a third allele here and there
    miss = rng.random((S, nS)) < 0.03                                        # missing GENOTYPES: both haplotypes of a sample
    g[np.repeat(miss, 2, axis=1)] = -1
    eng.upload(g, np.arange(1, S + 1, dtype=np.int32))
    eng.set_pops(hap_pop, P)
    lo = np.arange(0, S, 600, dtype=np.int64)
    hi = lo + 600
    eng.set_windows(lo, hi)
    for min_sites in (0, 590):
        r = eng.popgen(min_sites, 0.01, force_pairwise=True)
        assert np.all(r["path"] == 2)
        monkeypatch.setenv("PG_K2_POPC", "1")
        ref = eng.popgen(min_sites, 0.01, force_pairwise=True)
        monkeypatch.delenv("PG_K2_POPC")
        for key in ("pi", "dxy", "fst"):
            assert np.array_equal(np.isnan(r[key]), np.isnan(ref[key])), (key, min_sites)
            assert np.allclose(r[key], ref[key], rtol=1e-12, atol=1e-12, equal_nan=True), (key, min_sites)
        for w in range(min(nwin, 3)):
            pi, dxy = _direct_popgen(g, hap_pop, P, int(lo[w]), int(hi[w]), min_sites, 0.01)
            assert np.allclose(r["pi"][w], pi, rtol=1e-11, atol=1e-13, equal_nan=True), (w, min_sites)
            if P > 1:
                assert np.allclose(r["dxy"][w], dxy, rtol=1e-11, atol=1e-13, equal_nan=True), (w, min_sites)
