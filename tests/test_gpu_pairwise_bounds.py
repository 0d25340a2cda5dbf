"""The pairwise path (csrc/k2.cu, csrc/k2t.cu) at the boundaries where its behaviour changes, against plain float64 / int64
definitions of the same quantities:

  1. window batching: every caller of the pair matrices cuts its windows into batches that fit pair_batch_size()
     (PG_PAIR_SCRATCH_MB), pg_ind_het and pg_seq_nonnan into batches of 65535 windows; the batch rows are mapped back to the
     windows' own rows (routed subsets, duplicates, empty windows in between)
  2. the tile groups of the wgmma Gram kernels (gram_groups): widths around 16, 64, 128 and 256 rows, per-sample (R2 rows)
     and per-haplotype (R rows) co-valid Grams, odd widths (scalar stores), both stage widths of the co-valid Gram
  3. the switch from the tensor path to the POPC kernels at 16 * pitch + 8 * R > 96 KiB
  4. the switch from the sample-pair popgen epilogue to the per-pair block epilogue (P > 38, populations on odd rows)
  5. the plane span: site_base > 0, four alleles, allele sets {0,3} / {1,3}, pseudo-site prefixes on 64-multiples, the
     last partial chunk, and a span without any variable site
  6. the largest population the H12 clustering kernel accepts
  7. the order of the entry points' argument checks and early returns

Every case also asserts which branch it reached (kernel names and launch counts of eng.last_timings(), popgen's path), so
that a later change of a threshold cannot silently turn it into a copy of another case."""
import math
import re
import warnings

import numpy as np
import pytest

from helpers import assert_close, ref_counts
from oracle import dense_oracle as do

pytestmark = pytest.mark.gpu

# the knobs the library reads on every call; none of them may leak in from the environment or from one case into the next
KNOBS = ("PG_PAIR_SCRATCH_MB", "PG_K2_POPC", "PG_K2_NO_MASK_SHARING", "PG_K2T_CH", "PG_K2T_NSTAGES", "PG_K2T_NRAW",
         "PG_K2T_NO_PAIRS")


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


# ---- the library's thresholds, restated (the tests assert on which side of each one a case sits) ----------------------
def pitch_for(H):
    """ctx.cu pg_pitch_for: 16-byte column chunks, an odd number of them"""
    c = max(1, (H + 15) // 16)
    return (c + 1 if c % 2 == 0 else c) * 16


def tensor_fits(H, Hk):
    """pgwin_internal.h pg_k2t_fits: the tensor path's plane builders stage 16 bytes per column and 8 per plane row (96 KiB)"""
    return 16 * pitch_for(H) + (Hk + 15) // 16 * 16 * 8 <= 96 * 1024


def per_batch(budget_mb, Hk, n_ind=0):
    """windows per batch of pg_k2_popgen_windows / pg_hapstats / pg_pairdist_cat (n_ind = 0) and pg_pairdist"""
    return max(1, min((budget_mb << 20) // (Hk * Hk * 8 + n_ind * n_ind * 8), 65535))


def pairs_epilogue(Hk, pop_sizes, per_sample_rows):
    """k2.cu: the sample-pair epilogue needs per-sample co-valid rows, populations on even rows and nblk * 64 <= 48 KiB"""
    P = len(pop_sizes)
    starts = np.concatenate([[0], np.cumsum(pop_sizes)])
    return per_sample_rows and Hk % 2 == 0 and P * (P + 1) // 2 * 64 <= 48 * 1024 and bool(np.all(starts % 2 == 0))


def clustering_smem(N):
    """k2.cu pg_hapstats: match bits [N][ceil(N/32)] + alive + sizes of the k2_hap_epi kernel"""
    nwd = (N + 31) // 32
    return N * nwd * 4 + nwd * 4 + N * 4 + 64


def kernels(eng):
    return {k: v["launches"] for k, v in eng.last_timings().items()}


def assert_tensor_path(t, tensor, gram=True):
    """tensor: k2t_valid_class builds the planes (and k2t_gram_* run); else the POPC kernels k2_planes / k2_pair_*"""
    if tensor:
        assert "k2t_valid_class" in t and "k2_planes" not in t, t
        if gram:
            assert "k2t_gram_diff" in t and "k2t_gram_n" in t and "k2_pair_diff" not in t, t
    else:
        assert "k2_planes" in t and "k2t_valid_class" not in t, t
        if gram:
            assert "k2_pair_diff" in t and "k2_pair_n" in t and "k2t_gram_diff" not in t, t


def assert_int_equal(got, want, what):
    if not np.array_equal(got, want):
        bad = np.argwhere(got != want)
        i, j = bad[0]
        raise AssertionError("%s: %d entries differ, first (%d, %d): %d != %d" % (what, len(bad), i, j, got[i, j], want[i, j]))


# ---- plain float64 definitions ---------------------------------------------------------------------------------------
def dist_from_counts(d, n, min_sites=0):
    """d_ij = diff / n (genomics.py:1219-1221), nan where n_ij = 0 or n_ij < minSites (959-961); diagonal nan (963)"""
    with np.errstate(divide="ignore", invalid="ignore"):
        x = d.astype(np.float64) / n.astype(np.float64)
    x[n == 0] = np.nan
    if min_sites:
        x[n < min_sites] = np.nan
    np.fill_diagonal(x, np.nan)
    return x


def block_sums(x, groups):
    """sum and count of the non-nan entries of every (group a, group b) block of x"""
    assert all(len(ix) for ix in groups)
    order = np.concatenate(groups)
    starts = np.concatenate([[0], np.cumsum([len(ix) for ix in groups])[:-1]])
    if not np.array_equal(order, np.arange(len(x))):
        x = x[np.ix_(order, order)]
    fin = ~np.isnan(x)
    v = np.where(fin, x, 0.0)
    f = fin.astype(np.int64)
    s = np.add.reduceat(np.add.reduceat(v, starts, axis=0), starts, axis=1)
    c = np.add.reduceat(np.add.reduceat(f, starts, axis=0), starts, axis=1)
    return s, c


def nanmean_min(s, c, size, min_data):
    """genomics.py:88-90 on blocks with c non-nan entries summing to s out of `size` (element-wise)"""
    s, c, size = (np.asarray(v, dtype=np.float64) for v in (s, c, size))
    with np.errstate(divide="ignore", invalid="ignore"):
        ok = (size > 0) & ~(1 - (1.0 * (size - c) / size) < min_data) & (c > 0)
        return np.where(ok, s / np.maximum(c, 1), np.nan)


def popgen_ref(d, n, hap_pop, P, min_sites, min_data):
    """groupDistStats (genomics.py:956-995) from the integer pair matrices: (pi [P], dxy [npairs], fst [npairs]), pairs in
    itertools.combinations order"""
    x = dist_from_counts(d, n, min_sites)
    idx = [np.flatnonzero(hap_pop == X) for X in range(P)]
    s, c = block_sums(x, idx)
    N = np.array([len(ix) for ix in idx], dtype=np.float64)
    pi = nanmean_min(np.diag(s), np.diag(c), N * N, min_data)
    X, Y = np.triu_indices(P, 1)
    dxy = nanmean_min(s[X, Y], c[X, Y], N[X] * N[Y], min_data)
    pi_t = nanmean_min(s[X, X] + s[Y, Y] + 2 * s[X, Y], c[X, X] + c[Y, Y] + 2 * c[X, Y], (N[X] + N[Y]) ** 2, min_data)
    w = 1.0 * N[X] / (N[X] + N[Y])
    with np.errstate(divide="ignore", invalid="ignore"):
        fst = 1 - (w * pi[X] + (1 - w) * pi[Y]) / pi_t
    return pi, dxy, fst


def ind_dists_ref(d, n, hap_ind, n_ind):
    """indPairDists (genomics.py:934-954, distMat.py:42-45): nanmean of each individual x individual block, diagonal nan"""
    hap_ind = np.asarray(hap_ind)
    used = np.flatnonzero(hap_ind >= 0)
    x = dist_from_counts(d[np.ix_(used, used)], n[np.ix_(used, used)])
    s, c = block_sums(x, [np.flatnonzero(hap_ind[used] == a) for a in range(n_ind)])
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(c > 0, s / np.maximum(c, 1), np.nan)


def assert_popgen(r, w, pi, dxy, fst, what):
    assert_close(r["pi"][w], pi, "%s pi" % what, rtol=1e-10, atol=1e-13)
    assert_close(r["dxy"][w], dxy, "%s dxy" % what, rtol=1e-10, atol=1e-13)
    assert_close(r["fst"][w], fst, "%s fst" % what, rtol=1e-7, atol=1e-9)


# ---- genotype matrices -----------------------------------------------------------------------------------------------
def apply_missing(rng, g, miss, per_sample):
    """per_sample: both haplotypes of a sample (columns 2s, 2s + 1) are missing together; else every allele on its own"""
    S, H = g.shape
    if per_sample:
        m = np.repeat(rng.random((S, (H + 1) // 2)) < miss, 2, axis=1)[:, :H]
    else:
        m = rng.random((S, H)) < miss
    g[m] = -1
    return g


def random_geno(rng, S, H, miss, per_sample=True, nal=None):
    """int8 [S, H]: site s draws its haplotypes from nal[s] distinct alleles of {0..3} (any of them, e.g. {1, 3})"""
    if nal is None:
        nal = rng.choice(4, size=S, p=(0.15, 0.55, 0.2, 0.1)) + 1
    perm = np.argsort(rng.random((S, 4)), axis=1).astype(np.int8)
    k = rng.integers(0, np.asarray(nal)[:, None], size=(S, H))
    g = perm[np.arange(S)[:, None], k]
    return apply_missing(rng, g, miss, per_sample)


def n_alleles(g):
    """alleles present per site among the non-missing entries of g"""
    return sum((g == a).any(axis=1).astype(np.int64) for a in range(4))


def pseudo_prefix(g, base):
    """cps of k2t_inv: pseudo-sites (alleles present - 1) in [base, base + k) for every k"""
    return np.concatenate([[0], np.cumsum(np.maximum(n_alleles(g[base:]) - 1, 0))])


# ======================================================================================================================
# 1. window batching
# ======================================================================================================================
BATCH_S, BATCH_H = 3000, 320
MISSING_REGIONS = ((500, 900), (1600, 2000), (2800, 3000))    # missing genotypes only here: the other windows are complete
BATCH_WINDOWS = [(2500, 2600), (600, 800), (0, 300), (600, 800), (650, 700), (1000, 1000), (1700, 1701), (1200, 1500),
                 (1550, 1950), (2900, 3000), (300, 300), (850, 1250), (0, 3000), (1600, 1664), (37, 101), (2000, 2000),
                 (1601, 1990), (2790, 2801), (100, 200), (820, 900), (3000, 3000)]
# Hk haplotypes selected out of 320: 200 -> popgen / hapstats take 3 windows per 1 MB batch, pairdist 2; 320 -> 1 each
BATCH_SELECTIONS = pytest.mark.parametrize("Hk", [200, 320], ids=["3_per_batch", "1_per_batch"])


@pytest.fixture(scope="module")
def batch_data():
    rng = np.random.default_rng(20261015)
    g = random_geno(rng, BATCH_S, BATCH_H, 0.0)
    miss = np.zeros((BATCH_S, BATCH_H // 2), dtype=bool)
    for lo, hi in MISSING_REGIONS:
        miss[lo:hi] = rng.random((hi - lo, BATCH_H // 2)) < 0.03
        miss[np.arange(lo, hi), rng.integers(0, 100, hi - lo)] = True      # every site of a region misses a selected sample
    g[np.repeat(miss, 2, axis=1)] = -1
    lo = np.array([w[0] for w in BATCH_WINDOWS], dtype=np.int64)
    hi = np.array([w[1] for w in BATCH_WINDOWS], dtype=np.int64)
    return g, lo, hi


def batch_pops(Hk):
    hap_pop = np.full(BATCH_H, -1, dtype=np.int32)
    hap_pop[:Hk] = np.repeat(np.arange(4), Hk // 4)
    return hap_pop


def with_budget(monkeypatch, mb, fn):
    monkeypatch.setenv("PG_PAIR_SCRATCH_MB", str(mb))
    try:
        return fn()
    finally:
        monkeypatch.delenv("PG_PAIR_SCRATCH_MB")


@BATCH_SELECTIONS
def test_popgen_window_batches(eng, batch_data, Hk, monkeypatch):
    """pg_k2_popgen_windows over 1 MB batches: each batch re-uploads d_widx and the epilogue writes the windows' own record
    rows; routed (a non-contiguous subset of the windows) and forced through the pairwise path"""
    g, lo, hi = batch_data
    hap_pop = batch_pops(Hk)
    eng.upload(g, np.arange(1, BATCH_S + 1, dtype=np.int32))
    eng.set_pops(hap_pop, 4)
    eng.set_windows(lo, hi)
    pb = per_batch(1, Hk)
    assert pb == {200: 3, 320: 1}[Hk] and per_batch(3072, Hk) >= len(lo)
    used = hap_pop >= 0
    nmiss = (g[:, used] < 0).sum(axis=1)
    ragged = (nmiss > 0) & (nmiss < used.sum())
    for force in (False, True):
        ref = eng.popgen(1, 0.01, force_pairwise=force)                # default budget: one batch
        t_ref = kernels(eng)
        r = with_budget(monkeypatch, 1, lambda: eng.popgen(1, 0.01, force_pairwise=force))
        t = kernels(eng)
        path = np.array([0 if h == l else (2 if force or ragged[l:h].any() else 1) for l, h in zip(lo, hi)])
        assert np.array_equal(r["path"], path) and np.array_equal(ref["path"], path), (r["path"], path)
        k2 = np.flatnonzero(path == 2)
        if not force:   # the routed windows are a subset with gaps: batch row k is not window b0 + k
            assert (path == 1).any() and np.any(np.diff(k2) > 1)
        nbatch = math.ceil(len(k2) / pb)
        assert t_ref["k2t_gram_diff"] == 1 and t_ref["k2_popgen_epi_pairs"] == 1, t_ref
        assert t["k2t_gram_diff"] == t["k2t_gram_n"] == t["k2_popgen_epi_pairs"] == nbatch, (t, nbatch)
        for key in ("pi", "dxy", "fst", "sites", "pos_sum"):
            assert np.array_equal(r[key], ref[key], equal_nan=True), (key, force)
        for w, (l, h) in enumerate(zip(lo, hi)):
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                pi, dxy, fst = do.group_dist_stats(g[l:h], hap_pop, 4, 1, 0.01)
            assert_popgen(r, w, pi, dxy, fst, "window %d [%d, %d) force=%s" % (w, l, h, force))


@BATCH_SELECTIONS
def test_pairdist_and_hapstats_window_batches(eng, batch_data, Hk, monkeypatch):
    """pg_pairdist (staged copies, run by run of consecutive windows) and pg_hapstats (copy_rows_back) across batch
    boundaries, with empty windows between non-empty ones"""
    g, lo, hi = batch_data
    eng.upload(g, np.arange(1, BATCH_S + 1, dtype=np.int32))
    eng.set_windows(lo, hi)
    nonempty = [w for w in range(len(lo)) if hi[w] > lo[w]]
    counts = {w: ref_counts(g[lo[w]:hi[w]]) for w in nonempty}
    hap = np.arange(BATCH_H)
    hap_ind = np.where(hap < Hk, hap // 2, -1).astype(np.int32)
    n_ind = Hk // 2
    pbd = per_batch(1, Hk, n_ind)
    assert pbd == {200: 2, 320: 1}[Hk]
    ref = eng.pairdist(hap_ind, n_ind)
    assert kernels(eng)["k2t_gram_diff"] == 1
    r = with_budget(monkeypatch, 1, lambda: eng.pairdist(hap_ind, n_ind))
    t = kernels(eng)
    assert t["k2t_gram_diff"] == t["k2_ind_epi"] == math.ceil(len(nonempty) / pbd), t
    for key in ("dist", "sites", "pos_sum"):
        assert np.array_equal(r[key], ref[key], equal_nan=True), key
    for w in range(len(lo)):
        if w in counts:
            d, n = counts[w]
            assert_close(r["dist"][w], ind_dists_ref(d, n, hap_ind, n_ind), "pairdist window %d" % w, rtol=1e-11, atol=1e-14)
        else:
            assert np.all(np.isnan(r["dist"][w])), w

    hap_pop = batch_pops(Hk)
    eng.set_pops(hap_pop, 4)
    pb = per_batch(1, Hk)
    href = eng.hapstats(0.02)
    assert kernels(eng)["k2_hap_epi"] == 1
    h = with_budget(monkeypatch, 1, lambda: eng.hapstats(0.02))
    t = kernels(eng)
    assert t["k2t_gram_diff"] == t["k2_hap_epi"] == math.ceil(len(nonempty) / pb), t
    assert np.array_equal(h, href, equal_nan=True)
    for w in range(len(lo)):
        if w in counts:
            assert_close(h[w], do.h12_stats(g[lo[w]:hi[w]], hap_pop, 4, 0.02), "hapstats window %d" % w, rtol=1e-12)
        else:
            assert np.all(np.isnan(h[w])), w


@BATCH_SELECTIONS
def test_pairdist_cat_chunk_batches(eng, Hk, monkeypatch):
    """--windType cat: 100 000 sites = 4 chunks of 32 768; with 1 MB the chunks go 3 (or 1) per batch and the int64
    accumulator adds the batches"""
    S, CH = 100_000, 32768
    rng = np.random.default_rng(7 + Hk)
    g = random_geno(rng, S, BATCH_H, 0.02)
    eng.upload(g, np.arange(1, S + 1, dtype=np.int32))
    hap = np.arange(BATCH_H)
    hap_ind = np.where(hap < Hk, hap // 2, -1).astype(np.int32)
    n_ind = Hk // 2
    nchunks = math.ceil(S / CH)
    pb = per_batch(1, Hk)
    assert nchunks == 4 and pb == {200: 3, 320: 1}[Hk]
    ref, tot_ref = eng.pairdist_cat(hap_ind, n_ind)
    assert kernels(eng)["k2_reduce_pairs"] == 1
    dist, tot = with_budget(monkeypatch, 1, lambda: eng.pairdist_cat(hap_ind, n_ind))
    t = kernels(eng)
    assert t["k2t_gram_diff"] == t["k2_reduce_pairs"] == math.ceil(nchunks / pb), t
    assert tot == tot_ref == S
    assert np.array_equal(dist, ref, equal_nan=True)
    d, n = ref_counts(g[:, :Hk])
    assert_close(dist, ind_dists_ref(d, n, hap_ind[:Hk], n_ind), "pairdist_cat", rtol=1e-11, atol=1e-14)


def test_het_and_seq_nonnan_window_batches(eng, monkeypatch):
    """pg_ind_het and pg_seq_nonnan take 65 535 windows per batch: 70 000 windows of 3 sites, every 997th one empty (the
    copies back break there), are two batches, on the tensor path and on the POPC kernels"""
    W, H = 70_000, 8
    S = W + 2
    rng = np.random.default_rng(65535)
    g = random_geno(rng, S, H, 0.1)
    lo = np.arange(W, dtype=np.int64)
    hi = lo + 3
    hi[::997] = lo[::997]
    eng.upload(g, np.arange(1, S + 1, dtype=np.int32))
    eng.set_windows(lo, hi)
    nonempty = np.flatnonzero(hi > lo)
    assert 65535 < len(nonempty) <= 2 * 65535
    cum = np.concatenate([np.zeros((1, H), dtype=np.int64), np.cumsum(g >= 0, axis=0)])
    want_nn = cum[hi] - cum[lo]
    # het against the oracle at both ends, around the batch boundary and at random windows
    check = set(range(12)) | set(range(W - 12, W)) | set(nonempty[65525:65545].tolist())
    check |= set(rng.choice(W, 300, replace=False).tolist())
    hap_ind = (np.arange(H) // 2).astype(np.int32)
    for env in ({}, {"PG_K2_POPC": "1"}):
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        nn = eng.seq_nonnan()
        t = kernels(eng)
        assert_tensor_path(t, not env, gram=False)
        assert t["k2_seq_nonnan"] == 2, t
        assert np.array_equal(nn, want_nn), env
        for min_sites in (0, 3):
            het = eng.ind_het(hap_ind, H // 2, min_sites)
            t = kernels(eng)
            assert_tensor_path(t, not env, gram=False)
            assert t["k2_het"] == 2, t
            for w in sorted(w for w in check if hi[w] > lo[w]):
                assert_close(het[w], do.sample_het(g[lo[w]:hi[w]], hap_ind, H // 2, min_sites),
                             "het window %d min_sites %d %s" % (w, min_sites, env), rtol=1e-12)
            assert np.all(np.isnan(het[hi == lo]))
        for k in env:
            monkeypatch.delenv(k)


# ======================================================================================================================
# 2. tile groups of the Gram kernels
# ======================================================================================================================
# gram_groups cuts R = 16 ceil(Hk / 16) rows into 128-row A tiles x 256-row B ranges: R = 144 gives a diagonal group whose
# B range (16 rows) is shorter than the A tile, R = 272 a separate-A group with N = 64 over 16 live rows; odd widths take
# the scalar store; per-genotype missingness gives the co-valid Gram R2 = 16 ceil(Hk / 32) rows (Hk even), per-allele R
SWEEP_HK = [1, 2, 3, 15, 16, 17, 31, 33, 127, 128, 129, 130, 255, 256, 257, 258, 384, 385, 513, 514, 767, 768, 769, 1026]
SWEEP_S = 300                      # the last chunk (256..299) is partial
MONO = (192, 256)                  # one whole chunk of monomorphic sites
SWEEP_WINDOWS = [(0, SWEEP_S),     # the whole matrix
                 (70, 120),        # starts and ends inside chunk 1
                 (150, 151),       # one (tri-allelic) site
                 (200, 250)]       # only monomorphic sites: diff = 0, and the planes' span has no pseudo-site


def sweep_geno(Hk, mode):
    rng = np.random.default_rng(1000 + 2 * Hk + (mode == "per_allele"))
    nal = rng.choice(4, size=SWEEP_S, p=(0.15, 0.55, 0.2, 0.1)) + 1
    nal[MONO[0]:MONO[1]] = 1
    nal[150] = 3
    return random_geno(rng, SWEEP_S, Hk, 0.05, per_sample=(mode == "per_genotype"), nal=nal)


def span_is_variable(g, lo, hi):
    """does the planes' span [lo & ~63, end of hi's chunk) hold a site with two alleles? (k2t_build_pq runs iff so)"""
    sb = lo & ~63
    end = min(len(g), sb + (hi - sb + 63) // 64 * 64)
    return bool((n_alleles(g[sb:end]) >= 2).any())


@pytest.mark.parametrize("mode", ["per_genotype", "per_allele"])
@pytest.mark.parametrize("Hk", SWEEP_HK)
def test_pair_counts_tile_group_sweep(eng, Hk, mode, monkeypatch):
    g = sweep_geno(Hk, mode)
    valid = g >= 0
    shared = Hk % 2 == 0 and np.array_equal(valid[:, 0::2], valid[:, 1::2])
    # which co-valid Gram runs: per-sample rows (R2) exactly for even widths with per-genotype missingness
    assert shared == (mode == "per_genotype" and Hk % 2 == 0)
    assert tensor_fits(Hk, Hk)
    eng.upload(g, np.arange(1, SWEEP_S + 1, dtype=np.int32))
    eng.set_windows([w[0] for w in SWEEP_WINDOWS], [w[1] for w in SWEEP_WINDOWS])
    for w, (lo, hi) in enumerate(SWEEP_WINDOWS):
        rd, rn = ref_counts(g[lo:hi])
        variable = span_is_variable(g, lo, hi)
        if (lo, hi) == (200, 250):
            assert not rd.any() and not variable
        for env in ({}, {"PG_K2T_CH": "1"}, {"PG_K2_POPC": "1"}, {"PG_K2_POPC": "1", "PG_K2_NO_MASK_SHARING": "1"}):
            for k, v in env.items():
                monkeypatch.setenv(k, v)
            d, n = eng.pair_counts(w)
            t = kernels(eng)
            for k in env:
                monkeypatch.delenv(k)
            what = "Hk=%d %s window [%d, %d) %s" % (Hk, mode, lo, hi, env)
            assert_tensor_path(t, "PG_K2_POPC" not in env)
            if "PG_K2_POPC" not in env:
                assert ("k2t_build_pq" in t) == variable, (what, t)
            assert_int_equal(n, rn, what + " n")
            assert_int_equal(d, rd, what + " diff")


# non-identity plane order and unused columns: k2t_valid_class<false>, rows gathered through c2r
@pytest.mark.parametrize("Hk,perm", [(130, "samples"), (258, "samples"), (514, "samples"), (17, "haplotypes"),
                                     (129, "haplotypes"), (385, "haplotypes")])
def test_permuted_selection_with_unused_columns(eng, Hk, perm):
    """popgen / pairdist through the pairwise path on a shuffled selection with 14 unused columns: whole samples shuffled
    keep the per-sample co-valid rows (sample-pair epilogue), shuffled haplotypes do not (block epilogue)"""
    rng = np.random.default_rng(77 + Hk)
    H, S, P = Hk + 14, 400, 3
    g = random_geno(rng, S, H, 0.04)
    if perm == "samples":
        samples = rng.permutation(H // 2)[:Hk // 2]
        sel = np.stack([2 * samples, 2 * samples + 1], axis=1).ravel()
    else:
        sel = rng.permutation(H)[:Hk]
    unit = 2 if perm == "samples" else 1
    cuts = [len(sel) // unit * X // P * unit for X in range(P + 1)]
    hap_pop = np.full(H, -1, dtype=np.int32)
    for X in range(P):
        hap_pop[sel[cuts[X]:cuts[X + 1]]] = X
    hap_ind = np.full(H, -1, dtype=np.int32)
    hap_ind[sel] = np.arange(Hk) // 2              # "samples": an individual is a sample; else two random haplotypes
    n_ind = (Hk + 1) // 2
    wins = [(0, S), (45, 301), (130, 131)]
    eng.upload(g, np.arange(1, S + 1, dtype=np.int32))
    eng.set_pops(hap_pop, P)
    eng.set_windows([w[0] for w in wins], [w[1] for w in wins])
    counts = [ref_counts(g[lo:hi]) for lo, hi in wins]
    sizes = [int((hap_pop == X).sum()) for X in range(P)]
    # min_sites 236 masks about half of the pairs of the 256-site window (n_ij ~ 256 * 0.96^2), none of the first window's
    # and all of the 1-site window's; populations of > 32 haplotypes reach the second column of a block-walk step
    for min_sites in (0, 236):
        r = eng.popgen(min_sites, 0.01, force_pairwise=True)
        t = kernels(eng)
        assert np.array_equal(r["path"], [0 if hi - lo < min_sites else 2 for lo, hi in wins])    # fewer sites: path 0
        assert_tensor_path(t, True)
        # plane rows are sorted by population; a shuffled sample keeps its two haplotypes on rows 2k, 2k + 1
        assert ("k2_popgen_epi_pairs" in t) == (perm == "samples") == pairs_epilogue(Hk, sizes, perm == "samples"), t
        assert ("k2_popgen_epi_blocks" in t) == (perm != "samples"), t
        for w, (d, n) in enumerate(counts):
            assert_popgen(r, w, *popgen_ref(d, n, hap_pop, P, min_sites, 0.01),
                          "Hk=%d %s window %d min_sites %d" % (Hk, perm, w, min_sites))
        if min_sites:
            n1 = counts[1][1]
            assert np.any((n1 > 0) & (n1 < min_sites)) and np.any(n1 >= min_sites) and np.all(np.isnan(r["pi"][2]))
    pd = eng.pairdist(hap_ind, n_ind)
    assert_tensor_path(kernels(eng), True)
    for w, (d, n) in enumerate(counts):
        assert_close(pd["dist"][w], ind_dists_ref(d, n, hap_ind, n_ind), "pairdist Hk=%d %s window %d" % (Hk, perm, w),
                     rtol=1e-11, atol=1e-14)


# ======================================================================================================================
# 3. tensor / POPC width switch
# ======================================================================================================================
WIDE_S = 400
WIDE_WINDOWS = [(0, WIDE_S), (37, 333)]


@pytest.fixture(scope="module")
def wide_data():
    rng = np.random.default_rng(4096)
    g = random_geno(rng, WIDE_S, 4096, 0.02)
    counts = []
    for lo, hi in WIDE_WINDOWS:          # every column once: the three cases below take leading sub-matrices
        d, n = ref_counts(g[lo:hi])
        counts.append((d.astype(np.int32), n.astype(np.int32)))
    return g, counts


# pitch_for(4096) = 4112: 16 * 4112 + 8 * 4064 = 96 KiB exactly (tensor), 16 * 4112 + 8 * 4080 = 96 KiB + 128 (POPC);
# pitch_for(4080) = 4080: 16 * 4080 + 8 * 4080 < 96 KiB (tensor)
@pytest.mark.parametrize("H,Hk,tensor", [(4096, 4064, True), (4096, 4080, False), (4080, 4080, True)],
                         ids=["tensor_4064_of_4096", "popc_4080_of_4096", "tensor_4080_of_4080"])
def test_tensor_popc_width_switch(eng, wide_data, H, Hk, tensor):
    g_all, counts = wide_data
    assert tensor_fits(H, Hk) == tensor
    g = np.ascontiguousarray(g_all[:, :H])
    eng.upload(g, np.arange(1, WIDE_S + 1, dtype=np.int32))
    eng.set_windows([w[0] for w in WIDE_WINDOWS], [w[1] for w in WIDE_WINDOWS])
    hap_pop = np.full(H, -1, dtype=np.int32)
    hap_pop[:Hk] = np.repeat(np.arange(2), Hk // 2)
    eng.set_pops(hap_pop, 2)
    r = eng.popgen(0, 0.01, force_pairwise=True)
    assert np.all(r["path"] == 2)
    assert_tensor_path(kernels(eng), tensor)
    for w, (d, n) in enumerate(counts):
        assert_popgen(r, w, *popgen_ref(d[:Hk, :Hk], n[:Hk, :Hk], hap_pop[:Hk], 2, 0, 0.01), "%d of %d window %d" % (Hk, H, w))
    hap_ind = np.where(np.arange(H) < Hk, np.arange(H) // 2, -1).astype(np.int32)
    pd = eng.pairdist(hap_ind, Hk // 2)
    assert_tensor_path(kernels(eng), tensor)
    for w, (d, n) in enumerate(counts):
        assert_close(pd["dist"][w], ind_dists_ref(d[:Hk, :Hk], n[:Hk, :Hk], hap_ind[:Hk], Hk // 2),
                     "pairdist %d of %d window %d" % (Hk, H, w), rtol=1e-11, atol=1e-14)
    if Hk == H:
        for w, (d, n) in enumerate(counts):
            dd, nn = eng.pair_counts(w)
            assert_tensor_path(kernels(eng), tensor)
            assert_int_equal(nn, n[:H, :H], "n window %d" % w)
            assert_int_equal(dd, d[:H, :H], "diff window %d" % w)


# ======================================================================================================================
# 4. popgen epilogue switch
# ======================================================================================================================
def _epi_sizes(case):
    sizes = [4] * {"P38": 38, "P39": 39, "P64": 64, "P38_one_odd": 38, "P38_two_odd": 38}[case]
    if case in ("P38_one_odd", "P38_two_odd"):
        sizes[5] = 3                 # populations 6.. start on odd rows
    if case == "P38_two_odd":
        sizes[20] = 5                # Hk even again: per-sample co-valid rows, only the odd starts refuse the pair walk
    return sizes


# P = 38: nblk * 64 = 47 424 B fits 48 KiB (pair walk), P = 39: 49 920 B does not (block walk), P = 64 = PG_MAX_POPS;
# "few" windows deal the blocks of a window over nsplit > 1 CTAs, "many" (>= 8 x SMs of any H100) give nsplit = 1
@pytest.mark.parametrize("layout", ["few", "many"])
@pytest.mark.parametrize("case,pairs", [("P38", True), ("P39", False), ("P64", False), ("P38_one_odd", False),
                                        ("P38_two_odd", False)])
def test_popgen_epilogue_switch(eng, case, pairs, layout, monkeypatch):
    sizes = _epi_sizes(case)
    P, Hk = len(sizes), sum(sizes)
    hap_pop = np.repeat(np.arange(P), sizes).astype(np.int32)
    assert pairs_epilogue(Hk, sizes, Hk % 2 == 0) == pairs
    nwin, wlen, masking = (3, 400, 385) if layout == "few" else (1200, 8, 8)
    S = nwin * wlen
    rng = np.random.default_rng(P * 31 + Hk + nwin)
    g = random_geno(rng, S, Hk, 0.02)
    eng.upload(g, np.arange(1, S + 1, dtype=np.int32))
    eng.set_pops(hap_pop, P)
    lo = np.arange(0, S, wlen, dtype=np.int64)
    eng.set_windows(lo, lo + wlen)
    counts = [ref_counts(g[l:l + wlen]) for l in lo]
    for min_sites in (0, masking):
        r = eng.popgen(min_sites, 0.01, force_pairwise=True)
        t = kernels(eng)
        assert np.all(r["path"] == 2)
        assert_tensor_path(t, True)
        assert t.get("k2_popgen_epi_pairs" if pairs else "k2_popgen_epi_blocks") == 1, t
        monkeypatch.setenv("PG_K2_POPC", "1")
        ref = eng.popgen(min_sites, 0.01, force_pairwise=True)
        assert_tensor_path(kernels(eng), False)
        monkeypatch.delenv("PG_K2_POPC")
        for key in ("pi", "dxy", "fst"):
            assert_close(r[key], ref[key], "%s vs POPC min_sites=%d" % (key, min_sites), rtol=1e-12, atol=1e-12)
        if min_sites:     # the mask removes some pairs, not all
            n_all = np.stack([c[1] for c in counts])
            assert np.any((n_all > 0) & (n_all < min_sites)) and not np.all(np.isnan(r["pi"]))
        for w, (d, n) in enumerate(counts):
            assert_popgen(r, w, *popgen_ref(d, n, hap_pop, P, min_sites, 0.01), "%s window %d min_sites %d" % (case, w, min_sites))
        for w in (0, nwin - 1):
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                pi, dxy, fst = do.group_dist_stats(g[lo[w]:lo[w] + wlen], hap_pop, P, min_sites, 0.01)
            assert_popgen(r, w, pi, dxy, fst, "%s oracle window %d min_sites %d" % (case, w, min_sites))


# ======================================================================================================================
# 5. plane span and pseudo-site edges
# ======================================================================================================================
EDGE_H, EDGE_S = 40, 64 * 7 + 45
FOUR = (170, 171, 300, 470)                   # all four alleles
SET03, SET13 = (175, 176, 305, 475), (180, 310, 480)
DENSE = (320, 448)                            # tri-allelic: the pseudo-site prefix grows by exactly 2 per site


def edge_geno():
    """hand-built: every site's allele set is given and present (samples 0..3 carry it, both haplotypes)"""
    rng = np.random.default_rng(64)
    sets = []
    for s in range(EDGE_S):
        if s in FOUR:
            a = [0, 1, 2, 3]
        elif s in SET03:
            a = [0, 3]
        elif s in SET13:
            a = [1, 3]
        elif DENSE[0] <= s < DENSE[1]:
            a = sorted(rng.choice(4, 3, replace=False))
        else:
            a = sorted(rng.choice(4, rng.choice(4, p=(0.3, 0.45, 0.15, 0.1)) + 1, replace=False))
        sets.append(a)
    g = np.empty((EDGE_S, EDGE_H), dtype=np.int8)
    for s, a in enumerate(sets):
        g[s] = np.array(a)[rng.integers(0, len(a), EDGE_H)]
    apply_missing(rng, g, 0.05, True)
    for s, a in enumerate(sets):
        for j, x in enumerate(a):
            g[s, 2 * j:2 * j + 2] = x
    assert all(sorted(np.unique(g[s][g[s] >= 0])) == list(sets[s]) for s in range(EDGE_S))
    return g


def edge_windows(g):
    """the leftmost window starts at 64 k + 37 (site_base > 0); w3 has pseudo-site prefixes on 64-multiples in the span
    of the multi-window calls, w4 in its own span (pair_counts); w1, w2 lie in the last, partial chunk"""
    base = 165 & ~63
    cps = pseudo_prefix(g, base)
    lo3 = next(s for s in range(200, 330) if s % 64 and cps[s - base] % 64 == 0 and cps[s - base] > 0)
    hi3 = next(s for s in range(lo3 + 20, 448) if s % 64 and cps[s - base] % 64 == 0)
    own = pseudo_prefix(g, 320)
    assert own[352 - 320] == 64 and own[416 - 320] == 192
    return [(165, 230), (451, EDGE_S), (460, 470), (lo3, hi3), (352, 416), (170, 171), (175, 177), (300, 311)], base


def test_plane_span_edges(eng):
    g = edge_geno()
    wins, base = edge_windows(g)
    assert base == 128 and min(w[0] for w in wins) == 165 and EDGE_S % 64 != 0
    eng.upload(g, np.arange(1, EDGE_S + 1, dtype=np.int32))
    eng.set_windows([w[0] for w in wins], [w[1] for w in wins])
    for w, (lo, hi) in enumerate(wins):
        rd, rn = ref_counts(g[lo:hi])
        d, n = eng.pair_counts(w)
        assert_tensor_path(kernels(eng), True)
        assert_int_equal(n, rn, "n window [%d, %d)" % (lo, hi))
        assert_int_equal(d, rd, "diff window [%d, %d)" % (lo, hi))
    _check_plane_consumers(eng, g, wins)


def test_span_without_variable_sites(eng):
    """npseudo = 0: the P / Q planes are never built, k2t_het and the diff Gram still run over an empty pseudo-site range"""
    rng = np.random.default_rng(0)
    S, H = 150, 24
    g = np.repeat(rng.integers(0, 4, S)[:, None], H, axis=1).astype(np.int8)
    apply_missing(rng, g, 0.1, True)
    wins = [(0, S), (37, 100), (64, 128)]
    eng.upload(g, np.arange(1, S + 1, dtype=np.int32))
    eng.set_windows([w[0] for w in wins], [w[1] for w in wins])
    for w, (lo, hi) in enumerate(wins):
        d, n = eng.pair_counts(w)
        t = kernels(eng)
        assert "k2t_gram_diff" in t and "k2t_build_pq" not in t, t
        assert not d.any()
        assert_int_equal(n, ref_counts(g[lo:hi])[1], "n window %d" % w)
    _check_plane_consumers(eng, g, wins)
    assert "k2t_build_pq" not in kernels(eng)


def _check_plane_consumers(eng, g, wins):
    """ind_het (k2t_het: valid words + P / Q words over the window's pseudo-site range), seq_nonnan, hapstats"""
    H = g.shape[1]
    hap_ind = (np.arange(H) // 2).astype(np.int32)
    for min_sites in (0, 30):
        het = eng.ind_het(hap_ind, H // 2, min_sites)
        assert_tensor_path(kernels(eng), True, gram=False)
        for w, (lo, hi) in enumerate(wins):
            assert_close(het[w], do.sample_het(g[lo:hi], hap_ind, H // 2, min_sites), "het window %d" % w, rtol=1e-12)
    nn = eng.seq_nonnan()
    assert_tensor_path(kernels(eng), True, gram=False)
    for w, (lo, hi) in enumerate(wins):
        assert np.array_equal(nn[w], (g[lo:hi] >= 0).sum(axis=0)), w
    hap_pop = (np.arange(H) >= H // 2).astype(np.int32)
    eng.set_pops(hap_pop, 2)
    for max_dist, min_sites, diag_nan in ((0.1, 0, False), (0.0, 5, True)):
        hs = eng.hapstats(max_dist, min_sites, diag_nan)
        assert_tensor_path(kernels(eng), True)
        for w, (lo, hi) in enumerate(wins):
            want = do.h12_stats(g[lo:hi], hap_pop, 2, max_dist, min_sites, diag_nan)
            assert_close(hs[w], want, "hapstats window %d (%g, %d, %s)" % (w, max_dist, min_sites, diag_nan), rtol=1e-12)


# ======================================================================================================================
# 6. clustering width limit
# ======================================================================================================================
def test_hapstats_clustering_width_limit(eng):
    """1248 haplotypes in one population is the largest that k2_hap_epi's shared memory (200 KiB) holds; 1249 is refused
    on the host before any launch"""
    from genomics_general_b200._lib import PgError
    assert clustering_smem(1248) <= 200 * 1024 < clustering_smem(1249)
    rng = np.random.default_rng(1248)
    H, S = 1250, 40
    founders = rng.integers(0, 3, (24, S))
    g = founders[rng.integers(0, 24, H)].T.astype(np.int8)       # few haplotype families: large clusters
    mut = rng.random((S, H)) < 0.02
    g[mut] = rng.integers(0, 4, int(mut.sum()))
    apply_missing(rng, g, 0.01, True)
    g = np.ascontiguousarray(g)
    hap_pop = np.full(H, -1, dtype=np.int32)
    hap_pop[:1248] = 0
    wins = [(0, S), (5, 30)]
    eng.upload(g, np.arange(1, S + 1, dtype=np.int32))
    eng.set_pops(hap_pop, 1)
    eng.set_windows([w[0] for w in wins], [w[1] for w in wins])
    for max_dist in (0.0, 0.05):
        out = eng.hapstats(max_dist)
        t = kernels(eng)
        assert_tensor_path(t, True)
        assert t["k2_hap_epi"] == 1
        for w, (lo, hi) in enumerate(wins):
            want = do.h12_stats(g[lo:hi], hap_pop, 1, max_dist)
            assert want[0, 0] > 1.0 / 1248                             # not all singletons
            assert_close(out[w], want, "window %d max_dist %g" % (w, max_dist), rtol=1e-12)
    hap_pop[1248] = 0
    eng.set_pops(hap_pop, 1)
    with pytest.raises(PgError, match="too large"):
        eng.hapstats(0.0)
    assert eng.last_timings() == {}


# ======================================================================================================================
# 7. argument checks and early returns
# ======================================================================================================================
def test_checks_and_early_returns(eng):
    """the order of the entry points' checks and early returns, messages included: with no windows pg_pairdist and
    pg_ind_het return before they read hap_ind and pg_hapstats before its population check; with only empty windows nothing
    needs a haplotype; pg_pairdist_cat (one window over every site) checks its selection at once"""
    from genomics_general_b200._lib import PgError

    def raises(msg, fn):
        with pytest.raises(PgError, match=re.escape(msg)):
            fn()

    S, H = 100, 6
    g = random_geno(np.random.default_rng(11), S, H, 0.05)
    eng.upload(g, np.arange(1, S + 1, dtype=np.int32))
    bad = np.array([0, 0, 1, 1, 3, 2], dtype=np.int32)     # n_ind = 3: haplotype 4 is out of range
    none = np.full(H, -1, dtype=np.int32)
    raises("pg_pairdist: n_ind must be >= 1", lambda: eng.pairdist(bad, 0))
    raises("pg_ind_het: n_ind must be >= 1", lambda: eng.ind_het(bad, 0))
    raises("pg_pairdist_cat: n_ind must be >= 1", lambda: eng.pairdist_cat(bad, 0))
    raises("pg_pairdist_cat: hap_ind[4]=3 out of range", lambda: eng.pairdist_cat(bad, 3))
    raises("pg_pairdist_cat: no haplotypes selected", lambda: eng.pairdist_cat(none, 3))

    eng.set_windows(np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64))
    assert eng.pairdist(bad, 3)["dist"].shape == (0, 3, 3)
    assert eng.ind_het(bad, 3).shape == (0, 3)
    eng.set_pops(np.zeros(H, dtype=np.int32), 2)           # population 1 has no haplotypes
    assert eng.hapstats(0.0).shape == (0, 2, 3)
    assert eng.seq_nonnan().shape == (0, H)
    assert eng.last_timings() == {}

    eng.set_windows([0, 50], [0, 50])
    raises("pg_pairdist: hap_ind[4]=3 out of range", lambda: eng.pairdist(bad, 3))
    raises("pg_ind_het: hap_ind[4]=3 out of range", lambda: eng.ind_het(bad, 3))
    raises("pg_hapstats: population 1 has no haplotypes", lambda: eng.hapstats(0.0))
    r = eng.pairdist(none, 3)
    assert np.all(np.isnan(r["dist"])) and not r["sites"].any() and not r["pos_sum"].any()
    assert np.all(np.isnan(eng.ind_het(none, 3)))
    assert not eng.seq_nonnan().any()
    d, n = eng.pair_counts(1)
    assert not d.any() and not n.any() and eng.last_timings() == {}
    raises("pg_pair_counts: window 2 out of range", lambda: eng.pair_counts(2))
    raises("pg_pair_counts: window -1 out of range", lambda: eng.pair_counts(-1))

    eng.set_windows([0, 50], [0, 60])
    raises("pairwise path: no haplotypes selected", lambda: eng.pairdist(none, 3))
    het = eng.ind_het(none, 3)                              # no haplotype selected: all nan, nothing launched
    assert het.shape == (2, 3) and np.all(np.isnan(het)) and eng.last_timings() == {}
