"""The library's record paths on one GPU, against the direct calls on the same state:

  a. the pipelined gather (pg_popgen_gather_begin / _end) without a communicator: identical batches, window batches over one
     matrix, a change of populations, a batch with fewer windows than its slot held, the popFreq columns, W = 0 and S = 0
  b. the matrix replaced between two begins (an upload of the same shape, of another shape, a synth fill)
  c. a 1-rank NCCL communicator: the popgen, ABBA-BABA and fourPop all-gathers, and pairdist_cat
  d. the range ingest (pg_ingest_file_range + pg_ingest_meta) of 2, 3 and 5 ranks, run in turn on one context
  e. the halo append (pg_append_sites) as mgpu.assign_windows + mgpu.fetch_halo use it, and on its own

A record path and its direct call (pg_popgen, pg_abbababa, pg_fourpop, pg_pairdist_cat, a fresh upload) run the same kernels on
the same sites in the same tiling, so integer columns must be equal and fp64 columns bit-identical (compared as uint64).  A few
windows per case also check the direct call against oracle/dense_oracle.py, so that the two cannot be wrong together."""
import contextlib
import warnings

import numpy as np
import pytest

from helpers import assert_close
from oracle import dense_oracle as do

pytestmark = pytest.mark.gpu

MS, MD = 10, 0.01                 # min_sites, min_data of every popgen call
S_MAIN = 24000


@pytest.fixture(scope="module")
def eng():
    from genomics_general_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def synth_data(miss, seed, S=S_MAIN, n_pops=4, spp=8):
    from genomics_general_b200 import synth
    spec = synth.SynthSpec(n_pops, spp, miss=miss, seed=seed)
    return spec, synth.synth_genotypes(spec, 0, S), synth.synth_positions(S, seed=seed)


def mixed_data(seed, S=S_MAIN):
    """complete sites in the first half, 3 % missing genotypes in the second: closed-form and pairwise windows side by side
    (the generator draws the alleles first, so both halves come from one matrix)"""
    spec, g, pos = synth_data(0.0, seed, S)
    _, g3, _ = synth_data(0.03, seed, S)
    g[S // 2:] = g3[S // 2:]
    return spec, g, pos


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def direct(eng, lo, hi):
    eng.set_windows(np.asarray(lo, np.int64), np.asarray(hi, np.int64))
    return eng.popgen(MS, MD)


def n_pairwise(ref):
    return int((ref["path"] == 2).sum())


def check_rows(table, ref, P, what):
    """the first W records of a gathered table against pg_popgen: integers equal, fp64 bit-identical"""
    from genomics_general_b200 import multigpu
    W = len(ref["sites"])
    assert table.shape[1] == 4 + 5 * P + P * (P - 1), (what, table.shape, P)
    got = multigpu.unpack_device_records(np.ascontiguousarray(table[:W]), P)
    for k in ("sites", "pos_sum", "path"):
        bad = np.flatnonzero(got[k] != ref[k])
        assert bad.size == 0, "%s: %s differs in windows %s: %s vs %s" % (what, k, bad[:8], got[k][bad[:8]], ref[k][bad[:8]])
    for k in ("pi", "dxy", "fst"):
        bad = np.flatnonzero((bits(got[k]) != bits(ref[k])).any(axis=1)) if got[k].size else []
        assert len(bad) == 0, "%s: %s not bit-identical in windows %s" % (what, k, bad[:8])


def check_tail_zero(table, W, what):
    nz = np.flatnonzero(bits(table[W:]).any(axis=1))
    assert nz.size == 0, "%s: rows %s past the batch's %d windows are not zero" % (what, W + nz[:8], W)


def check_oracle(g, hap_pop, P, lo, hi, ref, ws):
    for w in ws:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            pi, dxy, fst = do.group_dist_stats(g[lo[w]:hi[w]], hap_pop, P, MS, MD)
        assert_close(ref["pi"][w], pi, "pi[%d]" % w, rtol=1e-9)
        assert_close(ref["dxy"][w], dxy, "dxy[%d]" % w, rtol=1e-9)
        assert_close(ref["fst"][w], fst, "fst[%d]" % w, rtol=1e-8)


def pipeline(eng, n, w_max, prepare):
    """prepare(0); begin(0); prepare(1); begin(1); end(0); prepare(2); begin(0); end(1); ... -> [(table copy, n_pairwise)]"""
    out = [None] * n
    prepare(0)
    eng.popgen_gather_begin(w_max, 0, MS, MD)
    for k in range(1, n):
        prepare(k)
        eng.popgen_gather_begin(w_max, k & 1, MS, MD)
        t, nk2 = eng.popgen_gather_end(w_max, (k - 1) & 1, with_pairwise=True)
        out[k - 1] = (t.copy(), nk2)
    t, nk2 = eng.popgen_gather_end(w_max, (n - 1) & 1, with_pairwise=True)
    out[n - 1] = (t.copy(), nk2)
    return out


def check_batches(outs, refs, Ps, what):
    for k, ((t, nk2), ref) in enumerate(zip(outs, refs)):
        check_rows(t, ref, Ps[k], "%s, batch %d" % (what, k))
        check_tail_zero(t, len(ref["sites"]), "%s, batch %d" % (what, k))
        assert nk2 == n_pairwise(ref), "%s, batch %d: n_pairwise %d, the batch has %d" % (what, k, nk2, n_pairwise(ref))


# ---- a. pipelined gather, no communicator -----------------------------------------------------------------------------
@pytest.mark.parametrize("miss", [0.0, 0.03])
def test_pipelined_identical_batches(eng, miss):
    """bench.py's pattern: one batch, five steps"""
    spec, g, pos = synth_data(miss, 11)
    hp = spec.hap_pop()
    eng.upload(g, pos)
    eng.set_pops(hp, 4)
    lo = np.arange(0, S_MAIN, 1000, dtype=np.int64)
    hi = lo + 1000
    ref = direct(eng, lo, hi)
    assert (n_pairwise(ref) == len(lo)) if miss else (n_pairwise(ref) == 0)
    check_oracle(g, hp, 4, lo, hi, ref, [0, 11, len(lo) - 1])
    outs = pipeline(eng, 5, len(lo) + 3, lambda k: None)
    check_batches(outs, [ref] * 5, [4] * 5, "identical batches, miss %g" % miss)


def window_batches():
    S = S_MAIN
    b = [(np.arange(0, S, 1000), np.arange(0, S, 1000) + 1000),                          # 24 tiling windows
         (np.arange(500, S - 1500, 700), np.arange(500, S - 1500, 700) + 1500),          # 32 overlapping windows
         (np.array([100, 13000, 5000, 20000]), np.array([100, 13020, 9000, S - 1])),     # an empty window, out of order
         (np.arange(12000, S, 200), np.arange(12000, S, 200) + 50),                      # 60 short windows, all ragged
         (np.array([0]), np.array([S]))]                                                  # one window over everything
    return [(np.asarray(lo, np.int64), np.asarray(hi, np.int64)) for lo, hi in b]


def test_pipelined_window_batches(eng):
    """each begin sees other windows over one resident matrix; set_windows runs between begin(k) and begin(k+1)"""
    spec, g, pos = mixed_data(5)
    hp = spec.hap_pop()
    eng.upload(g, pos)
    eng.set_pops(hp, 4)
    batches = window_batches()
    refs = [direct(eng, lo, hi) for lo, hi in batches]
    assert all(0 < n_pairwise(r) for r in refs[:4]) and n_pairwise(refs[0]) < len(batches[0][0])
    check_oracle(g, hp, 4, *batches[2], refs[2], [1, 2, 3])
    check_oracle(g, hp, 4, *batches[1], refs[1], [0, 17, 30])
    w_max = max(len(lo) for lo, _ in batches)
    outs = pipeline(eng, len(batches), w_max, lambda k: eng.set_windows(*batches[k]))
    check_batches(outs, refs, [4] * len(batches), "window batches")


def pop_maps():
    hp = np.repeat(np.arange(4, dtype=np.int32), 16)
    three = np.minimum(hp, 2)
    six = np.minimum(np.arange(64, dtype=np.int32) // 11, 5)
    return [(hp, 4), (three, 3), (six, 6), (hp, 4)]


def test_pipelined_population_change(eng):
    """set_pops between two begins: each slot keeps the record width of its own batch"""
    _, g, pos = synth_data(0.0, 13)
    eng.upload(g, pos)
    lo = np.arange(0, S_MAIN, 1500, dtype=np.int64)
    hi = lo + 1500
    maps = pop_maps()
    refs = []
    for hp, P in maps:
        eng.set_pops(hp, P)
        refs.append(direct(eng, lo, hi))
        assert n_pairwise(refs[-1]) == 0
    check_oracle(g, maps[2][0], 6, lo, hi, refs[2], [0, 9])
    outs = pipeline(eng, len(maps), len(lo), lambda k: eng.set_pops(*maps[k]))
    check_batches(outs, refs, [P for _, P in maps], "population change")


def test_pipelined_population_change_with_pairwise_windows_refuses(eng):
    """with ragged windows pending, the populations of the next batch cannot serve this slot's pairwise path: end refuses"""
    from genomics_general_b200._lib import PgError
    _, g, pos = mixed_data(17)
    eng.upload(g, pos)
    lo = np.arange(0, S_MAIN, 1500, dtype=np.int64)
    hi = lo + 1500
    (hpa, Pa), (hpb, Pb) = pop_maps()[:2]
    eng.set_pops(hpb, Pb)
    ref_b = direct(eng, lo, hi)
    eng.set_pops(hpa, Pa)
    eng.popgen_gather_begin(len(lo), 0, MS, MD)
    eng.set_pops(hpb, Pb)
    eng.popgen_gather_begin(len(lo), 1, MS, MD)
    with pytest.raises(PgError, match="changed after this slot's pg_popgen_gather_begin"):
        eng.popgen_gather_end(len(lo), 0)
    t, nk2 = eng.popgen_gather_end(len(lo), 1, with_pairwise=True)
    check_rows(t, ref_b, Pb, "the batch after the refused one")
    assert nk2 == n_pairwise(ref_b) > 0


def test_pipelined_fewer_windows_in_the_same_slot(eng):
    """a slot's rows W..w_max-1 must not keep an earlier batch's records, and n_pairwise counts this batch only"""
    spec, g, pos = mixed_data(19)
    hp = spec.hap_pop()
    eng.upload(g, pos)
    eng.set_pops(hp, 4)
    big = (np.arange(0, S_MAIN, 800, dtype=np.int64), np.arange(0, S_MAIN, 800, dtype=np.int64) + 800)
    big2 = (big[0] + 100, np.minimum(big[1] + 100, S_MAIN))
    small = (np.array([0, 3000, 9000, 12500, 15000, 18000, 21000], np.int64),
             np.array([900, 3900, 9900, 13400, 15900, 18900, 21900], np.int64))
    small2 = (small[0][:5] + 50, small[1][:5] + 50)
    w_max = len(big[0])
    refs = {k: direct(eng, *b) for k, b in dict(big=big, big2=big2, small=small, small2=small2).items()}
    assert 0 < n_pairwise(refs["small"]) < len(small[0]) and n_pairwise(refs["big"]) > n_pairwise(refs["small"])
    # one slot, one batch at a time
    for name, b in (("big", big), ("small", small)):
        eng.set_windows(*b)
        eng.popgen_gather_begin(w_max, 0, MS, MD)
        t, nk2 = eng.popgen_gather_end(w_max, 0, with_pairwise=True)
        check_tail_zero(t, len(b[0]), "sequential " + name)
        assert nk2 == n_pairwise(refs[name]), ("sequential " + name, nk2, n_pairwise(refs[name]))
        check_rows(t, refs[name], 4, "sequential " + name)
    # pipelined: slot 0 holds big, then small; slot 1 big2, then small2
    order = [big, big2, small, small2]
    outs = pipeline(eng, 4, w_max, lambda k: eng.set_windows(*order[k]))
    check_batches(outs, [refs["big"], refs["big2"], refs["small"], refs["small2"]], [4] * 4, "shrinking W")


def test_pipelined_freqstats_columns(eng):
    """set_freqstats(True): the popFreq columns of each slot's records equal popgen_freqstats() of its batch"""
    from genomics_general_b200 import multigpu
    spec, g, pos = mixed_data(23)
    eng.upload(g, pos)
    eng.set_pops(spec.hap_pop(), 4)
    batches = window_batches()[:3]
    eng.set_freqstats(True)
    try:
        refs, fss = [], []
        for lo, hi in batches:
            refs.append(direct(eng, lo, hi))
            fss.append(eng.popgen_freqstats())
        outs = pipeline(eng, len(batches), max(len(lo) for lo, _ in batches), lambda k: eng.set_windows(*batches[k]))
    finally:
        eng.set_freqstats(False)
    check_batches(outs, refs, [4] * 3, "freqstats")
    for k, ((t, _), fs) in enumerate(zip(outs, fss)):
        fq = multigpu.unpack_device_records(np.ascontiguousarray(t[:len(refs[k]["sites"])]), 4)["popfreq"]
        assert np.isfinite(fq[:, 0]).any(), "batch %d: no popFreq column was computed" % k
        assert np.array_equal(bits(fq[:, 0]), bits(fs["l"])), "batch %d: l" % k
        for j, name in enumerate(("S", "thetaPi", "thetaW", "TajD")):
            assert np.array_equal(bits(fq[:, 1 + 4 * j:5 + 4 * j]), bits(fs[name])), "batch %d: %s" % (k, name)


def test_pipelined_no_windows_and_no_sites(eng):
    """W = 0 leaves nothing to compute (the slot must read as zeros); S = 0 gives the host-built records of pg_popgen_enqueue"""
    spec, g, pos = mixed_data(29)
    hp = spec.hap_pop()
    eng.upload(g, pos)
    eng.set_pops(hp, 4)
    lo, hi = window_batches()[2]
    ref = direct(eng, lo, hi)
    eng.popgen_gather_begin(6, 0, MS, MD)
    t, nk2 = eng.popgen_gather_end(6, 0, with_pairwise=True)
    check_rows(t, ref, 4, "before W = 0")
    eng.set_windows(np.zeros(0, np.int64), np.zeros(0, np.int64))
    eng.popgen_gather_begin(6, 0, MS, MD)
    t, nk2 = eng.popgen_gather_end(6, 0, with_pairwise=True)
    check_tail_zero(t, 0, "W = 0")
    assert nk2 == 0
    # no sites: every window is empty
    eng.upload(np.zeros((0, g.shape[1]), np.int8), np.zeros(0, np.int32))
    eng.set_pops(hp, 4)
    z = np.zeros(3, np.int64)
    for ms in (MS, 0):
        eng.set_windows(z, z)
        ref = eng.popgen(ms, MD)
        assert np.all(ref["sites"] == 0) and np.all(ref["path"] == (0 if ms else 1)) and np.isnan(ref["pi"]).all()
        eng.popgen_gather_begin(5, 1, ms, MD)
        t, nk2 = eng.popgen_gather_end(5, 1, with_pairwise=True)
        check_rows(t, ref, 4, "S = 0, min_sites %d" % ms)
        check_tail_zero(t, 3, "S = 0, min_sites %d" % ms)
        assert nk2 == 0


# ---- b. the matrix replaced between two begins ------------------------------------------------------------------------
def load(eng, how, miss, seed):
    """upload (same or other shape) or synth_fill; returns (genotypes, hap_pop, windows)"""
    from genomics_general_b200 import synth
    S = S_MAIN if how != "upload_other_shape" else 15000
    spp = 8 if how != "upload_other_shape" else 6
    spec, g, pos = synth_data(miss, seed, S, 4, spp)
    if how == "synth_fill":
        eng.synth_fill(synth.SynthSpec(4, spp, miss=miss, seed=seed), S)
    else:
        eng.upload(g, pos)
    eng.set_pops(spec.hap_pop(), 4)
    lo = np.arange(0, S, 1300, dtype=np.int64)
    hi = np.minimum(lo + 1300, S)
    eng.set_windows(lo, hi)
    return g, spec.hap_pop(), (lo, hi)


@pytest.mark.parametrize("ragged", [False, True], ids=["complete", "ragged"])
@pytest.mark.parametrize("how", ["upload_same_shape", "upload_other_shape", "synth_fill"])
def test_pipelined_data_replaced_between_begins(eng, how, ragged):
    """complete data: both slots are right.  Ragged windows of batch 0 would need batch 0's matrix after batch 1 replaced it:
    end(0) refuses (PgError naming the cause) instead of returning rows computed from the other data"""
    from genomics_general_b200._lib import PgError
    miss = 0.03 if ragged else 0.0
    load(eng, "upload_same_shape", miss, 31)
    ref_a = eng.popgen(MS, MD)
    g_b, hp_b, wb = load(eng, how, miss, 37)
    ref_b = eng.popgen(MS, MD)
    check_oracle(g_b, hp_b, 4, *wb, ref_b, [0, len(wb[0]) - 1])
    assert (n_pairwise(ref_a) > 0) == ragged and (n_pairwise(ref_b) > 0) == ragged
    w_max = max(len(ref_a["sites"]), len(ref_b["sites"]))
    load(eng, "upload_same_shape", miss, 31)
    eng.popgen_gather_begin(w_max, 0, MS, MD)
    load(eng, how, miss, 37)
    eng.popgen_gather_begin(w_max, 1, MS, MD)
    if ragged:
        with pytest.raises(PgError, match="genotype matrix or the populations changed"):
            eng.popgen_gather_end(w_max, 0)
    else:
        t, nk2 = eng.popgen_gather_end(w_max, 0, with_pairwise=True)
        check_batches([(t, nk2)], [ref_a], [4], "batch before the %s" % how)
    t, nk2 = eng.popgen_gather_end(w_max, 1, with_pairwise=True)
    check_batches([(t, nk2)], [ref_b], [4], "batch after the %s" % how)


# ---- c. 1-rank NCCL communicator --------------------------------------------------------------------------------------
@contextlib.contextmanager
def one_rank(eng):
    """a communicator of this process alone (no other host is contacted); torch is imported first so that the library binds
    the libnccl torch has already loaded"""
    import torch  # noqa: F401
    from genomics_general_b200._lib import PgError
    try:
        eng.nccl_init(1, 0, eng.nccl_unique_id())
    except PgError as e:
        pytest.skip("NCCL is not available: %s" % e)
    try:
        yield
    finally:
        eng.nccl_finalize()


def test_nccl_pipelined_gather_collective_refusal(eng):
    """with a communicator, `end` agrees on a refusal through an all-reduce before the second gather: a slot with unchanged
    data is resolved, a slot whose pairwise windows need a replaced matrix is refused, and the next slot is still right"""
    from genomics_general_b200._lib import PgError
    load(eng, "upload_same_shape", 0.03, 31)
    ref_a = eng.popgen(MS, MD)
    load(eng, "upload_same_shape", 0.03, 37)
    ref_b = eng.popgen(MS, MD)
    assert n_pairwise(ref_a) > 0 and n_pairwise(ref_b) > 0
    w_max = len(ref_a["sites"]) + 2
    with one_rank(eng):
        load(eng, "upload_same_shape", 0.03, 31)
        eng.popgen_gather_begin(w_max, 0, MS, MD)
        check_batches([eng.popgen_gather_end(w_max, 0, with_pairwise=True)], [ref_a], [4], "unchanged data, one rank")
        eng.popgen_gather_begin(w_max, 0, MS, MD)
        load(eng, "upload_same_shape", 0.03, 37)
        eng.popgen_gather_begin(w_max, 1, MS, MD)
        with pytest.raises(PgError, match="genotype matrix or the populations changed"):
            eng.popgen_gather_end(w_max, 0)
        check_batches([eng.popgen_gather_end(w_max, 1, with_pairwise=True)], [ref_b], [4], "after the refusal, one rank")


@pytest.mark.parametrize("data", ["complete", "mixed"])
def test_nccl_popgen_allgather(eng, data):
    """one rank: the table is pg_popgen's records, rows past W zero; with missing data the resolve and second gather run,
    and a later call with fewer windows and the same w_max leaves no earlier record behind"""
    spec, g, pos = synth_data(0.0, 41) if data == "complete" else mixed_data(41)
    eng.upload(g, pos)
    eng.set_pops(spec.hap_pop(), 4)
    batches = window_batches()
    refs = [direct(eng, lo, hi) for lo, hi in batches]
    assert (n_pairwise(refs[0]) > 0) == (data == "mixed")
    w_max = 64
    with one_rank(eng):
        for k in (3, 0, 2, 4):                             # 60, 24, 4 (with an empty window) and 1 window
            eng.set_windows(*batches[k])
            table = np.full((w_max, eng.popgen_record_width()), np.nan)
            nk2 = eng.popgen_allgather(w_max, table, MS, MD)
            check_batches([(table, nk2)], [refs[k]], [4], "popgen_allgather, %s, batch %d" % (data, k))


def test_nccl_abba_fourpop_allgather_then_popgen(eng):
    """ABBA-BABA and fourPop (3 modes) records against the direct calls; then a popgen all-gather into the same buffer, with
    the same table size: its rows past W lie where ABBA-BABA records were, and the zeroing of rows W..w_max-1 in every
    popgen all-gather is what must clear them"""
    from genomics_general_b200 import multigpu
    spec, g, pos = mixed_data(43)
    hp = spec.hap_pop()
    eng.upload(g, pos)
    eng.set_pops(hp, 4)
    lo = np.arange(0, S_MAIN, 2400, dtype=np.int64)        # 10 windows
    hi = lo + 2400
    eng.set_windows(lo, hi)
    ref_p = eng.popgen(MS, MD)
    ref_a = eng.abbababa(0, 1, 2, 3, 0.5)
    ref_f = {m: eng.fourpop(0, 1, 2, 3, 0.5, **kw) for m, kw in (("default", {}), ("polarize", dict(polarize=True)),
                                                                 ("fixed", dict(fixed=True)))}
    for w in (0, 9):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ab = do.abbababa(g[lo[w]:hi[w]], hp, 0, 1, 2, 3, 0.5)
        for k in ("ABBA", "BABA", "D", "fd", "fdM"):
            assert_close(ref_a[k][w], ab[k], "abba %s[%d]" % (k, w), rtol=1e-9, atol=1e-9)
    w_abba = 81                                            # 81 * 8 words = 18 popgen records of 36 words
    with one_rank(eng):
        t8 = np.full((w_abba, 8), np.nan)
        eng.abbababa_allgather(0, 1, 2, 3, 0.5, w_abba, t8)
        got = multigpu.unpack_abba_records(t8[:len(lo)])
        for k in ("sites", "pos_sum"):
            assert np.array_equal(got[k], ref_a[k]), k
        for k in ("ABBA", "BABA", "D", "fd", "fdM", "sitesUsed"):
            assert np.array_equal(bits(got[k]), bits(ref_a[k])), k
        check_tail_zero(t8, len(lo), "abbababa_allgather")
        for m, kw in (("default", {}), ("polarize", dict(polarize=True)), ("fixed", dict(fixed=True))):
            t17 = np.full((len(lo) + 2, 17), np.nan)
            eng.fourpop_allgather(0, 1, 2, 3, 0.5, len(lo) + 2, t17, **kw)
            got = multigpu.unpack_fourpop_records(t17[:len(lo)])
            for k in ("sites", "pos_sum"):
                assert np.array_equal(got[k], ref_f[m][k]), (m, k)
            for k in multigpu.FOURPOP_KEYS + ("sitesUsed",):
                assert np.array_equal(bits(got[k]), bits(ref_f[m][k])), (m, k)
            check_tail_zero(t17, len(lo), "fourpop_allgather " + m)
        eng.abbababa_allgather(0, 1, 2, 3, 0.5, w_abba, t8)
        t36 = np.full((18, eng.popgen_record_width()), np.nan)
        assert t36.size == t8.size
        nk2 = eng.popgen_allgather(18, t36, MS, MD)
        check_batches([(t36, nk2)], [ref_p], [4], "popgen_allgather after abbababa_allgather")


def test_nccl_pairdist_cat(eng):
    """--windType cat: the all-reduce of one rank leaves the matrix of the local sites, bit-identical to the call without a
    communicator and to pg_pairdist on one window over every site"""
    spec, g, _ = synth_data(0.04, 47, 30001, 3, 6)
    hap_ind = (np.arange(g.shape[1]) // 2).astype(np.int32)
    n_ind = g.shape[1] // 2
    eng.upload(g, None)
    with one_rank(eng):
        got, tot = eng.pairdist_cat(hap_ind, n_ind, False)
        eng.nccl_finalize()
        ref, tot_ref = eng.pairdist_cat(hap_ind, n_ind, False)
    assert tot == tot_ref == g.shape[0]
    assert np.array_equal(bits(got), bits(ref))
    eng.set_windows([0], [g.shape[0]])
    one = eng.pairdist(hap_ind, n_ind, False)["dist"][0]
    assert np.array_equal(bits(one), bits(ref))


# ---- d. range ingest on one context -----------------------------------------------------------------------------------
SCAFFOLDS = (("chrA", 900), ("chrB", 1300), ("chrC", 800))     # no cut of 2, 3 or 5 ranks lands on a scaffold boundary


class GenoFile:
    def __init__(self, path, miss, seed):
        from genomics_general_b200 import geno_io, synth
        S = sum(n for _, n in SCAFFOLDS)
        spec, g, _ = synth_data(miss, seed, S, 4, 6)
        scaf = np.concatenate([[name] * n for name, n in SCAFFOLDS])
        pos = np.concatenate([synth.synth_positions(n, seed=seed + k) for k, (_, n) in enumerate(SCAFFOLDS)])
        synth.write_geno(path, g, pos, scaf, spec.sample_names())
        self.path, self.spec = str(path), spec
        self.whole = geno_io.parse_geno(self.path)
        assert np.array_equal(self.whole.geno, g) and np.array_equal(self.whole.pos, pos)
        data = open(self.path, "rb").read()
        nl = np.flatnonzero(np.frombuffer(data, np.uint8) == 10)
        self.body_off = int(nl[0]) + 1
        self.line_off = (nl[:-1] + 1).astype(np.int64)               # host offsets of the data lines
        sid = self.whole.scaf_ids
        self.newsc = np.concatenate([[1], sid[1:] != sid[:-1]]).astype(np.int8)
        file_names, samples, self.fmt, pl, col_take = geno_io._select(self.whole.header, "phased", None, None)
        self.col_hap, self.col_pl, _, self.H = geno_io._column_maps(file_names, samples, pl, col_take)

    def rows_of(self, lo, hi):
        return int(np.searchsorted(self.line_off, lo)), int(np.searchsorted(self.line_off, hi))

    def ingest(self, eng, lo, hi):
        return eng.ingest_file_range(self.path, lo, hi, self.fmt, self.col_hap, self.col_pl, self.H)


@pytest.fixture(scope="module", params=[0.0, 0.03], ids=["complete", "missing"])
def geno_file(request, tmp_path_factory):
    return GenoFile(tmp_path_factory.mktemp("geno") / "data.geno", request.param, 53)


@pytest.mark.parametrize("world", [2, 3, 5])
def test_ingest_file_range_ranks(eng, geno_file, world):
    from genomics_general_b200 import geno_io, mgpu
    gf, whole = geno_file, geno_file.whole
    ranges = mgpu.byte_ranges(gf.path, gf.body_off, world)
    cuts = [gf.rows_of(lo, hi)[0] for lo, hi in ranges[1:]]
    assert any(gf.newsc[c] == 0 for c in cuts), "no cut inside a scaffold"
    for r, (lo, hi) in enumerate(ranges):
        a, b = gf.rows_of(lo, hi)
        S = gf.ingest(eng, lo, hi)
        assert S == b - a, (world, r, S, b - a)
        g, pos = eng.download(0, S)
        assert np.array_equal(g, whole.geno[a:b]) and np.array_equal(pos, whole.pos[a:b]), (world, r)
        pos_m, newsc, off = eng.ingest_meta(S)
        assert np.array_equal(pos_m, whole.pos[a:b])
        assert np.array_equal(off + lo, gf.line_off[a:b]), (world, r, "line offsets")
        want = gf.newsc[a:b].copy()
        want[0] = 1
        assert np.array_equal(newsc, want), (world, r, "new_scaffold")

        def name_at(o):
            with open(gf.path, "rb") as f:
                f.seek(lo + o)
                return f.read(256)
        ids, names = geno_io._scaffold_runs(newsc, off, name_at)
        assert names == [whole.scaf_names[whole.scaf_ids[s]] for s in a + np.flatnonzero(want)], (world, r, names)
        assert np.array_equal(ids, np.cumsum(want) - 1)


def test_ingest_file_range_empty_and_open_ended(eng, geno_file):
    from genomics_general_b200 import mgpu
    gf = geno_file
    lo, hi = mgpu.byte_ranges(gf.path, gf.body_off, 3)[2]
    assert gf.ingest(eng, lo, lo) == 0
    assert eng.ingest_meta(0)[0].shape == (0,)
    a, b = gf.rows_of(lo, hi)
    assert gf.ingest(eng, lo, -1) == b - a == len(gf.line_off) - a
    g, pos = eng.download(0, b - a)
    assert np.array_equal(g, gf.whole.geno[a:]) and np.array_equal(pos, gf.whole.pos[a:])
    _, _, off = eng.ingest_meta(b - a)
    assert np.array_equal(off + lo, gf.line_off[a:])


# ---- e. append --------------------------------------------------------------------------------------------------------
def abba_close(got, ref, what):
    """a rank's matrix starts at another site than the whole file's: the fp64 ABBA / BABA sums of the site pass run in
    another order (tile and CTA boundaries move), so bitwise equality cannot hold; the tolerances of
    test_gpu_site_pass_bounds.py apply, with an absolute floor for the ratios"""
    for k in ("sites", "pos_sum"):
        assert np.array_equal(got[k], ref[k]), (what, k)
    for k in ("ABBA", "BABA", "sitesUsed"):
        assert_close(got[k], ref[k], "%s %s" % (what, k), rtol=1e-9, atol=1e-12)
    for k in ("D", "fd", "fdM"):
        assert_close(got[k], ref[k], "%s %s" % (what, k), rtol=1e-9, atol=1e-9)


def sub(d, idx):
    return {k: np.asarray(v)[idx] for k, v in d.items() if k != "pairs"}


@pytest.mark.parametrize("world", [2, 3])
def test_halo_append_as_a_rank_does(eng, geno_file, world):
    """every rank ingests its byte range, takes the windows whose first site it holds and appends the halo sites that its
    last windows reach into; its statistics equal the whole-file matrix's on those windows"""
    from genomics_general_b200 import mgpu, windows
    gf, whole = geno_file, geno_file.whole
    hp = gf.spec.hap_pop()
    ws = windows.sliding_coord_windows(whole.scaf_ids, whole.scaf_names, whole.pos, 2500, 1100)
    lo, hi = np.array(ws.lo, np.int64), np.array(ws.hi, np.int64)
    eng.upload(whole.geno, whole.pos)
    eng.set_pops(hp, 4)
    eng.set_windows(lo, hi)
    ref_p, ref_a, ref_c = eng.popgen(MS, MD), eng.abbababa(0, 1, 2, 3, 0.5), eng.site_counts()
    assert (n_pairwise(ref_p) > 0) == (gf.spec.miss > 0)
    ranges = mgpu.byte_ranges(gf.path, gf.body_off, world)
    starts = np.array([gf.rows_of(lo_, hi_)[0] for lo_, hi_ in ranges] + [len(gf.line_off)], np.int64)
    for c in starts[1:-1]:
        assert np.any((lo < c) & (hi > c)), "no window straddles the cut at site %d" % c
    gd = mgpu.GlobalGeno(whole.pos, whole.scaf_ids, whole.scaf_names, whole.names, whole.ploidy, whole.header)
    halos = []
    for r, (blo, bhi) in enumerate(ranges):
        S = gf.ingest(eng, blo, bhi)
        assert S == starts[r + 1] - starts[r]
        eng.ingest_meta(S)
        idx, llo, lhi, halo = mgpu.assign_windows(lo, hi, starts, r)
        mgpu.fetch_halo(eng, gf.path, gd, starts, gf.line_off, r, halo, "phased", None)
        halos.append(halo)
        assert eng.S == S + halo
        eng.set_pops(hp, 4)
        eng.set_windows(llo, lhi)
        got = eng.popgen(MS, MD)
        check_rows(_records(got), sub(ref_p, idx), 4, "rank %d of %d" % (r, world))
        abba_close(eng.abbababa(0, 1, 2, 3, 0.5), sub(ref_a, idx), "rank %d of %d" % (r, world))
        a = int(starts[r])
        assert np.array_equal(eng.site_counts(), ref_c[a:a + S + halo]), ("site_counts", r)
    assert all(h > 0 for h in halos[:-1]) and halos[-1] == 0, halos


def _records(res):
    """pg_popgen's dict as a record table (the layout check_rows reads)"""
    W, P = len(res["sites"]), res["pi"].shape[1]
    t = np.zeros((W, 4 + 5 * P + P * (P - 1)))
    t[:, :3] = np.stack([res["sites"], res["pos_sum"], res["path"].astype(np.int64)], axis=1).view(np.float64)
    npairs = P * (P - 1) // 2
    t[:, 3:3 + P], t[:, 3 + P:3 + P + npairs], t[:, 3 + P + npairs:3 + P + 2 * npairs] = res["pi"], res["dxy"], res["fst"]
    return t


def random_rows(rng, n, H, miss=0.03):
    g = rng.integers(0, 4, size=(n, H)).astype(np.int8)
    g[rng.random((n, H)) < miss] = -1
    return g


def check_against_fresh(e, g, pos, hp, what):
    """e holds g after appends: its contents and statistics equal a fresh upload of g on another context"""
    from genomics_general_b200.engine import Engine
    S = g.shape[0]
    got_g, got_p = e.download(0, S)
    assert np.array_equal(got_g, g) and np.array_equal(got_p, pos), what
    lo = np.array([0, S // 3, 0, S - 70, S - 1, 5], np.int64)
    hi = np.array([S, S, S // 2, S, S, S - 3], np.int64)
    res = []
    for x in (e, Engine(0)):
        if x is not e:
            x.upload(g, pos)
        x.set_pops(hp, 4)
        x.set_windows(lo, hi)
        res.append((x.popgen(MS, MD), x.abbababa(0, 1, 2, 3, 0.5), x.site_counts()))
        if x is not e:
            x.close()
    (p1, a1, c1), (p0, a0, c0) = res
    check_rows(_records(p1), p0, 4, what)
    assert n_pairwise(p0) > 0
    for k in ("sites", "pos_sum", "ABBA", "BABA", "D", "fd", "fdM", "sitesUsed"):
        assert np.array_equal(bits(a1[k]) if a1[k].dtype == np.float64 else a1[k],
                              bits(a0[k]) if a0[k].dtype == np.float64 else a0[k]), (what, k)
    assert np.array_equal(c1, c0), what


def test_append_sites_direct():
    """an append that reallocates; one that fits the capacity an earlier, wider matrix left (the appended rows lie past the
    slack that pg_alloc_sites zeroed, so their padding and the rows behind them keep the wider matrix's bytes: H = 38 leaves
    10 padding bytes per row, 300 rows > 64 slack rows); an append of 0 rows"""
    from genomics_general_b200.engine import Engine
    rng = np.random.default_rng(59)
    H = 38
    hp = (np.arange(H) * 4 // H).astype(np.int32)
    g = random_rows(rng, 450, H)
    pos = np.sort(rng.choice(10 ** 6, 450, replace=False)).astype(np.int32) + 1
    with Engine(0) as e:
        e.upload(g[:150], pos[:150])
        e.append_sites(g[150:], pos[150:])                  # (450 + 64) rows exceed the capacity of (150 + 64)
        check_against_fresh(e, g, pos, hp, "append that reallocates")
    with Engine(0) as e:
        wide = rng.integers(0, 4, size=(5000, 200)).astype(np.int8)     # no missing genotype: every byte nonzero
        e.upload(wide, np.arange(1, 5001, dtype=np.int32))
        e.upload(g[:150], pos[:150])
        e.append_sites(g[150:], pos[150:])
        check_against_fresh(e, g, pos, hp, "append inside the capacity of a wider matrix")
        e.append_sites(np.zeros((0, H), np.int8), np.zeros(0, np.int32))
        assert e.S == 450
        check_against_fresh(e, g, pos, hp, "append of 0 rows")
