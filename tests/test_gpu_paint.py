"""distPaint.py on the GPU: pg_distpaint against oracle/paint_oracle.py (assignments equal, means bitwise equal to
np.nanmean, p-values within 1e-12 of scipy's ranksums), its limits, the haploid token width test of the device ingest, and
the command line against the reference's fixtures byte for byte."""
import os

import numpy as np
import pytest

from oracle import paint_oracle as po
from test_paint_cpu import CASES, DIR, expected, run_cli

pytestmark = pytest.mark.gpu


def _data(rng, S, H, miss):
    """haplotypes drawn from four source populations whose allele frequencies differ per site, so that distances differ"""
    src = rng.integers(0, 4, H)
    freq = rng.choice([0.05, 0.3, 0.7, 0.95], size=(S, 4))
    alt = rng.random((S, H)) < freq[:, src]
    bases = rng.permuted(np.tile(np.arange(4, dtype=np.int8), (S, 1)), axis=1)[:, :2]
    g = np.where(alt, bases[:, 1:2], bases[:, 0:1]).astype(np.int8)
    g[rng.random((S, H)) < miss] = -1
    return g


def _pops(rng, H, P):
    """P member lists: sizes from 1 up, with duplicates, drawn from every haplotype"""
    pops = []
    for p in range(P):
        k = 1 if p == 0 else int(rng.integers(2, 12))
        pops.append([int(x) for x in rng.integers(0, H, k)])
    if P > 1:
        pops[-1] += pops[-1][:1]                     # a member listed twice
    return pops


def _windows(S):
    lo = [0, 5, 5, 40, 41, 0, 100, S - 60]
    hi = [37, 5, 6, 160, 260, S, 180, S]               # an empty and a single-site window among them
    return np.array(lo, dtype=np.int64), np.array(hi, dtype=np.int64)


def _same_bits(got, want, what):
    """equal bit for bit, nans aside: their sign bit is not part of np.nanmean's contract"""
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), what
    assert got[~nan].tobytes() == want[~nan].tobytes(), what


@pytest.mark.parametrize("H, P, miss, delta, seed", [
    (1, 1, 0.0, False, 1), (2, 2, 0.02, False, 2), (2, 2, 0.0, True, 3), (31, 5, 0.3, False, 4), (32, 32, 0.02, True, 5),
    (33, 32, 0.0, False, 6), (200, 5, 0.02, False, 7), (200, 2, 0.3, True, 8), (1000, 2, 0.02, False, 9),
])
def test_distpaint_equals_oracle(H, P, miss, delta, seed, monkeypatch):
    from genomics_general_b200.engine import Engine
    monkeypatch.setenv("PG_PAIR_SCRATCH_MB", "1")      # several window batches
    rng = np.random.default_rng(seed)
    S = 400
    g = _data(rng, S, H, miss)
    pops = _pops(rng, H, P)
    ref_off = np.cumsum([0] + [len(m) for m in pops]).astype(np.int32)
    ref_hap = np.array([j for m in pops for j in m], dtype=np.int32)
    query = rng.permutation(H).astype(np.int32)
    lo, hi = _windows(S)
    thr = 0.02 if delta else 0.05
    min_sites = 3
    with Engine(0) as eng:
        eng.upload(g, np.arange(S, dtype=np.int32) * 10 + 1)
        eng.set_windows(lo, hi)
        r = eng.distpaint(query, ref_off, ref_hap, min_sites, delta=delta, threshold=thr, noresult=-7, with_stats=True)
    n_checked = min(H, 120)                            # scipy's ranksums in the oracle sets the pace
    for w in range(len(lo)):
        if hi[w] == lo[w]:
            assert (r["assign"][w] == -7).all() and np.isnan(r["means"][w]).all()
            continue
        a, m, p = po.paint_window(g[lo[w]:hi[w]], list(query[:n_checked]), pops, min_sites, thr if delta else None, thr, -7)
        assert np.array_equal(r["assign"][w, :n_checked], a), w
        _same_bits(r["means"][w, :n_checked], m, w)
        got = r["pvals"][w, :n_checked]
        assert np.array_equal(np.isnan(got), np.isnan(p)), w
        ok = ~np.isnan(p)
        np.testing.assert_allclose(got[ok], p[ok], rtol=1e-12, atol=0)


def test_member_limit_and_population_limit():
    from genomics_general_b200._lib import PgError
    from genomics_general_b200.engine import Engine
    rng = np.random.default_rng(3)
    S, H = 64, 40
    g = _data(rng, S, H, 0.02)
    with Engine(0) as eng:
        eng.upload(g)
        eng.set_windows(np.array([0], np.int64), np.array([S], np.int64))
        for M in (1024, 1025):
            ref_hap = rng.integers(0, H, M).astype(np.int32)
            ref_off = np.array([0, M // 2, M], dtype=np.int32)
            if M == 1024:
                r = eng.distpaint(np.arange(H), ref_off, ref_hap, 1, with_stats=True)
                a, m, p = po.paint_window(g, list(range(H)), [list(ref_hap[:M // 2]), list(ref_hap[M // 2:])], 1)
                assert np.array_equal(r["assign"][0], a)
                _same_bits(r["means"][0], m, M)
                got = r["pvals"][0]                        # ranks over 512 + 512 members: 16 rounds of the lanes
                assert np.array_equal(np.isnan(got), np.isnan(p)) and (~np.isnan(p)).sum() == H
                np.testing.assert_allclose(got[~np.isnan(p)], p[~np.isnan(p)], rtol=1e-12, atol=0)
            else:
                with pytest.raises(PgError, match="1025 member entries; at most 1024"):
                    eng.distpaint(np.arange(H), ref_off, ref_hap, 1)
        with pytest.raises(PgError, match="P=33 populations"):
            eng.distpaint(np.arange(H), np.arange(34, dtype=np.int32), np.arange(33, dtype=np.int32), 1)
        with pytest.raises(PgError, match="needs two populations"):
            eng.distpaint(np.arange(H), np.array([0, 3], np.int32), np.arange(3, dtype=np.int32), 1, delta=True)


def test_wide_haploid_token_is_refused_with_its_line(tmp_path):
    from genomics_general_b200._lib import PgError
    from genomics_general_b200.cli import distPaint
    lines = open(os.path.join(DIR, "sorted.geno")).read().split("\n")
    f = lines[12].split("\t")
    f[4] = "AC"
    lines[12] = "\t".join(f)
    (tmp_path / "wide.geno").write_text("\n".join(lines))
    with pytest.raises(PgError, match="data line 12, genotype column 3"):
        distPaint.main(["-g", str(tmp_path / "wide.geno"), "-o", str(tmp_path / "o.tsv"), "-w", "1000", "-p", "A", "a01",
                        "-p", "B", "b01"])


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_cli_matches_reference_fixture(case, tmp_path):
    assert run_cli(case, tmp_path) == expected(case)


@pytest.mark.parametrize("case", [c for c in CASES if c["name"] in ("rank_unsorted", "delta_failed_windows")],
                         ids=lambda c: c["name"])
def test_cli_host_tokenizer_and_small_batches(case, tmp_path, monkeypatch):
    case = dict(case, args=case["args"] + ["--hostParse"])
    assert run_cli(case, tmp_path, monkeypatch, extra_env={"PG_PAIR_SCRATCH_MB": "1"}) == expected(case)
