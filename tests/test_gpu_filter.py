"""filterGenotypes.py on the GPU: the command line against the reference's fixtures byte for byte, the per-site statistics
and verdicts of k_filter_sites / k_filter_thin against the numpy restatement, and output that does not depend on the
ingest chunk or emit slab sizes."""
import random

import numpy as np
import pytest

from oracle import filter_oracle as fo
from test_filter_cpu import CASES, expected, run_cli

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_cli_matches_reference_fixture(case, tmp_path):
    assert run_cli(case, tmp_path) == expected(case)


@pytest.mark.parametrize("case", [c for c in CASES if c["name"] in ("include_thin_pods", "exclude_thin_notest",
                                                                      "phased_default", "alleles_tuple_varcount_het")],
                         ids=lambda c: c["name"])
def test_cli_tiny_chunks_and_slabs(case, tmp_path, monkeypatch):
    got = run_cli(case, tmp_path, monkeypatch, extra_env={"PG_FILTER_CHUNK_BYTES": "900", "PG_FILTER_SLAB_BYTES": "200"})
    assert got == expected(case)


def _text(rng, ploidy, n_sites):
    rows = []
    for i in range(n_sites):
        al = rng.sample("ACGT", rng.choice([1, 1, 2, 2, 3, 4]))
        miss = rng.choice([0.0, 0.05, 0.3])
        toks = []
        for pl in ploidy:
            a = [rng.choice(al) for _ in range(pl)]
            r = rng.random()
            if r < miss:
                a = ["N"] * pl
            elif r < 2 * miss and pl > 1:
                a[0] = "N"
            toks.append(rng.choice("|/").join(a))
        rows.append("\t".join(["chr%d" % (i // 50), str(10 * i + 1)] + toks))
    return ("\n".join(rows) + "\n").encode()


@pytest.mark.parametrize("n_samp, P, seed", [(1, 1, 1), (7, 2, 2), (40, 3, 3), (150, 5, 4), (1000, 8, 5), (1500, 4, 6)])
def test_keep_and_stats_equal_oracle(n_samp, P, seed):
    from genomics_general_b200.engine import Engine
    rng = random.Random(seed)
    ploidy = [rng.choice([1, 2, 2, 2, 3]) if n_samp < 1000 else 2 for _ in range(n_samp)]
    S = 120 if n_samp < 1000 else 40
    data = _text(rng, ploidy, S)
    hap0 = np.concatenate([[0], np.cumsum(ploidy)[:-1]]).astype(np.int32)
    H = int(sum(ploidy))
    # populations may overlap (a sample in several lists); with P > 1 the last one is empty: it stands for every sample
    pops = [sorted(rng.sample(range(n_samp), rng.randint(1, n_samp))) for _ in range(P)]
    if P > 1:
        pops[-1] = []
    with Engine(0) as eng:
        eng.set_strict_ingest(True)
        assert eng.ingest_text(data, 0, hap0, np.array(ploidy, np.int8), H) == S
        eng.ingest_meta(S, release=False)
        lines = data.decode().split("\n")[:S]
        for variant in range(4):
            spec = dict(samp_hap0=hap0, samp_ploidy=np.array(ploidy, np.int8), pops=pops,
                        min_calls=[1, 0, 2, n_samp // 2][variant], min_alleles=[1, 2, 1, 1][variant],
                        max_alleles=[float("inf"), 3, 2, float("inf")][variant], min_var_count=[None, 2, None, 1][variant],
                        max_het=[None, 0.5, 0.0, 0.9][variant], min_freq=[None, 0.1, None, 0.05][variant],
                        max_freq=[None, None, 0.45, 0.5][variant], min_pop_calls=[None, [1] * P, None, None][variant],
                        min_pop_alleles=[None, None, [1] * P, None][variant],
                        max_pop_alleles=[None, None, [2] * P, None][variant], fixed_diffs=variant == 3,
                        nearly_fixed_diff=[None, 0.3, None, None][variant], partial_to_missing=variant == 1)
            nk, _ = eng.filter(spec)
            st = eng.filter_stats()
            want = []
            for s, ln in enumerate(lines):
                gts = [fo.genotype(t, "phased", spec["partial_to_missing"]) for t in ln.split()[2:]]
                ok = fo.site_test(gts, pops, spec)
                want.append(ok)
                assert st["called"][s] == sum(not fo.is_missing(al) for al, _ in gts)
                assert st["het"][s] == sum(len(set(al)) > 1 for al, _ in gts)
                assert list(st["counts"][s]) == list(fo.counts(gts))
                for p in range(P):
                    m = pops[p]
                    assert st["pop_called"][s, p] == sum(not fo.is_missing(gts[i][0]) for i in m)
                    mask = sum(1 << a for a in np.flatnonzero(fo.counts(gts, m) > 0))
                    assert st["pop_mask"][s, p] == mask
                assert bool(st["flags"][s] & 1) == fo.is_tied(fo.counts(gts))
            assert list(st["keep"].astype(bool)) == want, variant
            assert nk == sum(want)


@pytest.mark.parametrize("n_samp, P", [(1, 0), (2, 0), (4, 0), (13, 1), (29, 5), (3, 2)])
def test_every_chunk_length_and_sample_table_size(n_samp, P):
    """the sample tables, member lists, scaffold ids and contig mask for chunks of 1 to 40 sites"""
    from genomics_general_b200.engine import Engine
    rng = random.Random(100 * n_samp + P)
    ploidy = [2] * n_samp
    hap0 = np.arange(0, 2 * n_samp, 2, dtype=np.int32)
    pops = [sorted(rng.sample(range(n_samp), rng.randint(1, n_samp))) for _ in range(P)]
    with Engine(0) as eng:
        eng.set_strict_ingest(True)
        for S in range(1, 41):
            data = _text(rng, ploidy, S)
            assert eng.ingest_text(data, 0, hap0, np.array(ploidy, np.int8), 2 * n_samp) == S
            eng.ingest_meta(S, release=False)
            lines = data.decode().split("\n")[:S]
            cmask = np.array([rng.random() < 0.7 for _ in range(S)], dtype=np.uint8)
            scaf = np.array([i // 50 for i in range(S)], dtype=np.int32)
            spec = dict(samp_hap0=hap0, samp_ploidy=np.array(ploidy, np.int8), pops=pops, min_calls=1,
                        min_pop_calls=[1] * P if P else None, thin_dist=15, pod_size=7)
            nk, _ = eng.filter(spec, contig_mask=cmask, scaf_id=scaf)
            want = []
            last = None
            for s, ln in enumerate(lines):
                if s % 7 == 0:
                    last = None
                if not cmask[s]:
                    continue
                pos = int(ln.split()[1])
                if last is None or scaf[s] != last[0]:
                    last = (scaf[s], pos)
                    continue
                if pos - last[1] < 15:
                    continue
                gts = [fo.genotype(t, "phased") for t in ln.split()[2:]]
                if fo.site_test(gts, pops, spec):
                    want.append(s)
                    last = (scaf[s], pos)
            st = eng.filter_stats()
            assert list(np.flatnonzero(st["final"])) == want, S
            assert nk == len(want)


def test_uniform_and_all_missing_sites():
    """sites where every haplotype is A, or every one is missing, next to varied ones"""
    from genomics_general_b200.engine import Engine
    ploidy = [2] * 20
    rows = []
    for i in range(64):
        g = ["A|A"] * 20 if i % 3 == 0 else (["N|N"] * 20 if i % 3 == 1 else ["A|T"] + ["T|T"] * 19)
        rows.append("\t".join(["c", str(i + 1)] + g))
    data = ("\n".join(rows) + "\n").encode()
    hap0 = np.arange(0, 40, 2, dtype=np.int32)
    with Engine(0) as eng:
        eng.set_strict_ingest(True)
        eng.ingest_text(data, 0, hap0, np.array(ploidy, np.int8), 40)
        eng.ingest_meta(64, release=False)
        nk, _ = eng.filter(dict(samp_hap0=hap0, samp_ploidy=np.array(ploidy, np.int8), P=0, min_calls=1))
        st = eng.filter_stats()
    assert nk == 64 - 64 // 3 - (1 if 64 % 3 > 1 else 0)
    assert list(st["keep"]) == [0 if i % 3 == 1 else 1 for i in range(64)]


@pytest.mark.parametrize("extra, msg", [
    (["-of", "randomAllele"], "randomAllele"),
    (["--HWE", "0.05", "both"], "HWE"),
    (["-p", "P1", "s1,s2", "-s", "s1,s3"], "not among the selected samples"),
    (["-of", "diplo"], "-of diplo needs diploid samples"),
])
def test_refusals(extra, msg, tmp_path):
    case = dict(name="refuse", input="phased.geno", args=extra, gz=False)
    with pytest.raises((SystemExit, RuntimeError)) as e:
        run_cli(case, tmp_path)
    assert msg in str(e.value)


def test_token_width_is_reported_with_its_line(tmp_path):
    case = dict(name="refuse", input="phased.geno", args=["--ploidy", "3"], gz=False)
    with pytest.raises(RuntimeError) as e:
        run_cli(case, tmp_path)
    assert "data line 1" in str(e.value)
