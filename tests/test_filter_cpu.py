"""filterGenotypes.py without a GPU: the numpy restatement of siteTest / asList against the reference's own fixtures and
against genomics.siteTest in process, and the command line's host logic on an oracle-backed engine."""
import gzip
import json
import os
import random
import sys

import numpy as np
import pytest

from helpers import GOLDEN

from oracle import filter_oracle as fo

CASES = json.load(open(os.path.join(GOLDEN, "cases6.json")))
DIR = os.path.join(GOLDEN, "filter6")
REF = os.path.join(os.path.dirname(GOLDEN), "..", "oracle", "_ref")


def run_cli(case, tmp_path, monkeypatch=None, engine=None, extra_env=None):
    from genomics_general_b200.cli import filterGenotypes as F
    if engine is not None:
        monkeypatch.setattr(F, "Engine", engine)
        from oracle_engine_filter import HostArray
        monkeypatch.setattr(F, "PinnedArray", HostArray)
    for k, v in (extra_env or {}).items():
        monkeypatch.setenv(k, v)
    out = str(tmp_path / (case["name"] + (".out.gz" if case["gz"] else ".out")))
    F.main(["-i", os.path.join(DIR, case["input"]), "-o", out] + case["args"])
    if case["gz"]:
        with gzip.open(out, "rb") as f:
            return f.read()
    return open(out, "rb").read()


def expected(case):
    return open(os.path.join(DIR, case["expected"]), "rb").read()


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_cli_on_oracle_engine_matches_reference(case, tmp_path, monkeypatch):
    from oracle_engine_filter import FilterOracleEngine
    assert run_cli(case, tmp_path, monkeypatch, FilterOracleEngine) == expected(case)


@pytest.mark.parametrize("case", [c for c in CASES if c["name"] in ("include_thin_pods", "phased_default", "bases_freq")],
                         ids=lambda c: c["name"])
def test_cli_output_does_not_depend_on_chunks_or_slabs(case, tmp_path, monkeypatch):
    from oracle_engine_filter import FilterOracleEngine
    got = run_cli(case, tmp_path, monkeypatch, FilterOracleEngine,
                  extra_env={"PG_FILTER_CHUNK_BYTES": "700", "PG_FILTER_SLAB_BYTES": "300"})
    assert got == expected(case)


def test_tie_rule_is_stable_argsort_and_matches_numpy_below_four_alleles():
    import itertools
    for c in itertools.product(range(5), repeat=4):
        c = np.array(c)
        k = int((c > 0).sum())
        idx = c > 0
        numpy_order = list(np.array(list("ACGT"))[idx][np.argsort(c[idx])[::-1]])
        if k <= 3:
            assert fo.freq_order(c) == numpy_order
        elif not fo.is_tied(c):
            assert fo.freq_order(c) == numpy_order


def _random_site(rng, ploidy, fmt):
    al = rng.sample("ACGT", rng.choice([1, 2, 3]))
    toks = []
    for pl in ploidy:
        a = [rng.choice(al) for _ in range(pl)]
        if rng.random() < 0.15:
            a[rng.randrange(pl)] = "N"
        toks.append(rng.choice("|/").join(a) if fmt == "phased" else "".join(a))
    return toks


@pytest.mark.skipif(not os.path.exists(os.path.join(REF, "genomics.py")), reason="reference genomics.py not staged")
def test_site_test_equals_reference_siteTest_in_process():
    sys.path.insert(0, REF)
    try:
        import genomics as G
    finally:
        sys.path.pop(0)
    rng = random.Random(5)
    names = ["a", "b", "c", "d", "e", "f"]
    ploidy = [2, 2, 1, 3, 2, 2]
    popDict = {"X": ["a", "b", "c"], "Y": ["d", "e"], "Z": []}
    pops = [[0, 1, 2], [3, 4], []]
    for it in range(600):
        toks = _random_site(rng, ploidy, "phased")
        p2m = it % 3 == 0
        spec = dict(min_calls=rng.choice([0, 1, 4]), min_alleles=rng.choice([1, 2]), max_alleles=rng.choice([2, float("inf")]),
                    min_var_count=rng.choice([None, 2]), max_het=rng.choice([None, 0.3, 0.6]),
                    min_freq=rng.choice([None, 0.2]), max_freq=rng.choice([None, 0.4]),
                    fixed_diffs=rng.random() < 0.2, nearly_fixed_diff=rng.choice([None, 0.0, 0.5]))
        mpc = rng.choice([None, [1, 1, 0]])
        mpa = rng.choice([None, ([1, 1, 0], [1, 2, 4])])
        spec["min_pop_calls"] = mpc
        spec["min_pop_alleles"], spec["max_pop_alleles"] = mpa if mpa else (None, None)
        site = G.GenomeSite(genotypes=toks, sampleNames=names, popDict=popDict, genoFormat="phased",
                            ploidyDict=dict(zip(names, ploidy)), partialToMissing=p2m)
        ref = G.siteTest(site, samples=names, minCalls=spec["min_calls"], minAlleles=spec["min_alleles"],
                         maxAlleles=spec["max_alleles"], minVarCount=spec["min_var_count"], maxHet=spec["max_het"],
                         minFreq=spec["min_freq"], maxFreq=spec["max_freq"], fixed=spec["fixed_diffs"],
                         nearlyFixedDiff=spec["nearly_fixed_diff"],
                         minPopCalls=dict(zip("XYZ", mpc)) if mpc else None,
                         minPopAlleles=dict(zip("XYZ", mpa[0])) if mpa else None,
                         maxPopAlleles=dict(zip("XYZ", mpa[1])) if mpa else None)
        gts = [fo.genotype(t, "phased", p2m) for t in toks]
        assert fo.site_test(gts, pops, spec) == ref, (toks, spec)
        c = fo.counts(gts)
        for mode in ("phased", "alleles", "bases"):
            assert [str(x) for x in site.asList(names, mode=mode)] == fo.as_list(gts, mode), (toks, mode)
        if not (fo.is_tied(c) and (c > 0).sum() == 4):
            assert [str(x) for x in site.asList(names, mode="alleles", alleleOrder="freq")] == \
                fo.as_list(gts, "alleles", "freq")
            assert [str(x) for x in site.asList(names, mode="coded")] == fo.as_list(gts, "coded")
            if c.sum():
                assert [str(x) for x in site.asList(names, mode="count")] == fo.as_list(gts, "count")


@pytest.mark.parametrize("extra, msg", [
    (["-of", "randomAllele"], "randomAllele"),
    (["--HWE", "0.05", "both"], "HWE"),
    (["-p", "P1", "s1,s2", "-s", "s1,s3"], "not among the selected samples"),
    (["-of", "diplo"], "-of diplo needs diploid samples"),
])
def test_refusals_before_any_launch(extra, msg, tmp_path, monkeypatch, capsys):
    from oracle_engine_filter import FilterOracleEngine
    case = dict(name="refuse", input="phased.geno", args=extra, gz=False)
    with pytest.raises((SystemExit, RuntimeError)) as e:
        run_cli(case, tmp_path, monkeypatch, FilterOracleEngine)
    assert msg in str(e.value)


def test_token_width_is_reported_by_the_ingest(tmp_path, monkeypatch):
    """a token whose width differs from --ploidy is refused by the (strict) ingest of the chunk, naming its data line"""
    from oracle_engine_filter import FilterOracleEngine
    case = dict(name="refuse", input="phased.geno", args=["--ploidy", "3"], gz=False)
    with pytest.raises(RuntimeError) as e:
        run_cli(case, tmp_path, monkeypatch, FilterOracleEngine)
    assert "data line 1" in str(e.value)


def test_first_data_line_longer_than_a_read_block():
    import io
    from genomics_general_b200.cli.filterGenotypes import _first_data_line
    long_line = b"c\t1\t" + b"\t".join([b"A|T"] * 400000)
    src = io.BytesIO(b"# note\n\n" + long_line + b"\nc\t2\t" + b"\t".join([b"A|A"] * 400000) + b"\n")
    body, first = _first_data_line(src)
    assert first == long_line and body.startswith(b"# note\n")


def test_thin_refuses_comment_lines(tmp_path, monkeypatch):
    from oracle_engine_filter import FilterOracleEngine
    text = open(os.path.join(DIR, "phased.geno")).read().split("\n")
    text.insert(5, "# a comment")
    p = tmp_path / "c.geno"
    p.write_text("\n".join(text))
    from genomics_general_b200.cli import filterGenotypes as F
    monkeypatch.setattr(F, "Engine", FilterOracleEngine)
    from oracle_engine_filter import HostArray
    monkeypatch.setattr(F, "PinnedArray", HostArray)
    with pytest.raises(SystemExit) as e:
        F.main(["-i", str(p), "-o", str(tmp_path / "o"), "--thinDist", "10"])
    assert "comment or blank lines" in str(e.value)
