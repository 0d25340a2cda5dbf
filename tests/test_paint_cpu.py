"""distPaint.py without a GPU: the command line's host logic on an oracle-backed engine against the reference's own output,
the summation and sort orders the kernel reproduces, and the refusals."""
import gzip
import json
import os
import random

import numpy as np
import pytest

from helpers import GOLDEN

from oracle import paint_oracle as po

CASES = json.load(open(os.path.join(GOLDEN, "cases7.json")))
DIR = os.path.join(GOLDEN, "paint7")
# populations of 9, 130 and 300 samples (oracle/make_golden8.py)
CASES8 = json.load(open(os.path.join(GOLDEN, "cases8.json")))
DIR8 = os.path.join(GOLDEN, "paint8")


def run_cli(case, tmp_path, monkeypatch=None, engine=None, extra_env=None, directory=DIR):
    from genomics_general_b200.cli import _common, distPaint
    if engine is not None:
        monkeypatch.setattr(distPaint, "Engine", engine)
        real = _common.load_geno
        monkeypatch.setattr(_common, "load_geno",
                            lambda args, samples, pl, header=None, engine=None: real(args, samples, pl, header, None))
    for k, v in (extra_env or {}).items():
        monkeypatch.setenv(k, v)
    out = str(tmp_path / (case["name"] + (".tsv.gz" if case["gz"] else ".tsv")))
    args = [os.path.join(directory, a) if a in ("windows.txt", "pops.txt") else a for a in case["args"]]
    distPaint.main(["-g", os.path.join(directory, case["input"]), "-o", out] + args)
    if case["gz"]:
        with gzip.open(out, "rb") as f:
            return f.read()
    return open(out, "rb").read()


def expected(case, directory=DIR):
    return open(os.path.join(directory, case["expected"]), "rb").read()


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_cli_on_oracle_engine_matches_reference(case, tmp_path, monkeypatch):
    from oracle_engine_paint import PaintOracleEngine
    assert run_cli(case, tmp_path, monkeypatch, PaintOracleEngine) == expected(case)


@pytest.mark.parametrize("case", CASES8, ids=[c["name"] for c in CASES8])
def test_cli_on_oracle_engine_matches_reference_at_large_populations(case, tmp_path, monkeypatch):
    from oracle_engine_paint import PaintOracleEngine
    assert run_cli(case, tmp_path, monkeypatch, PaintOracleEngine, directory=DIR8) == expected(case, DIR8)


def _values(rng, n):
    v = []
    for _ in range(n):
        r = rng.random()
        if r < 0.1:
            v.append(float("nan"))
        elif r < 0.4:
            v.append(rng.randint(0, 97) / rng.randint(1, 97))
        elif r < 0.7:
            v.append(rng.random() * 10.0 ** rng.randint(-12, 12))
        else:
            v.append(rng.random())
    return v


def test_pairwise_sum_equals_numpy_nansum_bitwise():
    rng = random.Random(11)
    lengths = list(range(1, 301)) + [7, 8, 9, 128, 129, 136] * 20
    for n in lengths:
        v = _values(rng, n)
        a = np.array(v)
        want = np.nansum(a)
        got = po.pairwise_sum([0.0 if x != x else x for x in v])
        assert np.float64(got).tobytes() == want.tobytes(), n
        with np.errstate(all="ignore"):
            import warnings
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                m = np.nanmean(a)
        assert np.float64(po.nanmean(v)).tobytes() == m.tobytes() or (np.isnan(m) and np.isnan(po.nanmean(v))), n


def test_cpython_sort_equals_sorted_with_nans():
    rng = random.Random(12)
    pool = [0.0, 0.25, 0.5, 1.0 / 3.0, float("nan")]
    for it in range(20000):
        n = rng.randint(1, 32)
        if it % 2:
            v = [rng.choice(pool) for _ in range(n)]
        else:
            v = [float("nan") if rng.random() < 0.2 else rng.random() for _ in range(n)]
        if it % 3 == 0:
            v = [np.float64(x) for x in v]          # what np.nanmean hands to sorted() in the reference
        want = sorted(v)
        got = po.cpython_sort(v)
        assert [repr(float(x)) for x in got] == [repr(float(x)) for x in want], v


def _refuse(tmp_path, monkeypatch, args, inp="sorted.geno"):
    from oracle_engine_paint import PaintOracleEngine
    case = dict(name="refuse", input=inp, args=args, gz=False)
    return run_cli(case, tmp_path, monkeypatch, PaintOracleEngine)


@pytest.mark.parametrize("args, msg", [
    (["-w", "1000", "--header", "a b c", "-p", "A", "a01"], "--header"),
    (["-w", "1000", "--delta_threshold", "0.1", "-p", "A", "a01,a02"], "needs at least two"),
    (["-w", "1000", "--devices", "2", "-p", "A", "a01", "-p", "B", "b01"], "--devices"),
])
def test_refusals_before_any_work(args, msg, tmp_path, monkeypatch):
    with pytest.raises(SystemExit) as e:
        _refuse(tmp_path, monkeypatch, args)
    assert msg in str(e.value)


def test_pops_file_blank_line_raises_as_in_the_reference(tmp_path, monkeypatch):
    pf = tmp_path / "pops.txt"
    pf.write_text("a01 A\n\nb01 B\n")
    with pytest.raises(ValueError):
        _refuse(tmp_path, monkeypatch, ["-w", "1000", "--popsFile", str(pf), "-p", "A", "-p", "B"])
    pf.write_text("a01 A extra\n")
    with pytest.raises(ValueError):
        _refuse(tmp_path, monkeypatch, ["-w", "1000", "--popsFile", str(pf), "-p", "A", "-p", "B"])


def test_population_without_members_is_refused(tmp_path, monkeypatch):
    with pytest.raises(AssertionError) as e:
        _refuse(tmp_path, monkeypatch, ["-w", "1000", "-p", "A", "a01", "-p", "B"])
    assert "Reference population B appears to have no individuals." in str(e.value)


def test_wide_token_is_refused_by_the_host_tokenizer_with_its_line(tmp_path, monkeypatch):
    lines = open(os.path.join(DIR, "sorted.geno")).read().split("\n")
    f = lines[7].split("\t")
    f[5] = "AC"
    lines[7] = "\t".join(f)
    (tmp_path / "wide.geno").write_text("\n".join(lines))
    from genomics_general_b200 import geno_io
    from genomics_general_b200.cli import distPaint
    with pytest.raises(geno_io.PgError) as e:
        distPaint.check_haplo_tokens(str(tmp_path / "wide.geno"))
    assert "data line 7, genotype column 4" in str(e.value)
