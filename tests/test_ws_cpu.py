"""windowStats.py without a GPU: the command line's host logic (flags, header, column plan, chunks, windows, refusals, rows) on
an oracle-backed engine (tests/oracle_engine_ws.py) against every output the unmodified reference wrote (tests/golden/ws13),
byte for byte after decompression, with normal and with tiny chunks."""
import gzip
import io
import json
import math
import os
import sys

import pytest

from helpers import GOLDEN

CASES = json.load(open(os.path.join(GOLDEN, "cases13.json")))
DIR = os.path.join(GOLDEN, "ws13")
OK = [c for c in CASES if "fails" not in c]
FAILS = [c for c in CASES if "fails" in c]
REFUSALS = {"fail_bad_token": "line 64: float() rejects the value 'NA' of column v, inside window 2",
            "fail_empty_min": "window 1 (c:1-20) has no value in column b",
            "fail_short_line": "line 3: the line's field count differs from the header's",
            "fail_columns_missing_on_line": "line 3: the line has no column b",
            "fail_column_not_in_header": "column zz is not in the header"}
TINY = {"PG_WS_CHUNK_BYTES": "200", "PG_WS_SORT_BYTES": "64"}


def expected(case):
    return gzip.decompress(open(os.path.join(DIR, case["output"]), "rb").read())


def same_up_to_zero_sign(a, b):
    """rows equal, cells compared up to the sign of a zero (min, max and quantile ties of -0.0 and 0.0)"""
    ra, rb = a.split(b"\n"), b.split(b"\n")
    if len(ra) != len(rb):
        return False
    for x, y in zip(ra, rb):
        if x != y:
            cx, cy = x.split(b","), y.split(b",")
            if len(cx) != len(cy) or any(u != v and not (u.lstrip(b"-") == v.lstrip(b"-") == b"0.0") for u, v in zip(cx, cy)):
                return False
    return True


def run_cli(args, tmp_path, monkeypatch, engine=None, extra_env=None, stdin=None):
    from genomics_general_b200.cli import windowStats as G
    if engine is not None:
        monkeypatch.setattr(G, "Engine", engine)
    for k, v in (extra_env or {}).items():
        monkeypatch.setenv(k, v)
    monkeypatch.chdir(DIR)
    out = io.TextIOWrapper(io.BytesIO())
    monkeypatch.setattr(sys, "stdout", out)
    if stdin is not None:
        monkeypatch.setattr(sys, "stdin", io.TextIOWrapper(open(stdin, "rb")))
    try:
        G.main(list(args))
    finally:
        out.flush()
        run_cli.got = out.buffer.getvalue()
    return run_cli.got


def case_args(case):
    return ["-i", case["input"]] + case["args"]


@pytest.mark.parametrize("tiny", [False, True])
@pytest.mark.parametrize("case", OK, ids=[c["name"] for c in OK])
def test_cli_on_oracle_engine_matches_reference(case, tiny, tmp_path, monkeypatch):
    from oracle_engine_ws import WsOracleEngine
    got = run_cli(case_args(case), tmp_path, monkeypatch, WsOracleEngine, TINY if tiny else None)
    assert same_up_to_zero_sign(got, expected(case))


@pytest.mark.parametrize("case", FAILS, ids=[c["name"] for c in FAILS])
def test_cli_refuses_before_any_output(case, tmp_path, monkeypatch):
    from oracle_engine_ws import WsOracleEngine
    with pytest.raises(SystemExit) as e:
        run_cli(case_args(case), tmp_path, monkeypatch, WsOracleEngine)
    assert str(e.value).startswith("windowStats: ") and REFUSALS[case["name"]] in str(e.value), str(e.value)
    assert run_cli.got == b""


def test_plain_input_file_output_gzip_output_and_stdin_match_stdout(tmp_path, monkeypatch):
    """the fixture's input is read as .gz; the same table read plain, from stdin, and written to -o / -o x.gz"""
    from oracle_engine_ws import WsOracleEngine
    case = next(c for c in OK if c["name"] == "sites")
    want = expected(case)
    plain = tmp_path / "main.tsv"
    plain.write_bytes(gzip.decompress(open(os.path.join(DIR, case["input"]), "rb").read()))
    args = case["args"]
    assert same_up_to_zero_sign(run_cli(["-i", str(plain)] + args, tmp_path, monkeypatch, WsOracleEngine), want)
    for name in ("out.csv", "out.csv.gz"):
        dest = tmp_path / name
        assert run_cli(["-i", str(plain), "-o", str(dest)] + args, tmp_path, monkeypatch, WsOracleEngine) == b""
        got = dest.read_bytes()
        assert same_up_to_zero_sign(gzip.decompress(got) if name.endswith(".gz") else got, want)
    got = run_cli(args, tmp_path, monkeypatch, WsOracleEngine, stdin=str(plain))
    assert same_up_to_zero_sign(got, want)


@pytest.mark.parametrize("body, what", [
    ("c\t1\t1.0\nc\t2\t\xe9\n", "line 3: a byte outside ASCII"),
    ("c\t1\t1.0\nc\t2\t3.0\r\t\n", "line 3: a '\\r' ends a line by itself"),
    ("c\t1\t1.0\nc\t1_0\t3.0\n", "line 3: the position is not an integer"),
    ("c\t5\t1.0\nc\t2\t3.0\n", "position 2 is below the one before it"),
])
def test_narrowings_are_refused(tmp_path, monkeypatch, body, what):
    from oracle_engine_ws import WsOracleEngine
    p = tmp_path / "t.tsv"
    p.write_bytes(("s\tp\tv\n" + body).encode("latin-1"))
    with pytest.raises(SystemExit) as e:
        run_cli(["-i", str(p), "-w", "10"], tmp_path, monkeypatch, WsOracleEngine)
    assert what in str(e.value), str(e.value)


def test_empty_input_is_refused_as_window_stats(tmp_path, monkeypatch):
    from oracle_engine_ws import WsOracleEngine
    p = tmp_path / "empty.tsv"
    p.write_bytes(b"")
    with pytest.raises(SystemExit) as e:
        run_cli(["-i", str(p), "-w", "10"], tmp_path, monkeypatch, WsOracleEngine)
    assert str(e.value).startswith("windowStats: the input is empty"), str(e.value)
    assert run_cli.got == b""


def test_blank_lines_skipped_and_flags_without_effect(tmp_path, monkeypatch):
    from oracle_engine_ws import WsOracleEngine
    p = tmp_path / "t.tsv"
    p.write_bytes(b"s\tp\tv\nc\t1\t1.5\n\n   \nc\t2\t2.5\n")
    got = run_cli(["-i", str(p), "-w", "10", "--verbose", "--writeFailedWindows", "--stats", "sum", "q25"], tmp_path,
                  monkeypatch, WsOracleEngine)
    assert got == b"scaffold,start,end,mid,sites,v_sum,v_q25\nc,1,10,2,2,4.0,1.75\n"
    with pytest.raises(SystemExit) as e:
        run_cli(["-i", str(p), "-w", "10", "--devices", "2"], tmp_path, monkeypatch, WsOracleEngine)
    assert "--devices" in str(e.value)


def test_plain_statement_rules():
    """worked examples of the statement: the pairwise split, sd rounding, median, lerped quantiles, the last value"""
    import numpy as np
    from oracle_engine_ws import stat
    rng = np.random.default_rng(3)
    for n in (1, 7, 8, 9, 127, 128, 129, 255, 256, 257, 1000, 4099):
        x = rng.normal(0, 1, n) * 10.0 ** rng.integers(-3, 9, n)
        xs = list(x)
        assert stat(xs, 5, 0) == np.sum(x) and stat(xs, 0, 0) == x.mean()
        assert stat(xs, 4, 0) == round(np.std(x), 6) and stat(xs, 1, 0) == np.median(x)
        for q in (0.05, 0.1, 0.25, 0.75, 0.9, 0.95):
            assert stat(xs, 6, q) == np.quantile(x, q)
    assert str(stat([-0.0], 6, 0.5)) == "-0.0" and math.isnan(stat([1.0, math.inf, math.inf], 6, 1.0))

