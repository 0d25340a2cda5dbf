"""mergeGeno.py without a GPU: the command line's host logic (flags, .fai, headers, chunks, rounds, slabs, refusals) on an
oracle-backed engine (tests/oracle_engine_merge.py) against every output the unmodified reference wrote (tests/golden/merge14),
byte for byte after decompression, with default and with tiny chunks and slabs."""
import gzip
import io
import json
import os
import sys

import pytest

from helpers import GOLDEN

CASES = json.load(open(os.path.join(GOLDEN, "cases14.json")))
DIR = os.path.join(GOLDEN, "merge14")
OK = [c for c in CASES if "fails" not in c]
FAILS = [c for c in CASES if "fails" in c]
TINY = {"PG_MERGE_CHUNK_BYTES": "64", "PG_MERGE_SLAB_BYTES": "40", "PG_MERGE_DENSE_ROWS": "7"}
REFUSED = {"fail_fai_short_line": "short.fai line 2 has fewer than 2 fields",
           "fail_fai_bad_length": "badint.fai line 2: the length 'abc' is not an integer",
           "fail_output_only_range": "--outputOnly 3: there are 2 input files",
           "fail_missing_input": "cannot open input"}


def expected(case):
    return gzip.decompress(open(os.path.join(DIR, case["output"]), "rb").read())


def case_argv(case):
    return [os.path.join(DIR, a) if k > 0 and case["args"][k - 1] in ("-i", "-f") else a for k, a in enumerate(case["args"])]


def run_cli(argv, dest, tmp_path, monkeypatch, engine=None, extra_env=None):
    """the command line with argv (and -o dest unless dest is "stdout") in tmp_path; returns what it wrote (decompressed)"""
    from genomics_general_b200.cli import mergeGeno as M
    if engine is not None:
        monkeypatch.setattr(M, "Engine", engine)
        from oracle_engine_filter import HostArray
        monkeypatch.setattr(M, "PinnedArray", HostArray)
    for k, v in (extra_env or {}).items():
        monkeypatch.setenv(k, v)
    work = tmp_path / "work"
    work.mkdir(exist_ok=True)
    monkeypatch.chdir(work)
    out = io.TextIOWrapper(io.BytesIO())
    monkeypatch.setattr(sys, "stdout", out)
    argv = list(argv) + ([] if dest == "stdout" else ["-o", dest])
    try:
        M.main(argv)
    finally:
        out.flush()
        got = out.buffer.getvalue()
        if dest != "stdout" and os.path.exists(work / dest):
            got = open(work / dest, "rb").read()
            got = gzip.decompress(got) if dest.endswith(".gz") else got
        run_cli.got = got
        run_cli.exists = dest != "stdout" and os.path.exists(work / dest)
    return got


@pytest.mark.parametrize("env", [None, TINY], ids=["default", "tiny"])
@pytest.mark.parametrize("case", OK, ids=[c["name"] for c in OK])
def test_cli_on_oracle_engine_matches_reference(case, env, tmp_path, monkeypatch):
    from oracle_engine_merge import MergeOracleEngine
    assert run_cli(case_argv(case), case["dest"], tmp_path, monkeypatch, MergeOracleEngine, env) == expected(case)


@pytest.mark.parametrize("case", FAILS, ids=[c["name"] for c in FAILS])
def test_reference_crashes_are_refused_before_any_output(case, tmp_path, monkeypatch):
    from oracle_engine_merge import MergeOracleEngine
    for dest in ("stdout", "out.geno"):
        with pytest.raises(SystemExit, match=REFUSED[case["name"]].replace("(", r"\(").replace("-", r"\-")):
            run_cli(case_argv(case), dest, tmp_path, monkeypatch, MergeOracleEngine)
        assert run_cli.got == b"" and not run_cli.exists


def _write(tmp_path, name, data):
    p = tmp_path / name
    p.write_bytes(data)
    return str(p)


FAI = b"c1\t20\nc2\t10\n"
HEAD = b"#CHROM\tPOS\ts\n"


@pytest.mark.parametrize("env", [None, TINY], ids=["default", "tiny"])
@pytest.mark.parametrize("body,line", [(b"c1\t1\tA\nc1\t2\t\xc3\xa9\nc1\t3\tA\n", 3),
                                       (b"c1\t1\tA\nc1\t2\tA\rc1\t3\tA\n", 3),
                                       (b"c1\t1\tA\nc1\t2\tA\nc9\xa0\t3\n", 4)])
def test_non_ascii_and_lone_cr_refused_where_the_walk_reaches(body, line, env, tmp_path, monkeypatch):
    from oracle_engine_merge import MergeOracleEngine
    fai = _write(tmp_path, "x.fai", FAI)
    a = _write(tmp_path, "a.geno", HEAD + body)
    for dest in ("stdout", "out.geno"):
        with pytest.raises(SystemExit, match="a.geno line %d: a byte outside ASCII" % line):
            run_cli(["-i", a, "-f", fai, "--method", "union"], dest, tmp_path, monkeypatch, MergeOracleEngine, env)
        if dest != "stdout":
            assert not run_cli.exists


def test_bad_bytes_after_the_stall_are_never_read(tmp_path, monkeypatch):
    from oracle_engine_merge import MergeOracleEngine
    fai = _write(tmp_path, "x.fai", FAI)
    a = _write(tmp_path, "a.geno", HEAD + b"c1\t1\tA\nc1\t1\tA\nc1\t2\t\xff\rB\n")
    got = run_cli(["-i", a, "-f", fai], "stdout", tmp_path, monkeypatch, MergeOracleEngine)
    assert got == b"#CHROM\tPOS\ts\nc1\t1\tA\n"


@pytest.mark.parametrize("fai,msg", [(b"c1\t5\nc2\t3\nc1\t4\n", "names scaffold c1 twice"),
                                     (b"c1\t%d\nc2\t%d\n" % (1 << 61, 1 << 61), "sum to 2\\^62 or more")])
def test_fai_narrowings_refused_before_any_output(fai, msg, tmp_path, monkeypatch):
    from oracle_engine_merge import MergeOracleEngine
    f = _write(tmp_path, "x.fai", fai)
    a = _write(tmp_path, "a.geno", HEAD + b"c1\t1\tA\n")
    with pytest.raises(SystemExit, match=msg):
        run_cli(["-i", a, "-f", f], "out.geno", tmp_path, monkeypatch, MergeOracleEngine)
    assert not run_cli.exists


def test_walk_just_below_the_limit_runs(tmp_path, monkeypatch):
    from oracle_engine_merge import MergeOracleEngine
    f = _write(tmp_path, "x.fai", b"c1\t%d\nc2\t%d\n" % ((1 << 61), (1 << 61) - 1))
    a = _write(tmp_path, "a.geno", HEAD + b"c2\t%d\tA\n" % ((1 << 61) - 1))
    got = run_cli(["-i", a, "-f", f], "stdout", tmp_path, monkeypatch, MergeOracleEngine)
    assert got == HEAD + b"c2\t%d\tA\n" % ((1 << 61) - 1)


@pytest.mark.parametrize("flag", [["--devices", "2"], ["--hostParse"], ["--cache"]])
def test_engine_flags_that_do_not_apply_are_refused(flag, tmp_path, monkeypatch):
    from oracle_engine_merge import MergeOracleEngine
    fai = _write(tmp_path, "x.fai", FAI)
    a = _write(tmp_path, "a.geno", HEAD)
    with pytest.raises(SystemExit, match="--devices|--hostParse"):
        run_cli(["-i", a, "-f", fai] + flag, "stdout", tmp_path, monkeypatch, MergeOracleEngine)


@pytest.mark.parametrize("dest", ["stdout", "o.geno", "o.geno.gz"])
def test_destinations_agree(dest, tmp_path, monkeypatch):
    from oracle_engine_merge import MergeOracleEngine
    case = next(c for c in OK if c["name"] == "method_union")
    assert run_cli(case_argv(case), dest, tmp_path, monkeypatch, MergeOracleEngine) == expected(case)


def test_crlf_cut_between_chunks_is_not_a_blank_line(tmp_path, monkeypatch):
    """a '\\r\\n' split across two chunks must not stall the file (parseVCF's chunks() would leave a blank line)"""
    from oracle_engine_merge import MergeOracleEngine
    fai = _write(tmp_path, "x.fai", FAI)
    body = b"".join(b"c1\t%d\tA\r\n" % p for p in range(1, 21))
    a = _write(tmp_path, "a.geno", HEAD + body)
    want = HEAD + b"".join(b"c1\t%d\tA\n" % p for p in range(1, 21))
    for size in range(5, 40):
        got = run_cli(["-i", a, "-f", fai], "stdout", tmp_path, monkeypatch, MergeOracleEngine,
                      {"PG_MERGE_CHUNK_BYTES": str(size), "PG_MERGE_SLAB_BYTES": "7"})
        assert got == want, size
