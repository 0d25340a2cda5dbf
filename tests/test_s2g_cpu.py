"""seqToGeno.py without a GPU: the command line's host logic (flags, refusals, FASTA records, PHYLIP structure, plan, slabs)
on an oracle-backed engine (tests/oracle_engine_s2g.py) against every output the unmodified reference wrote
(tests/golden/s2g12), byte for byte after decompression, with default and with 40-byte slabs."""
import gzip
import io
import json
import os
import sys

import pytest

from helpers import GOLDEN

CASES = json.load(open(os.path.join(GOLDEN, "cases12.json")))
DIR = os.path.join(GOLDEN, "s2g12")
OK = [c for c in CASES if "fails" not in c]
FAILS = [c for c in CASES if "fails" in c]
# every case the reference fails on is refused before any output
REFUSED = {"fail_single_ploidy": "a single -P value above 1",
           "fail_ploidy_sum": "sums to 5, the input gives 8 sequences",
           "fail_randomphase_ploidy": "--randomPhase with a ploidy above 1",
           "fail_multi_ploidy": "multi-PHYLIP input with a ploidy above 1",
           "fail_S_missing": "sequence zz is not in the input",
           "fail_multi_S_missing": "sequence zz is not in alignment 1",
           "fail_multi_counts": "hold different numbers of sequences (2, 3)",
           "fail_phylip_no_header": "has no header line",
           "fail_header_count_zero": "line 1: the header counts 0 sequences",
           "fail_header_few_lines": "line 1: the header counts 3 sequences, 2 lines follow it",
           "fail_one_field_line": "line 3: a sequence line with one field",
           "fail_fasta_no_newline": "record b has no newline",
           "fail_fasta_no_name": "the record at byte 8 has no name",
           "fail_samples_empty": "-M samples with no sequences",
           "fail_shorter_later": "column c holds 20 sites, the first holds 30",
           "fail_multi_shorter_later": "alignment 2: column b holds 3 sites, the first holds 4"}
TINY = {"PG_S2G_SLAB_BYTES": "40"}


def expected(case):
    return gzip.decompress(open(os.path.join(DIR, case["output"]), "rb").read())


def run_cli(case, tmp_path, monkeypatch, engine=None, extra_env=None, args=None, inp=None, stdin=None):
    """the command line on a fixture case (or on the file inp with args) in tmp_path; returns what it wrote (decompressed)"""
    from genomics_general_b200.cli import seqToGeno as G
    if engine is not None:
        monkeypatch.setattr(G, "Engine", engine)
        from oracle_engine_filter import HostArray
        monkeypatch.setattr(G, "PinnedArray", HostArray)
    for k, v in (extra_env or {}).items():
        monkeypatch.setenv(k, v)
    work = tmp_path / "work"
    work.mkdir(exist_ok=True)
    monkeypatch.chdir(work)
    out = io.TextIOWrapper(io.BytesIO())
    monkeypatch.setattr(sys, "stdout", out)
    if case is not None:
        argv = list(case["args"])
        if case["input"] == "-":
            monkeypatch.setattr(sys, "stdin", io.TextIOWrapper(open(os.path.join(DIR, "lf.fa"), "rb")))
        else:
            argv += ["-s", os.path.join(DIR, case["input"])]
        dest = case["dest"]
    else:
        argv, dest = list(args), "stdout"
        if inp is not None:
            argv += ["-s", inp]
        if stdin is not None:
            monkeypatch.setattr(sys, "stdin", io.TextIOWrapper(io.BytesIO(stdin)))
    if dest != "stdout":
        argv += ["-g", dest]
    try:
        G.main(argv)
    finally:
        out.flush()
        got = out.buffer.getvalue()
        if dest != "stdout" and os.path.exists(work / dest):
            got = open(work / dest, "rb").read()
            got = gzip.decompress(got) if dest.endswith(".gz") else got
        run_cli.got = got
    return got


@pytest.mark.parametrize("case", OK, ids=[c["name"] for c in OK])
def test_cli_on_oracle_engine_matches_reference(case, tmp_path, monkeypatch):
    from oracle_engine_s2g import S2gOracleEngine
    assert run_cli(case, tmp_path, monkeypatch, S2gOracleEngine) == expected(case)


@pytest.mark.parametrize("case", OK, ids=[c["name"] for c in OK])
def test_cli_on_oracle_engine_tiny_slabs(case, tmp_path, monkeypatch):
    from oracle_engine_s2g import S2gOracleEngine
    assert run_cli(case, tmp_path, monkeypatch, S2gOracleEngine, extra_env=TINY) == expected(case)


@pytest.mark.parametrize("case", FAILS, ids=[c["name"] for c in FAILS])
def test_cli_refuses_where_the_reference_fails(case, tmp_path, monkeypatch):
    from oracle_engine_s2g import S2gOracleEngine
    with pytest.raises(SystemExit) as e:
        run_cli(case, tmp_path, monkeypatch, S2gOracleEngine)
    msg = str(e.value)
    assert msg.startswith("seqToGeno: ")
    assert REFUSED[case["name"]] in msg, msg
    assert run_cli.got == b""


def _file(tmp_path, data, name="in.txt"):
    p = tmp_path / name
    p.write_bytes(data)
    return str(p)


# the narrowings: inputs the reference reads, which this engine refuses with the line
@pytest.mark.parametrize("data, args, what", [
    (b">a\nACGT\n>b\nAC\xc3\xa9T\n", [], "a byte outside ASCII at line 4"),
    (b"2 4\na ACGT\rb CCGT\n", ["-f", "phylip"], "line 2: a '\\r' ends a line by itself"),
    (b"2 4\n#a ACGT\nb CCGT\n", ["-f", "phylip"], "line 2 starts with '#'"),
    (b"#x\n2 4\na ACGT\nb CCGT\n", ["-f", "phylip"], "line 1 starts with '#'"),
    (b">a\nACGT\n>b\nTTGG\n", ["-S", "a", "b", "-P", "0", "2"], "-P values must be at least 1"),
    (b">a\nACGT\n>b\nTTGG\n", ["--devices", "2"], "--devices"),
])
def test_narrowings_are_refused(tmp_path, monkeypatch, data, args, what):
    from oracle_engine_s2g import S2gOracleEngine
    with pytest.raises(SystemExit) as e:
        run_cli(None, tmp_path, monkeypatch, S2gOracleEngine, args=args, inp=_file(tmp_path, data))
    assert str(e.value).startswith("seqToGeno: ") and what in str(e.value), str(e.value)
    assert run_cli.got == b""


def test_stdin_fasta_with_cr_is_refused(tmp_path, monkeypatch):
    """the reference reads stdin without universal newlines and keeps a '\\r' as a character"""
    from oracle_engine_s2g import S2gOracleEngine
    with pytest.raises(SystemExit) as e:
        run_cli(None, tmp_path, monkeypatch, S2gOracleEngine, args=[], stdin=b">a\r\nACGT\r\n")
    assert "line 1: a '\\r' in a FASTA read from stdin" in str(e.value), str(e.value)


def test_plain_statement_rules():
    """worked examples of the line table and the rows"""
    from oracle_engine_s2g import line_table, rows_of
    t = line_table(b"x\n +3  1_0 z\n#c\n a\tAC GT\n3 1__0\n\x1c\n")
    assert t.tolist() == [[0, 1, -1, 0, 1, 0, 0], [3, 2, 7, 3, 3, 4, 3], [17, 1, 19, 2, 3, 0, 0],
                          [25, 1, 27, 4, 2, 0, 0], [-1, 0, -1, 0, 0, 0, 0]]
    assert rows_of([b"AC", b"GT", b"T"], [b"c", b"d"], [2, 1], [[0, 1], [2]], [b"|\n", b"\n"]) == \
        b"c\t1\tA|G\nc\t2\tC|T\nd\t1\tT\n"
