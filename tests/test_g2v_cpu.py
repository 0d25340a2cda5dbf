"""genoToVCF.py without a GPU: the command line's host logic (flags, refusals, header, FASTA records, chunks, slabs, messages)
on an oracle-backed engine (tests/oracle_engine_g2v.py) against every output the unmodified reference wrote
(tests/golden/g2v11), byte for byte after decompression, with normal and with tiny chunks and slabs."""
import gzip
import io
import json
import os
import sys

import pytest

from helpers import GOLDEN

CASES = json.load(open(os.path.join(GOLDEN, "cases11.json")))
DIR = os.path.join(GOLDEN, "g2v11")
OK = [c for c in CASES if "fails" not in c]
FAILS = [c for c in CASES if "fails" in c]
# refused at a data line: the rows before it are written as the reference writes them
AT_LINE = {"fail_missing_column": "line 13: sample s5 has no genotype column",
           "fail_bad_diplo": "line 31: the genotype of sample d5 is not one of the diplo codes",
           "fail_scaffold_not_in_fasta": "line 16: scaffold chrZ is not a record of the reference FASTA",
           "fail_position_outside_contig": "line 10: position 201 is outside its reference contig"}
# refused before any output
UP_FRONT = {"fail_no_format": "-f/--genoFormat is required",
            "fail_sample_not_in_header": "sample zz is not in the header",
            "fail_no_names": "no samples",
            "fail_fai_short_line": "badfai.fa.fai line 2 has fewer than 2 fields",
            "fail_fasta_no_newline": "record chrB has no newline",
            "fail_fasta_no_token": "the record at byte 11 has no name",
            "fail_empty_input": "the input is empty"}
TINY = {"PG_G2V_CHUNK_BYTES": "300", "PG_G2V_SLAB_BYTES": "40"}


def expected(case):
    return gzip.decompress(open(os.path.join(DIR, case["output"]), "rb").read())


def run_cli(case, tmp_path, monkeypatch, engine=None, extra_env=None, args=None, inp=None):
    """the command line on a fixture case (or on the file inp with args) in tmp_path; returns what it wrote (decompressed)"""
    from genomics_general_b200.cli import genoToVCF as G
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
        argv = [os.path.join(DIR, a) if k > 0 and case["args"][k - 1] == "-r" else a for k, a in enumerate(case["args"])]
        if case["input"] == "-":
            monkeypatch.setattr(sys, "stdin", io.TextIOWrapper(open(os.path.join(DIR, "main.geno"), "rb")))
        else:
            argv += ["-g", os.path.join(DIR, case["input"])]
        dest = case["dest"]
    else:
        argv, dest = list(args) + ["-g", inp], "stdout"
    if dest != "stdout":
        argv += ["-o", dest]
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
    from oracle_engine_g2v import G2vOracleEngine
    assert run_cli(case, tmp_path, monkeypatch, G2vOracleEngine) == expected(case)


@pytest.mark.parametrize("case", OK, ids=[c["name"] for c in OK])
def test_cli_on_oracle_engine_tiny_chunks_and_slabs(case, tmp_path, monkeypatch):
    from oracle_engine_g2v import G2vOracleEngine
    assert run_cli(case, tmp_path, monkeypatch, G2vOracleEngine, extra_env=TINY) == expected(case)


@pytest.mark.parametrize("tiny", [False, True])
@pytest.mark.parametrize("case", FAILS, ids=[c["name"] for c in FAILS])
def test_cli_refuses_where_the_reference_fails(case, tiny, tmp_path, monkeypatch):
    """at a data line: the message names the file line (and the sample) and the rows before it are the reference's; before
    any output: nothing is written.  A blank data line is skipped (the reference fails on it)."""
    from oracle_engine_g2v import G2vOracleEngine
    env = TINY if tiny else None
    if case["name"] == "fail_blank_line":
        got = run_cli(case, tmp_path, monkeypatch, G2vOracleEngine, extra_env=env)
        assert got.startswith(expected(case)) and got.count(b"\n") == expected(case).count(b"\n") + 20 - 6
        return
    with pytest.raises(SystemExit) as e:
        run_cli(case, tmp_path, monkeypatch, G2vOracleEngine, extra_env=env)
    msg = str(e.value)
    assert msg.startswith("genoToVCF: ")
    if case["name"] in AT_LINE:
        assert AT_LINE[case["name"]] in msg, msg
        assert run_cli.got == expected(case)
    else:
        assert UP_FRONT[case["name"]] in msg, msg
        assert run_cli.got == b""


def _geno(tmp_path, text, name="in.geno"):
    p = tmp_path / name
    p.write_bytes(text.encode() if isinstance(text, str) else text)
    return str(p)


HEAD = "#CHROM\tPOS\ta\tb\n"


@pytest.mark.parametrize("body, line, what", [
    ("c\t1\tA|T\tG|G\nc\t1_000\tA|T\tG|G\n", 3, "not an integer of the form"),
    ("c\t1\tA|T\tG|G\n#x\nc\tx\tA|T\tG|G\n", 4, "not an integer of the form"),
    ("c\t1\tA|T\tG|G\nc\t9223372036854775808\tA|T\tG|G\n", 3, "int64"),
    ("c\t1\tA|T\tG|G\n\nc\t2\n", 4, "only two fields"),
    ("c\t1\tA|T\tG|G\nc\n", 3, "no position field"),
    ("c\t1\tA|T\tG|G\nc\t5\tA|T\tG|G\rc\t6\tA|T\tG|G\n", 3, "ends a line by itself"),
    ("c\t1\tA|T\tG|G\nc\t2\tA|\xe9\tG|G\n", 3, "outside ASCII"),
    ("c\t1\tA|T\tG|G\nc\t2\tA|T\n", 3, "sample b has no genotype column"),
])
def test_refusal_names_the_line(tmp_path, monkeypatch, body, line, what):
    from oracle_engine_g2v import G2vOracleEngine
    inp = _geno(tmp_path, HEAD + body)
    with pytest.raises(SystemExit) as e:
        run_cli(None, tmp_path, monkeypatch, G2vOracleEngine, args=["-f", "phased"], inp=inp)
    assert "line %d: " % line in str(e.value) and what in str(e.value), str(e.value)
    assert run_cli.got.endswith(b"\tFORMAT\ta\tb\nc\t1\t.\tG\tT,A\t.\t.\t.\tGT\t2|1\t0|0\n")


@pytest.mark.parametrize("args, what", [
    (["-f", "phased", "--devices", "2"], "--devices"),
    (["-f", "phased", "--hostParse"], "--hostParse"),
    (["-f", "phased", "-s", "a,"], "sample  is not in the header"),
])
def test_flag_refusals(tmp_path, monkeypatch, args, what):
    from oracle_engine_g2v import G2vOracleEngine
    inp = _geno(tmp_path, HEAD + "c\t1\tA|T\tG|G\n")
    with pytest.raises(SystemExit) as e:
        run_cli(None, tmp_path, monkeypatch, G2vOracleEngine, args=args, inp=inp)
    assert what in str(e.value), str(e.value)


def test_duplicate_header_name_takes_the_last_column_the_line_holds(tmp_path, monkeypatch):
    """dict(zip(names, GTs)): the last column of a name wins, among the columns the line has"""
    from oracle_engine_g2v import G2vOracleEngine
    inp = _geno(tmp_path, "#CHROM\tPOS\ta\tb\ta\nc\t1\tA|A\tC|C\tG|G\nc\t2\tA|A\tC|C\n")
    got = run_cli(None, tmp_path, monkeypatch, G2vOracleEngine, args=["-f", "phased", "-s", "a"], inp=inp)
    assert got.split(b"\n")[-3:] == [b"c\t1\t.\tG\t.\t.\t.\t.\tGT\t0|0", b"c\t2\t.\tA\t.\t.\t.\t.\tGT\t0|0", b""]


def test_plain_statement_rules():
    """worked examples of the allele list L and the coding: no counted base, a reference base, ties, phase, pairs"""
    from oracle_engine_g2v import site
    row, _ = site(b"c\t5\tN|N\tN|N", 0, [-1, -1], [0, 1], None)
    assert row == b"c\t5\t.\tN\t.\t.\t.\t.\tGT\t0|0\t0|0\n"
    row, _ = site(b"c\t5\tN|N", 0, [-1], [0], lambda s: "AAAAC")
    assert row == b"c\t5\t.\tC\tN\t.\t.\t.\tGT\t1|1\n"
    row, _ = site(b"c\t1\tA|N", 0, [-1], [0], lambda s: "N")
    assert row == b"c\t1\t.\tN\tA\t.\t.\t.\tGT\t1|0\n"
    row, _ = site(b"c\t1\tA|C\tC|A", 0, [-1, -1], [0, 1], None)                  # A=2 C=2: the later letter first
    assert row == b"c\t1\t.\tC\tA\t.\t.\t.\tGT\t1|0\t0|1\n"
    row, _ = site(b"c\t+007\tA/T|G\tAT", 0, [-1, -1], [0, 1], None)
    assert row == b"c\t7\t.\tA\tT,G\t.\t.\t.\tGT\t0/1/2\t0\n"
    row, _ = site(b"c\t1\tA/T\tGT", 2, [-1, -1], [0, 1], None)                    # pairs: '/' is an allele, never counted
    assert row == b"c\t1\t.\tT\tG\t.\t.\t.\tGT\t././.\t1/0\n"
