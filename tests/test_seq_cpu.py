"""genoToSeq.py without a GPU: the command line's host logic (flags, refusals, names, windows, output files and slabs) on an
oracle-backed engine (tests/oracle_engine_seq.py) against every file the unmodified reference wrote (tests/golden/seq10),
byte for byte after decompression."""
import gzip
import io
import json
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest

from helpers import GOLDEN

CASES = json.load(open(os.path.join(GOLDEN, "cases10.json")))
DIR = os.path.join(GOLDEN, "seq10")
OK = [c for c in CASES if "fails" not in c]
FAILS = [c for c in CASES if "fails" in c]


def expected(case):
    return {fn: gzip.decompress(open(os.path.join(DIR, fix), "rb").read()) for fn, fix in case["outputs"].items()}


def run_cli(case, tmp_path, monkeypatch, engine=None, extra_env=None, args=None, inp=None):
    """the command line on a fixture case (or on inp with args) in tmp_path; returns {file name: bytes} of what it wrote
    (decompressed), with "stdout" for standard output"""
    from genomics_general_b200.cli import genoToSeq as G
    if engine is not None:
        monkeypatch.setattr(G, "Engine", engine)
        from oracle_engine_filter import HostArray
        monkeypatch.setattr(G, "PinnedArray", HostArray)
    for k, v in (extra_env or {}).items():
        monkeypatch.setenv(k, v)
    work = tmp_path / "work"
    work.mkdir()
    monkeypatch.chdir(work)
    out = io.TextIOWrapper(io.BytesIO())
    monkeypatch.setattr(sys, "stdout", out)
    dest = case["dest"] if case else "out"
    argv = ["-g", inp or os.path.join(DIR, case["input"])] + (args if args is not None else case["args"])
    if dest != "stdout":
        argv += ["-s", dest]
    G.main(argv)
    got = {}
    if dest == "stdout":
        out.flush()
        got["stdout"] = out.buffer.getvalue()
    for fn in sorted(os.listdir(work)):
        data = open(os.path.join(work, fn), "rb").read()
        got[fn] = gzip.decompress(data) if fn.endswith(".gz") else data
    return got


@pytest.mark.parametrize("case", OK, ids=[c["name"] for c in OK])
def test_cli_on_oracle_engine_matches_reference(case, tmp_path, monkeypatch):
    from oracle_engine_seq import SeqOracleEngine
    assert run_cli(case, tmp_path, monkeypatch, SeqOracleEngine) == expected(case)


@pytest.mark.parametrize("case", [c for c in OK if c["name"] in ("cat_split", "contigs_separate", "windows_sites_separate",
                                                                  "crlf_phylip", "cat_gzip_flag")], ids=lambda c: c["name"])
def test_cli_on_oracle_engine_tiny_slabs(case, tmp_path, monkeypatch):
    """slabs of 40 bytes: rows cut after a site and resumed, files cut across slabs"""
    from oracle_engine_seq import SeqOracleEngine
    assert run_cli(case, tmp_path, monkeypatch, SeqOracleEngine, extra_env={"PG_SEQ_SLAB_BYTES": "40"}) == expected(case)


@pytest.mark.parametrize("case", FAILS, ids=[c["name"] for c in FAILS])
def test_cli_refuses_where_the_reference_fails(case, tmp_path, monkeypatch):
    from oracle_engine_seq import SeqOracleEngine
    with pytest.raises(SystemExit) as e:
        run_cli(case, tmp_path, monkeypatch, SeqOracleEngine)
    assert str(e.value).startswith("genoToSeq: ")


def _geno(tmp_path, text, name="in.geno"):
    p = tmp_path / name
    p.write_bytes(text.encode() if isinstance(text, str) else text)
    return str(p)


HEAD = "#CHROM\tPOS\ta\tb\n"


@pytest.mark.parametrize("body, line, what", [
    ("c\t1\tA|T\tG|G\nc\t2\tA|T\tGG\n", 2, "sample b is not as wide"),
    ("c\t1\tA|T\tG|G\nc\t2\tA|TT\tG|G\n", 2, "sample a is not as wide"),
    ("c\t1\tA|T\tG|G\n#x\nc\t2\tA|T\tG|G\tC|C\n", 2, "3 genotype columns"),
    ("c\t1\tA|T\tG|G\nc\tx\tA|T\tG|G\n", 2, "position is not an integer"),
    ("c\t1\tA|T\tG|G\nc\t5\tA|T\tG|G\rc\t6\tA|T\tG|G\n", 2, "ends a line by itself"),
    ("c\t1\tA|T\tG|G\nc\t2\tA|\xe9\tG|G\n", 2, "outside ASCII"),
    ("c\t1\tA|T\tG|G\nc\t3000000000\tA|T\tG|G\n", 2, "int32"),
])
def test_refusal_names_the_data_line_and_sample(tmp_path, monkeypatch, body, line, what):
    from oracle_engine_seq import SeqOracleEngine
    inp = _geno(tmp_path, HEAD + body)
    with pytest.raises(SystemExit) as e:
        run_cli(None, tmp_path, monkeypatch, SeqOracleEngine, args=[], inp=inp)
    assert "data line %d" % line in str(e.value) and what in str(e.value), str(e.value)


@pytest.mark.parametrize("args, what", [
    (["--splitPhased", "--ploidy", "3"], "holds 2 alleles, its ploidy is 3"),
    (["--splitPhased", "--ploidy", "2", "2", "2"], None),
    (["--splitPhased", "--ploidy", "2"], None),
    (["--splitPhased", "--ploidy", "2", "1"], "holds 2 alleles, its ploidy is 1"),
    (["--splitPhased", "--ploidy", "1", "2"], "ploidy is 1"),
    (["--splitPhased", "-S", "a", "--ploidy", "2", "2"], None),
    (["-S", "z"], "sample z is not in the header"),
    (["--devices", "2"], "--devices"),
    (["-M", "windows", "--windType", "sites", "--windSize", "5", "--overlap", "5", "--maxDist", "9"], "--overlap must be"),
    (["-M", "windows", "--windType", "coordinate"], "--windSize"),
])
def test_ploidy_and_flag_refusals(tmp_path, monkeypatch, args, what):
    """--splitPhased: each sample's ceil(width / 2) must equal its ploidy (the reference checks only the total)"""
    from oracle_engine_seq import SeqOracleEngine
    inp = _geno(tmp_path, HEAD + "c\t1\tA|T\tG|G\nc\t2\tA|C\tG|N\n")
    if what is None:
        got = run_cli(None, tmp_path, monkeypatch, SeqOracleEngine, args=args, inp=inp)
        assert got["out"].startswith(b">a_A\nAA\n")
        return
    with pytest.raises(SystemExit) as e:
        run_cli(None, tmp_path, monkeypatch, SeqOracleEngine, args=args, inp=inp)
    assert what in str(e.value), str(e.value)


def test_haploid_names_follow_the_reference():
    from genomics_general_b200.cli.genoToSeq import haploid_names
    assert haploid_names(["a", "b"], [2])[0] == ["a_A", "a_B", "b_A", "b_B"]
    assert haploid_names(["a", "b"], [1])[0] == ["a", "b"]
    assert haploid_names(["a", "b"], [1, 3])[0] == ["a_A", "b_A", "b_B", "b_C"]
    assert haploid_names(["a", "b"], [1, 1, 2])[0] == ["a_A", "b_A"]         # not all 1: zip keeps the first two
    with pytest.raises(KeyError):
        haploid_names(["a", "b", "c"], [2, 2])


def test_duplicate_header_names_take_the_first_column_without_S_and_the_last_with_it(tmp_path, monkeypatch):
    """seqDict looks names up with list.index (genomics.py:1792); -S reads dict(zip(names, GTs)), where the last wins"""
    from oracle_engine_seq import SeqOracleEngine
    inp = _geno(tmp_path, "#CHROM\tPOS\ta\ta\nc\t1\tA\tC\nc\t2\tG\tT\n")
    (tmp_path / "one").mkdir()
    got = run_cli(None, tmp_path / "one", monkeypatch, SeqOracleEngine, args=[], inp=inp)
    assert got["out"] == b">a\nAG\n>a\nAG\n"
    (tmp_path / "two").mkdir()
    got = run_cli(None, tmp_path / "two", monkeypatch, SeqOracleEngine, args=["-S", "a"], inp=inp)
    assert got["out"] == b">a\nCT\n"


def test_contig_windows_and_file_names():
    """-M contigs: 1e7 bp coordinate windows (a 2.5e7 bp contig gives three); --separateFiles names"""
    from genomics_general_b200.cli import genoToSeq as G
    pos = np.array([5, 9_999_999, 10_000_001, 24_000_000, 7], np.int32)
    newsc = np.array([1, 0, 0, 0, 1], np.int8)
    args = SimpleNamespace(mode="contigs", windType="sites", separateFiles=True, seqFile="x", format="phylip", gzip=True)
    names = {0: "long", 4: "short"}
    scaf, lo, hi = G.windows_for(args, 5, pos, newsc, lambda i: names[i])
    assert scaf == ["long", "long", "long", "short"]
    assert list(lo) == [0, 2, 3, 4] and list(hi) == [2, 3, 4, 5]
    w = G._Writer.__new__(G._Writer)
    w.args, w.scaffolds, w.lo, w.hi, w.pos = args, scaf, lo, hi, pos
    assert w._name(1) == "x.long.phy.gz"
    args.mode, args.gzip, args.format = "windows", False, "fasta"
    assert w._name(0) == "x.long_5_9999999.fa"


def test_coordinate_windows_without_step_refused_on_a_second_window():
    from genomics_general_b200.cli import genoToSeq as G
    args = SimpleNamespace(mode="windows", windType="coordinate", windSize=100, stepSize=None)
    pos = np.array([5, 50, 150], np.int32)
    newsc = np.array([1, 0, 0], np.int8)
    with pytest.raises(SystemExit, match="second coordinate window"):
        G.windows_for(args, 3, pos, newsc, lambda i: "c")
    args.stepSize = 100
    _, lo, hi = G.windows_for(args, 3, pos, newsc, lambda i: "c")
    assert list(lo) == [0, 2] and list(hi) == [2, 3]
    with pytest.raises(SystemExit, match="decreases"):
        G.windows_for(args, 3, np.array([5, 50, 40], np.int32), newsc, lambda i: "c")
