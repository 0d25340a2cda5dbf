"""parseVCF.py without a GPU: the plain-Python statement of the reference's semantics (oracle/vcf_oracle.py) against the
fixtures the unmodified reference wrote, the command line's host logic on an oracle-backed engine byte for byte (also with
tiny chunks and slabs), and the refusals."""
import gzip
import json
import os

import pytest

from helpers import GOLDEN

from oracle import vcf_oracle as vo

CASES = json.load(open(os.path.join(GOLDEN, "cases9.json")))
DIR = os.path.join(GOLDEN, "vcf9")


def read_input(name):
    """a fixture input's bytes (main.vcf is kept as main.vcf.gz only)"""
    path = os.path.join(DIR, name)
    if not os.path.exists(path):
        path += ".gz"
    data = open(path, "rb").read()
    return gzip.decompress(data) if path.endswith(".gz") else data


def input_path(name, tmp_path):
    """a path the command line can read the fixture input from: a plain copy in tmp_path when it is stored compressed"""
    if os.path.exists(os.path.join(DIR, name)):
        return os.path.join(DIR, name)
    p = tmp_path / name
    p.write_bytes(read_input(name))
    return str(p)


def expected(case):
    return gzip.decompress(open(os.path.join(DIR, case["expected"]), "rb").read())


def run_cli(case, tmp_path, monkeypatch, engine=None, extra_env=None, args=None, inp=None):
    """the command line on a fixture case (or on inp, a path, with args); returns the output bytes"""
    from genomics_general_b200.cli import parseVCF as P
    if engine is not None:
        monkeypatch.setattr(P, "Engine", engine)
        from oracle_engine_filter import HostArray
        monkeypatch.setattr(P, "PinnedArray", HostArray)
    for k, v in (extra_env or {}).items():
        monkeypatch.setenv(k, v)
    gz = case["gz"] if case else False
    out = str(tmp_path / ("out.geno.gz" if gz else "out.geno"))
    monkeypatch.chdir(DIR)              # the cases name their side files relative to the fixture directory
    P.main(["-i", inp or input_path(case["input"], tmp_path), "-o", out] + (args if args is not None else case["args"]))
    data = open(out, "rb").read()
    return gzip.decompress(data) if gz else data


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_oracle_matches_reference_fixture(case, monkeypatch):
    monkeypatch.chdir(DIR)
    assert vo.run(read_input(case["input"]), case["args"]) == expected(case)


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_cli_on_oracle_engine_matches_reference(case, tmp_path, monkeypatch):
    from oracle_engine_vcf import VcfOracleEngine
    assert run_cli(case, tmp_path, monkeypatch, VcfOracleEngine) == expected(case)


@pytest.mark.parametrize("case", [c for c in CASES if c["name"] in ("gtf_many", "dups_include", "field_phase_missing",
                                                                      "dupnames")], ids=lambda c: c["name"])
def test_cli_on_oracle_engine_tiny_chunks_and_slabs(case, tmp_path, monkeypatch):
    from oracle_engine_vcf import VcfOracleEngine
    got = run_cli(case, tmp_path, monkeypatch, VcfOracleEngine,
                  extra_env={"PG_VCF_CHUNK_BYTES": "300", "PG_VCF_SLAB_BYTES": "900"})
    assert got == expected(case)


HEAD = "##fileformat=VCFv4.2\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\ta\tb\n"


def bad_inputs():
    ok = "chr1\t5\t.\tA\tC\t.\tPASS\t.\tGT\t0/1\t1/1\n"
    return [
        ("short_line", HEAD + ok + "chr1\t6\t.\tA\tC\t.\tPASS\t.\tGT\t0/1\n", [], 2),
        ("no_format", HEAD + ok + ok + "chr1\t7\t.\tA\n", [], 3),
        ("bad_pos", HEAD + ok + "chr1\t6x\t.\tA\tC\t.\tPASS\t.\tGT\t0/1\t1/1\n", [], 2),
        ("pos_int64", HEAD + "chr1\t99999999999999999999\t.\tA\tC\t.\tPASS\t.\tGT\t0/1\t1/1\n", [], 1),
        ("no_gt", HEAD + ok + "chr1\t6\t.\tA\tC\t.\tPASS\t.\tDP:GT\t3\t1/1\n", [], 2),
        ("haploid_default_ploidy", HEAD + ok + ok + "chr1\t6\t.\tA\tC\t.\tPASS\t.\tGT\t0/1\t0\n", [], 3),
        ("nbsp_between_fields", HEAD + ok + "chr1\t6\t.\tA\tC\t.\tPASS\t.\tGT\t0/1 1/1\tx\n", [], 2),
        ("first_line_wins", HEAD + ok + "chr1\t6\t.\tA\tC\t.\tPASS\t.\tGT\t0/1\t0\n" +
         "chr1\t7x\t.\tA\tC\t.\tPASS\t.\tGT\t0/1\t1/1\n", [], 2),
    ]


@pytest.mark.parametrize("name, text, args, line", bad_inputs(), ids=[b[0] for b in bad_inputs()])
def test_oracle_refuses_at_the_line(name, text, args, line):
    with pytest.raises(vo.Refusal) as e:
        vo.run(text.encode(), args)
    assert e.value.line == line


@pytest.mark.parametrize("name, text, args, line", bad_inputs(), ids=[b[0] for b in bad_inputs()])
def test_cli_on_oracle_engine_refuses_at_the_line(name, text, args, line, tmp_path, monkeypatch):
    from oracle_engine_vcf import VcfOracleEngine
    p = tmp_path / "in.vcf"
    p.write_bytes(text.encode())
    with pytest.raises(SystemExit) as e:
        run_cli(None, tmp_path, monkeypatch, VcfOracleEngine, args=args, inp=str(p))
    assert "data line %d" % line in str(e.value)


@pytest.mark.parametrize("args", [["--simplifyALT"], ["--expandMulti"], ["--field", "alleles"], ["--devices", "2"],
                                  ["-s", "zz"], ["--gtf", "flag=DP", "min=1=2"], ["--gtf", "bogus=1"]])
def test_cli_refuses_flags_up_front(args, tmp_path, monkeypatch):
    p = tmp_path / "in.vcf"
    p.write_bytes((HEAD + "chr1\t5\t.\tA\tC\t.\tPASS\t.\tGT\t0/1\t1/1\n").encode())
    from genomics_general_b200.cli import parseVCF as P
    with pytest.raises(SystemExit) as e:
        P.main(["-i", str(p), "-o", str(tmp_path / "o")] + args)
    assert "parseVCF" in str(e.value)


def test_qual_threshold_is_the_exact_integer_comparison():
    from genomics_general_b200.cli.parseVCF import qual_threshold
    for m in [1, 20, -5, 2 ** 53 + 1, 10 ** 30 + 1, -(10 ** 30) - 1, 10 ** 400, -(10 ** 400)]:
        t = qual_threshold(m)
        for q in [t, float(m) if abs(m) < 1e300 else 0.0, -0.0, 1e308, float("inf"), float("-inf")]:
            assert (q < t) == (q < m), (m, q)
