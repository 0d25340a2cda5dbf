"""parseVCF.py on the GPU: every fixture case of the unmodified reference through the command line byte for byte, the same
with tiny chunks and slabs, and the error reports (the first offending line wins)."""
import pytest

from test_vcf_cpu import CASES, bad_inputs, expected, run_cli

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_cli_matches_reference_fixture(case, tmp_path, monkeypatch):
    assert run_cli(case, tmp_path, monkeypatch) == expected(case)


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_cli_tiny_chunks_and_slabs(case, tmp_path, monkeypatch):
    got = run_cli(case, tmp_path, monkeypatch, extra_env={"PG_VCF_CHUNK_BYTES": "700", "PG_VCF_SLAB_BYTES": "400"})
    assert got == expected(case)


@pytest.mark.parametrize("name, text, args, line", bad_inputs(), ids=[b[0] for b in bad_inputs()])
def test_cli_refuses_at_the_line(name, text, args, line, tmp_path, monkeypatch):
    p = tmp_path / "in.vcf"
    p.write_bytes(text.encode())
    with pytest.raises(SystemExit) as e:
        run_cli(None, tmp_path, monkeypatch, args=args, inp=str(p))
    assert "data line %d" % line in str(e.value)
