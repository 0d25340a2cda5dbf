"""genoToSeq.py on the GPU: every fixture case of the unmodified reference (tests/golden/seq10) through the command line byte
for byte, in every mode, format and --separateFiles layout, also with 40-byte slabs; and the refusals."""
import pytest

from test_seq_cpu import FAILS, OK, expected, run_cli

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", OK, ids=[c["name"] for c in OK])
def test_cli_matches_reference_fixture(case, tmp_path, monkeypatch):
    assert run_cli(case, tmp_path, monkeypatch) == expected(case)


@pytest.mark.parametrize("case", OK, ids=[c["name"] for c in OK])
def test_cli_tiny_slabs(case, tmp_path, monkeypatch):
    assert run_cli(case, tmp_path, monkeypatch, extra_env={"PG_SEQ_SLAB_BYTES": "40"}) == expected(case)


@pytest.mark.parametrize("case", FAILS, ids=[c["name"] for c in FAILS])
def test_cli_refuses_where_the_reference_fails(case, tmp_path, monkeypatch):
    with pytest.raises(SystemExit) as e:
        run_cli(case, tmp_path, monkeypatch)
    assert str(e.value).startswith("genoToSeq: ")
