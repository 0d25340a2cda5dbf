"""genoToVCF.py on the GPU: every fixture case of the unmodified reference (tests/golden/g2v11) through the command line byte
for byte, with normal and with tiny chunks and slabs, and its refusals; the device against the plain statement
(tests/oracle_engine_g2v.py) at the kernels' edges — sample counts around the warp width, token widths 1-15, rows longer than
a slab, chunk cuts inside scaffold runs and CRLF line ends, 20 k lines x 300 samples, positions near +-2^62, FASTA lookups at
a record's first and last base and from its end, the error order; and a round trip through the repository's parseVCF."""
import io
import random
import sys

import numpy as np
import pytest

from test_g2v_cpu import AT_LINE, FAILS, OK, TINY, UP_FRONT, expected, run_cli

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", OK, ids=[c["name"] for c in OK])
def test_cli_matches_reference_fixture(case, tmp_path, monkeypatch):
    assert run_cli(case, tmp_path, monkeypatch) == expected(case)


@pytest.mark.parametrize("case", OK, ids=[c["name"] for c in OK])
def test_cli_tiny_chunks_and_slabs(case, tmp_path, monkeypatch):
    assert run_cli(case, tmp_path, monkeypatch, extra_env=TINY) == expected(case)


@pytest.mark.parametrize("case", [c for c in FAILS if c["name"] != "fail_blank_line"], ids=lambda c: c["name"])
def test_cli_refuses_where_the_reference_fails(case, tmp_path, monkeypatch):
    with pytest.raises(SystemExit) as e:
        run_cli(case, tmp_path, monkeypatch, extra_env=TINY)
    msg = str(e.value)
    if case["name"] in AT_LINE:
        assert AT_LINE[case["name"]] in msg, msg
        assert run_cli.got == expected(case)
    else:
        assert UP_FRONT[case["name"]] in msg, msg
        assert run_cli.got == b""


# ---- the device against the plain statement ----------------------------------------------------------------------------

def _token(rng, fmt, w):
    if fmt == 1:
        return rng.choice("ACGKMNSRTWYACGT")
    chars = "ACGTACGTACGTNNa-/" if fmt == 2 else "ACGTACGTACGTNNa-"
    if fmt == 2:
        return "".join(rng.choice(chars) for _ in range(w))
    t = rng.choice(chars)
    for _ in range((w - 1) // 2):
        t += rng.choice("||/") + rng.choice(chars)
    return t + (rng.choice(chars) if w % 2 == 0 else "")


def _body(rng, n_lines, n_samp, fmt, widths, scafs=("c1", "c2"), run=7, pos=None, crlf=False, sep="\t"):
    lines = []
    for i in range(n_lines):
        sc = scafs[(i // run) % len(scafs)]
        p = pos(i) if pos else 1 + i % 50
        lines.append(sep.join([sc, str(p)] + [_token(rng, fmt, rng.choice(widths)) for _ in range(n_samp)]))
    eol = "\r\n" if crlf else "\n"
    return (eol.join(lines) + eol).encode()


def _run(eng, body, fmt, n_samp, sel=None, fasta=None, slab=1 << 20):
    """the engine's methods as the command line calls them, on one chunk: (VCF rows, error)"""
    sel = list(range(n_samp)) if sel is None else sel
    rec = {}
    if fasta is not None:
        from genomics_general_b200.cli.genoToVCF import fasta_records
        starts = eng.g2v_ref_load(fasta)
        names, lo, hi = fasta_records(fasta, starts)
        eng.g2v_ref_index(lo, hi)
        rec = {n: k for k, n in enumerate(names)}
    col_slot = [k if k in set(sel) else -1 for k in range(n_samp)]
    slot, k = [], 0
    for c in col_slot:
        slot.append(k if c >= 0 else -1)
        k += c >= 0
    eng.g2v_spec(fmt, slot, [-1] * n_samp, sel, bool(rec))
    S, run_line, run_off = eng.g2v_chunk(body)
    import re
    tok = re.compile(rb"[^ \t\n\r\x0b\x0c\x1c-\x1f]+")
    run_rec = [rec.get(tok.search(body, int(o)).group().decode(), -1) for o in run_off] if rec else []
    rows, nb, err = eng.g2v_sites(run_rec)
    out, at = b"", 0
    buf = np.zeros(slab, np.uint8)
    while at < nb:
        n = eng.g2v_emit(at, buf, slab)
        out += buf[:n].tobytes()
        at += n
    return out, err


def _both(body, fmt, n_samp, **kw):
    from oracle_engine_g2v import G2vOracleEngine

    from genomics_general_b200.engine import Engine
    with Engine(0) as eng:
        got = _run(eng, body, fmt, n_samp, **kw)
    want = _run(G2vOracleEngine(), body, fmt, n_samp, **kw)
    assert got[1] == want[1]
    assert got[0] == want[0]
    return got


@pytest.mark.parametrize("n_samp", [1, 2, 31, 32, 33, 64, 65, 70])
@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_sample_counts_around_the_warp(n_samp, fmt):
    rng = random.Random(n_samp * 3 + fmt)
    out, err = _both(_body(rng, 300, n_samp, fmt, [1, 2, 3, 4, 5]), fmt, n_samp)
    assert err[0] == 0 and out.count(b"\n") == 300


@pytest.mark.parametrize("fmt", [0, 2])
def test_token_widths_1_to_15_and_selected_subsets(fmt):
    rng = random.Random(15 + fmt)
    body = _body(rng, 400, 40, fmt, list(range(1, 16)))
    _both(body, fmt, 40)
    _both(body, fmt, 40, sel=[39, 3, 3, 0, 17])


def test_rows_longer_than_a_slab():
    rng = random.Random(3)
    body = _body(rng, 60, 70, 0, [3, 5, 9])
    for slab in (37, 64, 1000):
        _both(body, 0, 70, slab=slab)


def test_twenty_thousand_lines_by_300_samples():
    rng = random.Random(20)
    body = _body(rng, 20000, 300, 0, [3], scafs=("chr1", "chr2", "chr3"), run=5000)
    out, err = _both(body, 0, 300, slab=8 << 20)
    assert err[0] == 0 and out.count(b"\n") == 20000


def test_positions_near_two_to_the_62():
    rng = random.Random(62)
    vals = [2 ** 62, -2 ** 62, 2 ** 62 + 7, -(2 ** 62) - 7, 2 ** 63 - 1, -2 ** 63, 0, -1]
    body = _body(rng, len(vals), 3, 0, [3], pos=lambda i: vals[i])
    _both(body, 0, 3)
    body = _body(rng, 2, 3, 0, [3], pos=lambda i: [5, 2 ** 63][i])
    assert _both(body, 0, 3)[1][:3] == (3, 1, 0)


def test_fasta_lookups_at_the_ends_of_a_record_and_from_its_end():
    rng = random.Random(7)
    fasta = b"junk\n>r1 desc\nACGTN\r\nac gt\n>r2\nTTGCA\n>r3\n\n\nG\n"
    pos = [1, 9, 0, -8, -3, 1, 5, 0, -4, 1, 0]
    scaf = ["r1"] * 5 + ["r2"] * 4 + ["r3"] * 2
    lines = ["\t".join([s, str(p)] + [_token(rng, 0, 3) for _ in range(4)]) for s, p in zip(scaf, pos)]
    body = ("\n".join(lines) + "\n").encode()
    out, err = _both(body, 0, 4, fasta=fasta)
    assert err[0] == 0 and [r.split(b"\t")[3] for r in out.splitlines()] == \
        [b"A", b"t", b"t", b"A", b"a", b"T", b"A", b"A", b"T", b"G", b"G"]
    bad = body + b"r1\t10\tA|A\tA|A\tA|A\tA|A\nr1\t-9\tA|A\tA|A\tA|A\tA|A\n"
    assert _both(bad, 0, 4, fasta=fasta)[1][:3] == (10, 11, 5)


def test_error_order_the_earlier_line_then_the_earlier_column():
    rng = random.Random(9)
    lines = _body(rng, 200, 40, 1, [1]).split(b"\n")
    lines[150] = lines[150].replace(b"\t", b"\tX", 1)           # a position that is not an integer
    f = lines[90].split(b"\t")
    f[30], f[10] = b"Q", b"Z"                                   # two bad diplo tokens: sample 8 first
    lines[90] = b"\t".join(f)
    out, err = _both(b"\n".join(lines), 1, 40)
    assert err[:3] == (8, 90, 9) and out.count(b"\n") == 90


def test_chunk_cuts_inside_scaffold_runs_and_crlf(tmp_path, monkeypatch):
    """the command line with chunks of a few lines (cut inside a run, between '\\r' and '\\n') on the device and on the plain
    statement, with a FASTA"""
    from oracle_engine_g2v import G2vOracleEngine
    rng = random.Random(11)
    fa = tmp_path / "ref.fa"
    fa.write_bytes(b">c1\n" + bytes(rng.choice(b"ACGTNacgt") for _ in range(60)) + b"\n>c2\n" +
                   bytes(rng.choice(b"ACGTN") for _ in range(55)) + b"\n")
    head = b"#CHROM POS " + b" ".join(b"s%d" % i for i in range(5)) + b"\r\n"
    inp = tmp_path / "in.geno"
    inp.write_bytes(head + _body(rng, 500, 5, 0, [1, 3, 5], run=13, crlf=True, sep=" "))
    args = ["-f", "phased", "-r", str(fa)]
    for chunk in ("97", "250", "4096"):
        env = {"PG_G2V_CHUNK_BYTES": chunk, "PG_G2V_SLAB_BYTES": "113"}
        (tmp_path / chunk).mkdir()
        want = run_cli(None, tmp_path / chunk, monkeypatch, G2vOracleEngine, extra_env=env, args=args, inp=str(inp))
        from genomics_general_b200.engine import Engine, PinnedArray
        from genomics_general_b200.cli import genoToVCF as G
        monkeypatch.setattr(G, "Engine", Engine)
        monkeypatch.setattr(G, "PinnedArray", PinnedArray)
        got = run_cli(None, tmp_path / chunk, monkeypatch, extra_env=env, args=args, inp=str(inp))
        assert got == want and got.count(b"\n") == 504


def test_round_trip_through_parse_vcf(tmp_path, monkeypatch):
    """phased diploid A/C/G/T genotypes without missing data: parseVCF with default flags gives back the input rows"""
    rng = random.Random(5)
    names = ["s%d" % i for i in range(12)]
    rows = ["\t".join(["chr%d" % (1 + i // 300), str(1 + 10 * i)] +
                      ["%s|%s" % (rng.choice("ACGT"), rng.choice("ACGT")) for _ in names]) for i in range(900)]
    text = "#CHROM\tPOS\t" + "\t".join(names) + "\n" + "\n".join(rows) + "\n"
    inp = tmp_path / "in.geno"
    inp.write_text(text)
    vcf = tmp_path / "out.vcf"
    from genomics_general_b200.cli import genoToVCF, parseVCF
    genoToVCF.main(["-f", "phased", "-g", str(inp), "-o", str(vcf)])
    out = io.TextIOWrapper(io.BytesIO())
    monkeypatch.setattr(sys, "stdout", out)
    parseVCF.main(["-i", str(vcf)])
    out.flush()
    assert out.buffer.getvalue().decode() == text
