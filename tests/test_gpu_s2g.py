"""seqToGeno.py on the GPU: every fixture case of the unmodified reference (tests/golden/s2g12) through the command line
byte for byte, with default and with tiny slabs, and its refusals; the device against the plain statement
(tests/oracle_engine_s2g.py) at the transpose's edges — 1-70 sequences, lengths 0, 1, the tile width +-1 and 65 539, mixed
ploidy groups of 1-8, a 300-byte contig name, positions across every digit boundary up to 10^7, rows longer than a slab
and random slab sizes, 200 multi-PHYLIP alignments, interleaved PHYLIP with many blocks, FASTA line widths 1-200 with CRLF,
64 sequences x 2 M sites; and a round trip through the repository's genoToSeq."""
import io
import random
import sys

import numpy as np
import pytest

from test_s2g_cpu import FAILS, OK, REFUSED, TINY, expected, run_cli

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", OK, ids=[c["name"] for c in OK])
def test_cli_matches_reference_fixture(case, tmp_path, monkeypatch):
    assert run_cli(case, tmp_path, monkeypatch) == expected(case)


@pytest.mark.parametrize("case", OK, ids=[c["name"] for c in OK])
def test_cli_tiny_slabs(case, tmp_path, monkeypatch):
    assert run_cli(case, tmp_path, monkeypatch, extra_env=TINY) == expected(case)


@pytest.mark.parametrize("case", FAILS, ids=[c["name"] for c in FAILS])
def test_cli_refuses_where_the_reference_fails(case, tmp_path, monkeypatch):
    with pytest.raises(SystemExit) as e:
        run_cli(case, tmp_path, monkeypatch)
    assert REFUSED[case["name"]] in str(e.value), str(e.value)
    assert run_cli.got == b""


# ---- the device against the plain statement ----------------------------------------------------------------------------

def _seq(rng, n):
    return bytes(rng.choice(b"ACGTNacgt-RY") for _ in range(n))


def _fasta(rng, seqs, crlf=False, widths=(60,)):
    out = []
    for k, s in enumerate(seqs):
        out.append(b">q%d some description\n" % k)
        at = 0
        while at < len(s):
            w = rng.choice(widths)
            out.append(s[at:at + w] + (b"\r\n" if crlf else b"\n"))
            at += w
    return b"".join(out)


def _both(engine_calls, slab_sizes=(64 << 20,)):
    """run the same engine calls on the device and on the statement; returns (device bytes per slab size, statement bytes)"""
    from genomics_general_b200.engine import Engine
    from oracle_engine_s2g import S2gOracleEngine
    want = None
    got = []
    with Engine(0) as eng:
        for slab in slab_sizes:
            total = engine_calls(eng)
            buf = np.zeros(slab, np.uint8)
            parts, at = [], 0
            while at < total:
                nb = eng.s2g_emit(at, buf, slab)
                parts.append(buf[:nb].tobytes())
                at += nb
            got.append(b"".join(parts))
    o = S2gOracleEngine()
    total = engine_calls(o)
    want = o.out
    assert len(want) == total
    return got, want


def _fasta_calls(data, names_of, rows_of, members_of, seps_of):
    def calls(eng):
        starts = eng.s2g_fasta_load(data)
        from genomics_general_b200.cli._common import fasta_records
        _, lo, hi = fasta_records(data, starts, pytest.fail)
        eng.s2g_fasta_index(lo, hi)
        return eng.s2g_plan(names_of, rows_of, members_of, seps_of)
    return calls


def _samples_block(n, rows, name=b"contig0", groups=None):
    groups = groups or [1] * n
    mem, sep, at = [], [], 0
    for g, p in enumerate(groups):
        mem += list(range(at, at + p))
        sep += [b"|"] * (p - 1) + [b"\n" if g == len(groups) - 1 else b"\t"]
        at += p
    return [name], [rows], [mem], [b"".join(sep)]


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 63, 64, 65, 70])
@pytest.mark.parametrize("L", [0, 1, 63, 64, 65, 129])
def test_sequence_counts_and_lengths(n, L):
    rng = random.Random(n * 1000 + L)
    seqs = [_seq(rng, L) for _ in range(n)]
    got, want = _both(_fasta_calls(_fasta(rng, seqs), *_samples_block(n, L)), slab_sizes=(64 << 20, 37))
    assert got == [want, want]


def test_long_sequences_and_digit_boundaries():
    """65 539 sites, then positions across every digit boundary up to 10^7 (contigs mode: one member per block)"""
    rng = random.Random(3)
    seqs = [_seq(rng, 65539) for _ in range(3)]
    got, want = _both(_fasta_calls(_fasta(rng, seqs), *_samples_block(3, 65539)), slab_sizes=(1 << 20, 65536 + 7))
    assert got == [want, want]
    np_rng = np.random.default_rng(4)
    big = np_rng.choice(np.frombuffer(b"ACGT", np.uint8), 10 ** 7 + 3).tobytes()
    data = b">big\n" + big + b"\n>small\nAC\n"
    got, want = _both(_fasta_calls(data, [b"big", b"small"], [10 ** 7 + 3, 2], [[0], [1]], [b"\n", b"\n"]),
                      slab_sizes=(64 << 20, 9_999_991))
    assert got == [want, want]
    assert want.count(b"\n") == 10 ** 7 + 5


def test_mixed_ploidy_groups_long_name_and_random_slabs():
    rng = random.Random(5)
    groups = [1, 8, 2, 3, 1, 5, 7, 4, 6, 1, 2]
    n = sum(groups)
    seqs = [_seq(rng, 300 + rng.randrange(40)) for _ in range(n)]
    name = b"n" * 300
    calls = _fasta_calls(_fasta(rng, seqs), *_samples_block(n, 300, name=name, groups=groups))
    slabs = [1, 7, 64, 100, 777, 4096] + [rng.randrange(1, 50000) for _ in range(4)]
    got, want = _both(calls, slab_sizes=slabs)
    assert all(g == want for g in got)


def test_fasta_line_widths_and_crlf():
    rng = random.Random(6)
    seqs = [_seq(rng, 2000) for _ in range(9)]
    data = _fasta(rng, seqs, crlf=True, widths=tuple(range(1, 201)))
    got, want = _both(_fasta_calls(data, *_samples_block(9, 2000)))
    assert got == [want]
    assert want.split(b"\n")[0] == b"contig0\t1\t" + b"\t".join(s[:1] for s in seqs)


def _phylip_run(data, args, tmp_path, monkeypatch, slab="29"):
    """the command line on the device and on the statement, with default and with tiny slabs"""
    from oracle_engine_s2g import S2gOracleEngine
    p = tmp_path / "in.phy"
    p.write_bytes(data)
    want = run_cli(None, tmp_path, monkeypatch, S2gOracleEngine, args=args, inp=str(p))
    got = run_cli(None, tmp_path, monkeypatch, args=args, inp=str(p))
    tiny = run_cli(None, tmp_path, monkeypatch, args=args, inp=str(p), extra_env={"PG_S2G_SLAB_BYTES": slab})
    return got, tiny, want


def test_200_multi_phylip_alignments(tmp_path, monkeypatch):
    rng = random.Random(7)
    names = ["t%d" % k for k in range(12)]
    parts = []
    for i in range(200):
        order = names[:]
        rng.shuffle(order)
        L = rng.randrange(1, 40)
        parts.append("12 %d\n" % L + "".join("%s %s\n" % (n, _seq(rng, L).decode()) for n in order))
    data = "".join(parts).encode()
    for args in (["-f", "phylip"], ["-f", "phylip", "--merge", "-S", "t3", "t0", "t3"]):
        got, tiny, want = _phylip_run(data, args, tmp_path, monkeypatch)
        assert got == tiny == want


def test_interleaved_phylip_many_blocks(tmp_path, monkeypatch):
    rng = random.Random(8)
    n, blocks = 7, 150
    seqs = [[_seq(rng, rng.randrange(1, 12)) for _ in range(blocks)] for _ in range(n)]
    lines = [b"%d %d" % (n, 10)]
    for b in range(blocks):
        for k in range(n):
            lines.append((b"s%d " % k if b == 0 else b"%s " % _seq(rng, 3)) + seqs[k][b])
        if b % 10 == 0:
            lines.append(b"")
    data = b"\r\n".join(lines) + b"\r\n"
    for args in (["-f", "phylip", "-M", "contigs"], ["-f", "phylip", "-M", "contigs", "-P", "3", "4"]):
        got, tiny, want = _phylip_run(data, args, tmp_path, monkeypatch)
        assert got == tiny == want


def test_64_sequences_by_2M_sites():
    np_rng = np.random.default_rng(9)
    L = 2_000_000
    mat = np_rng.choice(np.frombuffer(b"ACGTN", np.uint8), (64, L))
    data = b"".join(b">q%d\n" % k + mat[k].tobytes() + b"\n" for k in range(64))
    from genomics_general_b200.engine import Engine
    with Engine(0) as eng:
        total = _fasta_calls(data, *_samples_block(64, L))(eng)
        buf = np.zeros(64 << 20, np.uint8)
        parts, at = [], 0
        while at < total:
            nb = eng.s2g_emit(at, buf, len(buf))
            parts.append(buf[:nb].copy())
            at += nb
    out = np.concatenate(parts)
    rows = out.tobytes().split(b"\n")[:-1]
    assert len(rows) == L
    for x in (0, 9, 10, 99_999, 1_999_999):
        f = rows[x].split(b"\t")
        assert f[0] == b"contig0" and f[1] == b"%d" % (x + 1) and b"".join(f[2:]) == mat[:, x].tobytes()


def test_round_trip_through_genoToSeq(tmp_path, monkeypatch):
    """a haploid .geno with contig0 and positions 1..L -> genoToSeq -M cat -> seqToGeno on the GPU: the same bytes"""
    from genomics_general_b200.cli import genoToSeq
    rng = random.Random(10)
    n, L = 13, 5000
    cols = [_seq(rng, L).upper().replace(b"-", b"N") for _ in range(n)]
    geno = b"#CHROM\tPOS\t" + b"\t".join(b"x%d" % k for k in range(n)) + b"\n" + \
        b"".join(b"contig0\t%d\t" % (x + 1) + b"\t".join(c[x:x + 1] for c in cols) + b"\n" for x in range(L))
    gp = tmp_path / "in.geno"
    gp.write_bytes(geno)
    fa = tmp_path / "out.fa"
    genoToSeq.main(["-g", str(gp), "-s", str(fa), "-M", "cat"])
    back = run_cli(None, tmp_path, monkeypatch, args=[], inp=str(fa))
    assert back == geno
