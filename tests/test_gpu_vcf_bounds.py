"""parseVCF.py on the GPU against the plain-Python statement of the reference (oracle/vcf_oracle.py) at the kernels' edges:
selected samples around a warp and past a thousand, out of column order; lines over 200 KB and alleles of 300 bp; more lines
than one records grid covers and more rows than one emit grid covers; slab caps of exactly k rows, one byte less, and a row
larger than the buffer; the number fast path's edges (2^53 +- 1, 1e22 / 1e23, 19 and 20 significant digits, subnormals),
which the host settles with float(); UTF-8 in INFO (accepted) and NBSP between fields (refused)."""
import math
import random

import pytest

from oracle import vcf_oracle as vo
from test_vcf_cpu import run_cli

pytestmark = pytest.mark.gpu

FIX = "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT"


def make_vcf(rng, n_samp, n_lines, alt_len=1, dp=None, info="."):
    names = ["s%d" % i for i in range(n_samp)]
    rows = ["##fileformat=VCFv4.2", "\t".join([FIX] + names)]
    for i in range(n_lines):
        ref = "".join(rng.choice("ACGT") for _ in range(alt_len))
        alts = ["".join(rng.choice("ACGT") for _ in range(rng.choice([alt_len, alt_len + 1]))) for _ in range(rng.randint(1, 3))]
        samp = []
        for _ in range(n_samp):
            gt = rng.choice("/|").join(str(rng.randrange(len(alts) + 1)) if rng.random() > 0.05 else "." for _ in range(2))
            samp.append("%s:%s:%d" % (gt, rng.choice(dp) if dp else str(rng.randint(0, 40)), rng.randint(0, 99)))
        rows.append("\t".join(["chr%d" % (i * 2 // max(n_lines, 1)), str(100 + 3 * i), ".", ref, ",".join(alts),
                               rng.choice([".", "50", "7.5"]), "PASS", info, "GT:DP:GQ"] + samp))
    return ("\n".join(rows) + "\n").encode(), names


def check(tmp_path, monkeypatch, data, args, env=None):
    p = tmp_path / "in.vcf"
    p.write_bytes(data)
    want = vo.run(data, args)
    got = run_cli(None, tmp_path, monkeypatch, args=args, inp=str(p), extra_env=env)
    assert got == want
    return want


@pytest.mark.parametrize("n_samp", [1, 31, 32, 33, 1100])
def test_selected_samples_out_of_column_order(n_samp, tmp_path, monkeypatch):
    rng = random.Random(n_samp)
    data, names = make_vcf(rng, n_samp, 40 if n_samp < 1000 else 12)
    sel = names[:]
    rng.shuffle(sel)
    check(tmp_path, monkeypatch, data, ["-s", ",".join(sel), "--gtf", "flag=DP", "min=5", "max=35"])
    check(tmp_path, monkeypatch, data, ["-s", ",".join(sel[: max(1, n_samp // 2)]), "--field", "GQ"])


def test_lines_over_200kb_and_300bp_alleles(tmp_path, monkeypatch):
    rng = random.Random(2)
    data, _ = make_vcf(rng, 40, 3, alt_len=300, info="NOTE=" + "A" * 210_000)
    assert max(len(x) for x in data.split(b"\n")) > 200_000
    check(tmp_path, monkeypatch, data, ["--skipIndels", "--addRefTrack"])


def test_more_lines_and_rows_than_one_grid(tmp_path, monkeypatch):
    # records: sm_count * 64 blocks of 8 warps; emit: sm_count * 32 blocks of 8 warps (132 SMs: 67584 / 33792 lines)
    rng = random.Random(3)
    data, _ = make_vcf(rng, 1, 80_000)
    check(tmp_path, monkeypatch, data, ["--minQual", "10"])


def test_slab_caps(tmp_path, monkeypatch):
    rng = random.Random(4)
    data, _ = make_vcf(rng, 3, 30)
    want = vo.run(data, ["--noHeader"])
    rows = want.split(b"\n")[:-1]
    k = 4
    cap = sum(len(r) + 1 for r in rows[:k])
    for c in (cap, cap - 1):
        check(tmp_path, monkeypatch, data, ["--noHeader"], env={"PG_VCF_SLAB_BYTES": str(c)})
    with pytest.raises(Exception) as e:
        check(tmp_path, monkeypatch, data, ["--noHeader"], env={"PG_VCF_SLAB_BYTES": str(len(rows[0]))})
    assert "more than" in str(e.value)


def test_number_fast_path_edges_and_host_settling(tmp_path, monkeypatch):
    vals = ["9007199254740992", "9007199254740993", "9007199254740991", "1e22", "1e23", "1234567890123456789",
            "12345678901234567890", "4.9e-324", "2.2250738585072014e-308", "1e-22", "1e-23", "0.1", "1_0", "٣",
            repr(math.nextafter(1e22, math.inf)), "1e400", "-inf", "nan", "5.", ".5", "0e999"]
    rng = random.Random(5)
    data, _ = make_vcf(rng, 4, 60, dp=vals)
    for lo, hi in [("1e22", "1e23"), ("9007199254740992", "9007199254740992"), ("0", "4.9e-324"), ("0.1", "1e22"),
                   ("-inf", "1_0")]:
        check(tmp_path, monkeypatch, data, ["--gtf", "flag=DP", "min=" + lo, "max=" + hi])


def test_utf8_in_info_is_accepted_and_nbsp_is_refused(tmp_path, monkeypatch):
    rng = random.Random(6)
    data, _ = make_vcf(rng, 5, 20, info="NOTE=café;Ω=1")
    check(tmp_path, monkeypatch, data, [])
    bad = data.replace(b"\tPASS\t", " PASS\t".encode(), 1)
    p = tmp_path / "bad.vcf"
    p.write_bytes(bad)
    with pytest.raises(SystemExit) as e:
        run_cli(None, tmp_path, monkeypatch, args=[], inp=str(p))
    assert "data line 1" in str(e.value)
