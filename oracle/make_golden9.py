#!/usr/bin/env python
"""TEST INFRASTRUCTURE — fixtures for parseVCF.py from the UNMODIFIED reference script.

    python oracle/make_golden9.py [/path/to/genomics_general]

Writes seeded VCFs under tests/golden/vcf9/ (main.vcf as main.vcf.gz only; tests/test_vcf_cpu.py unpacks a plain copy for
the cases that read it), runs the reference VCF_processing/parseVCF.py on every case of CASES and commits its output next to
them, gzip-compressed, with tests/golden/cases9.json listing the cases.  The inputs hold multi-allelic sites with
more than ten ALTs, indels, MNPs and '*', GTs such as './.', './1', '0|1/2', '00/1' and '+1/0', haploid and triploid
calls, truncated sample fields, a repeated FORMAT key, QUAL '.', genotype-filter values in every number form Python's
float() takes (and exactly on and one ulp beside the filter bounds), duplicate positions, POS with '+', leading zeros and
'_', two contigs, comment and blank lines after the header, CRLF and lone CR line ends, UTF-8 in INFO, a last line without
a newline, and (in dupnames.vcf) a repeated sample name with data lines shorter than the header."""
import gzip
import json
import math
import os
import random
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "..", "tests", "golden")
DIR = os.path.join(GOLD, "vcf9")

DIPLO = ["d%d" % i for i in range(8)]
HAPLO = ["h0", "h1"]
TRIPLO = ["t0"]
SAMPLES = DIPLO[:4] + HAPLO[:1] + DIPLO[4:] + TRIPLO + HAPLO[1:]
LO, HI = 10.0, 20.0
NUMBERS = ["10", "1_0", "+15", "-0", "15.", ".5", "1e1", "1E+1", "inf", "-Infinity", "NaN", "nan", "4.99999999999999999999",
           "1e400", "12", "19.999", "20", "17", "٣", "1_5.2_5", repr(math.nextafter(LO, -math.inf)),
           repr(math.nextafter(HI, math.inf)), repr(math.nextafter(LO, math.inf)), repr(math.nextafter(HI, -math.inf)), ".",
           "", "12,13", "12,25", "x", "9007199254740993", "1e22", "1e23", "0.1e-5", "123456789012345678901"]


def _alleles(rng, kind):
    b = "ACGT"
    if kind == "mono":
        return rng.choice(b), []
    if kind == "snp":
        ref = rng.choice(b)
        alts = rng.sample([x for x in b if x != ref], rng.randint(1, 3))
        if rng.random() < 0.2:
            alts.append("*")
        return ref, alts
    if kind == "mnp":
        n = rng.randint(2, 3)
        ref = "".join(rng.choice(b) for _ in range(n))
        return ref, ["".join(rng.choice(b) for _ in range(n)) for _ in range(rng.randint(1, 2))]
    if kind == "indel":
        ref = "".join(rng.choice(b) for _ in range(rng.randint(1, 4)))
        return ref, ["".join(rng.choice(b) for _ in range(rng.randint(1, 6))) for _ in range(rng.randint(1, 3))]
    if kind == "many":      # more than ten ALTs: two-digit allele keys
        two = [x + y for x in b for y in b]
        ref = two[0]
        alts = rng.sample(two[1:], rng.randint(11, 15))
        if rng.random() < 0.5:
            alts[-1] = "A"      # one of another length: an INDEL
        return ref, alts
    if kind == "nref":      # REF equal to the default missing string
        return "N", ["A"]
    raise ValueError(kind)


def _gt(rng, nal, ploidy):
    r = rng.random()
    sep = "|" if rng.random() < 0.4 else "/"
    if r < 0.08:
        return sep.join(["."] * ploidy)
    if r < 0.13 and ploidy > 1:
        return sep.join(["."] + [str(rng.randrange(nal))] * (ploidy - 1))
    if r < 0.15:
        return sep.join(["00"] + ["1"] * (ploidy - 1)) if nal > 1 else sep.join(["0"] * ploidy)
    if r < 0.16:
        return sep.join(["+1"] + ["0"] * (ploidy - 1))
    a = [str(rng.randrange(nal)) for _ in range(ploidy)]
    if ploidy == 3 and rng.random() < 0.3:
        return a[0] + "|" + a[1] + "/" + a[2]
    return sep.join(a)


def make_main(rng, n=260):
    head = ["##fileformat=VCFv4.2", "##contig=<ID=chr1,length=100000>", "##contig=<ID=chr2,length=100000>",
            '##INFO=<ID=DP,Number=1,Type=Integer,Description="Depth">',
            "\t".join(["#CHROM", "POS", "ID", "REF", "ALT", "QUAL", "FILTER", "INFO", "FORMAT"] + SAMPLES)]
    body = []
    pos = 100
    ploidy = {s: (1 if s in HAPLO else (3 if s in TRIPLO else 2)) for s in SAMPLES}
    for i in range(n):
        chrom = "chr1" if i < n // 2 else "chr2"
        if i == n // 2:
            pos = 50
        if rng.random() > 0.06:
            pos += rng.randint(1, 40)
        kind = rng.choices(["mono", "snp", "mnp", "indel", "many", "nref"], [1, 6, 1, 2, 1, 0.5])[0]
        ref, alts = _alleles(rng, kind)
        nal = 1 + len(alts)
        qual = rng.choice([".", "30", "12.5", "1e1", "nan", "55", "9"])
        fmt = rng.choice(["GT:AD:DP:GQ"] * 6 + ["GT:DP:GQ:DP", "DP:GT:GQ"])
        keys = fmt.split(":")
        samp = []
        for s in SAMPLES:
            vals = {"GT": _gt(rng, nal, ploidy[s]), "AD": ",".join(str(rng.randint(0, 30)) for _ in range(2)),
                    "DP": rng.choice(NUMBERS) if rng.random() < 0.5 else str(rng.randint(5, 25)), "GQ": str(rng.randint(0, 99))}
            f = [vals[k] if k != "DP" else (vals["DP"] if j < 2 else str(rng.randint(5, 25))) for j, k in enumerate(keys)]
            if fmt.startswith("GT") and rng.random() < 0.08:
                f = f[:rng.randint(1, len(f) - 1)]          # truncated sample field (GT kept)
            samp.append(":".join(f))
        p = str(pos)
        r = rng.random()
        if r < 0.03:
            p = "+00" + p
        elif r < 0.05:
            p = "0" + p
        elif r < 0.06 and len(p) > 1:
            p = p[0] + "_" + p[1:]
        info = "DP=%d" % rng.randint(10, 300) + (";NOTE=café" if rng.random() < 0.03 else "")
        body.append("\t".join([chrom, p, "." if rng.random() < 0.8 else "rs%d" % i, ref, ",".join(alts) or ".", qual, "PASS",
                               info, fmt] + samp))
        if rng.random() < 0.02:
            body.append(rng.choice(["#a comment after the header", "   #indented comment", "", "  \t "]))
    ends = []
    for k in range(len(body)):
        r = rng.random()
        ends.append("\r\n" if r < 0.1 else ("\r" if r < 0.13 else "\n"))
    text = "\n".join(head) + "\n" + "".join(b + e for b, e in zip(body, ends))
    return text[:-len(ends[-1])]            # the last line without a newline


def make_dupnames():
    """sample name 'a' twice (its last column counts, unless a line is too short for it); 'b' once"""
    head = "##fileformat=VCFv4.2\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\ta\tb\ta\n"
    rows = ["chr1\t1\t.\tA\tC\t.\tPASS\t.\tGT:DP\t0/1:5\t1/1:6\t0/0:7",
            "chr1\t2\t.\tA\tC\t.\tPASS\t.\tGT:DP\t1/1:5\t0/1:6",
            "chr1\t3\t.\tA\tC,G\t.\tPASS\t.\tGT\t2|1\t0|0\t1|1\textra",
            "chr1\t4\t.\tA\tG\t.\tPASS\t.\tGT:DP\t0/1\t./.:3"]
    return head + "\n".join(rows) + "\n"


SHUFFLED = "d5,d0,d7,d3,d1,d6,d2,d4"

CASES = [
    ("diploid_shuffled", "main.vcf", ["-s", SHUFFLED], False),
    ("ploidyfile_all", "main.vcf", ["--ploidyFile", "ploidy.txt"], False),
    ("p2m_all", "main.vcf", ["--ploidyMismatchToMissing"], False),
    ("gtf_dp_bounds", "main.vcf", ["-s", SHUFFLED, "--gtf", "flag=DP", "min=%r" % LO, "max=%r" % HI], False),
    ("gtf_many", "main.vcf", ["--ploidyFile", "ploidy.txt", "--gtf", "flag=GQ", "min=20", "siteTypes=SNP", "gtTypes=Het",
                              "--gtf", "flag=DP", "min=5", "max=inf", "samples=d1,d2,t0,h1", "--gtf", "flag=AD", "max=25",
                              "gtTypes=HomAlt,Missing", "--gtf", "min=3", "siteTypes=INDEL"], False),
    ("gtf_nan_bounds", "main.vcf", ["-s", SHUFFLED, "--gtf", "flag=DP", "min=-inf", "max=1e400"], False),
    ("skipindels", "main.vcf", ["-s", SHUFFLED, "--skipIndels"], False),
    ("skipindels_keeppartial", "main.vcf", ["--ploidyFile", "ploidy.txt", "--skipIndels", "--keepPartial"], False),
    ("missing_long_comma", "main.vcf", ["-s", SHUFFLED, "--missing", "NA", "--outSep", ",", "--addRefTrack"], False),
    ("missing_quirk_default_N", "main.vcf", ["-s", "d0,d1,d2", "--skipIndels", "--addRefTrack"], False),
    ("field_dp", "main.vcf", ["--field", "DP"], False),
    ("field_phase_missing", "main.vcf", ["--field", "phase", "--missing", "?"], False),
    ("field_ad_noheader", "main.vcf", ["-s", "t0,h0,d3", "--field", "AD", "--noHeader"], False),
    ("minqual_maxreflen", "main.vcf", ["-s", SHUFFLED, "--minQual", "20", "--maxREFlen", "2"], False),
    ("minqual_zero_falsy", "main.vcf", ["-s", SHUFFLED, "--minQual", "0", "--maxREFlen", "0"], False),
    ("dups_include", "main.vcf", ["-s", SHUFFLED, "--excludeDuplicates", "--include", "chr2"], False),
    ("exclude_file_gz", "main.vcf.gz", ["-s", SHUFFLED, "--excludeFile", "contigs.txt"], True),
    ("dupnames", "dupnames.vcf", [], False),
    ("dupnames_field", "dupnames.vcf", ["-s", "b,a,a", "--field", "DP"], False),
]


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
    script = os.path.join(ref, "VCF_processing", "parseVCF.py")
    os.makedirs(DIR, exist_ok=True)
    rng = random.Random(9)
    main_vcf = make_main(rng).encode()
    plain = os.path.join(DIR, "main.vcf")                  # the plain copy is only there while the reference runs
    with open(plain, "wb") as f:
        f.write(main_vcf)
    with open(os.path.join(DIR, "main.vcf.gz"), "wb") as f:
        f.write(gzip.compress(main_vcf, mtime=0))
    with open(os.path.join(DIR, "dupnames.vcf"), "wb") as f:
        f.write(make_dupnames().encode())
    with open(os.path.join(DIR, "ploidy.txt"), "wt") as f:
        f.write("h0 1\nh1 1\nt0 3\n")
    with open(os.path.join(DIR, "contigs.txt"), "wt") as f:
        f.write("chr1\n")
    cases = []
    try:
        for name, inp, args, gz in CASES:
            out = os.path.join(DIR, name + (".tmp.gz" if gz else ".tmp"))
            argv = [sys.executable, script, "-i", inp, "-o", out] + args
            r = subprocess.run(argv, cwd=DIR, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
            assert r.returncode == 0, (name, r.stderr.decode()[-2000:])
            data = gzip.open(out).read() if gz else open(out, "rb").read()
            os.remove(out)
            with open(os.path.join(DIR, name + ".out.gz"), "wb") as f:      # stored compressed, without a timestamp
                f.write(gzip.compress(data, mtime=0))
            cases.append(dict(name=name, input=inp, args=args, gz=gz, expected=name + ".out.gz"))
    finally:
        os.remove(plain)
    with open(os.path.join(GOLD, "cases9.json"), "wt") as f:
        f.write("[\n" + ",\n".join(json.dumps(c) for c in cases) + "\n]\n")
    print("wrote %d cases under %s" % (len(cases), DIR))


if __name__ == "__main__":
    main()
