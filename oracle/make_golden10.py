#!/usr/bin/env python
"""TEST INFRASTRUCTURE — fixtures for genoToSeq.py from the UNMODIFIED reference script.

    python oracle/make_golden10.py [/path/to/genomics_general]

Writes seeded .geno inputs under tests/golden/seq10/, runs the reference genoToSeq.py on every case of CASES in a scratch
directory and commits every file it writes (and its stdout), gzip-compressed, next to them, with tests/golden/cases10.json
listing the cases.  Cases where the reference fails record that it failed and the exception it raised.

The inputs hold phased diploid tokens with lowercase letters, '-', N and IUPAC codes, a comment line between data lines, a
contig longer than 1e7 bp (three -M contigs windows), samples of ploidy 1, 2 and 3, unphased tokens of unequal width in one
file, CRLF line ends, and a scaffold whose first site lies beyond the first coordinate window."""
import gzip
import json
import os
import random
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "..", "tests", "golden")
DIR = os.path.join(GOLD, "seq10")

BASES = "ACGTACGTACGTNacgtn-RYKM"


def _phased(rng, ploidy):
    return "|".join(rng.choice(BASES) for _ in range(ploidy))


def write_inputs():
    rng = random.Random(1010)
    names = ["s%d" % i for i in range(6)]
    lines = ["#CHROM\tPOS\t" + "\t".join(names)]
    # c1: dense, c2: longer than 2e7 bp (one site every 40 kb), c3: short
    for scaf, positions in (("c1", range(7, 3007, 10)), ("c2", range(1000, 25000000, 40000)), ("c3", range(5, 5005, 100))):
        for k, p in enumerate(positions):
            if scaf == "c1" and k == 40:
                lines.append("# a comment line between data lines")
            lines.append("\t".join([scaf, str(p)] + [_phased(rng, 2) for _ in names]))
    main = "\n".join(lines) + "\n"
    with open(os.path.join(DIR, "main.geno"), "w") as f:
        f.write(main)
    with gzip.GzipFile(os.path.join(DIR, "main.geno.gz"), "wb", mtime=0) as f:
        f.write(main.encode())
    # ploidies 1, 2, 3 (one sample each), and files of uniform ploidy 1 and 3
    for name, pls in (("mixed", [1, 2, 3, 2]), ("hap", [1, 1, 1]), ("trip", [3, 3])):
        sn = ["p%d" % i for i in range(len(pls))]
        ls = ["#CHROM\tPOS\t" + "\t".join(sn)]
        for k in range(120):
            ls.append("\t".join(["chrA" if k < 70 else "chrB", str(11 + 13 * k)] + [_phased(rng, p) for p in pls]))
        with open(os.path.join(DIR, name + ".geno"), "w") as f:
            f.write("\n".join(ls) + "\n")
    # unphased tokens of unequal width per column, CRLF line ends
    ls = ["#CHROM POS a b c"]
    for k in range(40):
        ls.append(" ".join(["u1", str(3 + 7 * k), rng.choice("ACGTNnRY-"), "".join(rng.choice("ACGTNk") for _ in range(2)),
                            _phased(rng, 2)]))
    with open(os.path.join(DIR, "crlf.geno"), "wb") as f:
        f.write(("\r\n".join(ls) + "\r\n").encode())
    # the first site of the second scaffold lies beyond the first 1000 bp window
    ls = ["#CHROM\tPOS\ts0\ts1", "k1\t10\tA|C\tG|T", "k1\t900\tA|A\tG|G", "k2\t5000\tC|C\tT|T", "k2\t5100\tA|C\tN|N"]
    with open(os.path.join(DIR, "gap.geno"), "w") as f:
        f.write("\n".join(ls) + "\n")
    # a data line with one genotype column fewer
    ls = ["#CHROM\tPOS\ts0\ts1", "k1\t10\tA|C\tG|T", "k1\t20\tA|A"]
    with open(os.path.join(DIR, "short.geno"), "w") as f:
        f.write("\n".join(ls) + "\n")


SITES = ["--windType", "sites", "--windSize", "50", "--overlap", "10", "--maxDist", "100000000", "--minSites", "20"]
CASES = [
    ("cat_fasta", "main.geno", []),
    ("cat_phylip", "main.geno", ["-f", "phylip"]),
    ("cat_stdout", "main.geno", ["-f", "phylip"], "stdout"),
    ("cat_split", "main.geno", ["--splitPhased"]),
    ("cat_split_phylip_ntogap", "main.geno", ["--splitPhased", "-f", "phylip", "--NtoGap"]),
    ("cat_samples_reorder", "main.geno", ["-S", "s4,s1,s2"]),
    ("cat_samples_split", "main.geno", ["-S", "s3,s0", "--splitPhased", "--NtoGap"]),
    ("cat_gz_in_gz_out", "main.geno.gz", [], "out.fa.gz"),
    ("cat_gzip_flag", "main.geno", ["--gzip", "-f", "phylip"], "out.phy"),
    ("ploidy1_split", "hap.geno", ["--splitPhased", "--ploidy", "1"]),
    ("ploidy3_split", "trip.geno", ["--splitPhased", "--ploidy", "3", "-f", "phylip"]),
    ("ploidy_list_split", "mixed.geno", ["--splitPhased", "--ploidy", "1", "2", "3", "2"]),
    ("mixed_widths_cat", "mixed.geno", ["-f", "phylip"]),
    ("crlf_unphased", "crlf.geno", ["--NtoGap"]),
    ("crlf_phylip", "crlf.geno", ["-f", "phylip"]),
    ("contigs", "main.geno", ["-M", "contigs"]),
    ("contigs_phylip_split", "main.geno", ["-M", "contigs", "-f", "phylip", "--splitPhased"]),
    ("contigs_separate", "main.geno", ["-M", "contigs", "--separateFiles"], "aln"),
    ("contigs_separate_gzip", "main.geno", ["-M", "contigs", "--separateFiles", "--gzip", "-f", "phylip"], "aln"),
    ("windows_coord", "main.geno", ["-M", "windows", "--windType", "coordinate", "--windSize", "100000", "--stepSize",
                                    "50000"]),
    ("windows_coord_phylip", "main.geno", ["-M", "windows", "--windType", "coordinate", "--windSize", "200000",
                                           "--stepSize", "200000", "-f", "phylip", "--splitPhased"]),
    ("windows_sites", "main.geno", ["-M", "windows"] + SITES),
    ("windows_sites_maxdist", "main.geno", ["-M", "windows", "--windType", "sites", "--windSize", "20", "--overlap", "5",
                                            "--maxDist", "100", "--minSites", "3"]),
    ("windows_sites_separate", "main.geno", ["-M", "windows", "--separateFiles", "-f", "phylip"] + SITES, "win"),
    ("windows_sites_separate_gzip", "mixed.geno", ["-M", "windows", "--separateFiles", "--gzip", "--windType", "sites",
                                                   "--windSize", "30", "--overlap", "0", "--maxDist", "1000000"], "w"),
    # the reference fails on these
    ("fail_seqname_contig", "main.geno", ["-M", "contigs", "--seqNameFormat", "contig"]),
    ("fail_seqname_sample_contig", "main.geno", ["-M", "contigs", "--seqNameFormat", "sample_contig"]),
    ("fail_seqname_scp", "main.geno", ["-M", "windows", "--seqNameFormat", "sample_contig_position"] + SITES),
    ("fail_samples_contigs", "main.geno", ["-M", "contigs", "-S", "s1"]),
    ("fail_sites_no_maxdist", "main.geno", ["-M", "windows", "--windType", "sites", "--windSize", "50", "--overlap", "5"]),
    ("fail_sites_no_overlap", "main.geno", ["-M", "windows", "--windType", "sites", "--windSize", "50", "--maxDist",
                                            "100000"]),
    ("fail_empty_coord_window", "gap.geno", ["-M", "windows", "--windType", "coordinate", "--windSize", "1000",
                                             "--stepSize", "1000"]),
    ("fail_separate_cat", "main.geno", ["--separateFiles"], "x"),
    ("fail_short_line", "short.geno", []),
]


def run_case(ref, case):
    name, inp, args = case[:3]
    dest = case[3] if len(case) > 3 else "out"
    work = tempfile.mkdtemp()
    try:
        cmd = [sys.executable, os.path.join(ref, "genoToSeq.py"), "-g", os.path.join(DIR, inp)] + list(args)
        if dest != "stdout":
            cmd += ["-s", os.path.join(work, dest)]
        r = subprocess.run(cmd, cwd=work, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=dict(os.environ, PYTHONPATH=ref))
        entry = dict(name=name, input=inp, args=list(args), dest=dest)
        if r.returncode != 0:
            entry["fails"] = r.stderr.decode().strip().splitlines()[-1]
            return entry
        files = {}
        if dest == "stdout":
            files["stdout"] = r.stdout
        for fn in sorted(os.listdir(work)):
            data = open(os.path.join(work, fn), "rb").read()
            files[fn] = gzip.decompress(data) if fn.endswith(".gz") else data
        entry["outputs"] = {}
        for k, (fn, data) in enumerate(sorted(files.items())):
            fix = "%s.%d.gz" % (name, k)
            with gzip.GzipFile(os.path.join(DIR, fix), "wb", mtime=0) as g:
                g.write(data)
            entry["outputs"][fn] = fix
        return entry
    finally:
        shutil.rmtree(work)


def main(ref):
    if os.path.isdir(DIR):
        shutil.rmtree(DIR)
    os.makedirs(DIR)
    write_inputs()
    cases = [run_case(ref, c) for c in CASES]
    with open(os.path.join(GOLD, "cases10.json"), "w") as f:
        json.dump(cases, f, indent=1)
    for c in cases:
        print(c["name"], "FAILS " + c["fails"] if "fails" in c else sorted(c["outputs"]))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
