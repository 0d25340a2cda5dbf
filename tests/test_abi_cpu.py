"""CPU tests: the C-ABI shared library loads and exports every symbol include/pgwin.h declares; entry points
that need a device fail loudly (no CPU fallback); host-only entry points (planner, .geno parser) work."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from genomics_general_b200 import _lib, engine, geno_io, synth

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    txt = open(os.path.join(REPO, "include", "pgwin.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(pg_[a-z0-9_]+)\s*\(", txt)))


def test_library_exports_every_declared_symbol():
    L = _lib.lib()
    names = declared_symbols()
    assert len(names) >= 20
    for n in names:
        assert hasattr(L, n), "libpgwin.so does not export %s" % n
    assert set(names) == set(_lib.EXPORTS), set(names) ^ set(_lib.EXPORTS)


def test_version_and_error_string():
    L = _lib.lib()
    assert L.pg_version() >= 100
    assert isinstance(L.pg_last_error(), bytes)


def test_no_cpu_fallback_without_device():
    import subprocess
    r = subprocess.run(["nvidia-smi", "-L"], stdout=subprocess.PIPE, stderr=subprocess.PIPE) if os.path.exists("/usr/bin/nvidia-smi") else None
    if r is not None and r.returncode == 0 and b"GPU" in r.stdout:
        pytest.skip("a GPU is present")
    with pytest.raises(_lib.PgError, match="no CUDA device|no CPU fallback"):
        engine.Engine(0)


def test_k1_plan_geometry():
    for S, H in ((10 ** 5, 40), (10 ** 7, 400), (2 * 10 ** 6, 1000), (10 ** 8, 1600), (100, 1), (1000, 3000), (10 ** 6, 16368),
                 (10 ** 6, 16369), (10 ** 6, 20000), (10 ** 6, 28272)):
        p = engine.k1_plan(S, H)
        assert p["ok"], (S, H, p)
        assert p["pitch"] % 16 == 0 and (p["pitch"] // 16) % 2 == 1 and p["pitch"] >= H      # odd 16-byte chunk count
        assert p["lanes_per_site"] in (1, 2, 4, 8, 16, 32)
        assert p["tile_sites"] % 4 == 0                          # positions ride behind the rows in 16-byte pieces
        assert p["tile_sites"] == 32 * p["warps_per_tile"] // p["lanes_per_site"] * p["sites_per_lane"]
        assert 8 % p["warps_per_tile"] == 0 and 1 <= p["ctas"] <= 132
        assert 2 <= p["stages"] <= 8
        assert p["tile_sites"] * p["pitch"] * p["stages"] <= p["smem_bytes"] <= 227 * 1024


def _write(tmp_path, spec, S, fmt="phased", scaffolds=("c1",), ploidy=2):
    g = synth.synth_genotypes(spec, 0, S)
    pos = synth.synth_positions(S)
    sc = [scaffolds[min(i * len(scaffolds) // S, len(scaffolds) - 1)] for i in range(S)]
    p = str(tmp_path / ("x_%s.geno" % fmt))
    synth.write_geno(p, g, pos, sc, spec.sample_names(), ploidy=ploidy, fmt=fmt)
    return p, g, pos, sc


def test_geno_parser_formats(tmp_path):
    spec = synth.SynthSpec(3, 4, miss=0.1, seed=3)
    p, g, pos, sc = _write(tmp_path, spec, 3000, "phased", ("c1", "c2", "c1"))
    gd = geno_io.parse_geno(p, "phased")
    assert np.array_equal(gd.geno, g) and np.array_equal(gd.pos, pos)
    assert gd.scaf_names == ["c1", "c2", "c1"] and np.array_equal(np.bincount(gd.scaf_ids), [1000, 1000, 1000])
    for threads in (1, 3, 16):
        assert np.array_equal(geno_io.parse_geno(p, "phased", threads=threads).geno, g)
    # sample subset in a different order
    sub = spec.sample_names()[::-2]
    cols = np.concatenate([[2 * spec.sample_names().index(s), 2 * spec.sample_names().index(s) + 1] for s in sub])
    assert np.array_equal(geno_io.parse_geno(p, "phased", samples=sub).geno, g[:, cols])
    p2, g2, _, _ = _write(tmp_path, spec, 500, "pairs")
    assert np.array_equal(geno_io.parse_geno(p2, "pairs").geno, g2)
    p3, g3, _, _ = _write(tmp_path, spec, 500, "diplo")
    a = np.sort(geno_io.parse_geno(p3, "diplo").geno.reshape(500, -1, 2), axis=2)
    b = g3.reshape(500, -1, 2).copy()
    b[(b < 0).any(axis=2)] = -1                       # IUPAC codes cannot hold half-missing genotypes
    assert np.array_equal(a, np.sort(b, axis=2))
    spec1 = synth.SynthSpec(2, 5, ploidy=1, miss=0.1)
    p4, g4, _, _ = _write(tmp_path, spec1, 200, "haplo", ploidy=1)
    assert np.array_equal(geno_io.parse_geno(p4, "haplo").geno, g4)


def test_geno_parser_edge_cases(tmp_path):
    txt = ("#CHROM\tPOS\ta\tb\n"
           "c1 5  A/T\tN/N\n"
           "# a comment line\n"
           "\n"
           "c1\t9\tC|C\tG/N\n"
           "c2\t1\tX/T\ta/c")                      # unknown letters and lower case are missing; no trailing newline
    p = tmp_path / "e.geno"
    p.write_text(txt)
    gd = geno_io.parse_geno(str(p), "phased")
    assert gd.geno.tolist() == [[0, 3, -1, -1], [1, 1, 2, -1], [-1, 3, -1, -1]]
    assert gd.pos.tolist() == [5, 9, 1] and gd.scaf_names == ["c1", "c2"]
    # haploid sample under -f phased must have one-allele tokens (genomics.py:1111)
    with pytest.raises(_lib.PgError, match="ploidy"):
        geno_io.parse_geno(str(p), "phased", ploidy={"a": 1, "b": 2})
    with pytest.raises(KeyError):
        geno_io.parse_geno(str(p), "phased", samples=["zz"])
    bad = tmp_path / "bad.geno"
    bad.write_text("#CHROM\tPOS\ta\tb\nc1\tfoo\tA/T\tA/T\n")
    with pytest.raises(_lib.PgError, match="position"):
        geno_io.parse_geno(str(bad), "phased")
    short = tmp_path / "short.geno"
    short.write_text("#CHROM\tPOS\ta\tb\nc1\t3\tA/T\n")
    with pytest.raises(_lib.PgError, match="requested samples"):
        geno_io.parse_geno(str(short), "phased")


def test_geno_parser_gz_and_header_override(tmp_path):
    import gzip
    spec = synth.SynthSpec(2, 3, miss=0.05, seed=9)
    p, g, pos, _ = _write(tmp_path, spec, 300)
    raw = open(p, "rb").read()
    gz = str(tmp_path / "x.geno.gz")
    with gzip.open(gz, "wb") as f:
        f.write(raw)
    assert np.array_equal(geno_io.parse_geno(gz, "phased").geno, g)
    body = raw.split(b"\n", 1)[1]
    gd = geno_io.parse_geno(body, "phased", header="#CHROM POS " + " ".join(spec.sample_names()))
    assert np.array_equal(gd.geno, g) and np.array_equal(gd.pos, pos)
