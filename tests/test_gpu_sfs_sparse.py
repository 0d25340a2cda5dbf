"""Sparse spectra on the H100 (pg_sfs_sparse / pg_sfs_tables_sparse): integer for integer the dense path's non-empty cells,
counts and first sites wherever the dense path runs; the command line above the dense limit against the unmodified
reference (tests/golden/cases5.json); quartets above the limit at scale against a vectorised numpy oracle; refusals."""
import ctypes as C
import itertools
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import GOLDEN

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle"))
import make_golden5 as mg5  # noqa: E402

C5 = json.load(open(os.path.join(GOLDEN, "cases5.json")))


def _engine(g, hp):
    from genomics_general_b200.engine import Engine
    eng = Engine(0)
    eng.upload(g)
    eng.set_pops(hp, 5)
    return eng


def _assert_same(sparse, dense):
    """sparse (coords, count, first) per spectrum == the dense histograms' non-empty cells in row-major order"""
    hists, firsts, n1 = dense
    assert sparse[1] == n1
    for (c, n, f), h, f1 in zip(sparse[0], hists, firsts, strict=True):
        nz = np.flatnonzero(h.reshape(-1))
        assert c.dtype == n.dtype == f.dtype == np.int64
        assert np.array_equal(c, np.argwhere(h > 0).reshape(c.shape))
        assert np.array_equal(n, h.reshape(-1)[nz]) and np.array_equal(f, f1.reshape(-1)[nz])


def _genotypes(S, seed=3):
    """populations of 5, 7, 6, 4 diploid samples + an outgroup of 3: biallelic sites, 1 % missing genotypes, third alleles"""
    rng = np.random.default_rng(seed)
    n_haps = [10, 14, 12, 8, 6]
    pop_of = np.repeat(np.arange(5), n_haps)
    anc = rng.integers(0, 4, S)
    alt = (anc + 1 + rng.integers(0, 3, S)) % 4
    freq = np.where((rng.random(S) < 0.7)[:, None], rng.random((S, 5)), 0.0)
    g = np.where(rng.random((S, sum(n_haps))) < freq[:, pop_of], alt[:, None], anc[:, None]).astype(np.int8)
    g[rng.random(g.shape) < 0.01] = -1
    g[rng.random(S) < 0.02, 0] = 3
    return g, pop_of.astype(np.int32), n_haps


GROUPS = {"1d": [(0,)], "2d": [(1, 2)], "3d": [(0, 1, 3)], "4d": [(0, 1, 2, 3)],
          "several": [(0,), (2,), (0, 1), (1, 2, 3), (3, 0, 2, 1)]}


@pytest.mark.parametrize("shape", list(GROUPS))
@pytest.mark.parametrize("polarized", [False, True])
@pytest.mark.parametrize("masked", [False, True])
def test_genotypes_sparse_equals_dense(shape, polarized, masked):
    g, hp, sizes = _genotypes(20000)
    kw = dict(outgroup=4 if polarized else -1,
              site_mask=(np.random.default_rng(1).random(len(g)) < 0.7).astype(np.uint8) if masked else None)
    with _engine(g, hp) as eng:
        _assert_same(eng.sfs_sparse(4, GROUPS[shape], sizes, **kw), eng.sfs(4, GROUPS[shape], sizes, **kw))


@pytest.mark.parametrize("slab", ["1", "37", "4096"])
def test_slab_seams(slab, monkeypatch):
    """slabs of `slab` sites (PG_SFS_SPARSE_SLAB): runs merged across slabs; genotypes and both table kinds"""
    g, hp, sizes = _genotypes(700 if slab == "1" else 9000, seed=9)
    groups = [(0,), (0, 1), (1, 2, 3), (0, 1, 2, 3)]
    mask = (np.random.default_rng(2).random(len(g)) < 0.8).astype(np.uint8)
    with _engine(g, hp) as eng:
        dense = eng.sfs(4, groups, sizes, outgroup=4, site_mask=mask)
        counts = eng.site_counts()
        tables = [("base", counts, 4), ("base", counts, -1), ("target", counts[:, :4].sum(axis=2) // 3, -1)]
        dense_t = [eng.sfs_tables(k, t, 4, groups, outgroup=og, site_mask=mask) for k, t, og in tables]
        monkeypatch.setenv("PG_SFS_SPARSE_SLAB", slab)
        _assert_same(eng.sfs_sparse(4, groups, sizes, outgroup=4, site_mask=mask), dense)
        for (k, t, og), d in zip(tables, dense_t):
            _assert_same(eng.sfs_tables_sparse(k, t, 4, groups, outgroup=og, site_mask=mask), d)


@pytest.mark.parametrize("case", ["no_sites", "all_masked", "none_counted", "base", "target"])
def test_tables_and_empty_inputs(case):
    g, hp, sizes = _genotypes(6000, seed=4)
    groups = [(0,), (1, 3), (0, 2, 3)]
    with _engine(g, hp) as eng:
        counts = eng.site_counts()
        if case in ("all_masked", "none_counted"):
            kw = dict(site_mask=np.zeros(len(g), np.uint8)) if case == "all_masked" else {}
            if case == "none_counted":                       # a missing in-group genotype at every site
                g[:, 0] = -1
                eng.upload(g)
                eng.set_pops(hp, 5)
            dense, sparse = eng.sfs(4, groups, sizes, **kw), eng.sfs_sparse(4, groups, sizes, **kw)
        else:
            kind, og = ("target", -1) if case == "target" else ("base", 4)
            t = counts[:, :4, 1].astype(np.int32) if kind == "target" else counts[:0 if case == "no_sites" else None]
            dense, sparse = eng.sfs_tables(kind, t, 4, groups, outgroup=og), eng.sfs_tables_sparse(kind, t, 4, groups, outgroup=og)
    assert (sparse[1] == 0) == (case in ("no_sites", "all_masked", "none_counted"))
    _assert_same(sparse, dense)


def test_fetch_once_and_refusals():
    """fetch: once, with the right total; a spectrum of 2^63 cells or more is refused before any launch, naming it;
    Engine.sfs / sfs_tables above the dense limit still raise"""
    from genomics_general_b200 import _lib
    from genomics_general_b200.engine import PgError
    g, hp, sizes = _genotypes(3000)
    with _engine(g, hp) as eng:
        L, p = _lib.lib(), lambda a: a.ctypes.data_as(C.c_void_p)
        nnz, n = np.zeros(1, np.int64), C.c_int64(0)
        _lib.check(L.pg_sfs_sparse(eng._ctx, 4, -1, 1, p(np.array([0, 2], np.int32)), p(np.array([0, 1], np.int32)), None,
                                   p(nnz), C.byref(n)))
        out = [np.empty(int(nnz[0]), np.int64) for _ in range(3)]
        assert L.pg_sfs_sparse_fetch(eng._ctx, int(nnz[0]) + 1, *map(p, out)) != 0
        assert L.pg_sfs_sparse_fetch(eng._ctx, int(nnz[0]), *map(p, out)) == 0 and out[1].sum() == n.value
        assert L.pg_sfs_sparse_fetch(eng._ctx, int(nnz[0]), *map(p, out)) != 0
        t = np.zeros((10, 3), np.int32)
        t[0] = 2 ** 30
        before = eng.launch_count()
        with pytest.raises(PgError, match="spectrum 1 has more than 2\\^63"):
            eng.sfs_tables_sparse("target", t, 3, [(0, 1), (0, 1, 2)])
        assert eng.launch_count() == before
        with pytest.raises(PgError, match="dense spectra are limited"):
            eng.sfs(4, [(0, 1, 2, 3)], [200] * 4)
        t = np.zeros((4, 3), np.int32)
        t[0] = 20000
        with pytest.raises(PgError, match="dense spectra are limited"):
            eng.sfs_tables("target", t, 3, [(0, 1)])
        (c, m, f), = eng.sfs_tables_sparse("target", t, 3, [(0, 1)])[0]
        assert c.tolist() == [[0, 0], [20000, 20000]] and m.tolist() == [3, 1] and f.tolist() == [1, 0]


@pytest.fixture(scope="module")
def inputs5(tmp_path_factory):
    assert json.loads(json.dumps(mg5.CFGS)) == C5["cfgs"]
    return mg5.inputs(str(tmp_path_factory.mktemp("golden5")))


@pytest.mark.parametrize("key", mg5.KEYS)
def test_cases5_command_line(inputs5, key, capsys):
    """the real command line above the dense limit: byte for byte the reference's output (its sha256)"""
    from genomics_general_b200.cli import sfs as sfs_cli
    capsys.readouterr()
    sfs_cli.main(["--pipe"] + mg5.argv(inputs5, key))
    assert mg5.digest(capsys.readouterr().out) == C5[key]


def test_quartets_above_the_limit_at_scale():
    """2 M sites, 6 populations x 36 diploid samples, singles + 15 quartets (4.3e8 cells): a vectorised numpy oracle"""
    from genomics_general_b200 import synth
    from genomics_general_b200.engine import Engine, sfs_unravel
    spec, S, P = synth.SynthSpec(6, 36, miss=0.002, seed=17), 2_000_000, 6
    groups = [(x,) for x in range(P)] + list(itertools.combinations(range(P), 4))
    hp = spec.hap_pop()
    cnt = np.zeros((S, P, 4), np.int64)
    with Engine(0) as eng:
        eng.synth_fill(spec, S)
        eng.set_pops(hp, P)
        sp, n = eng.sfs_sparse(P, groups, [72] * P)
        for lo in range(0, S, 250_000):                      # the oracle counts the genotypes itself
            g, _ = eng.download(lo, min(250_000, S - lo), want_pos=False)
            for x, a in itertools.product(range(P), range(4)):
                cnt[lo:lo + len(g), x, a] = (g[:, hp == x] == a).sum(axis=1)
    tot = cnt.sum(axis=1)
    n_all = (tot > 0).sum(axis=1)
    sites = np.flatnonzero((cnt.sum(axis=2) == 72).all(axis=1) & (n_all >= 1) & (n_all <= 2))
    target = np.argsort(tot, axis=1, kind="stable")[:, -2]              # the lower allele on an exact tie, as the device
    tc = np.take_along_axis(cnt, target[:, None, None].repeat(P, axis=1), axis=2)[:, :, 0]
    assert n == len(sites) > S // 4
    for (c, m, f), grp in zip(sp, groups, strict=True):
        key = np.zeros(len(sites), np.int64)
        for x in grp:
            key = key * 73 + tc[sites, x]
        cells, at, count = np.unique(key, return_index=True, return_counts=True)
        assert np.array_equal(c, sfs_unravel(cells, (73,) * len(grp))) and np.array_equal(m, count)
        assert np.array_equal(f, sites[at])


def test_devices_two_above_the_limit(inputs5):
    """sfs --devices 2 on the quartet case (--regions, --exclude) == the reference's single-device output"""
    from genomics_general_b200 import _lib
    n = C.c_int(0)
    _lib.lib().pg_device_count(C.byref(n))
    if n.value < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "genomics_general_b200.cli.sfs", "--pipe", "--devices", "2"]
                       + mg5.argv(inputs5, "geno6_quartets"), env=dict(os.environ, PYTHONPATH=os.path.dirname(HERE)),
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert mg5.digest(r.stdout) == C5["geno6_quartets"]
