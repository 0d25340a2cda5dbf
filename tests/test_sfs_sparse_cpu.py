"""sfs.py above the dense histograms' limit on the CPU: the sparse route of the command line with the oracle-backed engine
against the unmodified reference (tests/golden/cases5.json, oracle/make_golden5.py), the split of ordered_chains, and the
rank merge of `--devices N`."""
import itertools
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import GOLDEN
from oracle_engine import OracleEngine
from oracle_sparse import SparseOracleEngine

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle"))
import make_golden5 as mg5  # noqa: E402   (input generators only; the reference is not imported)

C5 = json.load(open(os.path.join(GOLDEN, "cases5.json")))


@pytest.fixture(scope="module")
def inputs5(tmp_path_factory):
    assert json.loads(json.dumps(mg5.CFGS)) == C5["cfgs"]
    return mg5.inputs(str(tmp_path_factory.mktemp("golden5")))


def _cli(monkeypatch, engine):
    from genomics_general_b200.cli import _common, sfs as sfs_cli
    monkeypatch.setattr(sfs_cli, "Engine", engine)
    real = _common.load_geno
    monkeypatch.setattr(_common, "load_geno", lambda args, samples, pl, header=None, engine=None: real(args, samples, pl, header, None))
    return sfs_cli


class SparseOnly(SparseOracleEngine):
    def sfs(self, *a, **k):
        raise AssertionError("dense path above the limit")

    sfs_tables = sfs


@pytest.mark.parametrize("key", mg5.KEYS)
def test_cases5_through_the_command_line(inputs5, key, monkeypatch, capsys):
    """byte for byte the reference's --pipe output (its sha256), without reaching a dense entry point"""
    sfs_cli = _cli(monkeypatch, SparseOnly)
    capsys.readouterr()
    sfs_cli.main(["--pipe"] + mg5.argv(inputs5, key))
    assert mg5.digest(capsys.readouterr().out) == C5[key]


def test_dense_requests_keep_the_dense_path(inputs5, monkeypatch, capsys):
    """the rule: sparse exactly where the summed cells of a request exceed SFS_MAX_CELLS"""
    from genomics_general_b200.engine import SFS_MAX_CELLS
    sfs_cli = _cli(monkeypatch, OracleEngine)                   # no sparse methods: a sparse call would fail
    assert not sfs_cli.use_sparse([(0,)], [SFS_MAX_CELLS]) and sfs_cli.use_sparse([(0,)], [SFS_MAX_CELLS + 1])
    assert not sfs_cli.use_sparse([(0, 1)], [2 ** 14, 2 ** 14]) and sfs_cli.use_sparse([(0,), (0, 1)], [2 ** 14, 2 ** 14])
    g4 = inputs5["geno4"]
    capsys.readouterr()
    sfs_cli.main(["--pipe", "-i", g4["geno"], "--popsFile", g4["pops"], "--inputType", "genotypes", "--FSpops", "A", "B", "C"])
    assert capsys.readouterr().out.count("\n") > 100


def _chains_by_dicts(cell, used, shape):
    """the reference's nested dicts (SparseFS.add + asChains, sfs.py:111-122) over the sites in order; used[i] = the sites
    of interval i, one count per interval"""
    rows = {}
    for s in range(len(cell)):
        if any(u[s] for u in used):
            key = tuple(int(v) for v in np.unravel_index(cell[s], shape))
            rows.setdefault(key, [0] * len(used))
            for i, u in enumerate(used):
                rows[key][i] += int(u[s])
    nested = {}
    for key, c in rows.items():                                  # insertion order = first appearance at every level
        d = nested
        for k in key[:-1]:
            d = d.setdefault(k, {})
        d[key[-1]] = c
    out = []

    def walk(d, prefix):
        for k, v in d.items():
            walk(v, prefix + [k]) if isinstance(v, dict) else out.append(prefix + [k] + v)
    walk(nested, [])
    return out


@pytest.mark.parametrize("shape,n_int", [((9,), 1), ((5, 7), 1), ((4, 3, 6), 1), ((3, 4, 2, 5), 1), ((6, 5), 3), ((3, 4, 5), 4)])
def test_split_ordered_chains(shape, n_int):
    """dense -> entries -> order (ordered_chains) and the intervals' sparse entries in any order (sparse_rows) both give the
    reference's rows"""
    from genomics_general_b200.cli import sfs as sfs_cli
    rng = np.random.default_rng(len(shape) * 10 + n_int)
    ncell = int(np.prod(shape))
    for n_sites in (0, 1, 40, 400):
        cell = rng.integers(0, ncell, n_sites)
        used = [rng.random(n_sites) < 0.6 for _ in range(n_int)]
        hists, firsts, sparse = [], [], []
        for u in used:
            s = np.flatnonzero(u)
            h = np.bincount(cell[s], minlength=ncell)
            f = np.full(ncell, -1)
            f[cell[s][::-1]] = s[::-1]
            nz = np.flatnonzero(h)
            p = rng.permutation(len(nz))
            hists.append(h.reshape(shape))
            firsts.append(f.reshape(shape))
            sparse.append(([(np.argwhere(h.reshape(shape) > 0)[p], h[nz][p], f[nz][p])], 0))
        want = _chains_by_dicts(cell, used, shape)
        assert sfs_cli.ordered_chains(hists if n_int > 1 else hists[0], firsts if n_int > 1 else firsts[0]) == want
        assert sfs_cli.sparse_rows(sparse, 1)[0] == want


@pytest.mark.parametrize("world", [2, 3])
def test_devices_sparse_rank_merge(inputs5, world, tmp_path):
    """the quartet case (--regions, --exclude) on `world` CPU ranks: each rank's cells with file-wide first sites, merged
    on rank 0, give the reference's output"""
    rdv, pref = str(tmp_path / "rdv"), str(tmp_path / "r.")
    os.makedirs(rdv)
    procs = [subprocess.Popen([sys.executable, os.path.join(HERE, "oracle_sparse.py")] + mg5.argv(inputs5, "geno6_quartets")
                              + ["--pref", pref], env=dict(os.environ, PG_MG_RANK=str(r), PG_MG_WORLD=str(world), PG_MG_DIR=rdv,
                                                            OMP_NUM_THREADS="1"),
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(world)]
    for p in procs:
        out, _ = p.communicate(timeout=600)
        assert p.returncode == 0, out[-3000:]
    names = inputs5["geno6"]["names"]
    groups = [[pn] for pn in names] + [list(c) for c in itertools.combinations(names, 4)]
    assert mg5.digest("".join(open(pref + "_".join(g) + ".sfs").read() for g in groups)) == C5["geno6_quartets"]
