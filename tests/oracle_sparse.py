"""TEST INFRASTRUCTURE — the oracle-backed engines with Engine.sfs_sparse / sfs_tables_sparse, built from the oracle's
per-site target counts with np.unique over row-major cell keys (never a dense array).  Never imported by the product.
As a script it is one `--devices N` rank of sfs.py on the CPU (what tests/_mgpu_cpu_worker.py is for the other command
lines): python oracle_sparse.py <argv ...>"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from oracle import dense_oracle as do  # noqa: E402
from oracle_engine import OracleEngine  # noqa: E402
from oracle_engine_mg import OracleEngineMG  # noqa: E402


class SparseMixin:
    @staticmethod
    def _sparse(tc, used, groups, dims, site_mask):
        from genomics_general_b200.engine import PgError, sfs_shapes, sfs_unravel
        if site_mask is not None:
            used = used & np.asarray(site_mask, dtype=bool)
        sites = np.flatnonzero(used)
        out = []
        for g, (grp, shape) in enumerate(zip(groups, sfs_shapes(groups, dims)[0])):
            if int(np.prod(shape, dtype=object)) > np.iinfo(np.int64).max:
                raise PgError("sfs: spectrum %d has more than 2^63 - 1 cells" % g)
            key = np.zeros(len(sites), dtype=np.int64)
            for x, d in zip(grp, shape):
                key = key * d + np.asarray(tc[sites, x], dtype=np.int64)
            cells, at, count = np.unique(key, return_index=True, return_counts=True)
            out.append((sfs_unravel(cells, shape), count.astype(np.int64), sites[at].astype(np.int64)))
        return out, int(used.sum())

    def sfs_sparse(self, n_in, groups, pop_sizes, outgroup=-1, site_mask=None):
        tc, used = do.sfs_target_counts(self.g, self.hap_pop, n_in, outgroup)
        return self._sparse(tc, used, groups, [int(n) + 1 for n in pop_sizes], site_mask)

    def sfs_tables_sparse(self, kind, table, n_in, groups, outgroup=-1, site_mask=None):
        from genomics_general_b200.engine import sfs_table_dims
        table = np.asarray(table)
        if kind == "base":
            tc, used = do.sfs_target_counts_from_counts(table, n_in, outgroup)
        else:
            tc, used = table, np.ones(len(table), dtype=bool)
        return self._sparse(tc, used, groups, sfs_table_dims(kind, table)[1], site_mask)


class SparseOracleEngine(SparseMixin, OracleEngine):
    pass


class SparseOracleEngineMG(SparseMixin, OracleEngineMG):
    pass


if __name__ == "__main__":
    from genomics_general_b200.cli import sfs as sfs_cli
    sfs_cli.Engine = SparseOracleEngineMG
    sfs_cli.main(sys.argv[1:])
