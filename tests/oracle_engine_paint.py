"""TEST INFRASTRUCTURE — Engine.distpaint backed by oracle/paint_oracle.py, so that the CPU tests run distPaint's command
line (flags, populations, row order, window rows) without a GPU.  Never imported by the product."""
import numpy as np

from oracle import paint_oracle as po
from oracle_engine import OracleEngine


class PaintOracleEngine(OracleEngine):
    def set_strict_ingest(self, on=True):
        self.strict = int(on)

    def distpaint(self, query_hap, ref_off, ref_hap, min_sites, delta=False, threshold=0.05, noresult=-1, with_stats=False):
        assert min_sites >= 1
        pops = [list(ref_hap[ref_off[p]:ref_off[p + 1]]) for p in range(len(ref_off) - 1)]
        assert not delta or len(pops) >= 2
        nq, P = len(query_hap), len(pops)
        assign = np.full((self.W, nq), noresult, dtype=np.int32)
        means = np.full((self.W, nq, P), np.nan)
        pvals = np.full((self.W, nq, P), np.nan)
        for w in range(self.W):
            if self.hi[w] > self.lo[w]:
                assign[w], means[w], pvals[w] = po.paint_window(self._win(w), list(query_hap), pops, min_sites,
                                                                threshold if delta else None, threshold, noresult)
        out = dict(assign=assign)
        if with_stats:
            out.update(means=means, pvals=pvals)
        return out
