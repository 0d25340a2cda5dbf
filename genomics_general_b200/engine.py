"""Thin object wrapper over the C-ABI: one ``Engine`` = one ``pg_ctx`` = one GPU.

All numerics run in libpgwin.so (hand-written CUDA, sm_90a).  numpy is used only for host
buffers.  Nothing here computes statistics on the CPU.
"""
from __future__ import annotations

import ctypes as C
import itertools

import numpy as np

from . import _lib
from ._lib import PgError, check


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _addr(buf):
    """the address of a numpy array or of any other writable buffer (the *_emit slabs)"""
    return C.c_void_p(buf.ctypes.data if hasattr(buf, "ctypes") else C.addressof(C.c_char.from_buffer(buf)))


class PinnedArray:
    """numpy view over cudaHostAlloc'd memory (freed on close/GC)."""

    def __init__(self, shape, dtype):
        self._lib = _lib.lib()
        self.shape = tuple(int(s) for s in shape)
        self.dtype = np.dtype(dtype)
        nbytes = int(np.prod(self.shape)) * self.dtype.itemsize
        p = C.c_void_p()
        check(self._lib.pg_host_alloc(C.byref(p), max(nbytes, 1)), "pg_host_alloc")
        self._p = p
        buf = (C.c_uint8 * max(nbytes, 1)).from_address(p.value)
        self.array = np.frombuffer(buf, dtype=self.dtype, count=int(np.prod(self.shape))).reshape(self.shape)

    def close(self):
        if self._p is not None:
            self.array = None
            self._lib.pg_host_free(self._p)
            self._p = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


SFS_MAX_CELLS = 1 << 28      # dense histograms of pg_sfs / pg_sfs_tables (k1.cu); the reference's sparse dicts have no such limit


def _check_sfs_cells(cells):
    """refuse before 16 bytes per cell are allocated on the host: e.g. a 4-D spectrum of > 127 haplotypes per population"""
    if sum(cells) > SFS_MAX_CELLS:
        raise PgError("sfs: %d histogram cells requested, the dense spectra are limited to %d in total (fewer dimensions, "
                      "fewer joint spectra per run, or --subsample smaller populations)" % (sum(cells), SFS_MAX_CELLS))


def sfs_shapes(groups, dims):
    """spectrum shapes (dims of each group's populations) and their cell counts (Python ints: no overflow)"""
    shapes = [tuple(int(dims[x]) for x in grp) for grp in groups]
    return shapes, [int(np.prod([int(d) for d in sh], dtype=object)) for sh in shapes]


def sfs_table_dims(kind, table):
    """the table as the engine reads it (uint16 [n,P,4] base counts | int32 [n,P] target counts) and the radix of every
    population: its largest count + 1"""
    if kind == "base":
        table = np.ascontiguousarray(table, dtype=np.uint16)
        n, P = table.shape[0], table.shape[1]
        dims = (table.sum(axis=2, dtype=np.int64).max(axis=0) + 1 if n else np.ones(P, np.int64)).astype(np.int32)
    else:
        table = np.ascontiguousarray(table, dtype=np.int32)
        n, P = table.shape
        dims = (table.max(axis=0) + 1 if n else np.ones(P, np.int64)).astype(np.int32)
        assert n == 0 or table.min() >= 0
    return table, dims


def _sfs_group_tables(groups):
    goff = np.zeros(len(groups) + 1, dtype=np.int32)
    for k, grp in enumerate(groups):
        goff[k + 1] = goff[k] + len(grp)
    return goff, np.array([x for grp in groups for x in grp], dtype=np.int32)


def sfs_unravel(cell, shape):
    """row-major flat cell indices -> int64 coordinates [n, len(shape)]"""
    cell = np.asarray(cell, dtype=np.int64)
    coords = np.empty((len(cell), len(shape)), dtype=np.int64)
    rest = cell.copy()
    for j in range(len(shape) - 1, -1, -1):
        coords[:, j] = rest % shape[j]
        rest //= shape[j]
    return coords


class Engine:
    def __init__(self, device: int = 0):
        self._lib = _lib.lib()
        ctx = C.c_void_p()
        check(self._lib.pg_ctx_create(int(device), C.byref(ctx)), "pg_ctx_create")
        self._ctx = ctx
        self.device = int(device)
        self.S = 0
        self.H = 0
        self.P = 0
        self.W = 0
        self._gslot_shape = {}     # table shape of each pipelined-gather slot, recorded at its begin

    # ---- lifetime ----
    def close(self):
        if getattr(self, "_ctx", None) is not None:
            self._lib.pg_ctx_destroy(self._ctx)
            self._ctx = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- data ----
    def upload(self, geno: np.ndarray, pos=None):
        """geno: int8 [S, H] site-major (A0 C1 G2 T3, negative = missing); pos: int32 [S]."""
        geno = np.ascontiguousarray(geno, dtype=np.int8)
        assert geno.ndim == 2
        S, H = geno.shape
        if pos is not None:
            pos = np.ascontiguousarray(pos, dtype=np.int32)
            assert pos.shape == (S,)
        check(self._lib.pg_upload(self._ctx, _ptr(geno), S, H, _ptr(pos)), "pg_upload")
        self.S, self.H = S, H
        self.W = 0

    def synth_fill(self, spec, n_sites: int, spacing: int = 10):
        tv, to, tt, tm = spec.thresholds()
        check(self._lib.pg_synth_fill(self._ctx, int(n_sites), spec.n_pops, spec.samples_per_pop, spec.ploidy,
                                      spec.seed, tv, to, tt, tm, int(spacing)), "pg_synth_fill")
        self.S, self.H = int(n_sites), spec.n_haps
        self.W = 0

    def download(self, site0: int, n: int, into_geno=None, into_pos=None, want_geno=True, want_pos=True):
        """Device -> host copy (decoded to A0 C1 G2 T3 / -1).  Destination arrays must be C-contiguous."""
        g = p = None
        if want_geno:
            g = into_geno if into_geno is not None else np.empty((n, self.H), dtype=np.int8)
            assert g.flags.c_contiguous and g.dtype == np.int8 and g.shape == (n, self.H)
        if want_pos:
            p = into_pos if into_pos is not None else np.empty(n, dtype=np.int32)
            assert p.flags.c_contiguous and p.dtype == np.int32 and p.shape == (n,)
        check(self._lib.pg_download(self._ctx, int(site0), int(n), _ptr(g), _ptr(p)), "pg_download")
        return g, p

    def set_pops(self, hap_pop, n_pops=None):
        hap_pop = np.ascontiguousarray(hap_pop, dtype=np.int32)
        assert hap_pop.shape == (self.H,), (hap_pop.shape, self.H)
        P = int(n_pops) if n_pops is not None else int(hap_pop.max()) + 1
        check(self._lib.pg_set_pops(self._ctx, P, _ptr(hap_pop)), "pg_set_pops")
        self.P = P

    def set_windows(self, lo, hi):
        lo = np.ascontiguousarray(lo, dtype=np.int64)
        hi = np.ascontiguousarray(hi, dtype=np.int64)
        assert lo.shape == hi.shape and lo.ndim == 1
        check(self._lib.pg_set_windows(self._ctx, len(lo), _ptr(lo), _ptr(hi)), "pg_set_windows")
        self.W = len(lo)

    # ---- statistics ----
    def set_freqstats(self, enable: bool = True):
        """Carry the popFreq counters (groupFreqStats) in the popgen site pass (opt-in: ~4 % of the pass)."""
        check(self._lib.pg_set_freqstats(self._ctx, 1 if enable else 0), "pg_set_freqstats")

    def popgen(self, min_sites: int = 1, min_data: float = 0.01, force_pairwise: bool = False):
        """-> dict(pi [W,P], dxy [W,npairs], fst [W,npairs], sites [W], pos_sum [W], path [W])."""
        W, P = self.W, self.P
        npairs = P * (P - 1) // 2
        pi = np.empty((W, P), dtype=np.float64)
        dxy = np.empty((W, npairs), dtype=np.float64)
        fst = np.empty((W, npairs), dtype=np.float64)
        sites = np.empty(W, dtype=np.int64)
        pos_sum = np.empty(W, dtype=np.int64)
        path = np.empty(W, dtype=np.int32)
        check(self._lib.pg_popgen(self._ctx, int(min_sites) if min_sites else 0, float(min_data),
                                  2 if force_pairwise else 0, _ptr(pi), _ptr(dxy), _ptr(fst), _ptr(sites),
                                  _ptr(pos_sum), _ptr(path)), "pg_popgen")
        return dict(pi=pi, dxy=dxy, fst=fst, sites=sites, pos_sum=pos_sum, path=path,
                    pairs=list(itertools.combinations(range(P), 2)))

    def popgen_record_width(self) -> int:
        return 4 + 5 * self.P + 2 * (self.P * (self.P - 1) // 2)

    def popgen_freqstats(self):
        """popFreq columns (Alignment.groupFreqStats) of the most recent popgen() call:
        dict(l [W], S, thetaPi, thetaW, TajD [W,P])."""
        W, P = self.W, self.P
        l = np.empty(W, dtype=np.float64)
        out = {k: np.empty((W, P), dtype=np.float64) for k in ("S", "thetaPi", "thetaW", "TajD")}
        check(self._lib.pg_popgen_freqstats(self._ctx, _ptr(l), _ptr(out["S"]), _ptr(out["thetaPi"]), _ptr(out["thetaW"]),
                                            _ptr(out["TajD"])), "pg_popgen_freqstats")
        out["l"] = l
        return out

    def popgen_device(self, d_rec_ptr: int, min_sites: int = 1, min_data: float = 0.01, force_pairwise: bool = False) -> int:
        """Statistics left on the device as fixed-width records (see pg_popgen_device); `d_rec_ptr` is a device
        pointer to W * popgen_record_width() 8-byte words.  Returns the number of windows that took the pairwise path."""
        n = C.c_int64(0)
        check(self._lib.pg_popgen_device(self._ctx, int(min_sites) if min_sites else 0, float(min_data),
                                         2 if force_pairwise else 0, C.c_void_p(int(d_rec_ptr)), C.byref(n)),
              "pg_popgen_device")
        return int(n.value)

    # ---- multi-GPU: native NCCL gather (one process per GPU) ----
    def nccl_unique_id(self) -> bytes:
        buf = (C.c_uint8 * 128)()
        check(self._lib.pg_nccl_unique_id(buf), "pg_nccl_unique_id")
        return bytes(buf)

    def nccl_init(self, world: int, rank: int, unique_id: bytes):
        assert len(unique_id) == 128
        buf = (C.c_uint8 * 128).from_buffer_copy(unique_id)
        check(self._lib.pg_nccl_init(self._ctx, int(world), int(rank), buf), "pg_nccl_init")
        self._world, self._rank = int(world), int(rank)

    def nccl_finalize(self):
        check(self._lib.pg_nccl_finalize(self._ctx), "pg_nccl_finalize")
        self._world, self._rank = 1, 0

    def popgen_allgather(self, w_max: int, table: np.ndarray, min_sites: int = 1, min_data: float = 0.01,
                         force_pairwise: bool = False) -> int:
        """Statistics of this rank's windows, then ONE ncclAllGather of every rank's records into `table`
        (float64 [world * w_max, popgen_record_width()], ideally pinned).  Returns this rank's pairwise-window count."""
        assert table.dtype == np.float64 and table.flags.c_contiguous
        assert table.shape == (self._world * int(w_max), self.popgen_record_width())
        n = C.c_int64(0)
        check(self._lib.pg_popgen_allgather(self._ctx, int(min_sites) if min_sites else 0, float(min_data),
                                            2 if force_pairwise else 0, int(w_max), _ptr(table), C.byref(n)),
              "pg_popgen_allgather")
        return int(n.value)

    def popgen_gather_begin(self, w_max: int, slot: int, min_sites: int = 1, min_data: float = 0.01):
        """Pipelined popgen_allgather: enqueue one batch (statistics on the main stream, all-gather + D2H on a side stream)."""
        check(self._lib.pg_popgen_gather_begin(self._ctx, int(min_sites) if min_sites else 0, float(min_data), int(w_max),
                                               int(slot)), "pg_popgen_gather_begin")
        world = getattr(self, "_world", 1) or 1
        self._gslot_shape[int(slot)] = (world * int(w_max), self.popgen_record_width())   # P may change before `end`

    def popgen_gather_end(self, w_max: int, slot: int, with_pairwise: bool = False):
        """-> float64 [world * w_max, record width at the slot's begin] view of the slot's pinned table (valid until its next
        begin); with_pairwise=True: (table, number of this rank's windows that took the pairwise path)."""
        p = C.c_void_p()
        n = C.c_int64(0)
        check(self._lib.pg_popgen_gather_end(self._ctx, int(slot), C.byref(p), C.byref(n)), "pg_popgen_gather_end")
        shape = self._gslot_shape[int(slot)]
        world = getattr(self, "_world", 1) or 1
        assert shape[0] == world * int(w_max), (shape, w_max)
        buf = (C.c_double * (shape[0] * shape[1])).from_address(p.value)
        table = np.frombuffer(buf, dtype=np.float64).reshape(shape)
        return (table, int(n.value)) if with_pairwise else table

    def abbababa_allgather(self, p1: int, p2: int, p3: int, o: int, min_data: float, w_max: int, table: np.ndarray):
        """ABBA-BABA statistics of this rank's windows + ONE ncclAllGather: `table` float64 [world * w_max, 8] receives
        [sites, pos_sum (int64 bit patterns), ABBA, BABA, D, fd, fdM, sitesUsed] per window (multigpu.unpack_abba_records)."""
        assert table.dtype == np.float64 and table.flags.c_contiguous and table.shape == (self._world * int(w_max), 8)
        check(self._lib.pg_abbababa_allgather(self._ctx, p1, p2, p3, o, float(min_data), int(w_max), _ptr(table)),
              "pg_abbababa_allgather")

    def fourpop_allgather(self, p1: int, p2: int, p3: int, p4: int, min_data: float, w_max: int, table: np.ndarray,
                          polarize: bool = False, fixed: bool = False):
        """genomics.fourPop of this rank's windows + ONE ncclAllGather: `table` float64 [world * w_max, 17]."""
        assert table.dtype == np.float64 and table.flags.c_contiguous and table.shape == (self._world * int(w_max), 17)
        mode = 1 if polarize else (2 if fixed else 0)
        check(self._lib.pg_fourpop_allgather(self._ctx, p1, p2, p3, p4, float(min_data), mode, int(w_max), _ptr(table)),
              "pg_fourpop_allgather")

    def abbababa(self, p1: int, p2: int, p3: int, o: int, min_data: float = 0.01):
        """-> dict(ABBA,BABA,D,fd,fdM [W], sitesUsed [W] (nan = no good site), sites, pos_sum)."""
        W = self.W
        out = np.empty((W, 5), dtype=np.float64)
        used = np.empty(W, dtype=np.float64)
        sites = np.empty(W, dtype=np.int64)
        pos_sum = np.empty(W, dtype=np.int64)
        check(self._lib.pg_abbababa(self._ctx, p1, p2, p3, o, float(min_data), _ptr(out), _ptr(used), _ptr(sites),
                                    _ptr(pos_sum)), "pg_abbababa")
        return dict(ABBA=out[:, 0], BABA=out[:, 1], D=out[:, 2], fd=out[:, 3], fdM=out[:, 4], sitesUsed=used,
                    sites=sites, pos_sum=pos_sum)

    FOURPOP_KEYS = ('fhom', "fhom'", 'D', 'fd', "fd'", 'fdm', "fdm'", 'fdh', 'fdh2', 'fh', "ABBA", "BABA", "ABAA", "BAAA")

    def fourpop(self, p1: int, p2: int, p3: int, p4: int, min_data: float = 0.01, polarize: bool = False,
                fixed: bool = False):
        """genomics.fourPop per window -> dict(<14 statistics> [W], sitesUsed [W], sites, pos_sum)."""
        W = self.W
        out = np.empty((W, 14), dtype=np.float64)
        used = np.empty(W, dtype=np.float64)
        sites = np.empty(W, dtype=np.int64)
        pos_sum = np.empty(W, dtype=np.int64)
        mode = 1 if polarize else (2 if fixed else 0)          # genomics.py:1610-1615: polarize wins over fixed
        check(self._lib.pg_fourpop(self._ctx, p1, p2, p3, p4, float(min_data), mode, _ptr(out), _ptr(used), _ptr(sites),
                                   _ptr(pos_sum)), "pg_fourpop")
        r = {k: out[:, i] for i, k in enumerate(self.FOURPOP_KEYS)}
        r.update(sitesUsed=used, sites=sites, pos_sum=pos_sum)
        return r

    def ingest_text(self, data: bytes, fmt: int, col_hap, col_ploidy, H: int, offset: int = 0) -> int:
        """Device-side .geno tokenizer (pg_ingest_text): data[offset:] = the file's data lines (no copy is made).
        Returns the number of sites now resident."""
        col_hap = np.ascontiguousarray(col_hap, dtype=np.int32)
        col_ploidy = np.ascontiguousarray(col_ploidy, dtype=np.int8)
        assert col_hap.shape == col_ploidy.shape
        n = C.c_int64(0)
        addr = C.cast(C.c_char_p(data), C.c_void_p).value or 0        # `data` stays referenced by the caller
        check(self._lib.pg_ingest_text(self._ctx, C.c_void_p(addr + offset), len(data) - offset, int(fmt), len(col_hap),
                                       _ptr(col_hap), _ptr(col_ploidy), int(H), C.byref(n)), "pg_ingest_text")
        self.S, self.H = int(n.value), int(H)
        return self.S

    def ingest_file(self, path: str, body_offset: int, fmt: int, col_hap, col_ploidy, H: int) -> int:
        """The same, reading the file straight into the pinned staging buffers (pg_ingest_file)."""
        col_hap = np.ascontiguousarray(col_hap, dtype=np.int32)
        col_ploidy = np.ascontiguousarray(col_ploidy, dtype=np.int8)
        n = C.c_int64(0)
        check(self._lib.pg_ingest_file(self._ctx, path.encode(), int(body_offset), int(fmt), len(col_hap), _ptr(col_hap),
                                       _ptr(col_ploidy), int(H), C.byref(n)), "pg_ingest_file")
        self.S, self.H = int(n.value), int(H)
        return self.S

    def ingest_file_range(self, path: str, byte_lo: int, byte_hi: int, fmt: int, col_hap, col_ploidy, H: int) -> int:
        """One rank's share of the file: bytes [byte_lo, byte_hi) (line starts; byte_hi < 0 = end of file)."""
        col_hap = np.ascontiguousarray(col_hap, dtype=np.int32)
        col_ploidy = np.ascontiguousarray(col_ploidy, dtype=np.int8)
        n = C.c_int64(0)
        check(self._lib.pg_ingest_file_range(self._ctx, path.encode(), int(byte_lo), int(byte_hi), int(fmt), len(col_hap),
                                             _ptr(col_hap), _ptr(col_ploidy), int(H), C.byref(n)), "pg_ingest_file_range")
        self.S, self.H = int(n.value), int(H)
        return self.S

    def append_sites(self, geno: np.ndarray, pos=None):
        """Append sites (int8 [n, H]) after the resident ones (halo of the next rank's first sites)."""
        geno = np.ascontiguousarray(geno, dtype=np.int8)
        assert geno.ndim == 2 and geno.shape[1] == self.H
        if pos is not None:
            pos = np.ascontiguousarray(pos, dtype=np.int32)
        check(self._lib.pg_append_sites(self._ctx, geno.shape[0], _ptr(geno), _ptr(pos)), "pg_append_sites")
        self.S += geno.shape[0]

    def ingest_meta(self, S: int, release: bool = True):
        """(pos int32 [S], new_scaffold int8 [S], line_off int64 [S]) of the last ingest_text.  The device copy of the text
        is freed unless release=False (filter_emit reads it)."""
        pos = np.empty(S, dtype=np.int32)
        newsc = np.empty(S, dtype=np.int8)
        off = np.empty(S, dtype=np.int64)
        check(self._lib.pg_ingest_meta(self._ctx, _ptr(pos), _ptr(newsc), _ptr(off)), "pg_ingest_meta")
        if release:
            check(self._lib.pg_ingest_release(self._ctx), "pg_ingest_release")
        return pos, newsc, off

    def ingest_geometry(self):
        """Geometry of the last ingest (pg_debug_ingest): slabs and slab bytes of the text copy, bytes per line-index block,
        warps of the line parse grid and threads of the scaffold-flag grid."""
        out = np.zeros(5, dtype=np.int64)
        check(self._lib.pg_debug_ingest(self._ctx, _ptr(out)), "pg_debug_ingest")
        return dict(zip(("slabs", "slab_bytes", "index_block_bytes", "parse_warps", "flag_threads"), (int(v) for v in out)))

    # ---- filterGenotypes.py ----
    FILTER_FORMATS = {"phased": 0, "diplo": 1, "bases": 2, "alleles": 3, "coded": 4, "count": 5}

    def set_strict_ingest(self, on=True):
        """Strict genotype tokens for the next ingests (pg_ingest_set_strict): True / 1 = widths and characters,
        2 = token widths only."""
        check(self._lib.pg_ingest_set_strict(self._ctx, int(on)), "pg_ingest_set_strict")

    def filter(self, spec: dict, contig_mask=None, scaf_id=None):
        """pg_filter over the sites of the last strict ingest.  spec keys: samp_hap0, samp_ploidy, pops (one list of sample
        indices per population, in -p order; may overlap) and the scalar / per-population settings of pg_filter_spec
        (None = off).  Returns (rows kept, OR of their flags)."""
        from ._lib import FilterSpec
        keep = []

        def arr(v, dt):
            if v is None:
                return None
            a = np.ascontiguousarray(v, dtype=dt)
            keep.append(a)
            return a.ctypes.data
        fs = FilterSpec()
        fs.n_samp = len(spec["samp_hap0"])
        fs.samp_hap0 = arr(spec["samp_hap0"], np.int32)
        fs.samp_ploidy = arr(spec["samp_ploidy"], np.int8)
        pops = [list(m) for m in (spec.get("pops") or [])]
        fs.P = len(pops)
        if fs.P:
            fs.pop_off = arr(np.concatenate([[0], np.cumsum([len(m) for m in pops])]), np.int32)
            fs.pop_members = arr(np.array([k for m in pops for k in m] or [0]), np.int32)
        fs.min_calls = int(spec.get("min_calls", 1))
        fs.min_alleles = int(spec.get("min_alleles", 1))
        fs.max_alleles = float(spec.get("max_alleles", float("inf")))
        fs.min_var_count = int(spec.get("min_var_count") or 0)
        fs.has_max_het = spec.get("max_het") is not None
        fs.max_het = float(spec.get("max_het") or 0.0)
        fs.min_freq = float(spec.get("min_freq") or 0.0)
        fs.max_freq = float(spec.get("max_freq") or 0.0)
        fs.min_pop_calls = arr(spec.get("min_pop_calls"), np.int32)
        fs.min_pop_alleles = arr(spec.get("min_pop_alleles"), np.int32)
        fs.max_pop_alleles = arr(spec.get("max_pop_alleles"), np.int32)
        fs.fixed_diffs = 1 if spec.get("fixed_diffs") else 0
        fs.has_nearly_fixed = spec.get("nearly_fixed_diff") is not None
        fs.nearly_fixed_diff = float(spec.get("nearly_fixed_diff") or 0.0)
        fs.partial_to_missing = 1 if spec.get("partial_to_missing") else 0
        fs.no_test = 1 if spec.get("no_test") else 0
        fs.thin_dist = int(spec.get("thin_dist") or 0)
        fs.pod_size = int(spec.get("pod_size") or 10000)
        cm = arr(contig_mask, np.uint8)
        sc = arr(scaf_id, np.int32)
        nk = C.c_int64(0)
        fo = C.c_uint8(0)
        check(self._lib.pg_filter(self._ctx, C.byref(fs), cm, sc, C.byref(nk), C.byref(fo)), "pg_filter")
        self._filter_P = fs.P
        return int(nk.value), int(fo.value)

    def filter_emit(self, fmt: str, freq_order: bool, row0: int, buf, cap: int):
        """Rows row0.. of the last filter as text into buf (a writable buffer of at least cap bytes, pinned for speed):
        (rows, bytes) written."""
        rows = C.c_int64(0)
        nb = C.c_size_t(0)
        check(self._lib.pg_filter_emit(self._ctx, self.FILTER_FORMATS[fmt], 1 if freq_order else 0, int(row0), _addr(buf),
                                       int(cap), C.byref(rows), C.byref(nb)), "pg_filter_emit")
        return int(rows.value), int(nb.value)

    def filter_stats(self, site0: int = 0, n: int | None = None):
        """Per-site statistics of the last filter (pg_filter_stats) as a dict of arrays."""
        if n is None:
            n = self.S - site0
        P = getattr(self, "_filter_P", 0)
        r = dict(called=np.empty(n, np.int32), het=np.empty(n, np.int32), counts=np.empty((n, 4), np.int32),
                 pop_called=np.empty((n, P), np.int32), pop_mask=np.empty((n, P), np.uint8), flags=np.empty(n, np.uint8),
                 keep=np.empty(n, np.uint8), final=np.empty(n, np.uint8))
        check(self._lib.pg_filter_stats(self._ctx, int(site0), int(n), *[_ptr(r[k]) for k in
                                        ("called", "het", "counts", "pop_called", "pop_mask", "flags", "keep", "final")]),
              "pg_filter_stats")
        return r

    # ---- parseVCF.py ----
    def vcf_set_spec(self, spec: dict):
        """pg_vcf_set_spec: the header's column tables, the FORMAT keys looked up (GT first), the selected samples, the
        --gtf filters and the output settings of one run (parseVCF.py:331-368)."""
        from ._lib import VcfSpec
        keep = []

        def arr(v, dt):
            a = np.ascontiguousarray(v if len(v) else np.zeros(1), dtype=dt)
            keep.append(a)
            return a.ctypes.data

        def text(b):
            keep.append(b)
            return C.cast(C.c_char_p(b), C.c_void_p).value
        keys = [k.encode() for k in spec["keys"]]
        vs = VcfSpec()
        vs.n_cols = len(spec["col_slot"])
        vs.col_slot = arr(spec["col_slot"], np.int32)
        vs.col_prev = arr(spec["col_prev"], np.int32)
        vs.n_keys = len(keys)
        vs.key_off = arr(np.concatenate([[0], np.cumsum([len(k) for k in keys])]), np.int32)
        vs.key_chars = text(b"".join(keys) + b"\0")
        vs.n_samp = len(spec["samp_col"])
        vs.samp_col = arr(spec["samp_col"], np.int32)
        vs.samp_ploidy = arr(spec["samp_ploidy"], np.int32)
        vs.field_key = int(spec["field_key"])
        vs.field_phase = 1 if spec.get("field_phase") else 0
        filt = spec["filters"]
        vs.n_filt = len(filt)
        vs.filt_key = arr([f["key"] for f in filt], np.int32)
        vs.filt_min = arr([f["min"] for f in filt], np.float64)
        vs.filt_max = arr([f["max"] for f in filt], np.float64)
        vs.filt_site = arr([f["site"] for f in filt], np.uint8)
        vs.filt_gt = arr([f["gt"] for f in filt], np.uint8)
        vs.filt_samp = arr(np.array([f["samples"] for f in filt], dtype=np.uint8).reshape(-1), np.uint8)
        vs.has_min_qual = 1 if spec.get("min_qual") is not None else 0
        vs.min_qual = float(spec.get("min_qual") or 0.0)
        vs.missing = text(spec["missing"] + b"\0")
        vs.missing_len = len(spec["missing"])
        vs.sep = text(spec["sep"] + b"\0")
        vs.sep_len = len(spec["sep"])
        vs.skip_indels = 1 if spec.get("skip_indels") else 0
        vs.keep_partial = 1 if spec.get("keep_partial") else 0
        vs.ploidy_mismatch_to_missing = 1 if spec.get("p2m") else 0
        vs.add_ref_track = 1 if spec.get("add_ref") else 0
        check(self._lib.pg_vcf_set_spec(self._ctx, C.byref(vs)), "pg_vcf_set_spec")

    def vcf_load(self, text: bytes, prev=None) -> int:
        """pg_vcf_load: complete lines of VCF body text; prev = (CHROM, POS) bytes of the data line before it, or None.
        Returns the number of data lines."""
        n = C.c_int64(0)
        pc, pp = (prev[0], prev[1]) if prev is not None else (b"", b"")
        check(self._lib.pg_vcf_load(self._ctx, text, len(text), (pc + pp) if prev is not None else None, len(pc), len(pp),
                                    C.byref(n)), "pg_vcf_load")
        self._vcf_lines = int(n.value)
        return self._vcf_lines

    def vcf_lines(self, line0: int = 0, n: int | None = None):
        """The pg_vcf_line records of the last load as a numpy record array (_lib.VCF_LINE)."""
        from ._lib import VCF_LINE
        if n is None:
            n = self._vcf_lines - line0
        out = np.zeros(n, dtype=VCF_LINE)
        check(self._lib.pg_vcf_lines(self._ctx, int(line0), int(n), _ptr(out)), "pg_vcf_lines")
        return out

    def vcf_genotypes(self, rows, pos):
        """pg_vcf_genotypes over the kept lines `rows` (with their POS): (genotypes left unresolved, error word)."""
        rows = np.ascontiguousarray(rows, dtype=np.int64)
        pos = np.ascontiguousarray(pos, dtype=np.int64)
        nu = C.c_int64(0)
        err = C.c_uint64(0)
        check(self._lib.pg_vcf_genotypes(self._ctx, len(rows), _ptr(rows), _ptr(pos), C.byref(nu), C.byref(err)),
              "pg_vcf_genotypes")
        return int(nu.value), int(err.value)

    def vcf_verdicts(self, n_rows: int, n_samp: int, put=None):
        """The verdict bytes [n_rows, n_samp] of the last vcf_genotypes; with put, replaces them first."""
        if put is not None:
            put = np.ascontiguousarray(put, dtype=np.uint8)
            check(self._lib.pg_vcf_verdicts(self._ctx, None, _ptr(put)), "pg_vcf_verdicts")
            return put
        out = np.zeros((n_rows, n_samp), dtype=np.uint8)
        check(self._lib.pg_vcf_verdicts(self._ctx, _ptr(out), None), "pg_vcf_verdicts")
        return out

    def vcf_emit(self, row0: int, buf, cap: int):
        """Rows row0.. of the last vcf_genotypes as .geno text into buf (at least cap bytes, pinned for speed):
        (rows, bytes) written."""
        rows = C.c_int64(0)
        nb = C.c_size_t(0)
        check(self._lib.pg_vcf_emit(self._ctx, int(row0), _addr(buf), int(cap), C.byref(rows), C.byref(nb)),
              "pg_vcf_emit")
        return int(rows.value), int(nb.value)

    def seq_index(self, col_slot, slot_width, exact: bool, data: bytes | None = None, path: str | None = None,
                  body_offset: int = 0):
        """pg_seq_index: the body (data, or bytes body_offset.. of the file path) to the device and the token start of every
        slotted column per data line.  Returns (data lines, (code, data line, genotype column)); code 0 = no error."""
        col_slot = np.ascontiguousarray(col_slot, dtype=np.int32)
        slot_width = np.ascontiguousarray(slot_width, dtype=np.int32)
        n = C.c_int64(0)
        err = np.zeros(3, dtype=np.int64)
        check(self._lib.pg_seq_index(self._ctx, data if path is None else None, 0 if data is None else len(data),
                                     None if path is None else path.encode(), int(body_offset), len(col_slot), _ptr(col_slot),
                                     len(slot_width), _ptr(slot_width), 1 if exact else 0, C.byref(n), _ptr(err)),
              "pg_seq_index")
        return int(n.value), tuple(int(v) for v in err)

    def seq_meta(self, S: int):
        """positions int32 [S], new-scaffold flags int8 [S] and line offsets int64 [S] of the last seq_index"""
        pos = np.zeros(S, np.int32)
        newsc = np.zeros(S, np.int8)
        off = np.zeros(S, np.int64)
        check(self._lib.pg_seq_meta(self._ctx, _ptr(pos), _ptr(newsc), _ptr(off)), "pg_seq_meta")
        return pos, newsc, off

    def seq_plan(self, fmt: str, nto_gap: bool, names, seq_slot, seq_byte, seq_width, lo, hi):
        """pg_seq_plan: alignments over the windows [lo, hi) of the last seq_index.  Returns (rows, bytes of every window)."""
        enc = [n.encode() for n in names]
        name_off = np.concatenate([[0], np.cumsum([len(b) for b in enc])]).astype(np.int64)
        seq_slot = np.ascontiguousarray(seq_slot, dtype=np.int32)
        seq_byte = np.ascontiguousarray(seq_byte, dtype=np.int32)
        seq_width = np.ascontiguousarray(seq_width, dtype=np.int32)
        lo = np.ascontiguousarray(lo, dtype=np.int64)
        hi = np.ascontiguousarray(hi, dtype=np.int64)
        wb = np.zeros(len(lo), np.int64)
        R = C.c_int64(0)
        check(self._lib.pg_seq_plan(self._ctx, {"fasta": 0, "phylip": 1}[fmt], 1 if nto_gap else 0, len(enc), b"".join(enc),
                                    _ptr(name_off), _ptr(seq_slot), _ptr(seq_byte), _ptr(seq_width), len(lo), _ptr(lo),
                                    _ptr(hi), C.byref(R), _ptr(wb)), "pg_seq_plan")
        return int(R.value), wb

    def seq_emit(self, row0: int, part0: int, buf, cap: int):
        """Alignment text of the last seq_plan from cell (row0, part0) into buf (cap bytes, pinned for speed):
        (row, part) to resume at, bytes written."""
        r1, p1 = C.c_int64(0), C.c_int64(0)
        nb = C.c_size_t(0)
        check(self._lib.pg_seq_emit(self._ctx, int(row0), int(part0), _addr(buf), int(cap), C.byref(r1), C.byref(p1),
                                    C.byref(nb)), "pg_seq_emit")
        return int(r1.value), int(p1.value), int(nb.value)

    def g2v_ref_load(self, text: bytes):
        """pg_g2v_ref_load + pg_g2v_ref_starts: the reference FASTA to the device; returns the byte offsets of its '>' bytes"""
        n = C.c_int64(0)
        check(self._lib.pg_g2v_ref_load(self._ctx, text, len(text), C.byref(n)), "pg_g2v_ref_load")
        starts = np.zeros(int(n.value), np.int64)
        check(self._lib.pg_g2v_ref_starts(self._ctx, _ptr(starts)), "pg_g2v_ref_starts")
        return starts

    def g2v_ref_index(self, lo, hi):
        """pg_g2v_ref_index: record k's sequence is FASTA bytes [lo[k], hi[k]) without newlines and spaces; returns the
        sequence lengths"""
        lo = np.ascontiguousarray(lo, dtype=np.int64)
        hi = np.ascontiguousarray(hi, dtype=np.int64)
        out = np.zeros(len(lo), np.int64)
        check(self._lib.pg_g2v_ref_index(self._ctx, len(lo), _ptr(lo), _ptr(hi), _ptr(out)), "pg_g2v_ref_index")
        return out

    def g2v_spec(self, fmt: int, col_slot, col_prev, sel_col, use_ref: bool):
        """pg_g2v_spec: format (0 phased, 1 diplo, 2 pairs), the header's column tables and the selected samples' columns"""
        col_slot = np.ascontiguousarray(col_slot, dtype=np.int32)
        col_prev = np.ascontiguousarray(col_prev, dtype=np.int32)
        sel_col = np.ascontiguousarray(sel_col, dtype=np.int32)
        check(self._lib.pg_g2v_spec(self._ctx, int(fmt), len(col_slot), _ptr(col_slot), _ptr(col_prev), len(sel_col),
                                    _ptr(sel_col), 1 if use_ref else 0), "pg_g2v_spec")

    def g2v_chunk(self, text: bytes):
        """pg_g2v_chunk + pg_g2v_runs: complete body lines to the device, tokenised.  Returns (data lines, first line of every
        scaffold run, its byte offset in text)."""
        S, nr = C.c_int64(0), C.c_int64(0)
        check(self._lib.pg_g2v_chunk(self._ctx, text, len(text), C.byref(S), C.byref(nr)), "pg_g2v_chunk")
        run_line = np.zeros(int(nr.value), np.int64)
        run_off = np.zeros(int(nr.value), np.int64)
        check(self._lib.pg_g2v_runs(self._ctx, _ptr(run_line), _ptr(run_off)), "pg_g2v_runs")
        return int(S.value), run_line, run_off

    def g2v_sites(self, run_rec):
        """pg_g2v_sites: the site pass over the last chunk, run_rec = FASTA record of every scaffold run (-1: none).  Returns
        (rows before the first error, their bytes, (code, data line, column, line offset)); code 0 = no error."""
        run_rec = np.ascontiguousarray(run_rec, dtype=np.int32)
        rows, nb = C.c_int64(0), C.c_int64(0)
        err = np.zeros(4, np.int64)
        check(self._lib.pg_g2v_sites(self._ctx, _ptr(run_rec) if len(run_rec) else None, C.byref(rows), C.byref(nb),
                                     _ptr(err)), "pg_g2v_sites")
        return int(rows.value), int(nb.value), tuple(int(v) for v in err)

    def g2v_emit(self, byte0: int, buf, cap: int) -> int:
        """Bytes byte0.. (at most cap) of the last g2v_sites' VCF rows into buf (pinned for speed); returns the bytes written"""
        nb = C.c_size_t(0)
        check(self._lib.pg_g2v_emit(self._ctx, int(byte0), _addr(buf), int(cap), C.byref(nb)), "pg_g2v_emit")
        return int(nb.value)

    def ws_spec(self, col_slot, n_slots: int, n_fields: int):
        """pg_ws_spec: value column c is parsed into slot col_slot[c] (-1: not read); n_fields >= 0: every line has exactly
        that many value fields, -1: every line holds every slot's column"""
        col_slot = np.ascontiguousarray(col_slot, dtype=np.int32)
        check(self._lib.pg_ws_spec(self._ctx, len(col_slot), _ptr(col_slot), int(n_slots), int(n_fields)), "pg_ws_spec")

    def ws_chunk(self, text: bytes):
        """pg_ws_chunk + pg_ws_chunk_info: complete body lines appended to the resident values.  Returns (data lines, first
        line of every scaffold run, its byte offset in text, flagged tokens as slot * lines + line, their records (offset << 32
        | length << 2 | status), (code, data line, slot) of the first bad line)."""
        S, nr, nf = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        err = np.zeros(3, np.int64)
        check(self._lib.pg_ws_chunk(self._ctx, text, len(text), C.byref(S), C.byref(nr), C.byref(nf), _ptr(err)),
              "pg_ws_chunk")
        run_line = np.zeros(int(nr.value), np.int64)
        run_off = np.zeros(int(nr.value), np.int64)
        fidx = np.zeros(int(nf.value), np.int64)
        ftok = np.zeros(int(nf.value), np.uint64)
        check(self._lib.pg_ws_chunk_info(self._ctx, _ptr(run_line), _ptr(run_off), _ptr(fidx), _ptr(ftok)), "pg_ws_chunk_info")
        return int(S.value), run_line, run_off, fidx, ftok, tuple(int(v) for v in err)

    def ws_set_values(self, line, slot, v):
        """pg_ws_set_values: slot[i]'s value on data line line[i] (over all chunks) = v[i]"""
        line = np.ascontiguousarray(line, dtype=np.int64)
        slot = np.ascontiguousarray(slot, dtype=np.int32)
        v = np.ascontiguousarray(v, dtype=np.float64)
        check(self._lib.pg_ws_set_values(self._ctx, len(line), _ptr(line), _ptr(slot), _ptr(v)), "pg_ws_set_values")

    def ws_meta(self):
        """pg_ws_meta: the positions of every data line so far (int64)"""
        S = C.c_int64(0)
        check(self._lib.pg_ws_meta(self._ctx, C.byref(S), None), "pg_ws_meta")
        pos = np.zeros(int(S.value), np.int64)
        check(self._lib.pg_ws_meta(self._ctx, C.byref(S), _ptr(pos)), "pg_ws_meta")
        return pos

    def ws_stats(self, lo, hi, codes, qs, n_slots: int, sort_budget: int = 1 << 30):
        """pg_ws_stats: windows [lo[w], hi[w]) of data lines -> (float64 [W x n_slots x K], non-NaN counts [W x n_slots]);
        codes: 0 mean, 1 median, 2 min, 3 max, 4 sd, 5 sum, 6 quantile qs[k]"""
        lo = np.ascontiguousarray(lo, dtype=np.int64)
        hi = np.ascontiguousarray(hi, dtype=np.int64)
        codes = np.ascontiguousarray(codes, dtype=np.int32)
        qs = np.ascontiguousarray(qs, dtype=np.float64)
        W, K = len(lo), len(codes)
        out = np.zeros((W, n_slots, K), np.float64)
        n = np.zeros((W, n_slots), np.int64)
        check(self._lib.pg_ws_stats(self._ctx, W, _ptr(lo), _ptr(hi), K, _ptr(codes), _ptr(qs), int(sort_budget), _ptr(out),
                                    _ptr(n)), "pg_ws_stats")
        return out, n

    def merge_setup(self, names, lengths, out, n_dummy, sep: bytes, missing: bytes, method: int, union_min: int,
                    must_include_first: int) -> bool:
        """pg_merge_setup: the .fai walk (names as bytes, lengths), per file whether its columns are written and its dummy
        genotype count, the separator, the missing genotype and the rule (method 0 intersect, 1 union, 2 all).  Returns
        True when every walk index is a row (the dense rule)."""
        name_off = np.zeros(len(names) + 1, np.int64)
        name_off[1:] = np.cumsum([len(n) for n in names])
        lengths = np.ascontiguousarray(lengths, dtype=np.int64)
        out = np.ascontiguousarray(out, dtype=np.int32)
        n_dummy = np.ascontiguousarray(n_dummy, dtype=np.int64)
        dense = C.c_int32(0)
        check(self._lib.pg_merge_setup(self._ctx, len(names), b"".join(names), _ptr(name_off), _ptr(lengths), len(out),
                                       _ptr(out), _ptr(n_dummy), sep, len(sep), missing, len(missing), int(method),
                                       int(union_min), int(must_include_first), C.byref(dense)), "pg_merge_setup")
        return bool(dense.value)

    def merge_load(self, file: int, text: bytes):
        """pg_merge_load: the next chunk of complete lines of a file's body.  Returns (lines, the first line that stalls the
        file (lines when none), 0 no stall / 1 stall / 2 that line is refused, walk index of the line before the stall)."""
        info = np.zeros(4, np.int64)
        check(self._lib.pg_merge_load(self._ctx, int(file), text, len(text), _ptr(info)), "pg_merge_load")
        return tuple(int(v) for v in info)

    def merge_rows(self, hi: int):
        """pg_merge_rows: the rows of walk indices (previous bound, hi]; returns (rows, bytes)"""
        n, nb = C.c_int64(0), C.c_int64(0)
        check(self._lib.pg_merge_rows(self._ctx, int(hi), C.byref(n), C.byref(nb)), "pg_merge_rows")
        return int(n.value), int(nb.value)

    def merge_emit(self, byte0: int, buf, cap: int) -> int:
        """Bytes byte0.. (at most cap) of the last merge_rows' rows into buf (pinned for speed); returns the bytes written"""
        nb = C.c_size_t(0)
        check(self._lib.pg_merge_emit(self._ctx, int(byte0), _addr(buf), int(cap), C.byref(nb)), "pg_merge_emit")
        return int(nb.value)

    def s2g_fasta_load(self, text: bytes):
        """pg_s2g_fasta_load + pg_s2g_fasta_starts: a FASTA to the device; returns the byte offsets of its '>' bytes"""
        n = C.c_int64(0)
        check(self._lib.pg_s2g_fasta_load(self._ctx, text, len(text), C.byref(n)), "pg_s2g_fasta_load")
        starts = np.zeros(int(n.value), np.int64)
        check(self._lib.pg_s2g_fasta_starts(self._ctx, _ptr(starts)), "pg_s2g_fasta_starts")
        return starts

    def s2g_fasta_index(self, lo, hi):
        """pg_s2g_fasta_index: record k's sequence is FASTA bytes [lo[k], hi[k]) without newlines and spaces; returns the
        sequence lengths"""
        lo = np.ascontiguousarray(lo, dtype=np.int64)
        hi = np.ascontiguousarray(hi, dtype=np.int64)
        out = np.zeros(len(lo), np.int64)
        check(self._lib.pg_s2g_fasta_index(self._ctx, len(lo), _ptr(lo), _ptr(hi), _ptr(out)), "pg_s2g_fasta_index")
        return out

    def s2g_phylip_load(self, text: bytes):
        """pg_s2g_phylip_load + pg_s2g_phylip_lines: a PHYLIP text to the device, one warp per line; returns the line table,
        int64 [lines, 7] = {field 0 start, its length, field 1 start, its length, fields, flags, header count}"""
        n = C.c_int64(0)
        check(self._lib.pg_s2g_phylip_load(self._ctx, text, len(text), C.byref(n)), "pg_s2g_phylip_load")
        lines = np.zeros((int(n.value), 7), np.int64)
        check(self._lib.pg_s2g_phylip_lines(self._ctx, _ptr(lines)), "pg_s2g_phylip_lines")
        return lines

    def s2g_phylip_pack(self, seq_len, spans):
        """pg_s2g_phylip_pack: the sequences (seq_len bytes each, one after another) from the field-1 spans, int64 [n, 3] =
        {text byte, sequence byte, bytes}"""
        seq_len = np.ascontiguousarray(seq_len, dtype=np.int64)
        spans = np.ascontiguousarray(spans, dtype=np.int64).reshape(-1, 3)
        check(self._lib.pg_s2g_phylip_pack(self._ctx, len(seq_len), _ptr(seq_len), len(spans), _ptr(spans)),
              "pg_s2g_phylip_pack")

    def s2g_plan(self, names, rows, members, seps):
        """pg_s2g_plan: one block per output contig — names[b] (bytes), rows[b], members[b] (sequence indices, in output
        order) and seps[b] (bytes, one per member: the byte that follows it).  Returns the bytes of all rows."""
        blk = np.zeros((len(names), 4), np.int64)
        blk[:, 1] = [len(n) for n in names]
        blk[:, 0] = np.concatenate([[0], np.cumsum(blk[:, 1])[:-1]]) if len(names) else []
        blk[:, 2] = rows
        blk[:, 3] = np.concatenate([[0], np.cumsum([len(m) for m in members])[:-1]]) if len(names) else []
        mem = np.ascontiguousarray(np.concatenate([np.asarray(m, np.int64) for m in members]) if members else [], np.int64)
        sep = np.frombuffer(b"".join(seps), np.uint8).copy()
        nb = C.c_int64(0)
        check(self._lib.pg_s2g_plan(self._ctx, len(names), _ptr(blk), b"".join(names), int(blk[:, 1].sum()), len(mem),
                                    _ptr(mem), _ptr(sep), C.byref(nb)), "pg_s2g_plan")
        return int(nb.value)

    def s2g_emit(self, byte0: int, buf, cap: int) -> int:
        """Bytes byte0.. (at most cap) of the last s2g_plan's rows into buf (pinned for speed); returns the bytes written"""
        nb = C.c_size_t(0)
        check(self._lib.pg_s2g_emit(self._ctx, int(byte0), _addr(buf), int(cap), C.byref(nb)), "pg_s2g_emit")
        return int(nb.value)

    def site_counts(self, site0: int = 0, n: int = None, out=None):
        """uint16 [n, P, 4] A,C,G,T counts per population (`out`: a caller-owned array to fill, e.g. one whose pages are
        already resident — a fresh 100 MB array costs more in page faults than the kernel and the copy together)."""
        n = self.S - site0 if n is None else int(n)
        if out is None:
            out = np.empty((n, self.P, 4), dtype=np.uint16)
        else:
            out = out[:n]
            assert out.dtype == np.uint16 and out.flags.c_contiguous and out.shape == (n, self.P, 4)
        check(self._lib.pg_site_counts(self._ctx, int(site0), n, _ptr(out)), "pg_site_counts")
        return out

    def site_target_freqs(self, target: str, site0: int = 0, n: int | None = None, min_data: float = 0.0,
                          as_counts: bool = False):
        """freq.py --target derived|minor -> (values float64 [n,P], tie bool [n])."""
        n = self.S - site0 if n is None else n
        out = np.empty((n, self.P), dtype=np.float64)
        tie = np.zeros(n, dtype=np.uint8)
        code = {"derived": 1, "minor": 2}[target]
        check(self._lib.pg_site_target_freqs(self._ctx, int(site0), int(n), code, float(min_data), 1 if as_counts else 0,
                                             _ptr(out), _ptr(tie)), "pg_site_target_freqs")
        return out, tie.astype(bool)

    def sfs(self, n_in: int, groups, pop_sizes, outgroup: int = -1, site_mask=None):
        """sfs.py for genotype input: `groups` = list of tuples of in-group population indices; pop_sizes[X] = haplotypes of
        population X.  Returns (list of dense int64 spectra shaped (N_k+1, ...), list of first-site arrays, sites counted)."""
        goff = np.zeros(len(groups) + 1, dtype=np.int32)
        for k, grp in enumerate(groups):
            goff[k + 1] = goff[k] + len(grp)
        gp = np.array([x for grp in groups for x in grp], dtype=np.int32)
        shapes = [tuple(int(pop_sizes[x]) + 1 for x in grp) for grp in groups]
        cells = [int(np.prod([int(d) for d in sh], dtype=object)) for sh in shapes]
        _check_sfs_cells(cells)
        hist = np.zeros(sum(cells), dtype=np.int64)
        first = np.zeros(sum(cells), dtype=np.int64)
        mask = None if site_mask is None else np.ascontiguousarray(site_mask, dtype=np.uint8)
        if mask is not None:
            assert mask.shape == (self.S,)
        n = C.c_int64(0)
        check(self._lib.pg_sfs(self._ctx, int(n_in), int(outgroup), len(groups), _ptr(goff), _ptr(gp), _ptr(mask), _ptr(hist),
                               _ptr(first), C.byref(n)), "pg_sfs")
        offs = np.concatenate([[0], np.cumsum(cells)])
        return ([hist[offs[k]:offs[k + 1]].reshape(shapes[k]) for k in range(len(groups))],
                [first[offs[k]:offs[k + 1]].reshape(shapes[k]) for k in range(len(groups))], int(n.value))

    def sfs_tables(self, kind: str, table, n_in: int, groups, outgroup: int = -1, site_mask=None):
        """sfs.py on count tables: kind "base" = uint16 [n,P,4] base counts per population, "target" = int32 [n,P] counts of
        the target allele.  Returns (dense spectra, first-site arrays, sites counted) like sfs()."""
        if kind == "base":
            table = np.ascontiguousarray(table, dtype=np.uint16)
            n, P = table.shape[0], table.shape[1]
            dims = (table.sum(axis=2, dtype=np.int64).max(axis=0) + 1 if n else np.ones(P, np.int64)).astype(np.int32)
        else:
            table = np.ascontiguousarray(table, dtype=np.int32)
            n, P = table.shape
            dims = (table.max(axis=0) + 1 if n else np.ones(P, np.int64)).astype(np.int32)
            assert n == 0 or table.min() >= 0
        goff = np.zeros(len(groups) + 1, dtype=np.int32)
        for k, grp in enumerate(groups):
            goff[k + 1] = goff[k] + len(grp)
        gp = np.array([x for grp in groups for x in grp], dtype=np.int32)
        shapes = [tuple(int(dims[x]) for x in grp) for grp in groups]
        cells = [int(np.prod([int(d) for d in sh], dtype=object)) for sh in shapes]
        _check_sfs_cells(cells)
        hist = np.zeros(sum(cells), dtype=np.int64)
        first = np.zeros(sum(cells), dtype=np.int64)
        mask = None if site_mask is None else np.ascontiguousarray(site_mask, dtype=np.uint8)
        cnt = C.c_int64(0)
        check(self._lib.pg_sfs_tables(self._ctx, 0 if kind == "base" else 1, _ptr(table), int(n), int(P), _ptr(dims), int(n_in),
                                      int(outgroup), len(groups), _ptr(goff), _ptr(gp), _ptr(mask), _ptr(hist), _ptr(first),
                                      C.byref(cnt)), "pg_sfs_tables")
        offs = np.concatenate([[0], np.cumsum(cells)])
        return ([hist[offs[k]:offs[k + 1]].reshape(shapes[k]) for k in range(len(groups))],
                [first[offs[k]:offs[k + 1]].reshape(shapes[k]) for k in range(len(groups))], int(cnt.value))

    def _sfs_sparse_fetch(self, nnz, shapes):
        total = int(nnz.sum())
        cell = np.empty(total, dtype=np.int64)
        count = np.empty(total, dtype=np.int64)
        first = np.empty(total, dtype=np.int64)
        check(self._lib.pg_sfs_sparse_fetch(self._ctx, total, _ptr(cell), _ptr(count), _ptr(first)), "pg_sfs_sparse_fetch")
        offs = np.concatenate([[0], np.cumsum(nnz)])
        return [(sfs_unravel(cell[offs[k]:offs[k + 1]], shapes[k]), count[offs[k]:offs[k + 1]], first[offs[k]:offs[k + 1]])
                for k in range(len(shapes))]

    def sfs_sparse(self, n_in: int, groups, pop_sizes, outgroup: int = -1, site_mask=None):
        """sfs() without dense histograms (any number of cells): returns (per spectrum (coords int64 [nnz, d], count int64
        [nnz], first site int64 [nnz]) with cells in row-major order, sites counted)."""
        goff, gp = _sfs_group_tables(groups)
        shapes, _ = sfs_shapes(groups, [int(x) + 1 for x in pop_sizes])
        mask = None if site_mask is None else np.ascontiguousarray(site_mask, dtype=np.uint8)
        if mask is not None:
            assert mask.shape == (self.S,)
        nnz = np.zeros(len(groups), dtype=np.int64)
        n = C.c_int64(0)
        check(self._lib.pg_sfs_sparse(self._ctx, int(n_in), int(outgroup), len(groups), _ptr(goff), _ptr(gp), _ptr(mask),
                                      _ptr(nnz), C.byref(n)), "pg_sfs_sparse")
        return self._sfs_sparse_fetch(nnz, shapes), int(n.value)

    def sfs_tables_sparse(self, kind: str, table, n_in: int, groups, outgroup: int = -1, site_mask=None):
        """sfs_tables() without dense histograms: returns (per spectrum (coords, count, first) as sfs_sparse(), sites
        counted)."""
        table, dims = sfs_table_dims(kind, table)
        n, P = table.shape[0], table.shape[1]
        goff, gp = _sfs_group_tables(groups)
        shapes, _ = sfs_shapes(groups, dims)
        mask = None if site_mask is None else np.ascontiguousarray(site_mask, dtype=np.uint8)
        nnz = np.zeros(len(groups), dtype=np.int64)
        cnt = C.c_int64(0)
        check(self._lib.pg_sfs_tables_sparse(self._ctx, 0 if kind == "base" else 1, _ptr(table), int(n), int(P), _ptr(dims),
                                             int(n_in), int(outgroup), len(groups), _ptr(goff), _ptr(gp), _ptr(mask),
                                             _ptr(nnz), C.byref(cnt)), "pg_sfs_tables_sparse")
        return self._sfs_sparse_fetch(nnz, shapes), int(cnt.value)

    def pairdist(self, hap_ind, n_ind: int, include_same_with_same: bool = False, min_sites: int = 0, out=None):
        """-> dict(dist [W,n_ind,n_ind], sites [W], pos_sum [W]).  min_sites > 0 masks haplotype pairs with fewer
        jointly non-missing sites (what an earlier groupDistStats does to the reference's cached matrix).
        `out`: a caller-owned float64 [W, n_ind, n_ind] array; a PinnedArray's `.array` is written by the copy engine
        directly (hundreds of MB of matrices otherwise spend most of their time in page faults of a fresh array)."""
        hap_ind = np.ascontiguousarray(hap_ind, dtype=np.int32)
        assert hap_ind.shape == (self.H,)
        W = self.W
        if out is not None:
            assert out.dtype == np.float64 and out.flags.c_contiguous and out.shape == (W, n_ind, n_ind)
        dist = out if out is not None else np.empty((W, n_ind, n_ind), dtype=np.float64)
        sites = np.empty(W, dtype=np.int64)
        pos_sum = np.empty(W, dtype=np.int64)
        check(self._lib.pg_pairdist(self._ctx, int(n_ind), _ptr(hap_ind), 1 if include_same_with_same else 0,
                                    int(min_sites or 0), _ptr(dist), _ptr(sites), _ptr(pos_sum)), "pg_pairdist")
        return dict(dist=dist, sites=sites, pos_sum=pos_sum)

    def distpaint(self, query_hap, ref_off, ref_hap, min_sites: int, delta: bool = False, threshold: float = 0.05,
                  noresult: int = -1, with_stats: bool = False):
        """distPaint.py's assignment of every query haplotype to its nearest reference population, per window ->
        dict(assign int32 [W, n_query]) and, with_stats, means / pvals float64 [W, n_query, P].  Populations are
        CSR: population p's member haplotypes are ref_hap[ref_off[p]:ref_off[p + 1]] (an ordered list; duplicates count
        twice).  delta: the delta rule with `threshold`, else the rank-sum rule with p-value threshold `threshold`.
        Windows without sites hold noresult (and nan statistics); the caller decides what to write for them."""
        query_hap = np.ascontiguousarray(query_hap, dtype=np.int32)
        ref_off = np.ascontiguousarray(ref_off, dtype=np.int32)
        ref_hap = np.ascontiguousarray(ref_hap, dtype=np.int32)
        W, nq, P = self.W, len(query_hap), len(ref_off) - 1
        assign = np.full((W, nq), int(noresult), dtype=np.int32)
        means = np.full((W, nq, P), np.nan) if with_stats else None
        pvals = np.full((W, nq, P), np.nan) if with_stats else None
        check(self._lib.pg_distpaint(self._ctx, nq, _ptr(query_hap), P, _ptr(ref_off), _ptr(ref_hap), int(min_sites),
                                     1 if delta else 0, float(threshold), int(noresult), _ptr(assign), _ptr(means),
                                     _ptr(pvals)), "pg_distpaint")
        out = dict(assign=assign)
        if with_stats:
            out.update(means=means, pvals=pvals)
        return out

    def pairdist_cat(self, hap_ind, n_ind: int, include_same_with_same: bool = False):
        """distMat.py --windType cat: one matrix over every uploaded site (summed over the ranks of the NCCL
        communicator when one is set) -> (dist [n_ind,n_ind], total_sites)."""
        hap_ind = np.ascontiguousarray(hap_ind, dtype=np.int32)
        assert hap_ind.shape == (self.H,)
        dist = np.empty((n_ind, n_ind), dtype=np.float64)
        tot = C.c_int64(0)
        check(self._lib.pg_pairdist_cat(self._ctx, int(n_ind), _ptr(hap_ind), 1 if include_same_with_same else 0,
                                        _ptr(dist), C.byref(tot)), "pg_pairdist_cat")
        return dist, int(tot.value)

    def seq_nonnan(self):
        """Alignment.seqNonNan() per window -> int64 [W, H]."""
        out = np.empty((self.W, self.H), dtype=np.int64)
        check(self._lib.pg_seq_nonnan(self._ctx, _ptr(out)), "pg_seq_nonnan")
        return out

    def ind_het(self, hap_ind, n_ind: int, min_sites: int = 0):
        """Alignment.sampleHet() per window -> [W, n_ind]."""
        hap_ind = np.ascontiguousarray(hap_ind, dtype=np.int32)
        assert hap_ind.shape == (self.H,)
        het = np.empty((self.W, n_ind), dtype=np.float64)
        check(self._lib.pg_ind_het(self._ctx, int(n_ind), _ptr(hap_ind), int(min_sites or 0), _ptr(het)), "pg_ind_het")
        return het

    def hapstats(self, max_dist: float = 0.0, min_sites: int = 0, diag_nan: bool = False):
        """Alignment.H12stats(maxDist) per window -> [W, P, 3] = H1, H12, H2."""
        out = np.empty((self.W, self.P, 3), dtype=np.float64)
        check(self._lib.pg_hapstats(self._ctx, float(max_dist), int(min_sites or 0), 1 if diag_nan else 0, _ptr(out)),
              "pg_hapstats")
        return out

    def pair_counts(self, window: int):
        """(diff, n) int32 [H,H] of one window (Alignment.distMatrix / pairNonNan numerators)."""
        diff = np.empty((self.H, self.H), dtype=np.int32)
        n = np.empty((self.H, self.H), dtype=np.int32)
        check(self._lib.pg_pair_counts(self._ctx, int(window), _ptr(diff), _ptr(n)), "pg_pair_counts")
        return diff, n

    # ---- introspection ----
    def last_timings(self):
        cap = 32
        names = (C.c_char * 32 * cap)()
        ms = (C.c_float * cap)()
        launches = (C.c_int32 * cap)()
        cnt = C.c_int32(0)
        check(self._lib.pg_last_timings(self._ctx, cap, names, ms, launches, C.byref(cnt)), "pg_last_timings")
        return {names[k].value.decode(): dict(ms=float(ms[k]), launches=int(launches[k])) for k in range(cnt.value)}

    def launch_count(self) -> int:
        n = C.c_int64(0)
        check(self._lib.pg_launch_count(self._ctx, C.byref(n)), "pg_launch_count")
        return int(n.value)

    def packed_rows(self, site0: int, n: int):
        """uint32 [n, 3, ceil(H / 32)] rows of the packed companion (valid bits, low and high allele-code bit; haplotype h at
        bit h % 32 of word h / 32), or None when the context has no companion."""
        words = C.c_int32(0)
        check(self._lib.pg_debug_packed(self._ctx, int(site0), int(n), C.byref(words), None), "pg_debug_packed")
        if words.value == 0:
            return None
        out = np.empty((n, words.value), dtype=np.uint32)
        check(self._lib.pg_debug_packed(self._ctx, int(site0), int(n), C.byref(words), _ptr(out)), "pg_debug_packed")
        wd = (self.H + 31) // 32
        return out[:, :3 * wd].reshape(n, 3, wd)

    def site_classes(self, site0: int, n: int):
        """uint8 [n] class bytes of the packed companion's rows (0 varied, 1..4 all A / C / G / T, 5 all missing, 6 / 7 every
        haplotype called and exactly two alleles, differing in the low / high allele-code bit), or None when it keeps none."""
        avail = C.c_int32(0)
        out = np.empty(int(n), dtype=np.uint8)
        check(self._lib.pg_debug_site_cls(self._ctx, int(site0), int(n), C.byref(avail), _ptr(out)), "pg_debug_site_cls")
        return out if avail.value else None

    def uniform_stream(self):
        """(in_use, varied_sites): whether the last popgen call's site pass streamed only the packed rows of the sites whose
        haplotypes are not all the same, and how many such sites it counted (S when it did not count them)."""
        in_use, varied = C.c_int32(0), C.c_int64(0)
        check(self._lib.pg_debug_uniform(self._ctx, C.byref(in_use), C.byref(varied)), "pg_debug_uniform")
        return bool(in_use.value), int(varied.value)

    def uniform_rows(self):
        """(one-plane rows, words of all rows) of the varied-row stream the last popgen call read ((0, 0) when it did not)."""
        n1, words = C.c_int64(0), C.c_int64(0)
        check(self._lib.pg_debug_uniform_rows(self._ctx, C.byref(n1), C.byref(words)), "pg_debug_uniform_rows")
        return int(n1.value), int(words.value)

    def uniform_tile(self):
        """(sites per tile, warps per tile) of the varied-row stream's launch plan, as the last popgen call on the packed
        companion made it ((0, 0) before any)."""
        v = (C.c_int32 * 2)()
        check(self._lib.pg_debug_uniform_tile(self._ctx, v), "pg_debug_uniform_tile")
        return int(v[0]), int(v[1])

    def uniform_ring(self):
        """(varied rows per tile at most, stages, bytes per stage) of the ring the last popgen call streamed the varied rows
        through ((0, 0, 0) when it did not read the stream)."""
        v = (C.c_int32 * 3)()
        check(self._lib.pg_debug_uniform_ring(self._ctx, v), "pg_debug_uniform_ring")
        return int(v[0]), int(v[1]), int(v[2])

    def uniform_launch(self):
        """(CTAs, consumer warps per CTA, 1 when the one-plane rows were summed as a Gram) of the varied-row stream's launch
        in the last popgen call ((0, 0, 0) when it did not read the stream)."""
        v = (C.c_int32 * 3)()
        check(self._lib.pg_debug_uniform_launch(self._ctx, v), "pg_debug_uniform_launch")
        return int(v[0]), int(v[1]), int(v[2])

    def uniform_tiles(self):
        """(R, Tmax, site_lo, row0) of the varied-row stream the last popgen call read: tile t covers the sites
        [site_lo[t], site_lo[t + 1]) and the varied rows [row0[t], row0[t + 1]); None when it did not read the stream."""
        nt, geo = C.c_int64(0), (C.c_int32 * 2)()
        check(self._lib.pg_debug_uniform_tiles(self._ctx, 0, None, None, C.byref(nt), geo), "pg_debug_uniform_tiles")
        if nt.value == 0:
            return None
        site_lo = np.empty(nt.value + 1, np.int64)
        row0 = np.empty(nt.value + 1, np.int64)
        check(self._lib.pg_debug_uniform_tiles(self._ctx, nt.value + 1, _ptr(site_lo), _ptr(row0), C.byref(nt), geo),
              "pg_debug_uniform_tiles")
        return int(geo[0]), int(geo[1]), site_lo, row0


def k1_plan(S: int, H: int, nw: int = 8, lanes: int = 0, table_bytes: int = 4096):
    """Host-only: the site-pass launch geometry for a shape (works without a GPU).  `nw` consumer warps per CTA (8, or 12
    for rows under 1 KiB by default), `lanes` > 0 forces the lanes per site (the lane-per-population variant uses one lane
    per population), `table_bytes` of mask tables share the shared memory.  The PG_K1_* geometry overrides apply, as they
    do to the launches.  `ok` is False for rows the site pass refuses."""
    v = (C.c_int32 * 9)()
    check(_lib.lib().pg_debug_k1_plan_ex(int(S), int(H), int(nw), int(lanes), int(table_bytes), v), "pg_debug_k1_plan_ex")
    return dict(pitch=v[0], lanes_per_site=v[1], warps_per_tile=v[2], sites_per_lane=v[3], tile_sites=v[4], stages=v[5],
                smem_bytes=v[6], ctas=v[7], ok=bool(v[8]))
