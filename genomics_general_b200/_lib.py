"""ctypes binding of libpgwin.so (C-ABI: include/pgwin.h).

There is no CPU fallback: if the shared library is missing, or no CUDA device is present when a
context is created, this raises.  ``build()`` compiles the library in-tree with nvcc for sm_90a (H100).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpgwin.so")
CSRC = os.path.join(_HERE, "csrc")

_lib = None


class PgError(RuntimeError):
    pass


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile csrc/*.cu -> libpgwin.so (nvcc, -gencode arch=compute_90a,code=sm_90a -lineinfo)."""
    srcs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".h", ".cpp"))]
    srcs.append(os.path.join(_HERE, "..", "include", "pgwin.h"))
    if not force and os.path.exists(LIB_PATH):
        newest = max(os.path.getmtime(s) for s in srcs)
        if os.path.getmtime(LIB_PATH) >= newest:
            return LIB_PATH
    cmd = ["make", "-C", CSRC, "-j4"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if verbose or r.returncode != 0:
        print(r.stdout)
    if r.returncode != 0:
        raise PgError("building libpgwin.so failed (nvcc for sm_90a)")
    return LIB_PATH


_SIGS = {
    "pg_version": (C.c_int, []),
    "pg_last_error": (C.c_char_p, []),
    "pg_device_count": (C.c_int, [C.POINTER(C.c_int)]),
    "pg_ctx_create": (C.c_int, [C.c_int, C.POINTER(C.c_void_p)]),
    "pg_ctx_destroy": (C.c_int, [C.c_void_p]),
    "pg_host_alloc": (C.c_int, [C.POINTER(C.c_void_p), C.c_size_t]),
    "pg_host_free": (C.c_int, [C.c_void_p]),
    "pg_upload": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]),
    "pg_alloc_sites": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32]),
    "pg_upload_range": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "pg_append_sites": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "pg_synth_fill": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_uint64, C.c_uint64,
                                C.c_uint64, C.c_uint64, C.c_uint64, C.c_int32]),
    "pg_download": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "pg_set_pops": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p]),
    "pg_set_windows": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "pg_popgen": (C.c_int, [C.c_void_p, C.c_int32, C.c_double, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                            C.c_void_p, C.c_void_p, C.c_void_p]),
    "pg_popgen_device": (C.c_int, [C.c_void_p, C.c_int32, C.c_double, C.c_int32, C.c_void_p, C.POINTER(C.c_int64)]),
    "pg_popgen_freqstats": (C.c_int, [C.c_void_p] * 6),
    "pg_set_freqstats": (C.c_int, [C.c_void_p, C.c_int32]),
    "pg_abbababa": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_void_p,
                              C.c_void_p, C.c_void_p, C.c_void_p]),
    "pg_fourpop": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_int32, C.c_void_p,
                             C.c_void_p, C.c_void_p, C.c_void_p]),
    "pg_site_counts": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]),
    "pg_site_target_freqs": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_double, C.c_int32, C.c_void_p,
                                       C.c_void_p]),
    "pg_sfs": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                         C.c_void_p, C.POINTER(C.c_int64)]),
    "pg_sfs_tables": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_int32,
                                C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64)]),
    "pg_sfs_sparse": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.POINTER(C.c_int64)]),
    "pg_sfs_tables_sparse": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32,
                                       C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.POINTER(C.c_int64)]),
    "pg_sfs_sparse_fetch": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pg_pairdist": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                              C.c_void_p]),
    "pg_distpaint": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                               C.c_double, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pg_pairdist_cat": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(C.c_int64)]),
    "pg_seq_nonnan": (C.c_int, [C.c_void_p, C.c_void_p]),
    "pg_ind_het": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "pg_hapstats": (C.c_int, [C.c_void_p, C.c_double, C.c_int32, C.c_int32, C.c_void_p]),
    "pg_pair_counts": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "pg_last_timings": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]),
    "pg_launch_count": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64)]),
    "pg_debug_k1_plan": (C.c_int, [C.c_int64, C.c_int32] + [C.POINTER(C.c_int32)] * 5),
    "pg_debug_k1_plan_ex": (C.c_int, [C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int32)]),
    "pg_debug_packed": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.POINTER(C.c_int32), C.c_void_p]),
    "pg_debug_site_cls": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.POINTER(C.c_int32), C.c_void_p]),
    "pg_debug_uniform": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]),
    "pg_debug_uniform_tile": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32)]),
    "pg_debug_uniform_rows": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "pg_debug_uniform_ring": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32)]),
    "pg_debug_uniform_launch": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32)]),
    "pg_debug_uniform_tiles": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64),
                                         C.POINTER(C.c_int32)]),
    "pg_nccl_unique_id": (C.c_int, [C.c_void_p]),
    "pg_nccl_init": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    "pg_nccl_finalize": (C.c_int, [C.c_void_p]),
    "pg_popgen_gather_begin": (C.c_int, [C.c_void_p, C.c_int32, C.c_double, C.c_int64, C.c_int32]),
    "pg_popgen_gather_end": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]),
    "pg_popgen_allgather": (C.c_int, [C.c_void_p, C.c_int32, C.c_double, C.c_int32, C.c_int64, C.c_void_p,
                                      C.POINTER(C.c_int64)]),
    "pg_ingest_file": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                                 C.POINTER(C.c_int64)]),
    "pg_ingest_file_range": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                       C.c_int32, C.POINTER(C.c_int64)]),
    "pg_ingest_text": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                                 C.POINTER(C.c_int64)]),
    "pg_ingest_meta": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pg_ingest_release": (C.c_int, [C.c_void_p]),
    "pg_ingest_set_strict": (C.c_int, [C.c_void_p, C.c_int32]),
    "pg_debug_ingest": (C.c_int, [C.c_void_p, C.c_void_p]),
    "pg_filter": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_uint8)]),
    "pg_filter_emit": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_void_p, C.c_size_t, C.POINTER(C.c_int64),
                                 C.POINTER(C.c_size_t)]),
    "pg_filter_stats": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64] + [C.c_void_p] * 8),
    "pg_format_freq_rows": (C.c_int, [C.c_int32, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_size_t, C.c_int32, C.c_void_p]),
    "pg_format_matrix_rows": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_size_t,
                                        C.c_int32, C.c_void_p]),
    "pg_abbababa_allgather": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_int64,
                                        C.c_void_p]),
    "pg_fourpop_allgather": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_int32,
                                       C.c_int64, C.c_void_p]),
    "pg_vcf_set_spec": (C.c_int, [C.c_void_p, C.c_void_p]),
    "pg_vcf_load": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, C.c_char_p, C.c_int32, C.c_int32, C.POINTER(C.c_int64)]),
    "pg_vcf_lines": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]),
    "pg_vcf_genotypes": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_uint64)]),
    "pg_vcf_verdicts": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "pg_vcf_emit": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_size_t, C.POINTER(C.c_int64), C.POINTER(C.c_size_t)]),
    "pg_seq_index": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, C.c_char_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32,
                               C.c_void_p, C.c_int32, C.POINTER(C.c_int64), C.c_void_p]),
    "pg_seq_meta": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pg_seq_plan": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_char_p, C.c_void_p, C.c_void_p, C.c_void_p,
                              C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.c_void_p]),
    "pg_seq_emit": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_size_t, C.POINTER(C.c_int64),
                              C.POINTER(C.c_int64), C.POINTER(C.c_size_t)]),
    "pg_g2v_ref_load": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, C.POINTER(C.c_int64)]),
    "pg_g2v_ref_starts": (C.c_int, [C.c_void_p, C.c_void_p]),
    "pg_g2v_ref_index": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pg_g2v_spec": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32]),
    "pg_g2v_chunk": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "pg_g2v_runs": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "pg_g2v_sites": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_void_p]),
    "pg_g2v_emit": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "pg_s2g_fasta_load": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, C.POINTER(C.c_int64)]),
    "pg_s2g_fasta_starts": (C.c_int, [C.c_void_p, C.c_void_p]),
    "pg_s2g_fasta_index": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pg_s2g_phylip_load": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, C.POINTER(C.c_int64)]),
    "pg_s2g_phylip_lines": (C.c_int, [C.c_void_p, C.c_void_p]),
    "pg_s2g_phylip_pack": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]),
    "pg_s2g_plan": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_char_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p,
                              C.POINTER(C.c_int64)]),
    "pg_s2g_emit": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "pg_ws_spec": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32]),
    "pg_ws_chunk": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                              C.POINTER(C.c_int64), C.c_void_p]),
    "pg_ws_chunk_info": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pg_ws_set_values": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pg_ws_meta": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64), C.c_void_p]),
    "pg_ws_stats": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64,
                              C.c_void_p, C.c_void_p]),
    "pg_merge_setup": (C.c_int, [C.c_void_p, C.c_int64, C.c_char_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                 C.c_void_p, C.c_char_p, C.c_int32, C.c_char_p, C.c_int32, C.c_int32, C.c_int64, C.c_int64,
                                 C.POINTER(C.c_int32)]),
    "pg_merge_load": (C.c_int, [C.c_void_p, C.c_int32, C.c_char_p, C.c_size_t, C.c_void_p]),
    "pg_merge_rows": (C.c_int, [C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "pg_merge_emit": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "pg_geno_count_lines": (C.c_int, [C.c_char_p, C.c_size_t, C.POINTER(C.c_int64)]),
    "pg_geno_parse": (C.c_int, [C.c_char_p, C.c_size_t, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                                C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32]),
}

EXPORTS = tuple(_SIGS)


class FilterSpec(C.Structure):
    """pg_filter_spec (include/pgwin.h)"""
    _fields_ = [("n_samp", C.c_int32), ("samp_hap0", C.c_void_p), ("samp_ploidy", C.c_void_p), ("P", C.c_int32),
                ("pop_off", C.c_void_p), ("pop_members", C.c_void_p), ("min_calls", C.c_int32), ("min_alleles", C.c_int32), ("max_alleles", C.c_double),
                ("min_var_count", C.c_int32), ("has_max_het", C.c_int32), ("max_het", C.c_double),
                ("min_freq", C.c_double), ("max_freq", C.c_double), ("min_pop_calls", C.c_void_p),
                ("min_pop_alleles", C.c_void_p), ("max_pop_alleles", C.c_void_p), ("fixed_diffs", C.c_int32),
                ("has_nearly_fixed", C.c_int32), ("nearly_fixed_diff", C.c_double), ("partial_to_missing", C.c_int32),
                ("no_test", C.c_int32), ("thin_dist", C.c_int32), ("pod_size", C.c_int32)]


class VcfSpec(C.Structure):
    """pg_vcf_spec (include/pgwin.h)"""
    _fields_ = [("n_cols", C.c_int32), ("col_slot", C.c_void_p), ("col_prev", C.c_void_p), ("n_keys", C.c_int32),
                ("key_off", C.c_void_p), ("key_chars", C.c_void_p), ("n_samp", C.c_int32), ("samp_col", C.c_void_p),
                ("samp_ploidy", C.c_void_p), ("field_key", C.c_int32), ("field_phase", C.c_int32), ("n_filt", C.c_int32),
                ("filt_key", C.c_void_p), ("filt_min", C.c_void_p), ("filt_max", C.c_void_p), ("filt_site", C.c_void_p),
                ("filt_gt", C.c_void_p), ("filt_samp", C.c_void_p), ("has_min_qual", C.c_int32), ("min_qual", C.c_double),
                ("missing", C.c_void_p), ("missing_len", C.c_int32), ("sep", C.c_void_p), ("sep_len", C.c_int32),
                ("skip_indels", C.c_int32), ("keep_partial", C.c_int32), ("ploidy_mismatch_to_missing", C.c_int32),
                ("add_ref_track", C.c_int32)]


# pg_vcf_line (include/pgwin.h) as a numpy record
VCF_LINE = np.dtype([("start", np.int64), ("end", np.int64), ("pos", np.int64)] +
                    [(n, np.uint32) for n in ("chrom_off", "chrom_len", "pos_off", "pos_len", "ref_off", "ref_len", "alt_off",
                                              "alt_len", "qual_off", "qual_len", "fmt_off", "fmt_len")] +
                    [("n_fields", np.int32), ("n_alt", np.int32), ("flags", np.uint32), ("reserved", np.uint32)])
VCF_NONASCII, VCF_POS_UNRESOLVED, VCF_QUAL_DROP, VCF_QUAL_UNRESOLVED, VCF_SAME_LEN, VCF_DUPLICATE, VCF_FORMAT_WIDE = \
    1, 2, 4, 8, 16, 32, 64


def lib():
    """Load libpgwin.so (once).  Raises PgError when it has not been built — never falls back."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise PgError("libpgwin.so is not built (%s). Run `python -c 'import __graft_entry__ as g; g.build()'` or "
                      "`make -C genomics_general_b200/csrc`. There is no CPU fallback." % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    for name, (res, args) in _SIGS.items():
        fn = getattr(L, name)          # AttributeError here means the header and the library diverged
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = lib().pg_last_error()
        raise PgError("%s failed: %s" % (what or "libpgwin call", msg.decode() if msg else "unknown error"))
