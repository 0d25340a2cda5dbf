/*
 * pgwin.h — C-ABI of libpgwin.so: the H100 (sm_90a) engine for the per-window / per-site numerics of
 * simonhmartin/genomics_general (popgenWindows.py / ABBABABAwindows.py / fourPopWindows.py / freq.py / sfs.py /
 * distMat.py) and for the .geno text parsing in front of them.
 *
 * The reference has no FFI: its seam is the Python API of genomics.py as used by the four scripts
 * (SURVEY.md §8b).  Each entry point below names the reference code it replaces
 * (genomics_general/<file>:<line>).  The binding a maintainer would add is a ctypes stub —
 * see INTEGRATION.md and genomics_general_b200/_lib.py.
 *
 * Conventions
 *   - every function returns 0 on success, non-zero on error; pg_last_error() gives the message of the
 *     last failure on the calling thread.
 *   - the caller owns every host buffer; the library owns device memory behind the opaque pg_ctx.
 *   - one ctx per device; calls on one ctx are not thread-safe; different ctxs are independent.
 *   - genotype codes: A=0 C=1 G=2 T=3, missing = any value with bit 7 set (canonically -1).
 *     This is Alignment.numArray (genomics.py:74-77, 834) narrowed to int8 and transposed to
 *     site-major: geno[site * H + hap].
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails.
 */
#ifndef PGWIN_H
#define PGWIN_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pg_ctx pg_ctx;

/* ---- library / context ------------------------------------------------------------------------ */
int         pg_version(void);
const char* pg_last_error(void);
int         pg_device_count(int* n);
int         pg_ctx_create(int device, pg_ctx** out);
int         pg_ctx_destroy(pg_ctx* ctx);
/* pinned host memory for the end-to-end path (H2D from pinned buffers) */
int         pg_host_alloc(void** ptr, size_t bytes);
int         pg_host_free(void* ptr);

/* ---- data in ---------------------------------------------------------------------------------- */
/* Replaces genoToAlignment + Alignment.__init__ (genomics.py:1101-1127, 813-869): the dense matrix of
 * a whole file (or shard).  geno: int8 [S x H] site-major, pos: int32 [S] (may be NULL -> zeros).
 * Copies host->device (pitched so that rows are 16-byte multiples). */
int pg_upload(pg_ctx* ctx, const int8_t* geno, int64_t S, int32_t H, const int32_t* pos);
/* Two-step variant: allocate, then fill site ranges (each call is an async H2D on the ctx stream). */
int pg_alloc_sites(pg_ctx* ctx, int64_t S, int32_t H);
int pg_upload_range(pg_ctx* ctx, int64_t site0, int64_t n, const int8_t* geno, const int32_t* pos);
/* Appends n sites (int8 [n x H], reference codes; pos int32 [n] or NULL) after the resident ones; the matrix grows.  Used by
 * the multi-GPU command lines for the halo sites of windows that reach into the next rank's share of the file. */
int pg_append_sites(pg_ctx* ctx, int64_t n, const int8_t* geno, const int32_t* pos);
/* Device-side synthetic data (SURVEY.md §8d distribution; bit-identical to synth.py::synth_genotypes /
 * synth_positions).  Thresholds are 32-bit integer probabilities (p * 2^32). */
int pg_synth_fill(pg_ctx* ctx, int64_t S, int32_t n_pops, int32_t samples_per_pop, int32_t ploidy,
                  uint64_t seed, uint64_t thr_var, uint64_t thr_out0, uint64_t thr_third, uint64_t thr_miss,
                  int32_t spacing);
/* Device -> host copy of a site range (tests / building host buffers for the e2e bench). */
int pg_download(pg_ctx* ctx, int64_t site0, int64_t n, int8_t* geno, int32_t* pos);

/* Replaces SampleData/Alignment.groups (genomics.py:1264-1290, 857-861): hap_pop[h] in [0,P) or -1. */
int pg_set_pops(pg_ctx* ctx, int32_t P, const int32_t* hap_pop);
/* Replaces the window generators' output (genomics.py:1971-2171): half-open site-index ranges
 * [lo[w], hi[w]) computed on the host with the generators' exact semantics (windows.py). Ranges may
 * overlap and may be empty. */
int pg_set_windows(pg_ctx* ctx, int64_t W, const int64_t* lo, const int64_t* hi);

/* ---- statistics ------------------------------------------------------------------------------- */
/* Replaces Alignment.groupDistStats (genomics.py:956-995) + the sites/mid bookkeeping of
 * popgenWindows.py:37-41 for every window.
 *   pi  [W x P], dxy/fst [W x P(P-1)/2] (pairs in (0,1),(0,2),..,(1,2).. order), n_sites [W],
 *   pos_sum [W] (sum of positions, for midPos genomics.py:1795), path [W]: 0 = failed (sites < minSites),
 *   1 = closed-form allele-count path (K1), 2 = pairwise path (K2).
 * force_path: 0 = route per window (K1 when exact, else K2), 2 = pairwise for every window.
 * min_sites <= 0 disables the n_ij < minSites mask (genomics.py:958). */
int pg_popgen(pg_ctx* ctx, int32_t min_sites, double min_data, int32_t force_path,
              double* pi, double* dxy, double* fst, int64_t* n_sites, int64_t* pos_sum, int32_t* path);

/* Same statistics, left on the DEVICE as fixed-width records (so that the multi-GPU all-gather can read
 * them in place): d_rec is a device buffer of W * (4 + 5P + 2*npairs) 8-byte words per window,
 *   [sites (int64), pos_sum (int64), path (int64), pi[P], dxy[npairs], fst[npairs],
 *    l, S[P], thetaPi[P], thetaW[P], TajD[P]] (statistics are doubles).
 * *n_pairwise (optional) receives the number of windows that went through the pairwise path. */
int pg_popgen_device(pg_ctx* ctx, int32_t min_sites, double min_data, int32_t force_path, void* d_rec,
                     int64_t* n_pairwise);

/* Replaces Alignment.groupFreqStats (genomics.py:1002-1028; popgenWindows --analysis popFreq): the columns
 * computed alongside by the most recent pg_popgen call on this ctx (after pg_set_freqstats(ctx, 1)).  l [W] = sites complete in every haplotype
 * that belongs to a population; S, theta_pi, theta_w, taj_d [W x P]. */
int pg_popgen_freqstats(pg_ctx* ctx, double* l, double* S, double* theta_pi, double* theta_w, double* taj_d);
/* The popFreq counters cost ~4 % of the site pass, so they are opt-in: enable before pg_popgen. */
int pg_set_freqstats(pg_ctx* ctx, int32_t enable);

/* Replaces genomics.ABBABABA (genomics.py:1647-1695, polarize=True) per window.
 * out [W x 5] = ABBA, BABA, D, fd, fdM; sites_used [W] (double: nan when the window has no good site,
 * genomics.py:1694-1695); n_sites/pos_sum as above. p1,p2,p3,o are population indices of pg_set_pops. */
int pg_abbababa(pg_ctx* ctx, int32_t p1, int32_t p2, int32_t p3, int32_t o, double min_data,
                double* out, double* sites_used, int64_t* n_sites, int64_t* pos_sum);

/* Replaces genomics.fourPop (genomics.py:1585-1643; fourPopWindows.py:27-52) per window.
 * out [W x 14] = fhom, fhom', D, fd, fd', fdm, fdm', fdh, fdh2, fh, ABBA, BABA, ABAA, BAAA; sites_used [W] (0 when the
 * window has no good site, 1641-1643).  mode 0 = default (the allele np.argsort(all4freqs)[:,2] picks, i.e. the rarer of
 * the two; on an exact tie the reference depends on numpy's sort implementation — here the lower allele index),
 * 1 = polarize (allele absent from P4), 2 = fixed (polarize + P1,P2,P3 each fixed). */
int pg_fourpop(pg_ctx* ctx, int32_t p1, int32_t p2, int32_t p3, int32_t p4, double min_data, int32_t mode,
               double* out, double* sites_used, int64_t* n_sites, int64_t* pos_sum);

/* Replaces Alignment.siteFreqs(asCounts=True) per population (genomics.py:1049-1052; freq.py:52-58):
 * counts uint16 [n x P x 4] (A,C,G,T) for sites site0 .. site0+n-1. */
int pg_site_counts(pg_ctx* ctx, int64_t site0, int64_t n, uint16_t* counts);

/* Replaces freq.py --target derived|minor (freq.py:62-92; derivedAllele / minorAllele genomics.py:636-668):
 * out double [n x P] = frequency (count/non-missing; nan = no value) or, with as_counts, count (0 = no value) of the
 * target allele in each population.  target 1 = derived (the LAST population is the outgroup), 2 = minor allele over
 * all populations' haplotypes.  min_data is compared with the population's non-missing COUNT, as the reference does
 * (freq.py:79).  The reference draws at random when the two alleles are exactly tied (genomics.py:667): here the
 * lower allele is used and tie[s] = 1 (tie may be NULL).  Values are not rounded (freq.py:91 rounds to 4 dp). */
int pg_site_target_freqs(pg_ctx* ctx, int64_t site0, int64_t n, int32_t target, double min_data, int32_t as_counts,
                         double* out, uint8_t* tie);

/* Replaces the per-site loop of sfs.py for --inputType genotypes without subsampling (sfs.py:430-470: population base
 * counts, the completeness test of 449, getTargetCounts 68-92) and the SparseFS accumulation (94-125, 484-487).
 * In-group = populations 0..n_in-1 of pg_set_pops; outgroup = a later population index (polarized spectra) or -1 (the
 * second most frequent allele, `totalBaseCounts.argsort()[-2]`; on an exact tie of the two alleles the reference depends
 * on numpy's sort, here the lower allele).  Spectrum g is over the populations group_pops[group_off[g] .. group_off[g+1]);
 * hist holds the spectra one after the other as dense row-major arrays of prod(N_k + 1) cells, first[cell] = index of
 * the first site that hit the cell (-1 = empty; gives the reference's first-appearance output order).
 * site_mask (may be NULL): only sites with mask 1 are counted (--include / --exclude).
 * The dense histograms are limited to 2^28 cells in total (PG_ERR above); pg_sfs_sparse has no such limit. */
int pg_sfs(pg_ctx* ctx, int32_t n_in, int32_t outgroup, int32_t n_groups, const int32_t* group_off,
           const int32_t* group_pops, const uint8_t* site_mask, int64_t* hist, int64_t* first, int64_t* n_counted);

/* The same spectra from TABLES of counts on the host (sfs.py --inputType baseCounts | targetCounts, sfs.py:456-474):
 * kind 0: table = uint16 [n x P x 4] base counts per population (the rows freq.py writes); kind 1: int32 [n x P] counts of
 * the target allele (sfs.py's default input, e.g. freq.py --target derived --asCounts).  No completeness test.
 * dims[X] = radix of population X in the dense histograms (its largest count + 1). */
int pg_sfs_tables(pg_ctx* ctx, int32_t kind, const void* table, int64_t n, int32_t P, const int32_t* dims, int32_t n_in,
                  int32_t outgroup, int32_t n_groups, const int32_t* group_off, const int32_t* group_pops,
                  const uint8_t* site_mask, int64_t* hist, int64_t* first, int64_t* n_counted);

/* Sparse spectra: the same per-site logic as pg_sfs / pg_sfs_tables (same arguments), kept the way sfs.py's nested
 * SparseFS dicts keep them (sfs.py:94-125, 484-487) — only the non-empty cells, so no limit on the cells of a spectrum
 * other than that prod(dims) of each must fit in 63 bits (PG_ERR before any launch, naming the spectrum).  Device memory
 * grows with the sites counted, not with the cells.  nnz[g] receives the non-empty cells of spectrum g; the cells
 * themselves stay in a buffer of the context until pg_sfs_sparse_fetch copies them out: total = sum(nnz), group-major,
 * cells ascending within a spectrum, cell = the dense row-major flat index pg_sfs would use, count = its sites,
 * first = the first site that hit it (the reference's first-appearance order).  A result is fetched once; the next
 * sparse call replaces a pending one, and fetch fails (PG_ERR) when total does not match or nothing is pending. */
int pg_sfs_sparse(pg_ctx* ctx, int32_t n_in, int32_t outgroup, int32_t n_groups, const int32_t* group_off,
                  const int32_t* group_pops, const uint8_t* site_mask, int64_t* nnz, int64_t* n_counted);
int pg_sfs_tables_sparse(pg_ctx* ctx, int32_t kind, const void* table, int64_t n, int32_t P, const int32_t* dims,
                         int32_t n_in, int32_t outgroup, int32_t n_groups, const int32_t* group_off,
                         const int32_t* group_pops, const uint8_t* site_mask, int64_t* nnz, int64_t* n_counted);
int pg_sfs_sparse_fetch(pg_ctx* ctx, int64_t total, int64_t* cell, int64_t* count, int64_t* first);

/* Replaces Alignment.indPairDists (genomics.py:934-954) as used by distMat.py:42-45 and popgenWindows.py:54-57.
 * hap_ind[h] = individual index in [0,n_ind) or -1; dist [W x n_ind x n_ind]; n_sites/pos_sum [W] (may be NULL).
 * min_sites > 0: haplotype pairs with n_ij < min_sites are nan — the state of the reference's cached matrix when
 * groupDistStats ran earlier on the same window (it masks in place, genomics.py:959-961); 0 = no mask (distMat.py). */
int pg_pairdist(pg_ctx* ctx, int32_t n_ind, const int32_t* hap_ind, int32_t include_same_with_same,
                int32_t min_sites, double* dist, int64_t* n_sites, int64_t* pos_sum);

/* Replaces distPaint.py's per-window loop (distPaint.py:26-44, 62-83): the nearest reference population of every query
 * haplotype in every window, by p-distance.  Haplotypes are upload-order indices: query_hap [n_query]; population p's
 * member entries are ref_hap[ref_off[p] .. ref_off[p+1]) (ordered, duplicates allowed; ref_off[0] = 0, every population
 * at least one entry).  d = diff_ij / n_ij, nan when n_ij < min_sites (>= 1); a query listed as a member is at 0.0 when
 * n_ii >= min_sites.  Population means are np.nanmean of the member distances, bit for bit; i = np.argmin of the means
 * (the first nan, else the first minimum).  mode 0 (rank-sum rule, which_lowest_test): out = noresult when
 * ranksums(x_i, x_j, "less").pvalue > threshold for some j != i (a list with a nan gives p = nan, which passes); mode 1
 * (delta rule, which_lowest_delta; P >= 2): out = noresult when sorted(means)[1] - sorted(means)[0] < threshold, sorted as
 * CPython's list.sort orders floats that may be nan.  Else out = i.  out int32 [W x n_query]; means, pvals double
 * [W x n_query x P] (either may be NULL; pvals[.., j] = the test against population j, nan for j = i, for lists with a nan
 * and in mode 1).  P <= 32 and ref_off[P] <= 1024 (PG_ERR before any launch).  Windows without sites are left as the
 * caller filled them. */
int pg_distpaint(pg_ctx* ctx, int32_t n_query, const int32_t* query_hap, int32_t P, const int32_t* ref_off,
                 const int32_t* ref_hap, int32_t min_sites, int32_t mode, double threshold, int32_t noresult, int32_t* out,
                 double* means, double* pvals);

/* Replaces distMat.py --windType cat (distMat.py:303-314: parseGenoFile turns the WHOLE file into one window, then
 * indPairDists): dist [n_ind x n_ind] over every uploaded site.  With a communicator (pg_nccl_init, nranks > 1) the
 * uploaded sites are this rank's shard of that window: the integer pair matrices diff_ij / n_ij are added across the
 * ranks with ONE ncclAllReduce (int64 sum) before the division, and every rank receives the same matrix.
 * *total_sites (may be NULL) = number of sites over all ranks. */
int pg_pairdist_cat(pg_ctx* ctx, int32_t n_ind, const int32_t* hap_ind, int32_t include_same_with_same,
                    double* dist, int64_t* total_sites);

/* Replaces Alignment.seqNonNan() (genomics.py:1038-1040) per window — the --minPerInd gate of distMat.py:40:
 * out int64 [W x H] = non-missing sites of each haplotype (upload order) inside each window. */
int pg_seq_nonnan(pg_ctx* ctx, int64_t* out);

/* Replaces Alignment.sampleHet() (genomics.py:918-929; popgenWindows.py:59-61 --analysis indHet): het [W x n_ind] =
 * p-distance between the two haplotypes of each individual; nan unless the individual has exactly two haplotypes
 * and bit 1 of n_ij is set (the reference's `len(x)==2 & n >= 1` is the chained comparison len(x) == (2 & n) >= 1).
 * min_sites as in pg_pairdist. */
int pg_ind_het(pg_ctx* ctx, int32_t n_ind, const int32_t* hap_ind, int32_t min_sites, double* het);

/* Replaces Alignment.H12stats(maxDist) + distMat_to_cluster_sizes (genomics.py:1079-1098, 1239-1261;
 * popgenWindows.py:63-64 --analysis hapStats): out [W x P x 3] = H1, H12, H2 for the populations of pg_set_pops.
 * min_sites as in pg_pairdist; diag_nan != 0 when an earlier groupDistStats / indPairDists of the same window set
 * the cached matrix's diagonal to nan (963, 940), which removes the self-matches from the greedy clustering. */
int pg_hapstats(pg_ctx* ctx, double max_dist, int32_t min_sites, int32_t diag_nan, double* out);

/* Replaces Alignment.distMatrix + pairNonNan (genomics.py:907-916, 1042-1047) for ONE window:
 * diff, n int32 [H x H] (symmetric, diagonal: diff 0, n = non-missing sites of the haplotype). */
int pg_pair_counts(pg_ctx* ctx, int64_t window, int32_t* diff, int32_t* n);

/* ---- multi-GPU: native NCCL all-gather of the per-window records -------------------------------- */
/* One process per GPU.  Windows shard across ranks with no data-path collective; the only exchange is ONE
 * ncclAllGather of the fixed-width records, enqueued on the ctx stream right behind the statistics kernels.
 * NCCL is bound at run time (dlopen): rank 0 creates the 128-byte id, the host distributes it by any means
 * (bench.py uses torch.distributed's broadcast), every rank calls pg_nccl_init.
 * pg_popgen_allgather: h_table (host) receives nranks * w_max * (4 + 5P + 2*npairs) 8-byte words in rank order
 * (record layout of pg_popgen_device; rows past a rank's own window count are zero); w_max >= every rank's W. */
int pg_nccl_unique_id(void* id128);
int pg_nccl_init(pg_ctx* ctx, int32_t nranks, int32_t rank, const void* id128);
int pg_nccl_finalize(pg_ctx* ctx);
int pg_popgen_allgather(pg_ctx* ctx, int32_t min_sites, double min_data, int32_t force_path, int64_t w_max,
                        void* h_table, int64_t* n_pairwise);
/* Pipelined form (two slots): `begin` enqueues site pass + finalize on the ctx stream and the exchange + read-back of the
 * table on a side stream; `end` waits for that batch and returns the slot's pinned table (nranks * w_max records, valid until
 * the slot's next `begin`).  begin(0); begin(1); end(0); begin(0); end(1); ... hides the all-gather and the D2H of one batch
 * under the site pass of the next (the reference's sorter + writer run concurrently with its workers,
 * popgenWindows.py:108-160).  Works without a communicator too (one rank).
 * `begin` records the batch: its windows and their bounds, the record width (P) and a generation of the resident matrix and
 * population map; this rank's rows W..w_max-1 of the slot are zeroed.  So between begin(k) and end(k) the caller may set the
 * next batch's windows or populations and call begin(k+1): `end` resolves the slot's pairwise windows (read off its own path
 * column, *n_pairwise = their number) with the recorded bounds.  When the matrix or the populations changed meanwhile
 * (upload, synth fill, ingest, append, pg_set_pops) and the slot has pairwise windows, `end` fails with PG_ERR rather
 * than compute them from the other batch's data; a slot without pairwise windows is complete at `begin` and is returned.
 * With a communicator the refusal is collective (one all-reduce of a flag, only when some rank has pairwise windows): every
 * rank returns PG_ERR, so none is left waiting in the second all-gather. */
int pg_popgen_gather_begin(pg_ctx* ctx, int32_t min_sites, double min_data, int64_t w_max, int32_t slot);
int pg_popgen_gather_end(pg_ctx* ctx, int32_t slot, const void** h_table, int64_t* n_pairwise);
/* The same for the ABBA-BABA statistics (ABBABABAwindows.py window-sharded over the GPUs): h_table receives
 * nranks * w_max * 8 words per window [sites (int64), pos_sum (int64), ABBA, BABA, D, fd, fdM, sitesUsed (doubles)],
 * and for genomics.fourPop: 17 words [sites, pos_sum, the 14 statistics in pg_fourpop's order, sitesUsed]. */
int pg_abbababa_allgather(pg_ctx* ctx, int32_t p1, int32_t p2, int32_t p3, int32_t o, double min_data, int64_t w_max,
                          void* h_table);
int pg_fourpop_allgather(pg_ctx* ctx, int32_t p1, int32_t p2, int32_t p3, int32_t p4, double min_data, int32_t mode,
                         int64_t w_max, void* h_table);

/* ---- host-side .geno text ingest (no CUDA) ------------------------------------------------------ */
/* Replaces parseGenoLine/GenoFileReader (genomics.py:1884-1945) + splitSeq/haplo/forceHomo (390-396, 27, 407)
 * + seqArrayToNumArray (74-77) for a whole file: `buf` holds complete data lines (no header line);
 * '#' lines and blank lines are skipped.  fmt: 0 phased, 1 diplo, 2 pairs, 3 haplo.
 * col_take[k] = genotype column (0-based, after scaffold and position) of output sample k, ploidy[k] its
 * haplotype count; output row layout: samples in the given order, haplotypes of a sample adjacent.
 * geno [n_lines x H_out] int8, pos [n_lines] int32, new_scaffold [n_lines] (1 where the scaffold field differs
 * from the previous data line), line_off [n_lines] byte offset of each data line in buf. */
int pg_geno_count_lines(const char* buf, size_t len, int64_t* n_lines);
int pg_geno_parse(const char* buf, size_t len, int32_t fmt, int32_t n_out, const int32_t* col_take,
                  const int8_t* ploidy, int32_t H_out, int64_t n_lines, int8_t* geno, int32_t* pos,
                  int8_t* new_scaffold, int64_t* line_off, int32_t n_threads);

/* ---- host-side output rows (no CUDA) ------------------------------------------------------------- */
/* Replaces the row assembly of freq.py (freq.py:100-111) for n sites: "<scaffold>\t<position>\t<col>...\n".
 * mode 0: data = counts uint16 [n x P x 4], a column is "cA,cC,cG,cT"; mode 1: data = double [n x P] printed like
 * numpy's float64 -> str ("0.25", "1.0", "nan"); mode 2: double [n x P] printed as integers (--asCounts).
 * keep (may be NULL): uint8 [n], rows with 0 are skipped.  Thread t formats its share of the sites into
 * out + t * seg_cap and reports the bytes written in seg_len[t]; the caller writes the segments in order. */
int pg_format_freq_rows(int32_t mode, const void* data, int64_t n, int32_t P, const int32_t* pos, const int32_t* scaf_id,
                        const char* const* scaf_names, const uint8_t* keep, char* out, size_t seg_cap, int32_t n_threads,
                        size_t* seg_len);

/* Rows of a float64 matrix [rows x cols] as text, "<prefix[r]><v0><sep><v1>...\n" with numbers printed like numpy's
 * float64 -> str: the " ".join(row) over ndarray.round(roundTo).astype(str) of makeDistMat*String (genomics.py:2288-2306)
 * for distMat.py's per-window matrices (the caller rounds).  prefix may be NULL.  Segments as in pg_format_freq_rows. */
int pg_format_matrix_rows(const double* v, int64_t rows, int32_t cols, int32_t sep, const char* const* prefix, char* out,
                          size_t seg_cap, int32_t n_threads, size_t* seg_len);

/* ---- device-side .geno text ingest --------------------------------------------------------------- */
/* Same job and grammar as pg_geno_parse, on the GPU: the text (complete data lines, no header line) is copied to
 * device memory as it is and tokenised there, straight into this ctx's resident matrix (replaces pg_geno_parse +
 * pg_upload when the text fits in device memory).  col_hap[c] = first output haplotype of genotype column c
 * (0-based, after scaffold and position) or -1 for a column that is not wanted; col_ploidy[c] its haplotype count.
 * *n_sites = number of data lines = sites now resident.  Errors (a token whose allele count does not match the
 * ploidy, genomics.py:1111; a non-integer position; a short line) name the offending data line. */
int pg_ingest_text(pg_ctx* ctx, const char* buf, size_t len, int32_t fmt, int32_t n_cols, const int32_t* col_hap,
                   const int8_t* col_ploidy, int32_t H_out, int64_t* n_sites);
/* The same for a file on disk: bytes [body_offset, EOF) of `path` (body_offset = length of the header line, or 0) are
 * read straight into the pinned staging buffers by a few host threads — the file is never copied whole into host
 * memory.  line_off values of pg_ingest_meta are relative to body_offset. */
int pg_ingest_file(pg_ctx* ctx, const char* path, int64_t body_offset, int32_t fmt, int32_t n_cols, const int32_t* col_hap,
                   const int8_t* col_ploidy, int32_t H_out, int64_t* n_sites);
/* One rank's share of a file in the multi-GPU command lines (replaces the single producer that feeds the -T workers,
 * popgenWindows.py:398-446): bytes [byte_lo, byte_hi) — both at line starts, byte_hi < 0 = end of file.  line_off values of
 * pg_ingest_meta are relative to byte_lo. */
int pg_ingest_file_range(pg_ctx* ctx, const char* path, int64_t byte_lo, int64_t byte_hi, int32_t fmt, int32_t n_cols,
                         const int32_t* col_hap, const int8_t* col_ploidy, int32_t H_out, int64_t* n_sites);
/* pos int32 [S], new_scaffold int8 [S], line_off int64 [S] of the last pg_ingest_text / pg_ingest_file (as pg_geno_parse returns them;
 * any pointer may be NULL). */
int pg_ingest_meta(pg_ctx* ctx, int32_t* pos, int8_t* new_scaffold, int64_t* line_off);
/* Frees the device copy of the text. */
int pg_ingest_release(pg_ctx* ctx);

/* Strict genotype tokens for the next ingests of this ctx (off by default; filterGenotypes turns it on with on = 1): a token must be
 * exactly as wide as its sample's ploidy (2p-1 characters phased, p alleles, one letter diplo with diploid samples only), and
 * hold only A C G T N (a diplo letter of genomics.py:14 DIPLOTYPES).  The reference makes a genotype with any other character
 * missing but writes the character back out (genomics.py:351-352), which the one-hot matrix cannot do; such a line is an
 * error naming its data line.  The ingest also keeps each sample's phase character (genomics.py:335) for pg_filter_emit.
 * on = 2 keeps only the width test (distPaint.py's haploid tokens: one character; other characters read as usual). */
int pg_ingest_set_strict(pg_ctx* ctx, int32_t on);
/* Geometry of the last text ingest of this ctx: out[0] = slabs of the host-to-device copy of the text, out[1] = bytes per
 * slab, out[2] = bytes per block of the line index, out[3] = warps of the line parse grid (one line per warp, grid-stride),
 * out[4] = threads of the scaffold-flag grid (one line per thread, grid-stride).  All 0 before any ingest. */
int pg_debug_ingest(pg_ctx* ctx, int64_t* out);

/* ---- filterGenotypes.py ------------------------------------------------------------------------ */
/* Filter settings (filterGenotypes.py:161-183 -> genomics.siteTest, genomics.py:742-799).  Samples are the selected
 * samples in output order; populations are indices in -p order.  Pointers are host memory. */
typedef struct pg_filter_spec {
    int32_t n_samp;
    const int32_t* samp_hap0;       /* [n_samp] first haplotype of the sample in the resident matrix */
    const int8_t* samp_ploidy;      /* [n_samp] */
    int32_t P;                      /* populations (<= 64), in -p order */
    const int32_t* pop_off;         /* [P + 1] population p's members are pop_members[pop_off[p] .. pop_off[p + 1]) */
    const int32_t* pop_members;     /* sample indices; a sample may be in several populations (siteTest visits each list
                                       on its own, genomics.py:774-796).  A population with no member stands for every
                                       sample, as GenomeSite.alleles / baseFreqs do for an empty list (genomics.py:521-523,
                                       544-545), except for its called count, which is 0.  NULL both when P == 0 */
    int32_t min_calls;              /* called samples (no missing allele) at least */
    int32_t min_alleles;
    double max_alleles;
    int32_t min_var_count;          /* 0 = off; second largest base count, variable sites only */
    int32_t has_max_het;
    double max_het;                 /* het samples / called samples (numpy division: 0/0 nan passes, k/0 inf fails) */
    double min_freq, max_freq;      /* 0 = off; second largest of count / n */
    const int32_t* min_pop_calls;   /* [P] or NULL */
    const int32_t* min_pop_alleles; /* [P] or NULL; min and max are both given or both NULL */
    const int32_t* max_pop_alleles;
    int32_t fixed_diffs;
    int32_t has_nearly_fixed;
    double nearly_fixed_diff;
    int32_t partial_to_missing;     /* a sample with any missing allele becomes all missing */
    int32_t no_test;                /* keep every site that survives the contig and thinning steps */
    int32_t thin_dist;              /* 0 = off */
    int32_t pod_size;               /* input lines per pod: thinning restarts at every pod; site 0 starts a pod */
} pg_filter_spec;

/* Replaces the per-line loop of filterGenotypes.py's analysisWrapper (filterGenotypes.py:33-55: the contig lists, the
 * thinning and genomics.siteTest) over the resident sites of the last text ingest.  contig_mask uint8 [S] (NULL = all 1):
 * 0 drops the line before anything else; scaf_id int32 [S]: equal ids = same scaffold (required with thin_dist).
 * *n_kept = rows to write; *flags_or (may be NULL) = OR of the flags (see pg_filter_stats) of the kept sites. */
int pg_filter(pg_ctx* ctx, const pg_filter_spec* spec, const uint8_t* contig_mask, const int32_t* scaf_id, int64_t* n_kept,
              uint8_t* flags_or);
/* Replaces the row assembly of filterGenotypes.py:53 (GenomeSite.asList, genomics.py:465-512) for the kept rows of the last
 * pg_filter: rows row0, row0 + 1, ... as many as fit in cap bytes of out (host memory).  fmt: 0 phased, 1 diplo, 2 bases,
 * 3 alleles, 4 coded, 5 count; freq_order = --alleleOrder freq.  Each row starts with the scaffold and position fields as
 * they are in the text.  *rows / *bytes = what was written; a single row larger than cap is an error. */
int pg_filter_emit(pg_ctx* ctx, int32_t fmt, int32_t freq_order, int64_t row0, char* out, size_t cap, int64_t* rows,
                   size_t* bytes);
/* Per-site statistics of the last pg_filter for sites [site0, site0 + n) (any pointer may be NULL): called, het int32 [n],
 * counts int32 [n x 4] (A C G T over the selected samples), pop_called int32 [n x P], pop_mask uint8 [n x P] (alleles of the
 * population, bit a = base a), flags uint8 [n] (1: two present alleles have the same count, so the frequency order is a tie
 * that numpy's sort may break either way; 2: a sample is partly missing; 4: no allele), keep uint8 [n] (the siteTest
 * verdict), final uint8 [n] (the row is written). */
int pg_filter_stats(pg_ctx* ctx, int64_t site0, int64_t n, int32_t* called, int32_t* het, int32_t* counts,
                    int32_t* pop_called, uint8_t* pop_mask, uint8_t* flags, uint8_t* keep, uint8_t* final_);

/* ---- parseVCF.py (csrc/vcf.cu) ------------------------------------------------------------------------------------- */
/* One data line of the last pg_vcf_load (offsets of the fields are from the line's first byte). */
typedef struct {
    int64_t start;              /* first byte of the line in the text */
    int64_t end;                /* its terminator ('\n' or '\r') */
    int64_t pos;                /* POS, unless flags & PG_VCF_POS_UNRESOLVED */
    uint32_t chrom_off, chrom_len, pos_off, pos_len, ref_off, ref_len, alt_off, alt_len, qual_off, qual_len, fmt_off, fmt_len;
    int32_t n_fields;           /* str.split() fields of the line */
    int32_t n_alt;              /* ALT alleles (0 for ".") */
    uint32_t flags;             /* PG_VCF_* */
    uint32_t reserved;
} pg_vcf_line;
#define PG_VCF_NONASCII 1u          /* a byte >= 0x80: the host checks str.split() against the ASCII split */
#define PG_VCF_POS_UNRESOLVED 2u    /* POS is not sign + ASCII digits ('_' between them) of at most 18 significant digits */
#define PG_VCF_QUAL_DROP 4u         /* float(QUAL) < min_qual */
#define PG_VCF_QUAL_UNRESOLVED 8u   /* QUAL off the fast number path: the host decides */
#define PG_VCF_SAME_LEN 16u         /* every ALT as long as REF (an ALT-less line has it too) */
#define PG_VCF_DUPLICATE 32u        /* CHROM and POS text equal to the data line before */
#define PG_VCF_FORMAT_WIDE 64u      /* a looked-up FORMAT key past the 64th */

/* What a run of parseVCF.py reads and writes (parseVCF.py:257-289, 350-391). */
typedef struct {
    int32_t n_cols;             /* #CHROM line tokens (the nine fixed columns, then the samples) */
    const int32_t* col_slot;    /* [n_cols] slot of a column a selected sample may read (0, 1, .. in column order), or -1 */
    const int32_t* col_prev;    /* [n_cols] the previous column of the same sample name, or -1 (also for columns < 9) */
    int32_t n_keys;             /* FORMAT keys looked up: key 0 is GT */
    const int32_t* key_off;     /* [n_keys + 1] into key_chars */
    const char* key_chars;
    int32_t n_samp;             /* selected samples, in -s order */
    const int32_t* samp_col;    /* [n_samp] last column of the sample's name */
    const int32_t* samp_ploidy; /* [n_samp] expected ploidy */
    int32_t field_key;          /* --field: its key; -1: genotypes */
    int32_t field_phase;        /* --field phase: the GT's phase character when the sample has a GT */
    int32_t n_filt;             /* --gtf filters, in command-line order */
    const int32_t* filt_key;    /* [n_filt] key of the flag; -1: the filter always fails */
    const double* filt_min;
    const double* filt_max;
    const uint8_t* filt_site;   /* [n_filt] site types it applies to: bit 0 MONO, 1 SNP, 2 INDEL */
    const uint8_t* filt_gt;     /* [n_filt] genotype types: bit 0 Het, 1 HomRef, 2 Missing, 3 HomAlt */
    const uint8_t* filt_samp;   /* [n_filt x n_samp] 1: it applies to the sample */
    int32_t has_min_qual;
    double min_qual;            /* drop a line whose float(QUAL) < min_qual */
    const char* missing;        /* the missing allele / field text */
    int32_t missing_len;
    const char* sep;            /* --outSep */
    int32_t sep_len;
    int32_t skip_indels, keep_partial, ploidy_mismatch_to_missing, add_ref_track;
} pg_vcf_spec;

/* Sets the run's spec (copied; the pointers need not outlive the call). */
int pg_vcf_set_spec(pg_ctx* ctx, const pg_vcf_spec* spec);
/* Complete lines of VCF body text (cut at line ends) -> device: data-line index and one pg_vcf_line per data line.  prev
 * (may be NULL) = the CHROM then POS text of the data line before this text (prev_chrom + prev_pos bytes, at most 4000), for
 * --excludeDuplicates.  *n_lines = data lines. */
int pg_vcf_load(pg_ctx* ctx, const char* text, size_t len, const char* prev, int32_t prev_chrom, int32_t prev_pos,
                int64_t* n_lines);
/* Lines [line0, line0 + n) of the last pg_vcf_load. */
int pg_vcf_lines(pg_ctx* ctx, int64_t line0, int64_t n, pg_vcf_line* out);
/* Replaces VcfSite.getGenotypes / getGenoField (parseVCF.py:107-190) for the kept lines rows[0..n_rows) (their POS in pos):
 * one verdict per (row, selected sample).  Every line must hold all of the header's sample names.  *n_unresolved = genotypes
 * whose filter values left the fast number path (verdict bit 2; settle them with pg_vcf_verdicts before pg_vcf_emit);
 * *error = 0, or the first offending genotype: ((line + 1) << 24) | (sample << 3) | code, code 1 = no GT, 2 = ploidy. */
int pg_vcf_genotypes(pg_ctx* ctx, int64_t n_rows, const int64_t* rows, const int64_t* pos, int64_t* n_unresolved,
                     uint64_t* error);
/* The verdict bytes [n_rows x n_samp] of the last pg_vcf_genotypes: copied out to get and/or replaced by put (either may be
 * NULL).  Bits: 1 a filter failed, 2 unresolved, 4 ploidy mismatch (to missing), 8 phased GT, 16 field absent. */
int pg_vcf_verdicts(pg_ctx* ctx, uint8_t* get, const uint8_t* put);
/* The .geno rows of the last pg_vcf_genotypes from row0 on, as many as fit in cap bytes of out (host memory): *rows, *bytes
 * written; a single row larger than cap is an error. */
int pg_vcf_emit(pg_ctx* ctx, int64_t row0, char* out, size_t cap, int64_t* rows, size_t* bytes);

/* ---- introspection ---------------------------------------------------------------------------- */
/* Device time (ms, CUDA events on the ctx stream) of the kernels launched by the last statistics call:
 * names[i] -> ms[i]; returns the number of entries through *count (at most cap). */
int pg_last_timings(pg_ctx* ctx, int32_t cap, char (*names)[32], float* ms, int32_t* launches, int32_t* count);
/* Total kernels launched by this ctx so far. */
int pg_launch_count(pg_ctx* ctx, int64_t* n);
/* Host-only planning self-test hook (no device needed): returns the K1 launch plan for a shape. */
int pg_debug_k1_plan(int64_t S, int32_t H, int32_t* pitch, int32_t* lanes_per_site, int32_t* tile_sites,
                     int32_t* stages, int32_t* smem_bytes);
/* The same for a given consumer-warp count (8 or 12), lanes per site forced to force_G (the lane-per-population variant;
 * 0 = chosen by row length) and table_bytes of mask tables in shared memory.  Reads the PG_K1_* geometry overrides like the
 * launches do.  out[9] = pitch, G, wpt, I, T (sites per tile), stages, smem_bytes, CTAs on 132 SMs, 1 if the site-pass
 * kernels accept the plan (0: such rows are refused). */
int pg_debug_k1_plan_ex(int64_t S, int32_t H, int32_t nw, int32_t force_G, int32_t table_bytes, int32_t* out);
/* The packed companion of the resident matrix (rows the popgen site pass reads): *row_words = 32-bit words per site row
 * (three planes of ceil(H / 32) words — valid bits, low and high bit of the allele code A0 C1 G2 T3 — then padding), 0 when
 * the context has no companion.  out (may be NULL) receives rows [site0, site0 + n). */
int pg_debug_packed(pg_ctx* ctx, int64_t site0, int64_t n, int32_t* row_words, uint32_t* out);
/* The class byte of each site of the packed companion, sites [site0, site0 + n) into out (may be NULL): 0 varied, 1..4 every
 * haplotype carries A / C / G / T, 5 every haplotype missing, 6 / 7 every haplotype called and exactly two alleles present,
 * told apart by the low / high allele-code bit.  *avail = 0 when the context keeps no classes. */
int pg_debug_site_cls(pg_ctx* ctx, int64_t site0, int64_t n, int32_t* avail, uint8_t* out);
/* The popgen pass's stream of varied rows as the last popgen call left it: *in_use = 1 when that call streamed only the
 * rows of sites whose haplotypes are not all the same (0: every packed row), *varied_sites = the varied sites it counted
 * (S when it did not count them). */
int pg_debug_uniform(pg_ctx* ctx, int32_t* in_use, int64_t* varied_sites);
/* Tile geometry of the varied-row stream after a popgen call: out[0] = sites per tile at most (Tmax), out[1] = warps per tile (0 before any
 * popgen call on the packed companion). */
int pg_debug_uniform_tile(pg_ctx* ctx, int32_t* out);
/* Ring of the varied-row stream's last popgen call: out[0] = varied rows a tile may hold (R), out[1] = stages, out[2] = bytes per
 * stage (all 0 when the last call did not read the stream). */
int pg_debug_uniform_ring(pg_ctx* ctx, int32_t* out);
/* Launch of the varied-row stream's last popgen call: out[0] = CTAs, out[1] = consumer warps per CTA, out[2] = 1 when the
 * one-plane rows were summed as a Gram (every population of at most 255 haplotypes), else 0 (all 0 when the last call did
 * not read the stream).  PG_K1_UNI_CTAS=n caps the stream's CTAs at n. */
int pg_debug_uniform_launch(pg_ctx* ctx, int32_t* out);
/* Tiles of the varied-row stream the last popgen call read: *ntiles, geometry[0] = R (varied rows per tile at most),
 * geometry[1] = Tmax (sites per tile at most); when cap >= *ntiles + 1, site_lo / row0 get each tile's first site / first
 * varied row and the totals (S, varied rows) at [ntiles].  All 0 when the last call did not read the stream. */
int pg_debug_uniform_tiles(pg_ctx* ctx, int64_t cap, int64_t* site_lo, int64_t* row0, int64_t* ntiles, int32_t* geometry);
/* Rows of the varied-row stream the last popgen call read: *one_plane_rows = complete biallelic rows streamed as one plane,
 * *words = 32-bit words of all its rows (both 0 when the last call did not read the stream). */
int pg_debug_uniform_rows(pg_ctx* ctx, int64_t* one_plane_rows, int64_t* words);

/* ---- genoToSeq.py (seq.cu) ---------------------------------------------------------------------------------------------
 * Replaces parseGenoFile / the window generators' line reading (genomics.py:1949-1967, 1971-2108), GenoWindow.seqDict
 * (1790-1793) and makeAlnString (2232-2251): the genotype tokens of a .geno body, transposed into alignment text. */

/* The body (text[0..len), or bytes [body_offset, EOF) of the file path when path is not NULL) -> device, its data lines
 * indexed as pg_ingest_text does, and the start of the token of every column with col_slot[c] >= 0 (n_cols genotype columns,
 * slots 0..n_slots-1, each of one column) recorded per line.  Every slot's token must be slot_width[slot] bytes wide (the
 * width on the first data line); with exact_cols a line holds exactly n_cols genotype columns, else at least every slot's.
 * *n_sites = data lines.  error[3] = {0, 0, 0}, or the first offending line: {code, data line, genotype column (0: none)},
 * both 1-based; codes 1 position not an integer, 2 no position, 3 position outside int32, 4 token width, 5 a slot's column
 * missing, 6 column count, 7 a byte >= 0x80, 8 a '\r' that ends a line by itself.  The text replaces the one of the last
 * pg_ingest_text on this ctx. */
int pg_seq_index(pg_ctx* ctx, const char* text, size_t len, const char* path, int64_t body_offset, int32_t n_cols,
                 const int32_t* col_slot, int32_t n_slots, const int32_t* slot_width, int32_t exact_cols, int64_t* n_sites,
                 int64_t* error);
/* pos int32 [S], new_scaffold int8 [S], line_off int64 [S] of the last pg_seq_index (any may be NULL). */
int pg_seq_meta(pg_ctx* ctx, int32_t* pos, int8_t* new_scaffold, int64_t* line_off);
/* The output rows of n_win alignments over data lines [lo[w], hi[w]): fmt 0 FASTA (">name\nseq\n" per sequence), 1 PHYLIP
 * (" n L\n", then "name   seq\n" per sequence, L the longest sequence).  Sequence k is named names[name_off[k] ..
 * name_off[k + 1]) and takes seq_width[k] bytes from byte seq_byte[k] of slot seq_slot[k]'s token at every site (the whole
 * token, or with --splitPhased one allele: seq_byte 2a, width 1); nto_gap maps N and n to '-' in the sequences.  A length
 * pass and a scan give every row's byte offset.  *n_rows = rows; win_bytes[w] = bytes of alignment w. */
int pg_seq_plan(pg_ctx* ctx, int32_t fmt, int32_t nto_gap, int32_t n_seq, const char* names, const int64_t* name_off,
                const int32_t* seq_slot, const int32_t* seq_byte, const int32_t* seq_width, int64_t n_win, const int64_t* lo,
                const int64_t* hi, int64_t* n_rows, int64_t* win_bytes);
/* The text of the last pg_seq_plan from cell (row0, part0) on into out (host memory, cap bytes): whole rows while they fit,
 * else row0 alone, cut after as many sites as fit.  part0 = -1 starts a row; k >= 0 resumes after its name and k sites.
 * (*row1, *part1) = where the next call resumes (*row1 = n_rows: done); *bytes = bytes written. */
int pg_seq_emit(pg_ctx* ctx, int64_t row0, int64_t part0, char* out, size_t cap, int64_t* row1, int64_t* part1, size_t* bytes);

/* ---- genoToVCF.py (geno2vcf.cu) ----------------------------------------------------------------------------------------
 * Replaces VCF_processing/genoToVCF.py makeVCFline, genomics.py GenomeSite / Genotype (317-378, 500-557) and parseFasta
 * (2256-2261): .geno genotypes -> VCF GT records, REF from a reference FASTA. */

/* The reference FASTA text[0..len) -> device; *n_rec = its '>' bytes (the starts of parseFasta's pieces). */
int pg_g2v_ref_load(pg_ctx* ctx, const char* text, size_t len, int64_t* n_rec);
/* The n_rec byte offsets of the '>' bytes of the last pg_g2v_ref_load, in order. */
int pg_g2v_ref_starts(pg_ctx* ctx, int64_t* starts);
/* Record k's sequence is bytes [lo[k], hi[k]) of the FASTA without '\n', '\r' and ' ' (lo = the piece's first newline, hi =
 * the next '>' or the end); the sequences are compacted into one resident buffer and the text is released.
 * rec_len[k] = length of record k's sequence. */
int pg_g2v_ref_index(pg_ctx* ctx, int64_t n_rec, const int64_t* lo, const int64_t* hi, int64_t* rec_len);
/* The conversion: fmt 0 phased, 1 diplo, 2 pairs; n_cols genotype columns of the header, col_slot[c] = the column's token
 * slot (the slotted columns numbered in order) or -1, col_prev[c] = the previous column of the same name or -1; selected
 * sample k reads column sel_col[k], or on a line with fewer columns the last column of its name the line holds (every column
 * of such a chain has a slot); use_ref: REF from the records of pg_g2v_ref_index. */
int pg_g2v_spec(pg_ctx* ctx, int32_t fmt, int32_t n_cols, const int32_t* col_slot, const int32_t* col_prev, int32_t n_sel,
                const int32_t* sel_col, int32_t use_ref);
/* A chunk of complete .geno body lines (no header line; below 4 GiB) -> device, its data lines indexed as pg_ingest_text
 * does and tokenised; *n_lines = data lines, *n_runs = runs of lines with the same scaffold name. */
int pg_g2v_chunk(pg_ctx* ctx, const char* text, size_t len, int64_t* n_lines, int64_t* n_runs);
/* The first data line of every scaffold run of the last pg_g2v_chunk and its byte offset in the chunk. */
int pg_g2v_runs(pg_ctx* ctx, int64_t* run_line, int64_t* run_off);
/* The site pass over the last chunk: with use_ref, run_rec[i] = the FASTA record of scaffold run i, or -1 (not in the FASTA).
 * Alleles, allele lists and row lengths, a scan for the row offsets.  *n_rows = the data lines before the first error (all
 * when none), *n_bytes = their VCF text.  error[4] = {0, 0, 0, 0}, or {code, data line (0-based in the chunk), column, byte
 * offset of the line in the chunk}; column 0 = the line itself, k + 1 = selected sample k, n_sel + 1 = the reference lookup;
 * codes 1 POS not [+-]?[0-9]+, 2 no POS field, 3 POS outside int64, 4 only two fields, 5 a byte >= 0x80, 6 a '\r' that ends a
 * line by itself, 7 the sample's column missing, 8 not a diplo code, 9 scaffold not in the FASTA, 10 POS outside the contig. */
int pg_g2v_sites(pg_ctx* ctx, const int32_t* run_rec, int64_t* n_rows, int64_t* n_bytes, int64_t* error);
/* Bytes [byte0, byte0 + cap) (at most to *n_bytes of pg_g2v_sites) of the VCF rows of the last site pass into out (host
 * memory); a row may be cut anywhere.  *bytes = bytes written. */
int pg_g2v_emit(pg_ctx* ctx, int64_t byte0, char* out, size_t cap, size_t* bytes);

/* ---- seqToGeno.py (seq2geno.cu, fasta.cu) ---------------------------------------------------------------------------------
 * Replaces seqToGeno.py:37-98 and genomics.py parseFasta / parsePhylip / haploToPhased (2256-2283, 412-446): FASTA / PHYLIP
 * alignments -> .geno rows.  The input must fit in device memory with 1 GiB to spare. */

/* A FASTA text[0..len) -> device; *n_rec = its '>' bytes (the starts of parseFasta's pieces). */
int pg_s2g_fasta_load(pg_ctx* ctx, const char* text, size_t len, int64_t* n_rec);
/* The n_rec byte offsets of the '>' bytes of the last pg_s2g_fasta_load, in order. */
int pg_s2g_fasta_starts(pg_ctx* ctx, int64_t* starts);
/* Record k's sequence is bytes [lo[k], hi[k]) of the FASTA without '\n', '\r' and ' '; the sequences are compacted into the
 * resident layout and the text is released.  rec_len[k] = length of record k's sequence. */
int pg_s2g_fasta_index(pg_ctx* ctx, int64_t n_rec, const int64_t* lo, const int64_t* hi, int64_t* rec_len);
/* A PHYLIP text[0..len) -> device, its lines indexed as pg_ingest_text does (so a line that starts with '#' is skipped: the
 * caller refuses such text) and classified, one warp per line; *n_lines = indexed lines. */
int pg_s2g_phylip_load(pg_ctx* ctx, const char* text, size_t len, int64_t* n_lines);
/* The line table of the last pg_s2g_phylip_load: 7 int64 per line, {field 0's first byte (-1: none), its length, field 1's
 * first byte (-1: none), its length, field count, flags (1 a byte >= 0x80, 2 a '\r' that ends a line by itself, 4 a header:
 * fields 0 and 1 pass Python's int()), the header's count (clamped to int64; 0 when not a header)}. */
int pg_s2g_phylip_lines(pg_ctx* ctx, int64_t* lines);
/* The resident layout of n_seq sequences of seq_len[k] bytes, one after another: span[3i .. 3i + 2] = {text byte, sequence
 * byte (in the concatenation), bytes} copies a field-1 span; the spans must fill the sequences exactly. */
int pg_s2g_phylip_pack(pg_ctx* ctx, int64_t n_seq, const int64_t* seq_len, int64_t n_span, const int64_t* span);
/* The rows: n_blk blocks, blk[4b .. 4b + 3] = {name offset in names, name length, rows, first member}; block b's members are
 * [first, next block's first or n_mem), mem_rec[m] = the member's sequence (at least `rows` long), mem_sep[m] = the byte
 * after it ('|', '\t' or '\n').  Row x of block b is "name\t<x + 1>\t" then every member's byte x and its mem_sep.
 * *n_bytes = the bytes of all rows. */
int pg_s2g_plan(pg_ctx* ctx, int64_t n_blk, const int64_t* blk, const char* names, int64_t names_len, int64_t n_mem,
                const int64_t* mem_rec, const uint8_t* mem_sep, int64_t* n_bytes);
/* Bytes [byte0, byte0 + cap) (at most to *n_bytes of pg_s2g_plan) of the rows into out (host memory); a row may be cut
 * anywhere.  *bytes = bytes written. */
int pg_s2g_emit(pg_ctx* ctx, int64_t byte0, char* out, size_t cap, size_t* bytes);

/* ---- windowStats.py (wstats.cu): per-window statistics of numeric columns ----
 * Spec: value column c (field 2 + c of a line) is parsed into slot col_slot[c] (-1: not read); every slot is read by exactly
 * one column.  n_fields >= 0: every data line must have exactly n_fields value fields (error 4); n_fields = -1: every line
 * must hold the columns of all slots (error 7 names the slot).  Drops the values of any earlier spec. */
int pg_ws_spec(pg_ctx* ctx, int32_t n_cols, const int32_t* col_slot, int32_t n_slots, int32_t n_fields);
/* Complete body lines (ASCII; '#' and blank lines skipped) appended to the resident values and positions.  *n_lines = data
 * lines, *n_runs = scaffold runs, *n_flag = tokens the parser rejected or left to the host; error = {code, data line of the
 * chunk, slot} of the first bad line (code 0: none; 1 position not [+-]?[0-9]+, 2 no position, 3 position outside int64,
 * 4 field count, 5 byte >= 0x80, 6 lone '\r', 7 missing column). */
int pg_ws_chunk(pg_ctx* ctx, const char* text, size_t len, int64_t* n_lines, int64_t* n_runs, int64_t* n_flag, int64_t* error);
/* Of the last pg_ws_chunk: the first data line of every scaffold run and its byte offset in the chunk; the flagged tokens as
 * slot * n_lines + line and {offset in the chunk << 32 | length << 2 | status (1 rejected, 2 left to the host)}.  Any NULL
 * pair is skipped. */
int pg_ws_chunk_info(pg_ctx* ctx, int64_t* run_line, int64_t* run_off, int64_t* flag_idx, uint64_t* flag_tok);
/* Set n values: slot[i]'s value on data line line[i] (counted over all chunks) = v[i]. */
int pg_ws_set_values(pg_ctx* ctx, int64_t n, const int64_t* line, const int32_t* slot, const double* v);
/* *n_lines = data lines so far; pos (may be NULL) = their positions. */
int pg_ws_meta(pg_ctx* ctx, int64_t* n_lines, int64_t* pos);
/* Window w = data lines [lo[w], hi[w]).  out[(w * n_slots + c) * K + k] = statistic code[k] of slot c's non-NaN values in the
 * window (0 mean, 1 median, 2 min, 3 max, 4 sd rounded to 6 decimals, 5 sum, 6 quantile q[k], numpy's linear method);
 * n_out[w * n_slots + c] = their count.  The first call compacts the values (no pg_ws_chunk after it); median and quantiles
 * sort the windows' values in batches of at most sort_budget bytes (one window at least). */
int pg_ws_stats(pg_ctx* ctx, int64_t W, const int64_t* lo, const int64_t* hi, int32_t K, const int32_t* code, const double* q,
                int64_t sort_budget, double* out, int64_t* n_out);

/* ---- mergeGeno.py (merge.cu): .geno files joined by position in the order of the .fai's walk ----
 * Replaces mergeGeno.py:41-88.  The walk visits every site 1..len of every scaffold in .fai order; walk index = the offset
 * of the scaffold (the lengths of the positive-length scaffolds before it) + site - 1.  A file's merged lines are the longest
 * prefix of its body whose lines have >= 2 fields, name a scaffold, hold its site as str(n) with 1 <= n <= len and lie
 * strictly after the line before in the walk. */

/* The walk and the rule.  n_scaf scaffolds: name s is bytes [name_off[s], name_off[s + 1]) of names (distinct), len[s] its
 * length (<= 0: no sites).  n_files inputs: out[x] = file x's columns are written, n_dummy[x] = its dummy genotypes (the
 * header's fields - 2).  Rows are sep-joined; a file that did not match adds n_dummy times sep + missing.  method 0
 * intersect, 1 union, 2 all, with the reference's unionMin and mustIncludeFirst.  *dense = 1 when every walk index is a row
 * (`all`, or `union` with max(unionMin, mustIncludeFirst) <= 0, and mustIncludeFirst <= 0).  Drops any earlier merge. */
int pg_merge_setup(pg_ctx* ctx, int64_t n_scaf, const char* names, const int64_t* name_off, const int64_t* len,
                   int32_t n_files, const int32_t* out, const int64_t* n_dummy, const char* sep, int32_t sep_len,
                   const char* missing, int32_t miss_len, int32_t method, int64_t union_min, int64_t must_include_first,
                   int32_t* dense);
/* The next chunk (complete '\n' lines; the last one may lack its '\n') of file `file`'s body, which must have merged every
 * line of its previous chunk.  info = {lines of the chunk, its first line that stalls the file (the line count when none),
 * 0 no stall / 1 the file stalls there / 2 that line is refused (a byte >= 0x80 or a lone '\r'), the walk index of the line
 * before the stall (that of the file's last line so far, -1 none)}. */
int pg_merge_load(pg_ctx* ctx, int32_t file, const char* text, size_t len, int64_t* info);
/* The rows of walk indices (previous bound, hi] (hi < the walk's length), from every file's waiting lines up to hi.
 * *n_rows = rows written, *n_bytes = their bytes. */
int pg_merge_rows(pg_ctx* ctx, int64_t hi, int64_t* n_rows, int64_t* n_bytes);
/* Bytes [byte0, byte0 + cap) (at most to *n_bytes of pg_merge_rows) of those rows into out (host memory); a row may be cut
 * anywhere.  *bytes = bytes written. */
int pg_merge_emit(pg_ctx* ctx, int64_t byte0, char* out, size_t cap, size_t* bytes);

#ifdef __cplusplus
}
#endif
#endif /* PGWIN_H */
