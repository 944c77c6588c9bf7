/*
 * squidpy_b200.h — C ABI of libsquidpy_b200.so: H100 (sm_90a) kernels for squidpy's spatial-statistics hot
 * path.  Plain pointers and sizes only (no torch / numpy types).  All array arguments are HOST pointers owned
 * by the caller unless a parameter is documented as a device pointer; the library never frees caller memory.
 *
 * Conventions
 *   - every function returns 0 (SQB_OK) or a negative sqb_status; sqb_last_error() returns a thread-local
 *     human-readable message for the last failure on the calling thread;
 *   - a sqb_ctx binds one CUDA device and one stream (caller-supplied cudaStream_t, or library-owned);
 *     object handles (sqb_nhood, sqb_autocorr) belong to the ctx they were created on; handles are not
 *     thread-safe, distinct ctx/handles may be used concurrently (one per GPU);
 *   - calls are synchronous with respect to the host unless the name ends in _async.
 *
 * Each entry point replaces one internal seam of the reference (paths relative to the squidpy tree):
 *   sqb_nhood_count            <- _test(indices, indptr, clustering)          src/squidpy/gr/_nhood.py:60-61,208-209
 *   sqb_nhood_permute*         <- _nhood_enrichment_helper(...)               src/squidpy/gr/_nhood.py:516-547
 *                                 (+ rng.shuffle / _shuffle_group             src/squidpy/gr/_utils.py:185-213,
 *                                    spawn_generators                         src/squidpy/_utils.py:240-241)
 *   sqb_interaction_matrix     <- _interaction_matrix(data, indices, indptr, cats, out) src/squidpy/gr/_nhood.py:401,412-429
 *   sqb_autocorr_*             <- scanpy.metrics.morans_i / gearys_c call     src/squidpy/gr/_ppatterns.py:216,267-272
 *   sqb_cooc_counts            <- _occur_count(x, y, thresholds, labs, n,k,l) src/squidpy/gr/_ppatterns.py:283-310
 *   sqb_pair_counts_f64        <- KDTree(points, metric=...).two_point_correlation(points, r)  src/squidpy/gr/_ripley.py:218-223
 *   sqb_ligrec_counts          <- _score_permutations(data, clustering, generators, ...)  src/squidpy/gr/_ligrec.py:616-676
 *   sqb_sepal                  <- _diffusion(conc, use_hex, n_iter, sat, sat_idx, unsat, unsat_idx, dt, thresh)  src/squidpy/gr/_sepal.py:186-233
 *   sqb_sepal_idxs             <- g.eliminate_zeros() + the max_neighs check + _compute_idxs  src/squidpy/gr/_sepal.py:308-361
 *   sqb_dense_gather_device   <- X.toarray() / np.asarray(X) + DataFrame.fillna(0.0) + column selection  src/squidpy/gr/_ligrec.py:203-218,
 *                                 vals[:, genes] of _diffusion_genes  src/squidpy/gr/_sepal.py:117-128,186-233
 *   sqb_ligrec_observed        <- data.groupby("clusters").mean() / the expression-fraction mask of _analysis  src/squidpy/gr/_ligrec.py:679-700
 *   sqb_ligrec_counts_dense    <- _score_permutations on a gathered device matrix  src/squidpy/gr/_ligrec.py:616-676
 *   sqb_sepal_dense            <- _diffusion on a gathered device matrix  src/squidpy/gr/_sepal.py:186-233
 *   sqb_nn_dist_hist_f64       <- NearestNeighbors(...).fit(ref).kneighbors(qry) + np.histogram  src/squidpy/gr/_ripley.py:140-150,160-169,206-209
 *   sqb_nn_min_dist_f64        <- KDTree(anchor_coord, metric=...).query(batch_coord)  src/squidpy/tl/_var_by_distance.py:129-134
 *   sqb_window_ranges          <- the per-window coordinate masks of sliding_window  src/squidpy/tl/_sliding_window.py:130-158
 *   sqb_knn_2d / sqb_radius_2d <- NearestNeighbors.kneighbors / radius_neighbors src/squidpy/gr/neighbors.py:192-209,253-270,395-419
 *   sqb_delaunay_2d            <- scipy.spatial.Delaunay(coords).vertex_neighbor_vertices  src/squidpy/gr/neighbors.py:318-332
 *   sqb_graph_*                <- GraphBuilder.build + GraphBuilderCSR.combine  src/squidpy/gr/neighbors.py:80-156,192-209,253-270,365-477
 *   sqb_interaction_matrix     <- _interaction_matrix(data, indices, indptr, cats, out)  src/squidpy/gr/_nhood.py:412-429
 *   sqb_centrality_scores      <- _build_graph + rx.group_degree_centrality / rx.group_closeness_centrality + _local_clustering
 *                                 src/squidpy/gr/_nhood.py:305-317,432-491
 *   sqb_niche_profile          <- _NhoodProfileEmbedder: _calculate_neighborhood_profile + the hop loop of get_embedding
 *                                 src/squidpy/gr/_niche.py:1117-1169,1176-1214
 *   sqb_niche_aggregate        <- normalize(A, "l1") @ X of _UtagEmbedder (:1259-1260); _setdiag, _hop, _normalize, _aggregate
 *                                 and hstack(...).toarray() of _CellcharterEmbedder (:1002-1054,1336-1355)
 *   sqb_mask_graph             <- _get_lines_coords + GeoDataFrame(LineString).within(polygon) + the masked assignments and
 *                                 eliminate_zeros of mask_graph  src/squidpy/gr/_build.py:853-966
 */
#ifndef SQUIDPY_B200_H
#define SQUIDPY_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SQB_ABI_VERSION 18

typedef enum {
    SQB_OK = 0,
    SQB_ERR_INVALID = -1, /* bad argument (message says which) */
    SQB_ERR_CUDA = -2,    /* CUDA runtime / launch failure */
    SQB_ERR_OOM = -3,     /* device allocation failed */
    SQB_ERR_UNSUPPORTED = -4,
    SQB_ERR_STATE = -5, /* call sequence error (e.g. run before upload) */
    SQB_ERR_LAYOUT = -6 /* a valid input in a layout the entry point does not take (message says which): use another path */
} sqb_status;

typedef struct sqb_ctx sqb_ctx;
typedef struct sqb_nhood sqb_nhood;
typedef struct sqb_autocorr sqb_autocorr;
typedef struct sqb_dense sqb_dense;

/* ---- library / context --------------------------------------------------------------------------- */
int sqb_abi_version(void);
const char* sqb_last_error(void);
int sqb_device_count(int* count);

/* stream: a cudaStream_t to launch on (e.g. torch's current stream), or NULL for a library-owned stream. */
int sqb_ctx_create(int device, void* stream, sqb_ctx** out);
int sqb_ctx_destroy(sqb_ctx* ctx);
int sqb_ctx_sync(sqb_ctx* ctx);
int sqb_ctx_stream(sqb_ctx* ctx, void** stream);
int sqb_ctx_sm_count(sqb_ctx* ctx, int* sm_count);
/* number of kernels this library launched on ctx so far */
int sqb_ctx_launch_count(sqb_ctx* ctx, int64_t* launches);
/* per-kernel-class event timing (synchronises every launch; for roofline passes, not for throughput runs) */
int sqb_ctx_profile(sqb_ctx* ctx, int enable);
int sqb_ctx_profile_reset(sqb_ctx* ctx);
/* kclass: 0 fill, 1 shuffle, 2 transpose, 3 count, 4 autocorr prep, 5 autocorr main, 6 autocorr final, 7 pairs, 8 misc */
int sqb_ctx_profile_get(sqb_ctx* ctx, int kclass, double* ms, int64_t* launches);

/* page-locked host memory for the host-facing API (so H2D/D2H copies run at full PCIe rate) */
int sqb_host_alloc(size_t bytes, void** ptr);
int sqb_host_free(void* ptr);

/* *device = the CUDA device ordinal that owns p (device or managed memory), or -1 for host / unregistered memory. */
int sqb_pointer_device(const void* p, int* device);

/* ---- nhood_enrichment ------------------------------------------------------------------------------
 * Graph = CSR of obsp['spatial_connectivities'] (data ignored; entries counted as stored; reference dtypes
 * uint32, _nhood.py:52,205).  n_cls = number of categories (labels in [0, n_cls)).                       */
int sqb_nhood_create(sqb_ctx* ctx, int64_t n, int64_t nnz, const uint32_t* indptr, const uint32_t* indices,
                     int n_cls, sqb_nhood** out);
/* The same from a graph already in device memory (e.g. a cupy / torch CSR of the caller): indptr (n + 1 entries) and
 * indices (nnz) are DEVICE pointers on the context's device with indptr_bits / index_bits 32 or 64 (signed).  The handle
 * converts them into its own uint32 copy on the device (the caller may free its buffers once the call returns; the library
 * never writes them); from there the graph is prepared exactly as by sqb_nhood_create.  indptr must run from 0 to nnz
 * without decreasing and every index must lie in [0, n) (negative ones included): both are checked on the device before
 * anything follows the arrays (SQB_ERR_INVALID).  producer_stream: as in sqb_autocorr_load_csr_device.  A CSC graph
 * passed here is the CSR of its transpose: every count it yields is the transpose of the graph's.                      */
int sqb_nhood_create_device(sqb_ctx* ctx, int64_t n, int64_t nnz, const void* indptr, int indptr_bits, const void* indices,
                            int index_bits, int n_cls, uintptr_t producer_stream, sqb_nhood** out);
int sqb_nhood_destroy(sqb_nhood* h);

/* observed count: out[a*n_cls+b] = #stored entries (i->j) with labels[i]=a, labels[j]=b   (uint32)       */
int sqb_nhood_count(sqb_nhood* h, const uint32_t* labels, uint32_t* out);

/* Base labels for the permutation test and the optional library partition (lib_codes[i] in [0,n_libs),
 * NULL/0 for none).  With libraries each category is shuffled separately, in category order, by the same
 * generator (gr/_utils.py:208-212).                                                                      */
int sqb_nhood_set_base(sqb_nhood* h, const uint32_t* base_labels, const int32_t* lib_codes, int n_libs);

/* Permutation test.  states: n_perms x 6 uint64 = numpy PCG64 state of generator p
 *   {state_hi, state_lo, inc_hi, inc_lo, has_uint32, uinteger}  (has_uint32 must be 0: fresh generators).
 * Permutation p replays numpy Generator.shuffle bit-exactly on the device and counts.
 * out_counts: n_perms x n_cls x n_cls uint32.                                                            */
int sqb_nhood_permute(sqb_nhood* h, const uint64_t* states, int64_t n_perms, uint32_t* out_counts);

/* The same in three steps, for measurement with inputs resident in HBM:
 * upload (H2D of the generator states), run (kernels only, asynchronous on the ctx stream, results stay on
 * the device), download (D2H of the counts, synchronises).                                               */
int sqb_nhood_permute_upload(sqb_nhood* h, const uint64_t* states, int64_t n_perms);
int sqb_nhood_permute_run_async(sqb_nhood* h);
int sqb_nhood_permute_download(sqb_nhood* h, uint32_t* out_counts);
/* Fast RNG mode (NOT the reference's permutations): permutation p (global index first_perm + p) of every library
 * segment is a keyed bijection — 4-round Feistel network with cycle walking, round keys = splitmix64(seed, global
 * permutation index, segment, round) — applied to the segment's labels sorted by class; labels are written straight into
 * the permutation-minor matrix the count kernel reads (no stream replay, no Fisher-Yates, no transposition).  Same
 * null distribution as numpy's shuffle, different draws: z-scores agree with the exact mode to O(n_perms^-1/2)
 * (SURVEY.md 8d "Fast-RNG validation"); tests/philox_ref.py is the executable specification.  After this upload,
 * run_async / download / stats / sums / var_chain / shuffled_labels work as in the exact mode.                     */
int sqb_nhood_permute_upload_philox(sqb_nhood* h, uint64_t seed, int64_t first_perm, int64_t n_perms);
/* Mean and standard deviation over the permutations of every count bin (n_cls x n_cls float64 each), computed on the
 * device in the operation order of numpy's perms.mean(axis=0) / perms.std(axis=0) on the float64 counts
 * (_nhood.py:231), i.e. bit-identical to the reference's host computation; saves the download of all counts.          */
int sqb_nhood_permute_stats(sqb_nhood* h, double* mean_out, double* std_out);
/* The same statistics when the permutations are sharded over several GPUs (contiguous shards in rank order):
 * sums: exact integer per-bin sums of this handle's permutations (all-reduce them, mean = sum / P_total);
 * var_chain: acc_out = acc_in continued with numpy's sequential sum((x - mean)^2) over this handle's permutations; rank r
 * passes acc_out to rank r+1, std = sqrt(acc_last / P_total): bit-identical to perms.std(axis=0) on the gathered counts.  */
int sqb_nhood_permute_sums(sqb_nhood* h, int64_t* sums_out);
int sqb_nhood_permute_var_chain(sqb_nhood* h, const double* mean, const double* acc_in, double* acc_out);

/* The same statistics with DEVICE pointers (n_cls*n_cls elements each), asynchronous on the ctx stream: for callers that
 * hand the buffers straight to a collective (torch tensors + NCCL) — no host round trip between count kernel and all-reduce. */
int sqb_nhood_permute_stats_dev(sqb_nhood* h, double* d_mean, double* d_std);
int sqb_nhood_permute_sums_dev(sqb_nhood* h, int64_t* d_sums);
int sqb_nhood_permute_var_chain_dev(sqb_nhood* h, const double* d_mean, const double* d_acc_in, double* d_acc_out);
/* Multi-GPU statistics by gathering (what squidpy_b200._dist does under NCCL): the per-permutation counts [n_perms][n_cls^2] as an
 * asynchronous device-to-device copy on the context's stream into a caller-owned buffer (the block a collective sends), and the
 * mean / std over the rows of any device array of counts (the gathered blocks, rows in global permutation order) -- the kernel of
 * sqb_nhood_permute_stats, i.e. `perms.mean(0)` / `perms.std(0)` of gr/_nhood.py:231 in numpy's operation order.          */
int sqb_nhood_permute_counts_dev(sqb_nhood* h, uint32_t* d_dst);
int sqb_nhood_stats_rows_dev(sqb_ctx* ctx, const uint32_t* d_counts, int64_t rows, int n_cls, double* d_mean, double* d_std);

/* Test hook: shuffled label vectors of permutations [p0, p1) of the last upload, recomputed on the device
 * (original node order), out: (p1-p0) x n uint32.                                                        */
int sqb_nhood_shuffled_labels(sqb_nhood* h, int64_t p0, int64_t p1, uint32_t* out);

/* Tuning / test options (all variants produce bit-identical results).
 *   "shuffle_algo"   -1 auto [default]: for many permutations of large arrays the partitioned region replay (9), or the
 *                    list replay (7) where a library segment exceeds its limits; else 1 / 2;
 *                    1 CTA per permutation; 2 warp per permutation; 7 two kernels (swap-target generation + list apply);
 *                    9 two kernels (swap targets partitioned by region of the array + region replay in shared memory; a
 *                    segment needing more than 16 regions or 2048-step blocks than threads makes the call use 7 instead).
 *                    Any other value is refused with SQB_ERR_INVALID.
 *   "shuffle_threads" 128/256/512/1024 (algos 1, 7), 512/1024 (9), "shuffle_r" 2/4/8 steps per thread (7),
 *   "shuffle_q"      1/2/4/8 PCG64 outputs per lane and batch (2, and the target generation of 7),
 *   "shuffle_low"    elements of every label array kept in shared memory by the apply kernel of 7 (-1 all that fits, 0 off),
 *   "shuffle_region" positions per region of 9 (0 = as many as shared memory holds; smaller values are a test hook),
 *   "shuffle_ctas"   persistent grid size = permutations in flight (0 = occupancy x SM count),
 *   "shuffle_stagger_us" start-up stagger of the persistent CTAs, "shuffle_wfactor_x100" window = min(i/4, f*sqrt(i)),
 *   "perm_chunk"     permutations resident at once (read at the next upload), "count_algo" 0 auto / 1 shared-memory histograms /
 *                    2 global atomics, "count_sym" -1 auto (row-record kernel; structurally symmetric graphs are counted from the entries with j >= i) /
 *                    0 always the CSR-row kernel on the full CSR, "count_un" row records (three entries each) a warp takes per pass in the count kernel (1 / 2 / 3 / 4),
 *   "count_single"   sqb_nhood_count: 1 dedicated single-vector kernel [default] / 0 the batched kernels (test hook). */
int sqb_nhood_set_option(sqb_nhood* h, const char* key, int64_t value);
/* algorithmic bytes per permutation, SURVEY.md 8(d): 4*nnz + 4*(n+1) + 8*n + 4*n_cls^2                   */
int sqb_nhood_bytes_per_perm(sqb_nhood* h, int64_t* bytes);

/* ---- interaction_matrix ------------------------------------------------------------------------------
 * Replaces _interaction_matrix(data, indices, indptr, cats, output) (src/squidpy/gr/_nhood.py:401,412-429) and the NaN
 * masking of interaction_matrix (:386-395).  codes[i] in [0, n_cls) or < 0 for an observation without label: stored
 * entries with an unlabelled end point are skipped (== restricting the graph to the labelled observations).
 * data_dtype -1 (weights=False, data unused): out_counts[a*n_cls+b] = number of stored entries (i->j) with code(i)=a,
 * code(j)=b (int64).  weights=True: data_dtype 3 = int32, 4 = int64, 5 = bool (one byte): out_counts = int64 sum of their
 * values, wrapping modulo 2^64 like numba's int64; 0 = f32, 1 = f64: out_weighted = float64 sum in the reference's order
 * (rows ascending, each row's entries in storage order), bit-identical to it and the same from run to run.            */
int sqb_interaction_matrix(sqb_ctx* ctx, int64_t n, int64_t nnz, const uint32_t* indptr, const uint32_t* indices,
                           const void* data, int data_dtype, const int32_t* codes, int n_cls, double* out_weighted,
                           int64_t* out_counts);
/* The same from a graph in device memory, read in place (no copy): indptr / indices / data are DEVICE pointers on the
 * context's device, indptr_bits / index_bits 32 or 64; codes and the outputs stay on the host.  csc != 0: the arrays are a
 * CSC graph's, i.e. the CSR of its transpose; out is then the transpose of the graph's result, and float sums follow the
 * order of the graph's tocsr() (rows ascending, columns ascending within a row, duplicates in storage order).  data_dtype
 * and outputs as above, plus 2 = f16 (float64 sums).  indptr is checked on the device before anything follows it; column indices outside
 * [0, n) and codes >= n_cls are detected by the kernel (SQB_ERR_INVALID, no result).  producer_stream: as in
 * sqb_autocorr_load_csr_device.  Returns after the device has stopped reading the caller's buffers.                   */
int sqb_interaction_matrix_device(sqb_ctx* ctx, int64_t n, int64_t nnz, const void* indptr, int indptr_bits, const void* indices,
                                  int index_bits, int csc, const void* data, int data_dtype, const int32_t* codes, int n_cls,
                                  double* out_weighted, int64_t* out_counts, uintptr_t producer_stream);

/* ---- centrality_scores -------------------------------------------------------------------------------------
 * The integer parts of the three group measures of centrality_scores (src/squidpy/gr/_nhood.py:245-346), over the graph
 * _build_graph makes (:432-454): A + Aᵀ with values summed in A's dtype, diagonal and zero sums dropped (an explicit zero or a
 * cancelling +w / -w pair removes the edge, a NaN sum keeps it).  The caller's CSR is taken as given, from the host
 * (device_input = 0: host pointers, uploaded) or from device memory (device_input = 1: DEVICE pointers on the context's
 * device, read in place; producer_stream as in sqb_autocorr_load_csr_device).  indptr_bits / index_bits 32 or 64;
 * data_dtype 0 = f32, 1 = f64, 3 = int32, 4 = int64, 5 = bool (one byte); an integer sum wraps at int_bits (8, 16, 32 or 64:
 * the width of the caller's dtype, whose values may arrive widened to int32 / int64).  nnz < 2^30; data may be NULL when nnz = 0.
 * codes[v] in [0, n_cls) is the cluster of observation v, -1 none (it is a node but in no group).  measures: a mask of
 *   1: out_reach1[k] = |N(S_k) \ S_k|                              (rx.group_degree_centrality numerator, :311-312)
 *   2: out_dist[k]   = sum over v not in S_k reachable from S_k of the hop distance d(S_k, v)
 *                      (rx.group_closeness_centrality denominator, :309-310); *out_levels = deepest BFS level reached
 *   4: out_cc[v]     = 2 T(v) / (k_v (k_v - 1)) in float64, 0 when k_v < 2  (_local_clustering, :457-491)
 * The divisions by n - |S_k| and the per-group means are the caller's.  Column indices outside [0, n) or an indptr not
 * running from 0 to nnz return SQB_ERR_INVALID.  Returns after the device has stopped reading the caller's buffers.          */
int sqb_centrality_scores(sqb_ctx* ctx, int64_t n, int64_t nnz, const void* indptr, int indptr_bits, const void* indices,
                          int index_bits, const void* data, int data_dtype, int int_bits, int device_input, const int32_t* codes,
                          int n_cls, int measures, int64_t* out_reach1, int64_t* out_dist, double* out_cc, int64_t* out_levels,
                          uintptr_t producer_stream);

/* ---- ligrec permutation test ------------------------------------------------------------------------------
 * _score_permutations of the reference (src/squidpy/gr/_ligrec.py:616-676) for a handle whose base labels are the cells'
 * cluster codes (sqb_nhood_set_base on a graph-less handle: nnz = 0) and whose numpy generator states are uploaded
 * (sqb_nhood_permute_upload).  data: n x n_genes float64 row-major; inv_counts: n_cls; mean_obs: n_cls x n_genes;
 * interactions: n_inter x 2 gene indices; inter_clusters: n_cpairs x 2 cluster indices; valid: n_inter x n_cpairs (uint8).
 * out_counts[i, j] = #permutations with  mean_perm[a, g0] + mean_perm[b, g1] > mean_obs[a, g0] + mean_obs[b, g1]
 * (int64; same float64 operation order as the reference, so the decisions are identical).                          */
int sqb_ligrec_counts(sqb_nhood* h, const double* data, int64_t n_genes, const double* inv_counts, const double* mean_obs,
                      const int32_t* interactions, int64_t n_inter, const int32_t* inter_clusters, int64_t n_cpairs,
                      const uint8_t* valid, int64_t* out_counts);

/* ---- expression matrix in GPU memory: ligrec and sepal -------------------------------------------------------------
 * sqb_dense_gather_device reads a caller's device-resident X (observations x genes: n_rows x n_cols) in place and writes the
 * selected rows x selected columns into a dense matrix owned by the returned handle (on the context's device).
 *   format 0 dense: x is the matrix with element strides stride_row / stride_col (C order, F order or a strided view);
 *   format 1 CSR / 2 CSC: x is the values array, indptr / indices DEVICE pointers with indptr_bits / index_bits 32 or 64, nnz
 *          the number of stored entries.  indptr must run from 0 to nnz without decreasing (checked on the device before
 *          anything follows it, one synchronisation); an index outside its range is rejected; two stored entries that fall
 *          into the same gathered cell are rejected (SQB_ERR_INVALID): scipy's toarray() sums such duplicates on the host, so
 *          sum them first.  Duplicates in rows or columns that are not gathered are never read.
 *   x_dtype: 0 = f32, 1 = f64, 2 = f16, 3 = int32, 4 = int64.
 *   rows (HOST, ascending, n_rows_out entries) or NULL for every row; cols (HOST, n_cols_out distinct input columns, in output
 *          order).
 *   layout 0: observations x genes row-major (what sqb_ligrec_observed / sqb_ligrec_counts_dense read); 1: genes x observations
 *          row-major (what sqb_sepal_dense reads).
 *   flags: 1 = write NaN as 0.0 (ligrec's fillna(0.0)); 2 = keep the input's value type (else every value is converted to
 *          float64 exactly, like astype(float64)).
 *   producer_stream: as in sqb_autocorr_load_csr_device.  Returns after the device has stopped reading the caller's buffers;
 *   on an error no handle is returned and the context stays usable.  The extra device memory is the gathered block.      */
int sqb_dense_gather_device(sqb_ctx* ctx, int format, const void* x, const void* indptr, int indptr_bits, const void* indices,
                            int index_bits, int64_t nnz, int x_dtype, int64_t n_rows, int64_t n_cols, int64_t stride_row,
                            int64_t stride_col, const int64_t* rows, int64_t n_rows_out, const int32_t* cols, int64_t n_cols_out,
                            int layout, int flags, uintptr_t producer_stream, sqb_dense** out);
/* The gathered values in their stored layout and type (n_rows_out x n_cols_out or its transpose) into HOST memory.          */
int sqb_dense_download(sqb_dense* d, void* out);
int sqb_dense_free(sqb_dense* d);
/* Observed statistics of ligrec on a layout-0 float64 gathered matrix with NaN written as 0: codes[i] in [0, n_cls) is the
 * cluster of observation i.  mean_out[k, g] = pandas' groupby mean (a Kahan sum over the cluster's observations in order,
 * the compensation reset when it is NaN, divided by the count), npos_out[k, g] = number of values > 0, sizes_out[k] = number
 * of observations of cluster k (all HOST, n_cls x n_genes / n_cls).                                                       */
int sqb_ligrec_observed(sqb_dense* d, const int32_t* codes, int n_cls, double* mean_out, int64_t* npos_out, int64_t* sizes_out);
/* sqb_ligrec_counts with the layout-0 float64 gathered matrix (observations = the handle's cells) in place of data.        */
int sqb_ligrec_counts_dense(sqb_nhood* h, const sqb_dense* x, const double* inv_counts, const double* mean_obs,
                            const int32_t* interactions, int64_t n_inter, const int32_t* inter_clusters, int64_t n_cpairs,
                            const uint8_t* valid, int64_t* out_counts);
/* sqb_sepal with a layout-1 float64 gathered matrix (one row per gene) in place of vals, on the matrix's context.          */
int sqb_sepal_dense(const sqb_dense* x, const int32_t* sat, int64_t n_sat, const int32_t* sat_idx, int max_neighs,
                    const int32_t* unsat, const int32_t* unsat_idx, int64_t n_unsat, int n_iter, double dt, double thresh,
                    double* out);

/* ---- spatial_autocorr (Moran's I / Geary's C) -------------------------------------------------------
 * W = obsp[connectivity_key] (after optional float32 row normalisation on the host) as CSR; w_dtype 0 = f32,
 * 1 = f64 (cast to f64 like scanpy does).  mode 0 = Moran's I, 1 = Geary's C.
 * X layout 0: features x obs (row-major dense, or CSR by feature); layout 1: obs x features (row-major
 * dense, or CSR by observation == CSC of the features x obs matrix, AnnData's native X).
 * x_dtype 0 = f32, 1 = f64.  row_perm (or NULL): length-n permutation p; row r of the permuted W is row p[r]
 * (g[idx_shuffle, :], _ppatterns.py:271-272).  out: n_features float64 (NaN for constant features).
 * Sparse X must not store an observation twice for one feature (scipy: sum_duplicates()); indices need not be
 * sorted.  Index ranges, indptr monotonicity and duplicates are checked on the device (SQB_ERR_INVALID).   */
int sqb_autocorr_create(sqb_ctx* ctx, int64_t n, int64_t nnz, const int32_t* w_indptr, const int32_t* w_indices,
                        const void* w_data, int w_dtype, sqb_autocorr** out);
/* The same from a weight matrix already in device memory (e.g. a torch sparse_csr or cupyx CSR of the caller), read in place
 * and never on the host: indptr (n + 1 entries), indices and data (nnz) are DEVICE pointers on the context's device,
 * indptr_bits / index_bits 32 or 64, value_code 0 = f32, 1 = f64.  Every row must be canonical (strictly increasing column
 * indices): indptr is checked first (SQB_ERR_INVALID unless it runs from 0 to nnz without decreasing), then every index must
 * lie in [0, n) (SQB_ERR_INVALID) and every row be canonical (SQB_ERR_LAYOUT: take the host path).  transformation != 0
 * row-normalises W like sklearn's normalize(W, norm="l1", axis=1) in W's dtype; NaN or infinite weights, which normalize rejects,
 * then return SQB_ERR_LAYOUT too.  data holds exactly nnz contiguous values.  The handle's W then equals, bit for bit, what
 * sqb_autocorr_create builds from the same (normalised) host CSR.  out_moments (host, 3): s0, s1, s2 of the normalised W
 * (_g_moments of the reference, src/squidpy/gr/_ppatterns.py:541-559) evaluated in W's dtype in scipy's operation order,
 * converted exactly to double.  producer_stream: as in sqb_autocorr_load_csr_device.  Returns after the device has stopped
 * reading the caller's buffers; on an error no handle is returned and the context stays usable.                             */
int sqb_autocorr_create_device(sqb_ctx* ctx, int64_t n, int64_t nnz, const void* indptr, int indptr_bits, const void* indices,
                               int index_bits, const void* data, int value_code, int transformation, uintptr_t producer_stream,
                               double* out_moments, sqb_autocorr** out);
/* How the handle's W is held: *w_format 0 packed rows of 8 slots, 1 packed rows of 16, 2 CSR walk, 3 compact rows (7 columns +
 * one common float32 weight); *s0_branch 0 = S0 summed exactly as an integer sum in parallel, 1 = one ordered thread.          */
int sqb_autocorr_w_info(sqb_autocorr* h, int* w_format, int* s0_branch);
int sqb_autocorr_destroy(sqb_autocorr* h);
int sqb_autocorr_load_dense(sqb_autocorr* h, const void* x, int x_dtype, int layout, int64_t n_features);
int sqb_autocorr_load_csr(sqb_autocorr* h, const int64_t* x_indptr, const int32_t* x_indices, const void* x_data,
                          int x_dtype, int layout, int64_t n_features);
/* Feature shard of a CSR-by-observation matrix (multi-GPU: every rank takes a contiguous range of features): uploads only
 * the columns col_lo <= c < col_hi of every row (rows must hold ascending column indices — scipy's sorted indices; the
 * slices are found with two binary searches per row and packed into pinned staging buffers by host threads) and loads them
 * as features 0 .. col_hi - col_lo.                                                                          */
int sqb_autocorr_load_csr_cols(sqb_autocorr* h, const int64_t* x_indptr, const int32_t* x_indices, const void* x_data,
                               int x_dtype, int64_t n_features_total, int64_t col_lo, int64_t col_hi);
/* Device-resident X (e.g. a cupy / torch array of the caller).  indptr, indices, data and x are DEVICE pointers on the
 * context's device; everything else is on the host.
 *   col_map (host, int32, one entry per input feature): the feature's index in [0, n_out) among the loaded features, or -1
 *           to skip it; every output index must occur exactly once.  One map expresses a gene subset in any order, a mask
 *           and a multi-GPU shard.
 *   data_dtype / x_dtype: 0 = f32, 1 = f64, 2 = f16, 3 = int32, 4 = int64.  f32 is loaded as f32, every other type is
 *           converted to f64 on the device (what the host path does on the host).
 *   producer_stream: the CUDA Array Interface v3 `stream` of the arrays: 0 = none, 1 = legacy default stream, 2 = per-thread
 *           default stream, else a cudaStream_t.  The context's stream waits on an event recorded there before it reads X.
 *   Both calls return after the device has finished reading the caller's buffers: the caller may then free or overwrite them.
 *   The library never writes caller memory.
 * CSR: indptr_bits / index_bits 32 or 64; layout as in sqb_autocorr_load_csr (1 = observations x features, AnnData's CSR X;
 *   0 = features x observations, AnnData's CSC X); n_cols = number of input features.  Indices need not be sorted.  Index
 *   ranges, indptr monotonicity (checked before anything follows indptr) and duplicates are validated on the device
 *   (SQB_ERR_INVALID).  The matrix is read in place: no staging copy; the extra device memory is the relaid-out copy of the
 *   selected features plus one transposition buffer of their entries (layout 1).
 * Dense: x is rows x cols with element strides stride_row / stride_col (C order, F order or a strided view; any sign);
 *   layout 1: rows = observations, 0: rows = features.  The selected features are gathered into the layout
 *   sqb_autocorr_load_dense produces for that layout.                                                          */
int sqb_autocorr_load_csr_device(sqb_autocorr* h, const void* indptr, int indptr_bits, const void* indices, int index_bits,
                                 const void* data, int data_dtype, int layout, int64_t n_cols, const int32_t* col_map, int64_t n_out,
                                 uintptr_t producer_stream);
int sqb_autocorr_load_dense_device(sqb_autocorr* h, const void* x, int x_dtype, int64_t rows, int64_t cols, int64_t stride_row,
                                   int64_t stride_col, int layout, const int32_t* col_map, int64_t n_out, uintptr_t producer_stream);
int sqb_autocorr_run_async(sqb_autocorr* h, int mode, const int64_t* row_perm);
int sqb_autocorr_download(sqb_autocorr* h, double* out);
/* The permutation variant in one call (_score_helper, _ppatterns.py:258-280): row_perms = n_perms x n int64 (row p is
 * idx_shuffle of permutation p), out = n_perms x n_features float64.  X stays resident; the permutations are validated
 * on the device (one error flag per batch) and every permutation is one kernel launch.                      */
int sqb_autocorr_run_perms(sqb_autocorr* h, int mode, const int64_t* row_perms, int64_t n_perms, double* out);
/* load + run + download */
int sqb_autocorr_dense(sqb_autocorr* h, int mode, const void* x, int x_dtype, int layout, int64_t n_features,
                       const int64_t* row_perm, double* out);
int sqb_autocorr_csr(sqb_autocorr* h, int mode, const int64_t* x_indptr, const int32_t* x_indices,
                     const void* x_data, int x_dtype, int layout, int64_t n_features, const int64_t* row_perm,
                     double* out);

/* ---- co_occurrence ------------------------------------------------------------------------------------
 * out[(a*k+b)*L + r] = #{ordered (i,j), i != j : labs[i]=a, labs[j]=b, d2_ij <= thr[r]}  (int64, cumulative in
 * r), float32 arithmetic with d2 = fma(dy,dy,dx*dx) (use_fma=1, what the reference's JIT emits on x86-64 with
 * FMA) or dx*dx+dy*dy (use_fma=0).  thr ascending.  Only tiles t with t % shard_count == shard_index are
 * evaluated (multi-GPU sharding; pass 0,1 for everything); partial results add up across shards.          */
int sqb_cooc_counts(sqb_ctx* ctx, const float* x, const float* y, int64_t n, const int32_t* labs, int k,
                    const float* thr, int L, int use_fma, int shard_index, int shard_count, int64_t* out);

/* ---- ripley L -------------------------------------------------------------------------------------------
 * For every group g (points group_ptr[g]..group_ptr[g+1] of pts, interleaved x,y float64):
 * out[g*S + s] = #{ordered (i,j) in group g, INCLUDING i == j : dist(i, j) <= support[s]}  (int64),
 * i.e. sklearn KDTree(points_g, metric=...).two_point_correlation(points_g, support).  support ascending, no NaN;
 * a negative radius counts nothing.  metric (the codes of sqb_nn_min_dist_f64) 0 euclidean sqrt(dx*dx + dy*dy) without
 * contraction, 1 manhattan |dx| + |dy|, 2 chebyshev max(|dx|, |dy|), in float64; any other code is SQB_ERR_INVALID.
 * Tiles t with t % shard_count == shard_index are evaluated, and shard 0 adds the self pairs (multi-GPU sharding;
 * pass 0,1 for everything); partial results add up across shards.                                           */
int sqb_pair_counts_f64(sqb_ctx* ctx, const double* pts, const int64_t* group_ptr, int n_groups,
                        const double* support, int S, int metric, int shard_index, int shard_count, int64_t* out);

/* ---- ripley F / G ----------------------------------------------------------------------------------------
 * Histograms of nearest-neighbour distances (src/squidpy/gr/_ripley.py:140-150,160-169: kneighbors of a query set against a
 * tree of a reference set, and :206-209: np.histogram of the distances).  pts: n_pts x 2 float64 point pool (interleaved x,y).
 * tasks: n_tasks x 6 int64 {ref_begin, ref_end, qry_begin, qry_end, k, out_row}, ranges into the pool: the k nearest
 * distances of every query point among the reference points (no point excluded: zero distances count) are binned into row
 * out_row.  Distances are sqrt(dx*dx + dy*dy) in float64 without contraction (scikit-learn's kd_tree).  Binning is
 * np.histogram(d, bins=support) for ascending support (S >= 2 edges): S - 1 bins, the last one closed, distances outside
 * [support[0], support[S-1]] dropped.  out: n_rows x (S - 1) int64, the sums over the tasks of each row.  k in [1, 64] and
 * k <= ref_end - ref_begin.  Query blocks of 1024 points, numbered over the tasks in order, are evaluated when
 * block % shard_count == shard_index (multi-GPU sharding; pass 0,1 for everything); partial results add up across shards. */
int sqb_nn_dist_hist_f64(sqb_ctx* ctx, const double* pts, int64_t n_pts, const int64_t* tasks, int64_t n_tasks,
                         const double* support, int S, int n_rows, int shard_index, int shard_count, int64_t* out);

/* ---- tl.var_by_distance ----------------------------------------------------------------------------------------------
 * Distance from every query point to its nearest reference point (src/squidpy/tl/_var_by_distance.py:129-134: KDTree of the
 * anchor coordinates, queried with every observation).  pts: n_pts x 2 float64 point pool (interleaved x,y), n_pts < 2^31, all
 * finite.  tasks: n_tasks x 5 int64 {ref_begin, ref_end, qry_begin, qry_end, out_begin}, ranges into the pool:
 * out[out_begin + (q - qry_begin)] = min over r in [ref_begin, ref_end) of dist(pts[q], pts[r]) for q in [qry_begin, qry_end)
 * (no point excluded: a query that is also a reference point gets 0).  metric 0 euclidean sqrt(dx*dx + dy*dy) without
 * contraction, 1 manhattan |dx| + |dy|, 2 chebyshev max(|dx|, |dy|): bit-identical to scikit-learn's KDTree.query.  Reference
 * ranges must be non-empty; output ranges must lie in [0, n_out) and not overlap.  out: n_out float64; positions no task
 * writes are NaN.                                                                                                         */
int sqb_nn_min_dist_f64(sqb_ctx* ctx, const double* pts, int64_t n_pts, const int64_t* tasks, int64_t n_tasks, int metric,
                        int64_t n_out, double* out);

/* ---- tl.sliding_window -------------------------------------------------------------------------------------------------
 * The windows that contain each observation (src/squidpy/tl/_sliding_window.py:130-158: one mask
 * x_start <= x <= x_end & y_start <= y <= y_end over the library's observations per window; the windows of a library are the
 * product of its x and y windows, :224-242).  xy: n x 2 coordinates (interleaved x,y), n < 2^31, in the dtype the comparisons
 * are made in: xy_dtype 0 float64, 1 int64; starts / ends hold the edges in the same dtype.  lib[i] in [-1, n_libs) is the
 * library of observation i, -1 none.  edge_off (2 n_libs + 1 entries, edge_off[0] = 0): the x edges of library l are
 * starts / ends [edge_off[2l], edge_off[2l+1]), its y edges [edge_off[2l+1], edge_off[2l+2]); within one such range both starts
 * and ends must be non-decreasing and not NaN (SQB_ERR_INVALID otherwise).  out: n x 4 int32 {lo_x, hi_x, lo_y, hi_y}, where
 * hi = the last window index whose start <= v and lo = the first whose end >= v: observation i lies in window (ix, iy) of its
 * library iff lo_x <= ix <= hi_x and lo_y <= iy <= hi_y.  An axis with lo > hi, a NaN coordinate or lib[i] = -1 (written as
 * {0, -1, 0, -1}) puts the observation in no window.                                                                       */
int sqb_window_ranges(sqb_ctx* ctx, const void* xy, int xy_dtype, int64_t n, const int32_t* lib, int n_libs, const int64_t* edge_off,
                      const void* starts, const void* ends, int32_t* out);

/* ---- sepal ---------------------------------------------------------------------------------------------------------
 * `_diffusion` for every gene (src/squidpy/gr/_sepal.py:186-289): vals = n_genes x n float64 (one row per gene), sat / unsat =
 * saturated / unsaturated node ids, sat_idx = n_sat x max_neighs neighbour ids, unsat_idx = nearest saturated node of every
 * unsaturated node (`_compute_idxs`, :292-306).  out[g] = dt * (first iteration whose entropy change is <= thresh), NaN if
 * n_iter iterations do not converge.                                                                                  */
int sqb_sepal(sqb_ctx* ctx, const double* vals, int64_t n_genes, int64_t n, const int32_t* sat, int64_t n_sat,
              const int32_t* sat_idx, int max_neighs, const int32_t* unsat, const int32_t* unsat_idx, int64_t n_unsat,
              int n_iter, double dt, double thresh, double* out);
/* The tables sqb_sepal reads (`_compute_idxs`, src/squidpy/gr/_sepal.py:308-361), built on the device.
 *   The graph: an n x n CSR (csc = 0) or CSC (csc = 1, read as scipy's tocsr) from the host (device_input = 0) or from device
 *   memory (device_input = 1: DEVICE pointers on the context's device, read in place after producer_stream, as in
 *   sqb_autocorr_load_csr_device).  indptr_bits / index_bits 32 or 64; data_dtype 0 f32, 1 f64, 3 i32, 4 i64, 5 bool; nnz < 2^31.
 *   Entries whose value is 0 are dropped in storage order (eliminate_zeros: NaN stays, -0.0 and False go); a node's degree is
 *   its count of remaining entries, duplicates included.
 *   *max_degree: the largest degree.  When it is not max_neighs (in [1, 1024]) the call returns here, nothing else written.
 *   Otherwise, in HOST buffers of n, n x max_neighs, n and n entries: sat = the ascending nodes of degree max_neighs (*n_sat),
 *   sat_idx = their remaining columns in storage order, unsat = the ascending other nodes (*n_unsat), unsat_idx = each one's
 *   first remaining column that is saturated, or for an orphan (no such column) the saturated node j minimising
 *   |x_o - x_j| + |y_o - y_j| in float64, numpy's argmin over the ascending saturated nodes (the first of equal distances, the
 *   first NaN distance before any other).
 *   xy: n x 2 coordinates, read only when orphans exist: host float64 C-contiguous (xy_device = 0, xy_dtype 1, strides 2 and 1),
 *   or a DEVICE pointer on the context's device (xy_device = 1, read after xy_stream) of xy_dtype 0 f32 / 1 f64 with element
 *   strides stride_row / stride_col.  *nonfinite = 1 when a coordinate of an orphan or of a saturated node was read and is NaN
 *   or infinite (scikit-learn's pairwise_distances refuses those), else 0.
 * Returns once the caller's arrays are no longer read; errors leave the context usable.                                  */
int sqb_sepal_idxs(sqb_ctx* ctx, int64_t n, int64_t nnz, const void* indptr, int indptr_bits, const void* indices, int index_bits,
                   const void* data, int data_dtype, int csc, int device_input, uintptr_t producer_stream, const void* xy, int xy_dtype,
                   int64_t stride_row, int64_t stride_col, int xy_device, uintptr_t xy_stream, int max_neighs, int64_t* max_degree,
                   int32_t* sat, int32_t* sat_idx, int32_t* unsat, int32_t* unsat_idx, int64_t* n_sat, int64_t* n_unsat, int* nonfinite);

/* ---- spatial neighbour graphs (what runs right before every hot-path call) ------------------------------------------
 * Exact k nearest neighbours of every observation among the others (2-D float64 coordinates, interleaved x,y), the query
 * itself excluded: NearestNeighbors(n_neighbors=k).fit(xy).kneighbors() of KNNBuilder.build_graph / GridBuilder._base_adjacency
 * (src/squidpy/gr/neighbors.py:192-209, :395-419).  out_idx / out_dist: n x k, every row ordered by ASCENDING NEIGHBOUR INDEX
 * (CSR-ready: indptr = k * arange(n + 1)); distances = sqrt(dx*dx + dy*dy) in float64 like sklearn's kd_tree.  Ties at the k-th
 * distance go to the smaller index.  median_out (or NULL): np.median of the n*k distances (GridBuilder's cut = 1.3 x that).   */
int sqb_knn_2d(sqb_ctx* ctx, const double* xy, int64_t n, int k, int32_t* out_idx, double* out_dist, double* median_out);
/* All neighbours within `radius` (dx*dx + dy*dy <= radius*radius, self excluded): radius_neighbors() of RadiusBuilder.build_graph
 * (neighbors.py:253-270).  Two calls: with out_idx == NULL only out_indptr (n + 1) and *nnz_out are produced; with buffers of
 * `capacity` >= nnz entries the rows are filled in ascending column order.                                                 */
int sqb_radius_2d(sqb_ctx* ctx, const double* xy, int64_t n, double radius, int64_t* out_indptr, int32_t* out_idx,
                  double* out_dist, int64_t capacity, int64_t* nnz_out);

/* The Delaunay graph of n points (DelaunayBuilder.build_graph, neighbors.py:318-332): row i lists the Delaunay neighbours of
 * observation i in ascending order.  Exact predicates; exactly cocircular points are resolved by a symbolic perturbation of
 * x^2 + y^2 by index (one fixed triangulation); exact duplicates are collapsed to the lowest index of their group, the other
 * copies get empty rows.  Two calls as sqb_radius_2d (out_idx == NULL: out_indptr and *nnz_out only; nnz < 6n always, so one
 * call with capacity 6n suffices).  Fewer than three distinct points or all distinct points collinear: SQB_ERR_INVALID with a
 * message starting "QhullError".  out_pass_counts: NULL or int64[2], the points finished by pass 1 and by pass 2.          */
int sqb_delaunay_2d(sqb_ctx* ctx, const double* xy, int64_t n, int64_t* out_indptr, int32_t* out_idx, int64_t capacity,
                    int64_t* nnz_out, int64_t* out_pass_counts);

/* ---- spatial neighbour graphs from coordinates in GPU memory, kept there ---------------------------------------------
 * The whole builder on the device: search, cut, ring expansion, diagonals, interval / percentile pruning, eliminate_zeros,
 * transform and the library block diagonal of KNNBuilder / GridBuilder / RadiusBuilder.build and GraphBuilderCSR.combine
 * (src/squidpy/gr/neighbors.py:80-156, :192-209, :253-270, :365-419, :423-477).  The result equals the host builders' after
 * sort_indices(), bit for bit.
 *   xy: DEVICE pointer on the context's device to n x 2 coordinates, xy_dtype 0 float32 / 1 float64, element strides
 *   stride_row / stride_col (any); never read on the host.  producer_stream: as in sqb_autocorr_load_csr_device.
 *   kind 0 kNN (n_neighbors in [1, 64]), 1 grid (n_neighbors, n_rings >= 1, 1.3 x median cut), 2 radius (radius; interval != 0
 *   prunes to [radius_min, radius_max] like a tuple radius), 3 Delaunay (as sqb_delaunay_2d; interval as for radius; the
 *   distances are computed in the coordinates' dtype, so float32 coordinates give float32 distances, and the interval bounds
 *   and the percentile follow numpy's float32 arithmetic).  set_diag as the builders'.  percentile: NaN for none (kNN /
 *   radius).  transform 0 none, 1 spectral, 2 cosine.
 *   lib_ptr / lib_rows (HOST, or NULL with n_libs = 0): library b is the ascending rows lib_rows[lib_ptr[b] .. lib_ptr[b+1]) of
 *   the coordinates; each is built as its own block, the blocks are combined in the order of the rows.
 * Returns a handle with *n_out rows (n, or the rows the libraries list), the entry counts of the connectivities (float32
 * values) and the distances (float64 values if *dst_f64, else float32).  Errors (non-finite coordinates, k >= n, ...) carry
 * the host path's messages and leave the context usable.                                                              */
typedef struct sqb_graph sqb_graph;
int sqb_graph_build_device(sqb_ctx* ctx, const void* xy, int xy_dtype, int64_t n, int64_t stride_row, int64_t stride_col,
                           uintptr_t producer_stream, int kind, int n_neighbors, int n_rings, double radius, int interval,
                           double radius_min, double radius_max, int set_diag, double percentile, int transform,
                           const int64_t* lib_ptr, const int32_t* lib_rows, int n_libs, sqb_graph** out, int64_t* n_out,
                           int64_t* adj_nnz, int64_t* dst_nnz, int* dst_f64);
/* Writes both CSR matrices into caller-allocated DEVICE buffers: indptr n_out + 1 int32, indices nnz int32, data nnz values.
 * consumer_stream (CUDA Array Interface convention) is the stream that allocated the buffers; it is waited on before the
 * copies.  The buffers are complete when the call returns.                                                             */
int sqb_graph_export(sqb_graph* g, int32_t* adj_indptr, int32_t* adj_indices, float* adj_data, int32_t* dst_indptr,
                     int32_t* dst_indices, void* dst_data, uintptr_t consumer_stream);
int sqb_graph_free(sqb_graph* g);

/* ---- post-processing a caller's spatial graph in GPU memory, kept there --------------------------------------------------
 * One post-processor of src/squidpy/gr/neighbors.py per call on a graph the caller built (a custom GraphBuilderCSR), with the
 * steps sqb_graph_build_device uses.  The result equals the reference post-processor applied to host copies of the same
 * matrices, after sort_indices(): the same stored entries, explicit zeros included, the same value dtypes and the same values
 * bit for bit (spectral on a weighted adjacency: column sums in float64, rounded to float32).
 *   The graph: n x n CSRs in DEVICE memory on the context's device, read in place after producer_stream (as in
 *   sqb_autocorr_load_csr_device); indptr_bits / index_bits 32 or 64; nnz < 2^31; columns strictly increasing in every row
 *   and inside [0, n) (else SQB_ERR_INVALID).  Connectivities float32; distances float64 if dst_f64, else float32.
 *   op 0, DistanceIntervalPostprocessor((a, b)) (:441-447): adj.data[t] and dst.data[t] become 0 where dst.data[t] < a or
 *     > b (by position: adj_nnz must equal dst_nnz), then every diagonal entry of adj is stored with its value from before,
 *     0 where none was stored.  Float32 distances are compared with the bounds rounded to float32, as numpy does.
 *   op 1, PercentilePostprocessor(a) (:450-458): threshold = np.percentile(dst.data, a) (method 'linear', in float32 for float32
 *     distances); every adj position where dst stores a value > threshold becomes 0, stored explicitly where adj had no
 *     entry; those distances become 0.  a in [0, 100]; an empty dst is SQB_ERR_INVALID and a threshold below 0 (scipy's
 *     `dst > threshold` then marks every implicit entry) SQB_ERR_UNSUPPORTED.
 *   op 2, TransformPostprocessor(transform) (:461-476): eliminate_zeros on both, then transform 0 none, 1 spectral, 2 cosine of
 *     the connectivities (float32 results).
 * Returns a sqb_graph handle (sqb_graph_export / sqb_graph_free) of n rows with the entry counts and the distances' dtype.
 * Errors leave the context usable.                                                                                        */
int sqb_graph_postprocess(sqb_ctx* ctx, int64_t n, int64_t adj_nnz, const void* adj_indptr, int adj_indptr_bits,
                          const void* adj_indices, int adj_index_bits, const float* adj_data, int64_t dst_nnz,
                          const void* dst_indptr, int dst_indptr_bits, const void* dst_indices, int dst_index_bits,
                          const void* dst_data, int dst_f64, uintptr_t producer_stream, int op, double a, double b, int transform,
                          sqb_graph** out, int64_t* adj_nnz_out, int64_t* dst_nnz_out, int* dst_f64_out);
/* GraphBuilderCSR.combine (neighbors.py:137-154) of per-library device graphs: the block diagonal, its rows and columns put in
 * the order of the observations.  Block b (block_n[b] >= 1 rows) is described by adj_blocks[6b .. 6b+6) and dst_blocks[6b ..
 * 6b+6) (HOST int64): nnz, indptr pointer, indptr_bits, indices pointer, index_bits, data pointer, each a CSR as for
 * sqb_graph_postprocess (float32 connectivities; distances float64 if dst_f64, else float32).  out_row (HOST int32, one per
 * block row in block order) is the output row of every block row, a permutation of [0, total rows): the rank of its
 * observation.  Explicit zeros are kept; columns come out ascending.  Returns a sqb_graph handle of *n_out rows.            */
int sqb_graph_combine(sqb_ctx* ctx, int n_blocks, const int64_t* block_n, const int64_t* adj_blocks, const int64_t* dst_blocks,
                      int dst_f64, uintptr_t producer_stream, const int32_t* out_row, sqb_graph** out, int64_t* n_out,
                      int64_t* adj_nnz_out, int64_t* dst_nnz_out, int* dst_f64_out);

/* ---- calculate_niche embeddings -----------------------------------------------------------------------------------
 * The graph (both entry points): an n x n CSR (csc = 0) or CSC (csc = 1) from the host (device_input = 0) or from device memory
 * (device_input = 1: DEVICE pointers on the context's device, read in place after producer_stream, as in
 * sqb_autocorr_load_csr_device).  indptr_bits / index_bits 32 or 64; data_dtype 0 f32, 1 f64, 3 i32, 4 i64 (boolean graphs are
 * refused: scipy combines them with logical and / or); nnz < 2^31; data may be NULL when nnz = 0.  Integer values are taken as
 * their float64 values, exact while the reference's integer sums do not overflow the graph's dtype.  Duplicates are summed
 * (in float32 for a float32 graph) where the reference's scipy calls sum them.  Both return once the device has stopped
 * reading the caller's buffers.
 *
 * sqb_niche_profile: the neighbourhood-profile embedding (src/squidpy/gr/_niche.py:1117-1214).  codes[v] in [-1, n_cls): the
 * category of observation v (-1: NaN, a row that counts towards no column).  P_1 = A Y (Y the one-hot codes), P_k = A P_{k-1},
 * summed in float64 over ascending columns.  Per hop p_k = P_k (abs_nhood) or P_k / (row total), NaN (a zero total) -> 0.
 * out (HOST, n x n_cls float64 row-major) = p_1 when distance = 1, else w_0 p_1 + w_1 p_2 + ... (weights: distance entries,
 * already extended), divided by weight_sum (the sum of every weight given) unless abs_nhood.
 * Exactness: bit for bit with the reference for integer-valued graphs whose path sums stay below 2^24; for other weights within
 * float32 rounding of it, and bit for bit with this float64 statement.
 *
 * sqb_niche_aggregate: X is n x m, dense row-major contiguous (x_format 0) or CSR (x_format 1: x = values, x_indptr / x_indices
 * of x_indptr_bits / x_index_bits), float32 (x_f32 = 1) or float64 values, on the host (x_device = 0) or the device (x_device = 1,
 * after x_stream).  Duplicate X entries add up.  out (HOST, row-major) is float32 (out_f32) or float64: the dtype numpy's upcast gives.
 *   mode 0, UTAG (:1259-1260): normalize(A, "l1", axis=1) in the graph's storage order (a CSC transposed as scipy's tocsr
 *     does it): row sum of |a| in float64, a / sum rounded once to the value type, a zero row unchanged; out (n x m) = N X
 *     accumulated over each row's entries in that order, in float32 when N and X are float32, else float64.  Bit for bit.
 *   modes 1 (mean) / 2 (variance), CellCharter (:1336-1355): from the canonical A, hop_1 = A without diagonal and zeros,
 *     visited = A with diagonal 1, hop_k = (hop_{k-1} A) > visited compared on path sums in the value type, visited += hop_k.
 *     out (n x (distance + 1) m) = [X, agg_1, ..., agg_distance] where agg_k = N_k X (mean) or N_k (X∘X) - (N_k X)² (variance),
 *     N_1 = diag(1 / deg) hop_1 in the value type (deg: numpy's pairwise row sum) taken in reverse column order as scipy's SpGEMM
 *     stores it, N_k (k >= 2) = 1 / |row| over the hop set in ascending columns, in float64.  out_hop_nnz[k - 1] = nnz of hop_k.
 *     hop_1's aggregate is bit for bit; hop sets are identical; hop >= 2 aggregates are bit for bit with this statement (the
 *     reference's own order, fixed by scipy's non-canonical sparse binops, differs within 1e-12 relative).                  */
int sqb_niche_profile(sqb_ctx* ctx, int64_t n, int64_t nnz, const void* indptr, int indptr_bits, const void* indices, int index_bits,
                      const void* data, int data_dtype, int csc, int device_input, uintptr_t producer_stream, const int32_t* codes,
                      int n_cls, int distance, const double* weights, double weight_sum, int abs_nhood, double* out);
int sqb_niche_aggregate(sqb_ctx* ctx, int64_t n, int64_t nnz, const void* indptr, int indptr_bits, const void* indices, int index_bits,
                        const void* data, int data_dtype, int csc, int device_input, uintptr_t producer_stream, const void* x,
                        const void* x_indptr, const void* x_indices, int64_t x_nnz, int x_format, int x_indptr_bits, int x_index_bits,
                        int x_f32, int64_t m, int x_device, uintptr_t x_stream, int mode, int distance, int out_f32, void* out,
                        int64_t* out_hop_nnz);

/* ---- mask_graph ------------------------------------------------------------------------------------------------------
 * Keeps or drops the stored entries of a spatial graph by a polygon (src/squidpy/gr/_build.py:853-966).  Entry (i, j) of the
 * connectivities is the segment xy[i] -> xy[j]; it is within the polygon P when no point of it lies in P's exterior and some point
 * of its open part in P's interior (shapely's LineString.within, DE-9IM T*F**F***); a zero-length segment is within iff its point
 * is in P's interior.  Decided by exact orientation signs (mask_pred.h).  negative = 0 drops the entries that are not within,
 * 1 those that are.  The distances lose the entries at the same (row, col) positions, and then both matrices every entry whose
 * value is zero (scipy's eliminate_zeros; NaN is kept).  Values, their dtype and the order within each row are unchanged.
 *   The graphs: n x n CSRs (indptr_bits / index_bits 32 or 64; data_dtype 0 f32, 1 f64, 3 i32, 4 i64, 5 bool), both on the host
 *   (graph_device = 0) or both in device memory on the context's device (graph_device = 1, read in place after graph_stream, as
 *   in sqb_autocorr_load_csr_device).  nnz < 2^31; an index outside [0, n) or a (row, col) stored twice is SQB_ERR_INVALID.
 *   xy: n x 2 coordinates: host float64 C-contiguous (xy_device = 0, xy_dtype 1, strides 2 and 1), or a DEVICE pointer on the
 *   context's device (xy_device = 1, read after xy_stream) of xy_dtype 0 f32 / 1 f64 with element strides stride_row /
 *   stride_col.  Non-finite coordinates, or coordinates / polygon vertices neither 0 nor of magnitude in [2^-120, 2^120], are
 *   SQB_ERR_INVALID.
 *   The polygon: n_rings rings, ring r = the vertices ring_ptr[r] .. ring_ptr[r+1] of ring_xy (HOST, interleaved x, y), a hole of
 *   the polygon before it when ring_hole[r] != 0, else the shell of a polygon; the polygons are the parts of a MultiPolygon.
 *   Closing and repeated consecutive vertices are allowed; the polygon must be valid (shapely's is_valid), which is not checked.
 * Returns a handle holding both masked CSRs and their entry counts.                                                         */
typedef struct sqb_masked sqb_masked;
int sqb_mask_graph(sqb_ctx* ctx, int64_t n, int64_t adj_nnz, const void* adj_indptr, int adj_indptr_bits, const void* adj_indices,
                   int adj_index_bits, const void* adj_data, int adj_dtype, int64_t dst_nnz, const void* dst_indptr, int dst_indptr_bits,
                   const void* dst_indices, int dst_index_bits, const void* dst_data, int dst_dtype, int graph_device, uintptr_t graph_stream,
                   const void* xy, int xy_dtype, int64_t stride_row, int64_t stride_col, int xy_device, uintptr_t xy_stream, const double* ring_xy,
                   const int64_t* ring_ptr, const uint8_t* ring_hole, int64_t n_rings, int negative, sqb_masked** out, int64_t* adj_nnz_out,
                   int64_t* dst_nnz_out);
/* Writes both masked CSRs (indptr n + 1 int32, indices int32, values in the input's dtype) into caller buffers in host or device
 * memory.  consumer_stream: as in sqb_graph_export (0 for host buffers).  The buffers are complete when the call returns.     */
int sqb_mask_export(sqb_masked* m, int32_t* adj_indptr, int32_t* adj_indices, void* adj_data, int32_t* dst_indptr, int32_t* dst_indices,
                    void* dst_data, uintptr_t consumer_stream);
int sqb_mask_free(sqb_masked* m);

#ifdef __cplusplus
}
#endif
#endif /* SQUIDPY_B200_H */
