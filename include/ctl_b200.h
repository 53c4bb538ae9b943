/* libctl_b200.so -- C ABI of the H100-native centroid-triplet re-ID hot path.
 *
 * The reference (mikwieczorek/centroids-reid @ a1825b7) is pure Python: the path it exposes
 * is a Python module/class API called by PyTorch-Lightning hooks, there is no FFI of its
 * own.  This header is the boundary a maintainer binds instead of the torch/numpy calls at
 * the cited reference lines (see INTEGRATION.md for the ctypes stub); the Python package
 * `centroids-reid_b200` is that binding plus drop-in classes with the reference's names.
 *
 * Conventions
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless marked host;
 *     buffers are caller-owned (the Python shim allocates them with torch's caching
 *     allocator) and must be contiguous and 16-byte aligned;
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, nothing
 *     synchronises unless stated;
 *   - return value: 0 = ok, negative = CTL_ERR_* (argument / capacity error),
 *     positive = cudaError_t; ctl_last_error() returns a thread-local description;
 *   - there is NO CPU fallback: without an sm_90 device every compute entry point fails.
 */
#ifndef CTL_H100_H_
#define CTL_H100_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CTL_ABI_VERSION 5

#define CTL_OK 0
#define CTL_ERR_INVALID_ARGUMENT (-1)
#define CTL_ERR_WORKSPACE (-2)   /* workspace too small; ctl_last_error() names the size */
#define CTL_ERR_UNSUPPORTED (-3)
#define CTL_ERR_CAPACITY (-4)    /* a device-side list overflowed (see the entry point) */
#define CTL_ERR_NO_DEVICE (-5)

typedef void* ctl_stream_t; /* cudaStream_t */

const char* ctl_last_error(void);
int ctl_abi_version(void);
/* 0 when the current device is sm_90 (H100); CTL_ERR_NO_DEVICE otherwise. */
int ctl_device_check(void);

/* ------------------------------------------------------------------------------------------
 * Query x gallery distances, top-k and streamed CMC / mAP ranks
 * replaces: utils/reid_metric.py:25-33 (get_euclidean), :51-59 (get_cosine), :112-136
 * (R1_mAP.compute: normalize, distmat, np.argsort), utils/eval_reid.py:25-92 (eval_func),
 * inference/get_similar.py:104-128 (dist + argsort + [:, :topk]).
 * ---------------------------------------------------------------------------------------- */
#define CTL_DIST_EUCLIDEAN 0 /* squared L2, unclamped: |q|^2 + |g|^2 - 2 q.g */
#define CTL_DIST_COSINE 1    /* clamp(|1 - cos|, 1e-12) */
#define CTL_FLAG_NORMALIZE 2 /* torch.nn.functional.normalize(x, dim=1, p=2) first */
#define CTL_DIST_SQRT 4      /* euclidean only: sqrt(clamp(d, 1e-12)) -- losses/triplet_loss.py:27-41 */

/* Row planes: the fp32 rows split into two fp16 planes (hi + 2^-11 lo, per-row power-of-two
 * scale) plus fp32 squared norms, the operand format of the tensor-core distance kernel.
 * Opaque to the caller; ctl_planes_bytes() gives the buffer size. */
size_t ctl_planes_bytes(int64_t n, int32_t d);
int ctl_planes_build(const float* x, int64_t n, int32_t d, int32_t flags, void* planes, ctl_stream_t stream);

/* out[nq, ld_out] = dist(q, g): the full matrix (get_euclidean / get_cosine drop-in). */
int ctl_dist_matrix(const void* q_planes, int64_t nq, const void* g_planes, int64_t ng, int32_t d, int32_t flags,
                    float* out, int64_t ld_out, ctl_stream_t stream);

/* Streamed top-k and evaluation: passes of the distance GEMM (ctl_dist_pass) whose epilogues reduce each tile instead
 * of storing it, so the [nq, ng] matrix is never materialised.  Keys are uint64 (distance, gallery index) pairs whose
 * integer order is the ascending (distance, index) order (ctl_key_encode); the index is gallery row + g_index_offset,
 * or g_index_map[row].
 *
 * Top-k: the k <= ng smallest distances per query, in that order, for the plan of ctl_topk_plan:
 *   pass 1: gmin -> ctl_select_tau: tau = the k-th smallest group minimum, an upper bound of the k-th distance.  Any
 *           subset of the groups gives such a bound, so pass 1 may run a tile list of every ctl_dist_subset_stride-th
 *           gallery tile (gmin pre-filled with +inf): a looser tau, longer candidate lists, the same results.  With
 *           emit_all there is no pass 1 and tau = +inf (ctl_fill_f32);
 *   pass 2: tau + cand_keys -> ctl_sort_key_rows of the candidates -> ctl_topk_emit.
 *   The caller zeroes cand_count and *overflow.  *overflow becomes non-zero if more rows than the candidate capacity
 *   tie exactly at tau; the results are then invalid.
 *
 * Evaluation (eval_func semantics).  Identity / camera arrays: q_pid, g_pid int32;
 * q_cam = dense camera index in [0,64); g_cammask = bit set of the cameras a gallery row
 * (or centroid, utils/eval_reid.py:52-56 respect_camids) was built from.  A gallery row is
 * junk for a query iff same pid and bit q_cam of its mask is set; it is a positive iff
 * same pid and not junk.
 *   collect : pos_keys[nq, max_pos] <- keys of each query's positives (unordered), pos_count[nq] (zeroed by the
 *             caller); *overflow is set when a query has more than max_pos;
 *   sort    : ctl_sort_key_rows of the positives -> the threshold list thr_keys / thr_count;
 *   count   : buckets[nq, max_pos + 1] (zeroed by the caller) += for every kept gallery row,
 *             the index of the first positive that sorts after it;
 *   finalize: ctl_eval_finalize_packed.
 * Collect shares pass 1 with the top-k, count shares pass 2.
 * With a gallery sharded over ranks, each rank's keys carrying global gallery indices: collect per shard, all-gather +
 * sort the keys, count per shard, all-reduce(sum) the buckets, finalize; for the top-k, all-gather every rank's first k
 * sorted candidates and sort + emit those rows again. */
/* One pass of the distance GEMM with any combination of the streamed epilogues.  NULL pointers disable a feature.
 * With both top-k and evaluation wanted, TWO passes serve both:
 *   pass 1: gmin (+ pos_keys/pos_count)            -> ctl_select_tau, ctl_sort_key_rows
 *   pass 2: tau + cand_keys (+ thr_keys + buckets) -> ctl_sort_key_rows, ctl_topk_emit,
 *                                                     ctl_eval_finalize_packed */
typedef struct ctl_pass_desc {
  float* dist_out;            /* [nq, ld_out] full matrix */
  int64_t ld_out;
  float* gmin;                /* [nq, n_groups] minima of 16-column groups, n_groups = ceil(ng/16) */
  const float* tau;           /* [nq] candidate threshold */
  uint64_t* cand_keys;        /* [nq, cand_cap] rows with dist <= tau */
  int32_t* cand_count;        /* [nq], zeroed by the caller */
  int32_t cand_cap;
  const int32_t* q_pid;       /* identities: see the evaluation above */
  const int32_t* q_cam;
  const int32_t* g_pid;
  const uint64_t* g_cammask;
  uint64_t* pos_keys;         /* [nq, max_pos] (collect) */
  int32_t* pos_count;         /* [nq], zeroed by the caller */
  int32_t max_pos;
  const uint64_t* thr_keys;   /* [nq, max_pos] sorted positives (count) */
  const int32_t* thr_count;
  int32_t* buckets;           /* [nq, max_pos + 1], zeroed by the caller */
  int32_t* overflow;          /* device int, set non-zero when a list overflows */
  int64_t g_index_offset;
  /* Optional (NULL = off). */
  const int32_t* tile_list;    /* ctl_dist_worklist: run only these 128 x 128 tiles.  For passes whose outputs do not need
                                  every tile: pos_keys / pos_count (tiles that can hold a positive) and gmin (any subset of
                                  the groups still bounds the k-th distance from above; the caller pre-fills gmin with
                                  +inf).  Rejected with dist_out, cand_keys or buckets. */
  const int32_t* g_index_map;  /* [ng] index written into the keys for gallery row i (instead of i + g_index_offset):
                                  lets the rows be stored in another order (e.g. sorted by pid) with unchanged results */
} ctl_pass_desc;
int ctl_dist_pass(const void* q_planes, int64_t nq, const void* g_planes, int64_t ng, int32_t d, int32_t flags,
                  const ctl_pass_desc* desc, ctl_stream_t stream);
/* ascending sort of every row of a key matrix (counts[i] valid entries; row_stride <= 16384) */
int ctl_sort_key_rows(uint64_t* keys, const int32_t* counts, int64_t rows, int32_t row_stride, ctl_stream_t stream);
/* top-k plan for (ng, k): emit_all != 0 means "skip pass 1, tau = +inf". */
int ctl_topk_plan(int64_t ng, int32_t k, int32_t* emit_all, int32_t* n_groups, int32_t* merge, int32_t* cand_cap);
int ctl_select_tau(const float* gmin, int64_t nq, int32_t n_groups, int32_t merge, int32_t k, float* tau,
                   ctl_stream_t stream);
/* Tile list for ctl_pass_desc.tile_list: tile_list[0] = count, then the kept tile ids (ascending; id = gallery tile *
 * ceil(nq/128) + query tile).  A tile is kept if
 * the identity ranges of its 128 query rows and its 128 gallery rows intersect (q_pid / g_pid in the planes' row order;
 * both NULL = no identities) or if its gallery-tile index is a multiple of keep_stride (0 = none).  With both operands
 * stored in identity order the first set is a few per cent of the matrix.  ctl_dist_subset_stride(ng, k): the stride that
 * leaves ~2.5 k column groups for ctl_select_tau (1 = use every tile).  Limits: <= 2^20 tiles, <= 5632 row tiles
 * (CTL_ERR_UNSUPPORTED beyond: run the pass without a list). */
size_t ctl_dist_worklist_bytes(int64_t nq, int64_t ng);
int ctl_dist_subset_stride(int64_t ng, int32_t k);
int ctl_dist_worklist(const int32_t* q_pid, int64_t nq, const int32_t* g_pid, int64_t ng, int32_t keep_stride,
                      int32_t* tile_list, ctl_stream_t stream);
int ctl_fill_f32(float* p, int64_t n, float value, ctl_stream_t stream);
int ctl_topk_emit(const uint64_t* cand_keys_sorted, const int32_t* cand_count, int64_t nq, int32_t cand_cap, int32_t k,
                  int64_t* out_idx, float* out_dist, int32_t* overflow, ctl_stream_t stream);
/* finalize: ranks[nq, max_pos] (1-based rank of each positive among kept rows), ap[nq] (float64, eval_reid.py:75-79),
 * -1 / NaN for queries without positives; and, unless `packed` is NULL, packed[nq + 1][3] doubles: per query AP,
 * first-hit rank (-1: none), number of positives; last row: {*overflow (0 for a NULL overflow), 0, 0} -- everything
 * eval_func's final reductions (utils/eval_reid.py:86-92) need, so the host does ONE device->host copy per evaluation. */
int ctl_eval_finalize_packed(const int32_t* buckets, const int32_t* pos_count, int64_t nq, int32_t max_pos, int32_t* ranks,
                             double* ap, double* packed, const int32_t* overflow, ctl_stream_t stream);
/* key <-> (distance, index) helpers for host-side merges of per-shard results */
uint64_t ctl_key_encode(float dist, uint32_t index);
void ctl_key_decode(uint64_t key, float* dist, uint32_t* index);

/* ------------------------------------------------------------------------------------------
 * CMC / mAP over a materialised distance matrix
 * replaces: utils/eval_reid.py:25-92 (eval_func) for a [nq, ld] fp32 matrix the caller computed (re-ranked distances,
 * or any other): np.argsort + the per-query loop.  The collect and count passes of ctl_dist_pass reading the matrix
 * instead of forming it: same identity arrays and junk rule (see ctl_dist_pass), same (distance, column) keys, so
 * ctl_sort_key_rows and ctl_eval_finalize_packed complete them unchanged.  pos_count and buckets are zeroed by the caller.
 * ---------------------------------------------------------------------------------------- */
int ctl_eval_matrix_collect(const float* dist, int64_t nq, int64_t ng, int64_t ld, const int32_t* q_pid,
                            const int32_t* q_cam, const int32_t* g_pid, const uint64_t* g_cammask, int32_t max_pos,
                            uint64_t* pos_keys, int32_t* pos_count, int32_t* overflow, ctl_stream_t stream);
int ctl_eval_matrix_count(const float* dist, int64_t nq, int64_t ng, int64_t ld, const int32_t* q_pid,
                          const int32_t* q_cam, const int32_t* g_pid, const uint64_t* g_cammask, int32_t max_pos,
                          const uint64_t* pos_keys_sorted, const int32_t* pos_count, int32_t* buckets,
                          ctl_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * k-reciprocal re-ranking (Zhong, Zheng, Cao, Li, CVPR 2017)
 * replaces: re_ranking(probFea, galFea, k1, k2, lambda_value) of the reid-strong-baseline lineage credited in
 * utils/reid_metric.py (the CTL reference dropped it): dense N x N float16 V, Python loops over the N rows, Jaccard
 * through an inverted index.
 * F = [q; g] (planes of nq + ng rows built with CTL_DIST_EUCLIDEAN [| CTL_FLAG_NORMALIZE]), N = nq + ng:
 *   1. D = ctl_dist_matrix(F, F), squared euclidean, unclamped, materialised (N^2 * 4 bytes of the workspace);
 *   2. nd[i, :] = D[i, :] / max_j D[i, j] (fp32 division); a row maximum <= 0 sets bit 0 of *status;
 *   3. rank[i, :kr] = the first kr = max(k1 + 1, k2) columns of row i sorted by (nd, column index);
 *   4. R(i) = {j in rank[i, :k1+1] : i in rank[j, :k1+1]}; h = round-half-even(k1 / 2); R_h(c) likewise with h + 1
 *      neighbours; E(i) = R(i) united with every R_h(c), c in R(i), for which 3 |R_h(c) & R(i)| > 2 |R_h(c)|;
 *      V[i, j] = exp(-nd[i, j]) / sum_{j' in E(i)} exp(-nd[i, j']) on E(i), 0 elsewhere;
 *   5. k2 > 1: V[i] <- mean over t < k2 of V[rank[i, t]];
 *   6. out[i, j] = (1 - lambda) (1 - s / (2 - s)) + lambda nd[i, nq + j], s = sum_c min(V[i, c], V[nq + j, c]).
 * V and its sums are fp32; rows are padded (index, value) lists in ascending column order, capacities from
 * ctl_rerank_plan.  No host synchronisation, no data-dependent allocation, fixed accumulation order (bit-identical
 * repeats and graph replays).  ctl_rerank zeroes *status; the caller reads it back and rejects the result if non-zero.
 * ctl_rerank_plan / ctl_rerank_workspace_bytes are host-only; unsupported arguments (k1 < 1, k2 < 1, N < 2, or beyond
 * kr <= 128, (k1 + 1)(h + 2) <= 8192, k2 (k1 + 1)(h + 2) <= 16384) give CTL_ERR_* / 0 bytes. */
int ctl_rerank_plan(int64_t nq, int64_t ng, int32_t k1, int32_t k2, int32_t* kr, int32_t* h, int32_t* v_cap,
                    int32_t* q_cap);
size_t ctl_rerank_workspace_bytes(int64_t nq, int64_t ng, int32_t k1, int32_t k2);
int ctl_rerank(const void* planes, int64_t nq, int64_t ng, int32_t d, int32_t flags, int32_t k1, int32_t k2,
               float lambda_value, float* out, int64_t ld_out, int32_t* status, void* workspace, size_t workspace_bytes,
               ctl_stream_t stream);
/* The stages of ctl_rerank, each on the previous stage's device output (buffers as laid out by ctl_rerank_plan):
 *   rank   : steps 2 + 3, dist [n, ld] -> nd in place, rank [n, kr] (-1 beyond n columns); *status is OR-ed;
 *   expand : step 4, V rows v_idx / v_val [n, v_cap], v_cnt [n];
 *   qe     : step 5 (k2 > 1), rows [n, q_cap];
 *   invert : CSC of the gallery rows (nq <= r < nq + ng) of a row-padded V of capacity cap: col_ptr [nq + ng + 1],
 *            inv_row (gallery-local row) / inv_val [ng * cap]; cursor [nq + ng] is scratch.  The set of each column is
 *            fixed, the order inside a column is not (it does not enter the Jaccard sums);
 *   jaccard: step 6, out [nq, ld_out]. */
int ctl_rerank_rank(float* dist, int64_t n, int64_t ld, int32_t kr, int32_t* rank, int32_t* status, ctl_stream_t stream);
int ctl_rerank_expand(const float* nd, int64_t n, int64_t ld, const int32_t* rank, int32_t k1, int32_t k2,
                      int32_t* v_idx, float* v_val, int32_t* v_cnt, ctl_stream_t stream);
int ctl_rerank_qe(const int32_t* rank, int64_t n, int32_t k1, int32_t k2, const int32_t* v_idx, const float* v_val,
                  const int32_t* v_cnt, int32_t* q_idx, float* q_val, int32_t* q_cnt, ctl_stream_t stream);
int ctl_rerank_invert(int64_t nq, int64_t ng, const int32_t* idx, const float* val, const int32_t* cnt, int32_t cap,
                      int32_t* col_ptr, int32_t* cursor, int32_t* inv_row, float* inv_val, ctl_stream_t stream);
int ctl_rerank_jaccard(int64_t nq, int64_t ng, const int32_t* idx, const float* val, const int32_t* cnt, int32_t cap,
                       const int32_t* col_ptr, const int32_t* inv_row, const float* inv_val, const float* nd,
                       int64_t ld_nd, float lambda_value, float* out, int64_t ld_out, ctl_stream_t stream);

/* Row-blocked re-ranking: the steps above with at most a [block_rows, N] slice of the distance matrix alive, so the
 * workspace grows linearly in N (ctl_rerank's grows as N^2), and only each query's top-k of the re-ranked [Q, G] matrix
 * (and, optionally, the evaluation passes over it) is kept.  Bit-identical to ctl_rerank for every block_rows:
 *   sweep A, each row block: D rows (ctl_dist_matrix rows of [q; g] against all N) -> row maxima, nd, rank;
 *   sweep B, each row block: the same D rows again, normalised by the stored maxima -> expansion (V) of those rows
 *            (it reads nd at 2-hop candidates, which are not in the row's own rank list, hence a second sweep);
 *   qe and invert once, as in ctl_rerank;
 *   sweep C, each block of query rows: D against the gallery rows, normalised -> Jaccard + blend -> the k smallest
 *            (distance, gallery column) -> out_idx / out_dist [nq, k], ascending; with identities (q_pid != NULL) also
 *            the collect / sort / count passes of ctl_eval_matrix_* on those rows (the caller completes them with
 *            ctl_eval_finalize_packed).
 * The GEMM runs one plan and k-order for every shape, so a distance depends only on its two rows; the row maximum is
 * exact; the normalisation is the same IEEE division; the later kernels are ctl_rerank's.
 * ctl_rerank_topk zeroes *status, pos_count, buckets and *overflow; no host synchronisation, no allocation (capturable
 * in a CUDA graph).  ctl_rerank_topk_workspace_bytes is host-only: 0 for what ctl_rerank_plan rejects, and for d not a
 * positive multiple of 8, k < 1, k > min(128, ng) or block_rows < 1. */
size_t ctl_rerank_topk_workspace_bytes(int64_t nq, int64_t ng, int32_t d, int32_t k1, int32_t k2, int32_t k,
                                       int64_t block_rows);
int ctl_rerank_topk(const void* planes, int64_t nq, int64_t ng, int32_t d, int32_t flags, int32_t k1, int32_t k2,
                    float lambda_value, int32_t k, int64_t block_rows, int64_t* out_idx, float* out_dist,
                    const int32_t* q_pid, const int32_t* q_cam, const int32_t* g_pid, const uint64_t* g_cammask,
                    int32_t max_pos, uint64_t* pos_keys, int32_t* pos_count, int32_t* buckets, int32_t* overflow,
                    int32_t* status, void* workspace, size_t workspace_bytes, ctl_stream_t stream);
/* The row-block stages ctl_rerank_topk composes.  Every table (rank [n, kr], rowmax [n], V, out_idx / out_dist
 * [nq, k]) is the global one; a block covers rows [r0, r0 + rows) (queries [q0, q0 + rows) for jaccard) and its
 * matrix argument holds just those rows:
 *   dist_rows   : rows [r0, r0 + rows) of the planes (n rows) against rows [c0, c0 + cols) -> out [rows, ld_out];
 *                 with rowmax != NULL divided by rowmax[r0 + i] as the rank stage does (nd);
 *   rank_rows   : steps 2 + 3 of a [rows, n] block: nd in place, rank and rowmax of its rows, *status OR-ed;
 *   expand_rows : step 4 of the block's rows (its nd [rows, n]), into the global V;
 *   jaccard_rows: step 6 of the queries, nd [rows, ld_nd] holding the gallery columns only, out [rows, ld_out];
 *   topk_rows   : the k <= min(128, n) smallest (value, column) of each row of a [rows, n] block, ascending.
 * With the rows sharded over ranks (each holding the planes of all N rows): sweep A on the rank's contiguous rows,
 * all-gather rank and rowmax, OR (MAX) the status words; sweep B on the same rows (expand_rows reads the rank lists of
 * other rows), all-gather V; qe and invert on every rank over the whole V; sweep C on the rank's contiguous queries
 * against all ng gallery rows, then the collect / sort / count passes and ctl_eval_finalize_packed on those queries
 * alone, and all-gather idx / dist, ranks and the packed rows.  Each stage writes only its own rows of the global
 * tables, so the gathered tables and results equal the one-rank run's bit for bit; the entry points above need no
 * offset beyond r0 / q0. */
int ctl_rerank_dist_rows(const void* planes, int64_t n, int32_t d, int32_t flags, int64_t r0, int64_t rows, int64_t c0,
                         int64_t cols, const float* rowmax, float* out, int64_t ld_out, ctl_stream_t stream);
int ctl_rerank_rank_rows(float* dist, int64_t r0, int64_t rows, int64_t n, int64_t ld, int32_t kr, int32_t* rank,
                         float* rowmax, int32_t* status, ctl_stream_t stream);
int ctl_rerank_expand_rows(const float* nd, int64_t r0, int64_t rows, int64_t n, int64_t ld, const int32_t* rank,
                           int32_t k1, int32_t k2, int32_t* v_idx, float* v_val, int32_t* v_cnt, ctl_stream_t stream);
int ctl_rerank_jaccard_rows(int64_t nq, int64_t ng, int64_t q0, int64_t rows, const int32_t* idx, const float* val,
                            const int32_t* cnt, int32_t cap, const int32_t* col_ptr, const int32_t* inv_row,
                            const float* inv_val, const float* nd, int64_t ld_nd, float lambda_value, float* out,
                            int64_t ld_out, ctl_stream_t stream);
int ctl_rerank_topk_rows(float* dist, int64_t r0, int64_t rows, int64_t n, int64_t ld, int32_t k, int64_t* out_idx,
                         float* out_dist, ctl_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Per-identity centroid mean (segmented reduction)
 * replaces: modelling/bases.py:92-95 (_calculate_centroids), the tensor part of
 * :179-262 (validation_create_centroids), inference/inference_utils.py:147-159.
 * out[s, :] = sum_{j in [indptr[s], indptr[s+1])} x[indices[j], :] / count  (CSR groups;
 * indices == NULL means contiguous rows j).
 * ---------------------------------------------------------------------------------------- */
int ctl_segment_mean(const float* x, int64_t n, int32_t d, const int64_t* indptr, const int64_t* indices,
                     int64_t n_seg, float* out, ctl_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * CTL training-step losses, forward + backward in one enqueue
 * replaces: train_ctl_model.py:54-152 (everything between the trunk and manual_backward) and
 * the gradients autograd derives from it; modelling/bases.py:359-384 (create_masks_train);
 * losses/triplet_loss.py:27-41,68-173,194-205; losses/center_loss.py:26-45.
 * Batch contract (datasets/bases.py:346-406): B = P*K rows, pid-major blocks of K, padded rows
 * (is_real = 0) at the end of a block, every pid keeps >= 2 real rows.  labels[B] = class
 * index in [0, C).  All matrices fp32 row-major.
 * out_losses[8] = total, xent, triplet, center, ctl, dist_ap, dist_an, l2_mean_centroid (each
 * already multiplied by its SOLVER weight, like the reference's logged values).
 * Gradients are those of `total`: d_feats[B,D], d_centers[C,D] (dense, NOT yet rescaled by
 * 1/center_weight -- train_ctl_model.py:157-158 does that in the step), d_bn_weight[D],
 * d_fc_weight[C,D].  bn_running_mean/var are updated in place (momentum, unbiased var).
 * ---------------------------------------------------------------------------------------- */
typedef struct ctl_loss_config {
  int32_t B, D, P, K, C;
  float margin;         /* SOLVER.MARGIN (MarginRankingLoss) */
  float center_weight;  /* SOLVER.CENTER_LOSS_WEIGHT */
  float xent_weight;    /* SOLVER.QUERY_XENT_WEIGHT */
  float triplet_weight; /* SOLVER.QUERY_CONTRASTIVE_WEIGHT */
  float ctl_weight;     /* SOLVER.CENTROID_CONTRASTIVE_WEIGHT */
  float bn_eps;         /* 1e-5 */
  float bn_momentum;    /* 0.1 */
  float label_smooth;   /* 0.1 */
} ctl_loss_config;

size_t ctl_loss_workspace_bytes(const ctl_loss_config* cfg);
int ctl_loss_step(const ctl_loss_config* cfg, const float* feats, const int32_t* labels, const uint8_t* is_real,
                  const float* centers, const float* bn_weight, const float* bn_bias, float* bn_running_mean,
                  float* bn_running_var, const float* fc_weight, float* out_losses, float* d_feats, float* d_centers,
                  float* d_bn_weight, float* d_fc_weight, void* workspace, size_t workspace_bytes,
                  ctl_stream_t stream);

/* Stand-alone drop-ins (forward value + gradient of that value in one call):
 *   TripletLoss.__call__ (losses/triplet_loss.py:139-173; euclidean, margin ranking, optional
 *   anchor mask; any label multiset), CenterLoss.forward (losses/center_loss.py:26-45),
 *   CrossEntropyLabelSmooth.forward (losses/triplet_loss.py:194-205). */
size_t ctl_triplet_workspace_bytes(int32_t n, int32_t d);
int ctl_triplet_step(const float* feats, int32_t n, int32_t d, const int32_t* labels, const uint8_t* anchor_mask,
                     float margin, float* out_loss, float* out_dist_ap, float* out_dist_an, float* d_feats,
                     void* workspace, size_t workspace_bytes, ctl_stream_t stream);
/* The two remaining variants of TripletLoss (losses/triplet_loss.py:127-137,157-158): soft_margin != 0 = SoftMarginLoss
 * on (dist_an - dist_ap) (TripletLoss(margin=None): log(1 + exp(d_ap - d_an)), `margin` ignored); cosine != 0 =
 * dist_func 'cosine' (clamp(|1 - cos(x_i, x_j)|, 1e-12) with rows divided by max(|x|, 1e-12), triplet_loss.py:44-65),
 * gradient through the normalisation included. */
int ctl_triplet_step_ex(const float* feats, int32_t n, int32_t d, const int32_t* labels, const uint8_t* anchor_mask,
                        float margin, int32_t soft_margin, int32_t cosine, float* out_loss, float* out_dist_ap,
                        float* out_dist_an, float* d_feats, void* workspace, size_t workspace_bytes, ctl_stream_t stream);
int ctl_center_loss_step(const float* x, int32_t b, int32_t d, const int32_t* labels, const float* centers, int32_t c,
                         float* out_loss, float* d_x, float* d_centers, void* workspace, size_t workspace_bytes,
                         ctl_stream_t stream);
int ctl_xent_smooth_step(const float* logits, int32_t b, int32_t c, const int32_t* targets, float epsilon,
                         float* out_loss, float* d_logits, void* workspace, size_t workspace_bytes,
                         ctl_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Base-model training-step losses (the paper's baseline: no centroid rounds), forward + backward in one enqueue
 * replaces: train_base_model.py:38-96 (everything between the trunk and manual_backward, and the gradients autograd
 * derives from it); losses/triplet_loss.py:27-65,68-173,194-205; losses/center_loss.py:26-45.
 * Rows: B feature rows, mock rows (is_real = 0) included; any label multiset, labels[B] in [0, C).
 *   query triplet : batch-hard mining over all B rows (train_base_model.py:60-65), anchors masked to is_real; every
 *                   TripletLoss variant: euclidean or cosine distance, MarginRankingLoss(margin) or SoftMarginLoss
 *                   (soft_margin != 0, `margin` ignored);
 *   center loss   : all B rows (:67-69), the clamp adds (C-1)*1e-12 per row;
 *   head          : BatchNorm1d with batch statistics over all B rows (running statistics updated in place with
 *                   n = B, unbiased var; both NULL = not tracked) -> bias-free fc -> label-smoothed CE over all B rows
 *                   (:70-73).
 * out_losses[6] = total (:75, center + xent + triplet), xent, triplet, center (each multiplied by its SOLVER weight),
 * dist_ap, dist_an (means over the real anchors, :91-94).  Gradients are those of `total`: d_feats[B,D],
 * d_centers[C,D] (dense, NOT yet rescaled by 1/center_weight -- train_base_model.py:80-81 does that in the step),
 * d_bn_weight[D], d_fc_weight[C,D].  No host synchronisation, graph-capturable, fixed-order reductions (two calls give
 * identical bits).  A label outside [0, C) writes a NaN with payload 1 to every out_losses entry; the centers and
 * logits are never indexed out of range.
 * ---------------------------------------------------------------------------------------- */
typedef struct ctl_base_loss_config {
  int32_t B, D, C;
  float margin;           /* SOLVER.MARGIN; ignored when soft_margin != 0 */
  int32_t soft_margin;    /* SOLVER.MARGIN is None -> SoftMarginLoss */
  int32_t cosine;         /* SOLVER.DISTANCE_FUNC == 'cosine' */
  float center_weight;    /* SOLVER.CENTER_LOSS_WEIGHT */
  float xent_weight;      /* SOLVER.QUERY_XENT_WEIGHT */
  float triplet_weight;   /* SOLVER.QUERY_CONTRASTIVE_WEIGHT */
  float bn_eps;           /* 1e-5 */
  float bn_momentum;      /* 0.1 */
  float label_smooth;     /* 0.1 */
} ctl_base_loss_config;

size_t ctl_base_loss_workspace_bytes(const ctl_base_loss_config* cfg);
int ctl_base_loss_step(const ctl_base_loss_config* cfg, const float* feats, const int32_t* labels,
                       const uint8_t* is_real, const float* centers, const float* bn_weight, const float* bn_bias,
                       float* bn_running_mean, float* bn_running_var, const float* fc_weight, float* out_losses,
                       float* d_feats, float* d_centers, float* d_bn_weight, float* d_fc_weight, void* workspace,
                       size_t workspace_bytes, ctl_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Trunk inference forward (ResNet50 / ResNet50-IBN-A), NHWC fp16 activations
 * replaces: modelling/backbones/resnet.py:51-133, resnet_ibn_a.py:18-141,
 * modelling/baseline.py:91-96, modelling/bases.py:169-177, inference/inference_utils.py:104-113.
 *   conv2d   : out = [relu]( conv(x, weight) + bias [+ residual] ), weight [Cout][k][k][Cin] fp16
 *              (eval BatchNorm folded in), 1x1 or 3x3 (pad k/2), stride 1 or 2, Cin/Cout % 64 == 0;
 *              ReLU (if relu != 0) is applied to output channels >= relu_from only (IBN: the
 *              InstanceNorm half of bn1 is left raw for ctl_instnorm_relu);
 *   stem     : conv 7x7/2 pad 3 (3 -> 64) + folded BN [+ ReLU] from NCHW fp32 to NHWC fp16;
 *   maxpool  : 3x3 / 2, pad 1;
 *   gap_bn   : feat = mean over H*W (fp32), emb = feat * bn_scale + bn_shift (eval BatchNorm1d);
 *   instnorm : per-(image, channel) InstanceNorm(affine) + ReLU in place on channels [0, half).
 * ---------------------------------------------------------------------------------------- */
int ctl_conv2d_nhwc_f16(const void* x, int32_t n, int32_t h, int32_t w, int32_t cin, const void* weight,
                        const float* bias, const void* residual, void* out, int32_t cout, int32_t ksize,
                        int32_t stride, int32_t relu, int32_t relu_from, ctl_stream_t stream);
/* Two 1x1 convolutions summed in ONE GEMM over the concatenated K dimension -- the last layer of a bottleneck's
 * first block, out = act(bn3(conv3(x1)) + bn_d(downsample(x2))) (resnet.py:75-85 with a downsample branch):
 *   out[n][i][j][:] = act( W[:, :cin1] x1[n][i][j][:] + W[:, cin1:] x2[n][i*stride2][j*stride2][:] + bias )
 * x1: NHWC fp16 [n][h2/stride2][w2/stride2][cin1]; x2: NHWC fp16 [n][h2][w2][cin2]; weight_cat: [cout][cin1 + cin2]
 * fp16 (both folded weight matrices side by side), bias = sum of the two folded biases.  The shortcut tensor is
 * never written to or re-read from HBM. */
int ctl_conv1x1_dual_nhwc_f16(const void* x1, int32_t cin1, const void* x2, int32_t h2, int32_t w2, int32_t cin2,
                              int32_t stride2, int32_t n, const void* weight_cat, const float* bias, void* out,
                              int32_t cout, int32_t relu, ctl_stream_t stream);
/* The 3x3 counterpart: a 3x3 / 1 convolution (pad 1) and a 1x1 convolution summed in ONE GEMM -- the last layer of a
 * BasicBlock's first block, out = act(bn2(conv2(x1)) + bn_d(downsample(x2))) (resnet.py:31-47 with a downsample branch):
 *   out[n][i][j][:] = act( sum_{r,s} W[:, (3r + s) cin1 ..][:cin1] x1[n][i + r - 1][j + s - 1][:]
 *                          + W[:, 9 cin1:] x2[n][i*stride2][j*stride2][:] + bias )
 * x1: NHWC fp16 [n][h2/stride2][w2/stride2][cin1] (zero outside); x2: NHWC fp16 [n][h2][w2][cin2]; weight_cat:
 * [cout][9 cin1 + cin2] fp16 (the folded [cout][3][3][cin1] weights, then the folded shortcut), bias = sum of the two
 * folded biases.  The shortcut tensor is never written to or re-read from HBM. */
int ctl_conv3x3_dual_nhwc_f16(const void* x1, int32_t cin1, const void* x2, int32_t h2, int32_t w2, int32_t cin2,
                              int32_t stride2, int32_t n, const void* weight_cat, const float* bias, void* out,
                              int32_t cout, int32_t relu, ctl_stream_t stream);
/* The last 1x1 of a bottleneck and the first 1x1 of the next one in ONE launch (the block output is not re-read):
 *   out [n][i][j][:] = relu( W[:, :cin1] x1[n][i][j][:] [+ W[:, cin1:] x2[n][i*stride2][j*stride2][:]] + bias
 *                            [+ residual[n][i][j][:]] )
 *   out2[n][i][j][c] = act_c( W2[c][:] out[n][i][j][:] + bias2[c] ),  act_c = ReLU for c >= relu_from2, identity below
 * x2 != NULL is the K-concatenated form of ctl_conv1x1_dual_nhwc_f16 (no residual); x2 == NULL: x1 alone (stride2 = 1,
 * cin2 ignored) with an optional residual [n][h2][w2][cout].  x1: [n][h2/stride2][w2/stride2][cin1]; weight
 * [cout][cin1 (+ cin2)], weight2 [cout2][cout] fp16; out2 NHWC [n][h2/stride2][w2/stride2][cout2].  Both outputs are
 * bit-identical to the two stand-alone launches.  Only shapes with ctl_conv1x1_chain_supported(cout, cout2) != 0 are
 * accepted. */
int32_t ctl_conv1x1_chain_supported(int32_t cout, int32_t cout2);
int ctl_conv1x1_chain_nhwc_f16(const void* x1, int32_t cin1, const void* x2, int32_t h2, int32_t w2, int32_t cin2,
                               int32_t stride2, int32_t n, const void* weight, const float* bias, const void* residual,
                               void* out, int32_t cout, const void* weight2, const float* bias2, int32_t cout2,
                               int32_t relu_from2, void* out2, ctl_stream_t stream);
/* tensor-core stem: weight_k192_f16 = [64][192] fp16, k = (c*7 + r)*8 + s (s = 7 and k >= 168 zero) */
int ctl_stem_conv7x7_tc(const float* x_nchw, int32_t n, int32_t h, int32_t w, const void* weight_k192_f16,
                        const float* bias, int32_t relu, void* out_nhwc_f16, ctl_stream_t stream);
/* Fused stem for inputs up to 128 pixels wide (h % 4 == 0, w even): conv1 7x7/2 + folded bn1 (+ReLU for IBN-a) +
 * maxpool 3x3/2 in one pass; replaces resnet.py:123-126 / resnet_ibn_a.py:127-130.  `xpad` is a caller-owned
 * workspace of ctl_stem_pad_bytes(n, h, w) bytes that must have been zero-filled ONCE before its first use with a
 * given (n, h, w) (the call rewrites only the interior: zero-bordered NHWC4 fp16 copy of x).  `weight_packed_f16`
 * is [28][64][8] fp16: element (c, o, e) = folded weight w[o][ch = e % 4][r = c / 4][s = 2 * (c % 4) + e / 4],
 * zero for ch == 3 or s == 7.  Output: pooled NHWC fp16 [n][h/4][(w/2 - 1)/2 + 1][64]. */
size_t ctl_stem_pad_bytes(int32_t n, int32_t h, int32_t w);
int ctl_stem_pool_fused(const float* x_nchw, int32_t n, int32_t h, int32_t w, void* xpad, const void* weight_packed_f16,
                        const float* bias, int32_t relu, void* out_pooled_nhwc_f16, ctl_stream_t stream);
/* ctl_stem_pool_fused from uint8 HWC crops [n][h][w][3]: ToTensor + Normalize ((u / 255 - mean) / std, IEEE fp32 -- the
 * arithmetic of ctl_augment_batch_u8 without flip / crop / erasing; datasets/transforms/build.py:29-33) folded into the
 * stem's input packing, so a validation loader that ships uint8 crops never materialises the fp32 NCHW tensor.
 * Bit-identical to ctl_augment_batch_u8 (neutral parameters) followed by ctl_stem_pool_fused. */
int ctl_stem_pool_fused_u8(const void* x_u8_nhwc, int32_t n, int32_t h, int32_t w, const float* mean3_host,
                           const float* std3_host, void* xpad, const void* weight_packed_f16, const float* bias, int32_t relu,
                           void* out_pooled_nhwc_f16, ctl_stream_t stream);
int ctl_maxpool3x3s2_nhwc_f16(const void* x, int32_t n, int32_t h, int32_t w, int32_t c, void* out,
                              ctl_stream_t stream);
int ctl_gap_bn_nhwc_f16(const void* x, int32_t n, int32_t hw, int32_t c, const float* bn_scale, const float* bn_shift,
                        float* feat, float* emb, ctl_stream_t stream);
int ctl_instnorm_relu_nhwc_f16(void* x, int32_t n, int32_t hw, int32_t c, int32_t half, const float* gamma,
                               const float* beta, float eps, ctl_stream_t stream);

/* ---- whole-trunk entry points (SURVEY 8b): the eval embedding path bn(backbone(x)) behind an opaque handle ----
 * replaces: ResNet.forward / ResNet_IBN.forward (modelling/backbones/resnet.py:122-133, resnet_ibn_a.py:126-141),
 * Baseline.forward's pooling (modelling/baseline.py:91-96), ModelBase.validation_step / inference_utils._inference
 * (modelling/bases.py:169-177, inference/inference_utils.py:104-113).  This is the eval trunk's only driver;
 * modelling/backbones/engine.py::TrunkEngine is its ctypes form.
 *   ctl_trunk_create   : ResNet of `block` = CTL_BLOCK_BOTTLENECK (resnet.py:51-87) or CTL_BLOCK_BASIC (resnet.py:19-48)
 *                        blocks with `stage_blocks` blocks per stage (bottleneck: {3, 4, 6, 3} = ResNet50, {3, 4, 23, 3} =
 *                        ResNet101, {3, 8, 36, 3} = ResNet152; basic: {2, 2, 2, 2} = ResNet18, {3, 4, 6, 3} = ResNet34;
 *                        each >= 1), IBN-a when `ibn` != 0 (bottleneck only), MODEL.LAST_STRIDE 1 or 2.  An unknown
 *                        `block`, or a basic block with `ibn` != 0, is CTL_ERR_INVALID_ARGUMENT before any device work.
 *   ctl_trunk_feature_dim: width of the trunk output and of the features below: 2048 (bottleneck) or 512 (basic).
 *                        Host only.
 *   ctl_weights_pack   : `tensors` = the reference's `base.*`-stripped state_dict as DEVICE fp32 pointers, by name
 *                        ("conv1.weight", "bn1.running_var", "layer3.0.downsample.1.bias", "layer1.0.bn1.IN.weight", ...),
 *                        plus optionally "bn_head.weight|bias|running_mean|running_var" (ModelBase.bn, [feature_dim]).
 *                        Folds every eval BatchNorm into fp16 weights + fp32 biases on the device and keeps the packed
 *                        operands in the handle.  Call again whenever the parameters change (after opt.step(), load_state_dict).
 *   ctl_embed_forward  : x NCHW fp32 [n][3][h][w] on the device -> out_feat [n][feature_dim] (global_feat) and / or out_emb
 *                        [n][feature_dim] (= eval BatchNorm1d(global_feat); needs the bn_head.* tensors).  Activations live in the
 *                        caller's workspace of ctl_embed_workspace_bytes(h, n, h, w) bytes.  The entry point for C hosts:
 *                        stem -> blocks -> head below in one call.
 * The same forward in three stages, for hosts that capture or time them separately; NHWC fp16 tensors between them are
 * the caller's:
 *   ctl_embed_stem     : conv1 7x7/2 + bn1 (+ReLU for IBN-a) + maxpool 3x3/2 -> out [n][hp][wp][64], hp = (h/2 - 1)/2 + 1
 *                        with h/2 = (h - 1)/2 + 1 (wp alike).  x is fp32 NCHW [n][3][h][w], or with mean3_host and std3_host
 *                        uint8 NHWC [n][h][w][3] crops normalised as ctl_stem_pool_fused_u8 does (h % 4 == 0, even w <= 128).
 *                        Workspace: ctl_embed_workspace_bytes(h, n, h, w) bytes (the tensor-core stem's temporary).
 *   ctl_embed_blocks   : x [n][hp][wp][64] -> out [n][ho][wo][feature_dim] (ho = hp / 4, / 8 with last_stride 2).  Never
 *                        writes x.  Workspace: ctl_embed_workspace_bytes(h, n, 4 * hp, 4 * wp) bytes, no more than the image
 *                        size needs.
 *   ctl_embed_head     : x [n][hw][feature_dim] -> out_feat and / or out_emb as ctl_embed_forward.
 *   ctl_embed_launches : kernels launched by the handle's last ctl_embed_* call.
 * The fused stem (h % 4 == 0, even w <= 128) stages its input in a zero-bordered buffer that the handle allocates at the
 * first call with each (n, h, w) and keeps until ctl_trunk_destroy; a call that would allocate one while `stream` is
 * capturing a graph is CTL_ERR_INVALID_ARGUMENT, so capture after one eager call at the same shape.
 * The handle is per device and not thread-safe; all launches go to `stream`; a missing / mis-sized tensor is
 * CTL_ERR_INVALID_ARGUMENT naming it. */
typedef struct ctl_trunk ctl_trunk;
typedef struct ctl_named_tensor {
  const char* name;
  const float* data; /* device pointer */
  int64_t numel;
} ctl_named_tensor;
#define CTL_BLOCK_BOTTLENECK 0
#define CTL_BLOCK_BASIC 1
int ctl_trunk_create(ctl_trunk** out, int32_t block, int32_t ibn, int32_t last_stride, const int32_t stage_blocks[4]);
int32_t ctl_trunk_feature_dim(const ctl_trunk* h);
void ctl_trunk_destroy(ctl_trunk* h);
int ctl_weights_pack(ctl_trunk* h, const ctl_named_tensor* tensors, int32_t n_tensors, ctl_stream_t stream);
size_t ctl_embed_workspace_bytes(const ctl_trunk* h, int32_t n, int32_t height, int32_t width);
int ctl_embed_forward(ctl_trunk* h, const float* x_nchw, int32_t n, int32_t height, int32_t width, float* out_feat,
                      float* out_emb, void* workspace, size_t workspace_bytes, ctl_stream_t stream);
int ctl_embed_stem(ctl_trunk* h, const void* x, int32_t n, int32_t height, int32_t width, const float* mean3_host,
                   const float* std3_host, void* out_nhwc, void* workspace, size_t workspace_bytes, ctl_stream_t stream);
int ctl_embed_blocks(ctl_trunk* h, const void* x_nhwc, int32_t n, int32_t height, int32_t width, void* out_nhwc,
                     void* workspace, size_t workspace_bytes, ctl_stream_t stream);
int ctl_embed_head(ctl_trunk* h, const void* x_nhwc, int32_t n, int32_t hw, float* out_feat, float* out_emb,
                   ctl_stream_t stream);
int32_t ctl_embed_launches(const ctl_trunk* h);

/* ---- training-side trunk kernels (autograd through modelling/backbones/resnet.py:67-87 in train mode) ---- */

/* Weight gradient of ctl_conv2d_nhwc_f16's convolution (torch.nn.Conv2d backward w.r.t. weight):
 *   dw[co][r][s][ci] = sum_{n,ho,wo} dy[n][ho][wo][co] * x[n][ho*stride + r - pad][wo*stride + s - pad][ci]
 * x: NHWC fp16 [n][h][w][cin]; dy: NHWC fp16 [n][ho][wo][cout]; dw: fp32 [cout][k][k][cin] (the layout of the
 * forward's weight operand).  fp32 accumulation, deterministic (fixed split + fixed-order reduction).
 * `workspace` holds the per-split partial tiles: ctl_conv2d_wgrad_workspace_bytes(...) bytes. */
size_t ctl_conv2d_wgrad_workspace_bytes(int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t ksize,
                                        int32_t stride);
int ctl_conv2d_wgrad_nhwc_f16(const void* x, int32_t n, int32_t h, int32_t w, int32_t cin, const void* dy, int32_t cout,
                              int32_t ksize, int32_t stride, void* workspace, size_t workspace_bytes, float* dw,
                              ctl_stream_t stream);
/* Same, with the epilogue a training step needs folded into the split-K reduction: dw is multiplied by out_scale (the
 * 1 / loss-scale un-scaling) and, with param_layout != 0, written as [cout][cin][k][k] -- torch.nn.Conv2d.weight's own
 * layout -- so the gradient needs no permute / mul pass. */
int ctl_conv2d_wgrad_nhwc_f16_ex(const void* x, int32_t n, int32_t h, int32_t w, int32_t cin, const void* dy, int32_t cout,
                                 int32_t ksize, int32_t stride, void* workspace, size_t workspace_bytes, float* dw,
                                 float out_scale, int32_t param_layout, ctl_stream_t stream);
/* Operand packs of every convolution of a training step in ONE launch: table = device array of
 * {const float* src [cout][cin][k][k]; void* fwd fp16 [cout][k][k][cin]; void* dgrad fp16 [cin][k][k][cout] with flipped
 * taps (may be NULL); int32 cout, cin, k, pad; int64 chunk_begin} (48 bytes; chunk_begin = running sum of
 * ceil(numel / CTL_PACK_CHUNK) over the preceding entries). */
#define CTL_PACK_CHUNK 8192
int ctl_train_pack_weights(const void* table_device, int32_t n_tensors, int64_t n_chunks, ctl_stream_t stream);

/* BatchNorm2d with batch statistics (torch.nn.BatchNorm2d in train mode, resnet.py:72-85) over NHWC fp16
 * [rows = N*H*W] rows of `pitch` elements, normalising the c channels that start at the given pointers (pitch == c
 * for a dense tensor; pitch > c addresses a channel slice, e.g. the BatchNorm half of an IBN layer); c a power of two
 * in [32, 2048].  forward: mean / biased variance over the rows (fp32 partial
 * sums combined in double, deterministic), running statistics updated in place when given (momentum, unbiased
 * variance), out = [relu](gamma * (y - mean) * invstd + beta [+ residual]) rounded to fp16; save_mean / save_invstd
 * feed the backward.  backward: g = dz * (z > 0) when the ReLU output z is given (g is written to g_out, which may
 * alias dz) else g = dz; dgamma = sum g * xhat, dbeta = sum g (both multiplied by grad_unscale, fp32);
 * dy = gamma * invstd * (g - mean_rows(g) - xhat * mean_rows(g * xhat)) rounded to fp16.
 * Workspace: ctl_bn_workspace_bytes(rows, c). */
size_t ctl_bn_workspace_bytes(int64_t rows, int32_t c);
int ctl_bn_train_forward_nhwc_f16(const void* y, int64_t rows, int32_t c, int32_t pitch, const float* gamma, const float* beta, float eps,
                                  float momentum, float* running_mean, float* running_var, const void* residual,
                                  int32_t relu, void* workspace, size_t workspace_bytes, float* save_mean,
                                  float* save_invstd, void* out, ctl_stream_t stream);
int ctl_bn_train_backward_nhwc_f16(const void* dz, const void* z, const void* y, int64_t rows, int32_t c, int32_t pitch, const float* gamma,
                                   const float* save_mean, const float* save_invstd, float grad_unscale, void* workspace,
                                   size_t workspace_bytes, void* g_out, float* dgamma, float* dbeta, void* dy,
                                   ctl_stream_t stream);
/* InstanceNorm2d(affine) + ReLU of an IBN layer's first `half` channels in train mode (resnet_ibn_a.py:18-32): y, out,
 * dz, z, dy are NHWC fp16 with rows of `pitch` elements ([n][hw][pitch]); instance statistics (biased variance) per
 * (image, channel) are saved as [n][half] fp32, unless save_mean and save_invstd are both null; out may equal y (in place,
 * as ctl_instnorm_relu_nhwc_f16 runs it).  backward: g = dz * (z > 0) is written back over dz; dgamma_part /
 * dbeta_part are per-image partials [n][half] (sum over n = the parameter gradient), multiplied by grad_unscale. */
int ctl_instnorm_train_forward_nhwc_f16(const void* y, int32_t n, int32_t hw, int32_t pitch, int32_t half, const float* gamma,
                                        const float* beta, float eps, float* save_mean, float* save_invstd, void* out,
                                        ctl_stream_t stream);
int ctl_instnorm_train_backward_nhwc_f16(void* dz, const void* z, const void* y, int32_t n, int32_t hw, int32_t pitch,
                                         int32_t half, const float* gamma, const float* save_mean, const float* save_invstd,
                                         float grad_unscale, float* dgamma_part, float* dbeta_part, void* dy,
                                         ctl_stream_t stream);
/* Backward helpers of the trunk: global average pool (out[n][p][c] = dfeat[n][c] * scale, fp16), max-pool 3x3/2 pad 1
 * (gradient routed to the first maximum of every window, like torch), zero-insertion upsampling
 * out[n][2i][2j] = x[n][i][j] (+ add) (the transpose of a stride-2 subsampling), and the stem's im2col
 * ([n*ho*wo][192] fp16, k = (c*7 + r)*8 + s) that turns the 7x7 weight gradient into ctl_conv2d_wgrad_nhwc_f16
 * with cin = 192, ksize = 1. */
int ctl_gap_backward_nhwc_f16(const float* dfeat, int32_t n, int32_t hw, int32_t c, float scale, void* out,
                              ctl_stream_t stream);
int ctl_maxpool3x3s2_backward_nhwc_f16(const void* x, const void* dy, int32_t n, int32_t h, int32_t w, int32_t c, void* dx,
                                       ctl_stream_t stream);
/* Training pair of the pool: the forward also records which window tap (r*3 + s, one byte per output element,
 * [n][ho][wo][c] uint8) held the first maximum; the backward gathers from the <= 4 windows of a pixel. */
int ctl_maxpool3x3s2_argmax_nhwc_f16(const void* x, int32_t n, int32_t h, int32_t w, int32_t c, void* out, void* arg_u8,
                                     ctl_stream_t stream);
int ctl_maxpool3x3s2_backward_argmax_nhwc_f16(const void* arg_u8, const void* dy, int32_t n, int32_t h, int32_t w, int32_t c,
                                              void* dx, ctl_stream_t stream);
int ctl_upsample2_zero_nhwc_f16(const void* x, int32_t n, int32_t h, int32_t w, int32_t c, const void* add, void* out,
                                ctl_stream_t stream);
int ctl_stem_im2col_f16(const float* x_nchw, int32_t n, int32_t h, int32_t w, void* out, ctl_stream_t stream);

/* ---- train-mode trunk behind an opaque handle (SURVEY 8b: the train forward / backward variants) ----
 * replaces: torch autograd through ResNet.forward / ResNet_IBN.forward in train mode (modelling/backbones/resnet.py:67-87,
 * 122-133, resnet_ibn_a.py:18-32,126-141) + Baseline.forward's pooling (modelling/baseline.py:91-96) inside
 * CTLModel.training_step (train_ctl_model.py:38-179): x -> global_feat [n][feature_dim], then d(loss)/d(global_feat) ->
 * every parameter gradient.  This is the training trunk's only driver; modelling/backbones/engine_train.py::TrunkTrainer
 * is its ctypes form.
 *   ctl_trainer_create      : ResNet of `block` (CTL_BLOCK_BOTTLENECK or CTL_BLOCK_BASIC) blocks with `stage_blocks`
 *                             blocks per stage ({3, 4, 6, 3} = ResNet50 / ResNet34, {3, 4, 23, 3} = ResNet101,
 *                             {2, 2, 2, 2} = ResNet18, each >= 1), IBN-a when `ibn` != 0 (bottleneck only),
 *                             MODEL.LAST_STRIDE 1 or 2, BatchNorm momentum in (0, 1].  Argument errors as ctl_trunk_create.
 *   ctl_trainer_feature_dim : 2048 (bottleneck) or 512 (basic).  Host only.
 *   ctl_trainer_bind        : `params` = the `base.*`-stripped fp32 parameters AND BatchNorm running buffers as device
 *                             pointers, by name (running_mean / running_var optional per layer, updated in place like
 *                             torch); `grads` = one fp32 output per PARAMETER, same name, the parameter's own layout
 *                             (conv [Cout][Cin][k][k]).  The handle keeps the pointers: re-bind when storage moves.
 *   ctl_train_workspace_bytes: bytes of the caller's workspace for one (n, h, w) step: the saved activations of the
 *                             forward + the scratch of the backward (≈ 60 MB per 256x128 image).
 *   ctl_train_forward       : x NCHW fp32 -> out_feat [n][feature_dim] fp32 (global_feat); saved tensors stay in
 *                             `workspace`.
 *   ctl_train_backward      : dfeat [n][feature_dim] fp32 = dLoss/dglobal_feat.  Activation gradients are computed on
 *                             grad_scale * dfeat in fp16 (loss scaling, the role of PL's GradScaler, utils/misc.py:111);
 *                             the parameter gradients are written UN-scaled.  Same workspace as the forward, once per forward.
 *   ctl_train_saved         : inspection call for checkers: the fp16 NHWC tensors the last completed forward saved in
 *                             its workspace, raw conv output `y` and normalised output `z`, with their shape `nhwc`.
 *                             index 0 = the stem, 1... = every conv + BatchNorm in forward order: per bottleneck conv1,
 *                             conv2, [downsample], conv3; per basic block conv1, [downsample], conv2 (conv2's BatchNorm
 *                             adds the shortcut, so the downsample runs before it).  An error before a forward or out of
 *                             range.
 * Not thread-safe; all launches go to `stream`; 256-byte aligned workspace. */
typedef struct ctl_trainer ctl_trainer;
typedef struct ctl_named_buffer {
  const char* name;
  float* data; /* device pointer, written */
  int64_t numel;
} ctl_named_buffer;
int ctl_trainer_create(ctl_trainer** out, int32_t block, int32_t ibn, int32_t last_stride, float momentum,
                       const int32_t stage_blocks[4]);
int32_t ctl_trainer_feature_dim(const ctl_trainer* t);
void ctl_trainer_destroy(ctl_trainer* t);
int ctl_trainer_bind(ctl_trainer* t, const ctl_named_tensor* params, int32_t n_params, const ctl_named_buffer* grads,
                     int32_t n_grads);
size_t ctl_train_workspace_bytes(const ctl_trainer* t, int32_t n, int32_t height, int32_t width);
int ctl_train_forward(ctl_trainer* t, const float* x_nchw, int32_t n, int32_t height, int32_t width, float* out_feat,
                      void* workspace, size_t workspace_bytes, ctl_stream_t stream);
int ctl_train_backward(ctl_trainer* t, const float* dfeat, float grad_scale, void* workspace, size_t workspace_bytes,
                       ctl_stream_t stream);
int ctl_train_saved(const ctl_trainer* t, int32_t index, const void** y, const void** z, int32_t nhwc[4]);

/* ---- optimizer step (solver/build.py:9-47, train_ctl_model.py:155-159, modelling/bases.py:102-133) ---- */

/* One table entry per parameter tensor, resident on the device; chunk_begin = running sum of
 * ceil(numel / CTL_OPT_CHUNK) over the preceding entries. */
#define CTL_OPT_CHUNK 8192
typedef struct ctl_adam_entry {
  float* param;
  const float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  int64_t numel;
  int64_t chunk_begin;
} ctl_adam_entry;
/* torch.optim.Adam (L2 weight decay added to the gradient, bias-corrected, no amsgrad) on every tensor of the table
 * in one launch; `step` is the 1-based step count after this update; gradients are read as grad * grad_mul. */
int ctl_adam_multi_step(const void* table_device, int32_t n_tensors, int64_t n_chunks, float lr, float beta1, float beta2,
                        float eps, float weight_decay, int64_t step, float grad_mul, const int32_t* skip_flag,
                        ctl_stream_t stream);
/* torch.optim.SGD without momentum: param -= lr * grad * grad_mul (the center parameters; grad_mul =
 * 1 / SOLVER.CENTER_LOSS_WEIGHT, train_ctl_model.py:157-158). */
int ctl_sgd_step(float* param, const float* grad, int64_t numel, float lr, float grad_mul, const int32_t* skip_flag,
                 ctl_stream_t stream);
/* `skip_flag` (device int, may be NULL) of the two optimizer entry points: when non-zero at execution time the kernel
 * returns without touching parameters or moments -- GradScaler.step's "skip the step on inf / NaN gradients" without a
 * host synchronisation.  ctl_loss_scale_update is GradScaler.update() on the device: state3 = {scale, scale / base_scale,
 * base_scale / scale}; *found_inf is copied to *last_found and cleared. */
int ctl_loss_scale_update(float* state3, int32_t* tracker, int32_t* found_inf, int32_t* last_found, float base_scale,
                          float growth_factor, float backoff_factor, int32_t growth_interval, ctl_stream_t stream);
/* Gradient overflow check of dynamic loss scaling (torch.cuda.amp.GradScaler.unscale_ in the reference's PL AMP trainer,
 * utils/misc.py:111): table = device array of {float* grad; int64 numel; int64 chunk_begin} (chunks of 8192 elements, like
 * ctl_adam_multi_step); every gradient is multiplied in place by `mul` * (*mul_device if non-NULL: a device scalar such as
 * base_scale / scale) -- skipped when that factor is exactly 1 -- and *found_inf (device int,
 * OR-accumulated, cleared by the caller) becomes 1 if any element is inf or NaN. */
int ctl_grad_check_multi(const void* table_device, int32_t n_tensors, int64_t n_chunks, float mul, const float* mul_device,
                         int32_t* found_inf, ctl_stream_t stream);

/* ---- training-time augmentation (datasets/transforms/build.py:15-27, random_erasing.py:30-55) ---- */

/* images: uint8 NHWC [n][h][w][3], already resized (T.Resize stays on the host); params_device: int32 [n][8] =
 * {flip, crop_top, crop_left (offsets inside the padded image, 0..2*pad), erase_row, erase_col, erase_h, erase_w
 * (erase_h == 0: none), is_real (0: mock image -> zeros)}; mean / std: 3 floats on the HOST.
 * out = RandomErasing(Normalize(ToTensor(RandomCrop(Pad(Flip(image)))))) as fp32 NCHW [n][3][h][w]. */
int ctl_augment_batch_u8(const void* images_u8_nhwc, int32_t n, int32_t h, int32_t w, int32_t pad, const int32_t* params_device,
                         const float* mean3_host, const float* std3_host, float* out_nchw, ctl_stream_t stream);

/* ---- T.Resize((out_h, out_w)) of native-size images (datasets/transforms/build.py:19,29) ----
 * The reference resizes PIL RGB images (datasets/bases.py:32-33, inference/inference_utils.py:33-34), so T.Resize is
 * Image.resize((out_w, out_h), BILINEAR).  This reproduces it bit for bit.  PIL resamples the width first, then the
 * height of the width pass's output clipped to uint8; per axis (`in` -> `out` pixels), in IEEE double without FMA:
 *   scale = in / out, support = max(scale, 1), ss = 1 / support, center = (o + 0.5) scale,
 *   xmin = max((int)(center - support + 0.5), 0), taps = min((int)(center + support + 0.5), in) - xmin,
 *   w[t] = tri((t + xmin - center + 0.5) ss) (tri(x) = max(1 - |x|, 0)), each divided by their sum taken in tap order,
 *   k[t] = (int)(0.5 + w[t] 2^22), pixel = clamp((2^21 + sum_t src[xmin + t] k[t]) >> 22, 0, 255) per channel.
 * src: HWC RGB uint8 images packed back to back in src_bytes bytes, any byte alignment; table_device: n entries
 * struct ctl_resize_entry below.  out_u8_nhwc: uint8 [n][out_h][out_w][3].  An entry with h == 0 or w == 0 is a mock
 * row (zeros).  An entry whose h * w * 3 bytes at `offset` do not fit in src_bytes (or with a negative or > 2^24 side)
 * gives zeros and sets bit 0 of *status; nothing outside src_bytes is read.
 * workspace: the uint8 intermediate [sum of the h of the real entries][out_w][3], planned by
 * ctl_resize_bilinear_u8_workspace_bytes(total_rows = that sum, ...), which is host-only and 0 for a negative
 * total_rows or an output size the call rejects.  An image whose rows do not fit in the workspace gives zeros and sets
 * bit 1 of *status.  Two launches (width pass, height pass); the call zeroes *status first.  No host synchronisation,
 * no allocation: capturable in a CUDA graph.  A null pointer, n < 1, an output side outside 1..16384, or a workspace
 * shorter than one intermediate row is CTL_ERR_INVALID_ARGUMENT before any device work. */
typedef struct ctl_resize_entry {
  int64_t offset; /* first byte of the image in src */
  int64_t h;
  int64_t w;
} ctl_resize_entry;
size_t ctl_resize_bilinear_u8_workspace_bytes(int64_t total_rows, int32_t out_h, int32_t out_w);
int ctl_resize_bilinear_u8(const void* src, int64_t src_bytes, const void* table_device, int64_t n, int32_t out_h,
                           int32_t out_w, void* out_u8_nhwc, int32_t* status, void* workspace, size_t workspace_bytes,
                           ctl_stream_t stream);

/* ---- JPEG decode: Image.open(p).convert("RGB") (datasets/bases.py:32-33, inference/inference_utils.py:33-34) ----
 * Pillow decodes with libjpeg-turbo's defaults (JDCT_ISLOW, fancy upsampling), fixed integer arithmetic that this
 * reproduces bit for bit for baseline (SOF0) and extended-sequential Huffman (SOF1) files with 8-bit samples and one
 * interleaved scan, grayscale or YCbCr, any integral sampling factors (4:4:4, 4:2:2, 4:2:0, 4:4:0, 4:1:1), with or
 * without restart intervals, 8- or 16-bit quantisation tables and any Huffman tables:
 *   - coefficients: Huffman decode with byte stuffing, RSTn resync and DC-predictor resets;
 *   - jpeg_idct_islow (jidctint.c): coef * (short)quantval, CONST_BITS 13, PASS1_BITS 2, 64-bit products, an int
 *     workspace, then x = sample - 128 clamped: sample = min(max(x + 128, 0), 255).  Pillow runs libjpeg-turbo's
 *     SIMD IDCT, which saturates; the C path's range_limit[x & 1023] (jdmaster.c prepare_range_limit_table) agrees
 *     on [-384, 512) and wraps outside it, which encoder output does not reach;
 *   - upsampling per component (jdsample.c): h2v1 / h2v2 triangle ("fancy") filters when the component's downsampled
 *     width is > 2, replication otherwise; h1v2 fancy always; replication for other integral ratios.  Neighbours are
 *     clamped to the component's real downsampled width and height; rounding +1/+2 (h2v1, h1v2), +8/+7 (h2v2);
 *   - ycc_rgb_convert (jdcolor.c): R = Y + ((91881 Cr' + 2^15) >> 16), G = Y + ((-46802 Cr' - 22554 Cb' + 2^15) >> 16),
 *     B = Y + ((116130 Cb' + 2^15) >> 16) (Cb' = Cb - 128, Cr' = Cr - 128), each clamped to 0..255; grayscale gives
 *     R = G = B = Y, as convert("RGB") of an "L" image does.
 *
 * ctl_jpeg_parse (host-only) reads the marker segments of one file up to SOS, never its entropy-coded data, and fills
 * *desc (and *h, *w when not null).  It returns 0, or CTL_ERR_UNSUPPORTED for a JPEG this decode does not cover
 * (progressive, lossless, hierarchical, arithmetic coding, not 8-bit, CMYK / YCCK, Adobe RGB (transform 0) or
 * R/G/B component ids without JFIF, a first scan without every component, non-integral sampling factors), or
 * CTL_ERR_INVALID_ARGUMENT for data that is not a JPEG or whose header is truncated or corrupt; ctl_last_error()
 * names the reason.  The colour space follows libjpeg's guess: JFIF, Adobe transform 1 or other ids mean YCbCr.
 * Offsets in the descriptor count from the file's first byte; the tables are the last definitions before SOS. */
typedef struct ctl_jpeg_desc {
  int32_t h, w;
  uint32_t scan_begin, scan_end; /* entropy-coded data: from after SOS to the end of the file */
  uint32_t dqt[3];               /* per component: its 64 quantisation values, zig-zag order */
  uint32_t dht_dc[3], dht_ac[3]; /* per component: its DHT tables' 16 code-length counts, then their symbols */
  uint16_t restart_interval;     /* MCUs per interval, 0: none */
  uint8_t ncomp;                 /* 1 (grayscale) or 3 (YCbCr) */
  uint8_t dqt16;                 /* bit c: component c's quantisation values are 16-bit big-endian */
  uint8_t hs[3], vs[3];          /* sampling factors; 1 for grayscale */
  uint8_t reserved[2];
} ctl_jpeg_desc;

#define CTL_JPEG_ENTRY_JPEG 0 /* a JPEG file described by desc */
#define CTL_JPEG_ENTRY_RAW 1  /* HWC RGB uint8 bytes of desc.h x desc.w, copied through */
#define CTL_JPEG_ENTRY_MOCK 2 /* a mock row: no bytes, an output entry with h = w = 0 */

typedef struct ctl_jpeg_entry {
  int64_t offset; /* first byte of the entry in src */
  int64_t nbytes;
  int32_t kind;   /* CTL_JPEG_ENTRY_* */
  int32_t reserved;
  ctl_jpeg_desc desc;
} ctl_jpeg_entry;

/* ctl_jpeg_decode: src holds n entries packed back to back at any byte alignment (entries_device: n struct
 * ctl_jpeg_entry in device memory).  Entry i is written as HWC RGB uint8 at out_u8 + out_table_device[i].offset
 * (struct ctl_resize_entry, whose h and w must be the entry's: 0 for a mock row), so the output is the ragged
 * input of ctl_resize_bilinear_u8.  status: int32 [n] on the device, written for every entry (the call needs no
 * clearing): 0 or an OR of 1 (entropy-coded data ending before the last MCU, a Huffman code that does not exist, a
 * coefficient index > 63, a missing RSTn marker), 2 (an entry outside src_bytes, or a descriptor ctl_jpeg_parse
 * cannot have written), 4 (an output entry of another size or outside out_bytes), 8 (a workspace too short for the
 * entry).  Such an entry's output is zeros (status 4: untouched); the others are unaffected, and nothing outside the
 * buffers is read or written.  workspace: planned by ctl_jpeg_decode_workspace_bytes (host-only, from the host copy
 * of the entries; 0 for null or n < 1): an offset per entry, then per JPEG its int16 coefficients and uint8
 * component planes (3 bytes per coefficient).  Three launches (entropy decode, one CTA per image decoding up to 256
 * subsequences of its entropy-coded data in parallel; IDCT; upsample + colour convert); no host synchronisation, no
 * allocation: capturable in a CUDA graph.  A null pointer, n < 1, a negative buffer size or a workspace shorter than
 * its header is CTL_ERR_INVALID_ARGUMENT before any device work. */
int ctl_jpeg_parse(const void* bytes, int64_t nbytes, ctl_jpeg_desc* desc, int32_t* h, int32_t* w);
size_t ctl_jpeg_decode_workspace_bytes(const ctl_jpeg_entry* entries_host, int64_t n);
int ctl_jpeg_decode(const void* src, int64_t src_bytes, const void* entries_device, int64_t n,
                    const void* out_table_device, void* out_u8, int64_t out_bytes, int32_t* status, void* workspace,
                    size_t workspace_bytes, ctl_stream_t stream);

/* ---- Ranked-result grids: visualize_ranked_results (utils/visrank.py:23-244) ----
 * The reference reads each image with cv2.imread (the same pixels as Pillow's decode, in BGR order; the calls below
 * work in RGB), then per grid cell runs cv2.resize(img, (w, h)), cv2.copyMakeBorder(3 px, colour), cv2.resize(.., (w, h))
 * (visrank.py:168-174, 206-211) and pastes the cell into a white grid (visrank.py:176-184, 212-220).
 *
 * ctl_resize_linear_cv_u8: cv2.resize(img, (out_w, out_h)) with INTER_LINEAR on HWC uint8 3-channel images, bit for
 * bit.  Per axis (`in` -> `out` pixels, o the output index): f = (float)((o + 0.5) * (in / out) - 0.5) in double,
 * s = floor(f), f -= s in float, a0 = rint((float)(1 - f) * 2048) (half to even), a1 = 2048 - a0.  Along x the weights
 * are clamped (s < 0: s = 0, f = 0; s >= in - 1: s = in - 1, f = 0); along y they are not, and the two source rows are
 * clamped to [0, in - 1].  Per channel: hrow(y) = S[y][s] a0 + S[y][min(s + 1, in - 1)] a1,
 * out = min((((b0 (hrow(y0) >> 4)) >> 16) + ((b1 (hrow(y1) >> 4)) >> 16) + 2) >> 2, 255).
 * src / table_device: the ragged batch of ctl_resize_bilinear_u8 (struct ctl_resize_entry).  out_u8_nhwc: uint8
 * [n][out_h][out_w][3].  status: int32 [n] on the device, written for every entry: 0, or 1 for an entry whose bytes
 * do not fit in src_bytes (or with a negative or > 2^24 side); such an entry and a mock row (h or w == 0) give zeros.
 * One launch, no workspace, no host synchronisation: capturable in a CUDA graph.  A null pointer, n < 1 or an output
 * side outside 1..16384 is CTL_ERR_INVALID_ARGUMENT before any device work.
 *
 * ctl_visrank_compose: the grids uint8 [n_grids][h][Wg][3], Wg = (topk + 1) w + 2 topk + 8, from the images of
 * ctl_resize_linear_cv_u8 (resized_u8: uint8 [n_rows][h][w][3]).  cells_device: int32 [n_cells][4] = {row of
 * resized_u8, grid, column, border colour 0xRRGGBB}.  Every grid is first filled with 255; the cell of column c is
 * cv2.resize(copyMakeBorder(row, 3, 3, 3, 3, colour), (w, h)), computed without an intermediate, at x = 0 for c = 0
 * (the query) and x = c w + 2 c + 8 otherwise.  A cell with a row, grid or column (0..topk) out of range is skipped
 * and sets *status (zeroed by the call) to 1.  No host synchronisation: capturable in a CUDA graph.
 *
 * ctl_visrank_select: the ranked list of visrank.py:192-232.  topk_idx: int64 [nq][k], each query's k nearest
 * gallery rows in ascending (distance, index) order; identities as in struct ctl_pass_desc: q_pid, q_cam int32 [nq];
 * g_pid int32 [ng]; g_cammask uint64 [ng].  A row is junk when g_pid == q_pid and bit q_cam of g_cammask is set
 * (same pid and camera, or with camera sets the query's camera is in the centroid's set, visrank.py:196-200).
 * Writes the first topk non-junk rows of each query to out_idx int64 [nq][topk] and out_matched int8 [nq][topk]
 * (1 when g_pid == q_pid), padded with -1 / 0 when fewer remain.  k must cover topk plus the query's junk rows for the
 * list to be complete.  An index outside [0, ng) stops that query and sets *status (zeroed by the call) to 1. */
int ctl_resize_linear_cv_u8(const void* src, int64_t src_bytes, const void* table_device, int64_t n, int32_t out_h,
                            int32_t out_w, void* out_u8_nhwc, int32_t* status, ctl_stream_t stream);
int ctl_visrank_compose(const void* resized_u8, int64_t n_rows, int32_t h, int32_t w, const int32_t* cells_device,
                        int64_t n_cells, int64_t n_grids, int32_t topk, void* out_u8, int32_t* status,
                        ctl_stream_t stream);
int ctl_visrank_select(const int64_t* topk_idx, int64_t nq, int32_t k, const int32_t* q_pid, const int32_t* q_cam,
                       const int32_t* g_pid, const uint64_t* g_cammask, int64_t ng, int32_t topk, int64_t* out_idx,
                       int8_t* out_matched, int32_t* status, ctl_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* CTL_H100_H_ */
