/*
 * tensorrec_b200.h -- C ABI of the H100-native (sm_90a) predict / predict_rank hot path of jfkirk/tensorrec.
 *
 * The reference (pure Python over TensorFlow 1.x, commit 80690737) has no FFI of its own; the boundary a
 * maintainer would bind is the set of TF ops its graph evaluates on this path.  Each entry point below
 * replaces one of those graph nodes (reference file:line given per function; paths relative to the
 * reference root).  INTEGRATION.md shows the ctypes binding on the reference side.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless named host_*; the caller owns every buffer;
 *   - matrices are dense row-major; indices are int32; values float32;
 *   - `stream` is a cudaStream_t passed as void* (NULL = default stream); calls are asynchronous;
 *   - return value: 0 = ok, negative = TRK_ERR_*; trk_last_error() gives the text for this thread;
 *   - nothing here allocates persistent device memory; workspace sizes are queried and caller-provided;
 *   - there is no CPU fallback: without a CUDA device every compute entry point returns TRK_ERR_CUDA.
 */
#ifndef TENSORREC_B200_H_
#define TENSORREC_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TRK_OK 0
#define TRK_ERR_ARG (-1)         /* bad argument (null pointer, size, alignment, unsupported shape) */
#define TRK_ERR_CUDA (-2)        /* a CUDA runtime / driver call failed */
#define TRK_ERR_UNSUPPORTED (-3) /* shape outside what the fused tensor-core kernel supports */

/* ABI version of this header (major*1000 + minor). */
int trk_version(void);

/* Text of the last error raised on the calling thread ("" if none). */
const char* trk_last_error(void);

/* ------------------------------------------------------------------------------------------------------
 * K1  sparse features -> dense representation (CSR x dense gather-reduce)
 *
 * replaces tf.sparse_tensor_dense_matmul in LinearRepresentationGraph.connect_representation_graph
 * (tensorrec/representation_graphs.py:32-43, the matmul is :40) and, with n_normalize >= 1, the
 * tf.nn.l2_normalize of NormalizedLinearRepresentationGraph (:53-58, :57) and of relative_cosine
 * (tensorrec/recommendation_graphs.py:119-120).
 *
 *   out[r, :] = sum over p in [indptr[r], indptr[r+1])  val[p] * weights[col[p], :]     (fp32, CSR order)
 *   then n_normalize times:  out[r, :] *= rsqrt(max(sum(out[r, :]^2), 1e-12))
 *
 * CSR entries of one row are accumulated sequentially in storage order (duplicates are summed), so the
 * result is run-to-run bit-identical (reference requirement: test/test_tensorrec.py:418-458).
 *
 * Outputs (either may be NULL, not both):
 *   out_f32   [rows, d]            the representation as the reference returns it;
 *   out_split [rows, 2*d_pad] f16  the operand layout of the tensor-core score kernel: columns [0,d_pad) hold
 *                                  hi = fp16(x * 2^e_r), columns [d_pad, 2*d_pad) hold lo = fp16(x * 2^e_r - hi),
 *                                  zero padded from d to d_pad (d_pad a multiple of 64);
 *   out_scale [rows]               2^-e_r, the exact power of two that undoes the per-row scaling
 *                                  (required when out_split is given);
 *   out_norm  [rows] (optional)    |out[r, :]|_2 inflated by 2^-9: an UPPER bound, the factor of the filter's error bound;
 *   stats     [3]    (optional)    zeroed by this call, then stats[0] = max out_norm, stats[1] = max out_scale over the
 *                                  non-zero rows (atomic max on the float bits: order independent); stats[2] is left
 *                                  for trk_pack_item_bias.  The row is still in registers when these are formed: the
 *                                  separate pass of trk_operand_stats over the operand is not needed after K1.
 * ---------------------------------------------------------------------------------------------------- */
int trk_csr_gather_reduce_f32(const int32_t* indptr, const int32_t* col, const float* val,
                              const float* weights, int64_t rows, int32_t n_features, int32_t d,
                              int32_t n_normalize, float* out_f32, void* out_split, int32_t d_pad,
                              float* out_scale, float* out_norm, float* stats, void* stream);

/* Converts an existing dense fp32 representation [rows, d] into the split-fp16 operand + scales
 * (same layout as above).  Used when a representation comes from a user-defined plugin graph. */
int trk_split_f32_to_f16x2(const float* repr, int64_t rows, int32_t d, int32_t n_normalize, void* out_split,
                           int32_t d_pad, float* out_scale, void* stream);

/* L2-normalises rows of a dense fp32 matrix in place: tf.nn.l2_normalize(x, 1)
 * (tensorrec/recommendation_graphs.py:119-120). */
int trk_l2_normalize_rows_f32(float* x, int64_t rows, int32_t d, void* stream);

/* ------------------------------------------------------------------------------------------------------
 * project_biases (tensorrec/recommendation_graphs.py:4-19):
 *   out[r] = sum over the row's entries  val[p] * feature_biases[col[p]]      (fp32, CSR order)
 * ---------------------------------------------------------------------------------------------------- */
int trk_csr_project_biases_f32(const int32_t* indptr, const int32_t* col, const float* val,
                               const float* feature_biases, int64_t rows, float* out, void* stream);

/* ------------------------------------------------------------------------------------------------------
 * K2 (exact fp32, CUDA cores)  dense prediction for every user x item pair, any shape
 *
 * replaces tf.matmul(user, item, transpose_b=True) of DotProductPredictionGraph.connect_dense_prediction_graph
 * (tensorrec/prediction_graphs.py:49-50) / relative_cosine (tensorrec/recommendation_graphs.py:121, inputs
 * pre-normalised by K1), followed by collapse_mixture_of_tastes without attention (max over tastes,
 * tensorrec/recommendation_graphs.py:107) and bias_prediction_dense (:41):
 *
 *   out[u, i] = max_t ( sum_k user_repr[t, u, k] * item_repr[i, k] )  + user_bias[u] + item_bias[i]
 *
 * user_repr is [n_tastes, n_users, d]; user_bias / item_bias may be NULL (unbiased model).
 * mode: 0 = dot product, 1 = negative euclidean distance (EuclideanSimilarityPredictionGraph,
 * tensorrec/prediction_graphs.py:84-100).
 * ---------------------------------------------------------------------------------------------------- */
int trk_score_f32(const float* user_repr, const float* item_repr, const float* user_bias,
                  const float* item_bias, float* out, int64_t n_users, int64_t n_items, int32_t d,
                  int32_t n_tastes, int32_t mode, void* stream);

/* Attention variant of the taste collapse (tensorrec/recommendation_graphs.py:96-103):
 *   out[u,i] = sum_t softmax_t(att[t,u,i]) * pred[t,u,i]  (+ biases), pred/att = dot products of
 *   user_repr[t] / attention_repr[t] with item_repr. */
int trk_score_attention_f32(const float* user_repr, const float* attention_repr, const float* item_repr,
                            const float* user_bias, const float* item_bias, float* out, int64_t n_users,
                            int64_t n_items, int32_t d, int32_t n_tastes, void* stream);

/* ------------------------------------------------------------------------------------------------------
 * K3 (full)  rank_predictions (tensorrec/recommendation_graphs.py:73-82): the reference's double
 * tf.nn.top_k(k = n_items) == for every user row
 *     rank[u, i] = 1 + #{j : s[u,j] > s[u,i]} + #{j < i : s[u,j] == s[u,i]}          (int32, 1-based)
 * computed by a per-row sort of (score descending, index ascending) keys.
 * workspace: trk_rank_full_workspace_bytes(n_users, n_items) bytes of device memory.
 * ---------------------------------------------------------------------------------------------------- */
size_t trk_rank_full_workspace_bytes(int64_t n_users, int64_t n_items);
int trk_rank_full(const float* scores, int32_t* ranks, int64_t n_users, int64_t n_items, void* workspace,
                  size_t workspace_bytes, void* stream);
/* order[ranks[i] - 1] = i for ONE row of ranks: the items of that row listed by reference rank (tf.nn.top_k order).
 * trk_rank_full on the 1 x n_items row of item biases followed by this call is the stable descending sort that fixes the
 * filter kernel's processing order (no library sort of the items or of any score on the predict path; the only sort is
 * the O(nnz) ordering of exclusion lists, see trk_exclusion_positions). */
int trk_order_from_ranks(const int32_t* ranks, int64_t n, int32_t* order, void* stream);

/* ------------------------------------------------------------------------------------------------------
 * K2+K3 fused (tensor cores, sm_90a)   scores and per-user top-k without materialising [n_users, n_items]
 *
 * replaces the chain  tf.matmul (prediction_graphs.py:49-50)  ->  bias_prediction_dense
 * (recommendation_graphs.py:41)  ->  rank_predictions (recommendation_graphs.py:73-82) restricted to the
 * entries with rank <= k (the only ones tensorrec/eval.py:23,49,68-69 ever reads).
 *
 * Operands are the split-fp16 layout produced by K1 (hi/lo halves, per-row power-of-two scale); the score is
 *   s[u,i] = (hi_u.hi_i + hi_u.lo_i + lo_u.hi_i) * scale_u * scale_i + user_bias[u] + item_bias[i]
 * accumulated in fp32 in registers (three groups of wgmma per k-block; relative error vs an fp32 dot
 * product <= 2^-21 of |u|.|i|, and exact for integer-valued representations).
 *
 * The item axis is cut into n_splits contiguous ranges (parallelism when n_users is small; shards when the
 * item axis is distributed over GPUs).  For each (user, split) the kernel emits the k best candidates ordered by
 * (score descending, item id ascending):
 *   cand_score [n_users, n_splits, k] f32,  cand_item [n_users, n_splits, k] i32 (GLOBAL ids = local + item_id_offset;
 *   unused slots: score = -inf, id = INT32_MAX).
 * item_meta [n_items_padded256, 2] f32 = {item scale, item bias} per item, rows beyond n_items = {0, -inf}
 * (build with trk_pack_item_meta).  user_bias may be NULL.
 * Constraints: d_pad in {64, 128}; 1 <= k <= trk_score_topk_max_k(d_pad).
 * n_users_live (device int32, may be NULL): only the first *n_users_live user rows hold work -- user blocks beyond
 * them are skipped on the device.  This is how the rows the filter's certificate rejects are re-scored without a
 * host round trip (their count exists only on the device, see trk_select_flagged_rows).
 * ---------------------------------------------------------------------------------------------------- */
int trk_score_topk_max_k(int32_t d_pad);
int trk_pack_item_meta(const float* item_scale, const float* item_bias, int64_t n_items, float* item_meta,
                       int64_t n_items_padded, void* stream);
int trk_score_topk_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                         const void* item_split, const float* item_meta, int64_t n_users, int64_t n_items,
                         int32_t d_pad, int32_t k, int32_t n_splits, int32_t item_id_offset,
                         float* cand_score, int32_t* cand_item, const int32_t* n_users_live, void* stream);

/* ------------------------------------------------------------------------------------------------------
 * Exclusion: the top-k among the items a user has NOT interacted with (serving, and the held-out evaluation protocol
 * of tensorrec/eval.py:23,49,68-69 with the training interactions removed).  The result is the chain above on a model
 * whose excluded pairs score -inf, with excluded items never reported: for every user the k best non-excluded items in
 * tf.nn.top_k order (score descending, lower item id first); a user with fewer than k eligible items gets the sentinel
 * (-inf, INT32_MAX) in the remaining slots.  An empty list leaves a row's result bit-identical to the calls without
 * exclusion.
 *
 * Lists are CSR over the launch's user rows: int32 excl_indptr [rows + 1], int32 values per row strictly ascending.
 *   trk_score_topk_f16x3_excl  the arguments of trk_score_topk_f16x3 plus excl_ids = LOCAL item ids (global id -
 *                              item_id_offset, in [0, n_items)) and excl_row_map (may be NULL): user row u of the
 *                              launch reads list row excl_row_map[u] -- the idx array of trk_select_flagged_rows, so
 *                              the device-side fallback over gathered rows needs no gathered lists.  Rows at or beyond
 *                              *n_users_live exclude nothing (their results are discarded).
 *   trk_exclusion_positions    the filter kernel walks items in PROCESSING order (item_perm: position -> local id), so
 *                              it takes each row's list as processing positions: inv_perm (int32 [n_items], workspace)
 *                              = the inverse of item_perm, then out_keys[e] (int64 [nnz]) = (row << 32) | inv_perm[id]
 *                              for every entry e of row `row` (item_perm NULL = identity, inv_perm unused).  Sorting
 *                              out_keys ascending orders every row (rows are contiguous: excl_indptr is unchanged); the
 *                              low 32 bits of the sorted keys are excl_pos.  That O(nnz) sort prepares the lists -- it
 *                              is not part of the scoring.
 *   trk_score_filter_f16_excl  the arguments of trk_score_filter_f16 plus excl_pos (processing positions, ascending).
 *                              Excluded items leave the candidate universe (also in the first tile the starting
 *                              threshold is taken from); the certificate of trk_rescore_topk_split is unchanged, and
 *                              rows it flags are re-run through trk_score_topk_f16x3_excl with the same lists.
 * ---------------------------------------------------------------------------------------------------- */
int trk_score_topk_f16x3_excl(const void* user_split, const float* user_scale, const float* user_bias,
                              const void* item_split, const float* item_meta, int64_t n_users, int64_t n_items,
                              int32_t d_pad, int32_t k, int32_t n_splits, int32_t item_id_offset,
                              float* cand_score, int32_t* cand_item, const int32_t* n_users_live,
                              const int32_t* excl_indptr, const int32_t* excl_ids, const int32_t* excl_row_map,
                              void* stream);
int trk_exclusion_positions(const int32_t* item_perm, int64_t n_items, int32_t* inv_perm, const int32_t* excl_indptr,
                            const int32_t* excl_ids, int64_t n_rows, int64_t* out_keys, void* stream);

/* ------------------------------------------------------------------------------------------------------
 * K2+K3 fused, FILTER form (the throughput path of predict_rank(k)): one tensor-core pass over the fp16 "hi"
 * halves gives approximate scores with a proven error bound m = 1.5*2^-10 * |u|_2 * max_j |i_j|_2 (+ bias
 * rounding); per user the kernel keeps every item whose approximate score is within 2.25 m of the running k-th best.
 * trk_rescore_topk_split then scores the survivors from the full split operands (22-bit operands, fp32 accumulate: the
 * arithmetic of trk_score_topk_f16x3; reference chain tensorrec/prediction_graphs.py:49-50 and
 * recommendation_graphs.py:41), ranks them in tf.nn.top_k order (recommendation_graphs.py:81) and verifies the
 * bound; users it flags are re-run through trk_score_topk_f16x3 (device-side routing below).  Same reference chain
 * as trk_score_topk_f16x3, one third of its tensor work.
 *
 * Preparation (all device-side, no host sync):
 *   K1 (trk_csr_gather_reduce_f32) already yields the user norms and the item statistics; for operands that do not
 *   come from K1 (user-defined representation graphs):
 *   trk_operand_stats      norm[r] = |row r|_2 (upper bound) of a split operand; stats[0] = max norm, stats[1] = max
 *                          row scale, both by atomic max (stats[3] must be zeroed by the caller; either output may be
 *                          NULL)
 *   trk_rescale_hi_global  item "hi" half re-expressed with ONE scale for the whole matrix and laid out in PROCESSING
 *                          order: out_hi[p, :] (f16 [rows, d_pad]) = hi[perm[p], :] * (scale[perm[p]] / stats[1]) (exact
 *                          power-of-two factors; perm NULL = identity)
 *   trk_pack_item_bias     out[p] = bias[perm[p]], padded with -inf to n_padded (multiple of 256) entries; stats[2] =
 *                          max |bias|; block_max[b] / block_min[b] = max / min bias of positions [128 b, 128 b + 128)
 *                          (min = -inf as soon as the block holds padding; block_min may be NULL)
 * Processing order: the host sorts the items by DESCENDING bias (perm = stable argsort) so that the biases inside a
 * 128-item block are nearly equal and the running k-th best rises early; the kernel's hot loop then bounds
 * acc_j + bias_j / c by max_j acc_j + block_max / c and touches neither the biases nor an FFMA per score.  With
 * block_bias_min the kernel also starts every (user, split) sweep from a threshold derived from the first tile
 * (k-th largest of 16 group maxima + block minimum) instead of -inf.  Candidate ids are reported in ORIGINAL numbering.
 * Filter outputs, one list per (user, split): cand_* [n_users, n_splits, 16] (approximate score, global id;
 * unused = (-inf, INT32_MAX)), row_theta [n_users, n_splits].
 * Constraints: d_pad in {64, 128}; 1 <= k <= trk_score_filter_max_k().
 * ---------------------------------------------------------------------------------------------------- */
int trk_score_filter_max_k(void);
int trk_score_filter_list_width(void); /* candidates per list: 16 (one list per (user, split)) */
int trk_operand_stats(const void* split, const float* scale, int64_t rows, int32_t d_pad, float* out_norm,
                      float* stats, void* stream);
int trk_rescale_hi_global(const void* split, const float* scale, const float* stats, const int32_t* perm,
                          int64_t rows, int32_t d_pad, void* out_hi, void* stream);
int trk_pack_item_bias(const float* item_bias, const int32_t* perm, int64_t n_items, float* out,
                       int64_t n_items_padded, float* stats, float* block_max, float* block_min, void* stream);
int trk_score_filter_f16(const void* user_split, const float* user_scale, const float* user_bias,
                         const float* user_norm, const void* item_hi_global, const float* item_stats,
                         const float* item_bias_padded, const float* block_bias_max, const float* block_bias_min,
                         const int32_t* item_perm, int64_t n_users, int64_t n_items, int32_t d_pad, int32_t k,
                         int32_t n_splits, int32_t item_id_offset, float* cand_score, int32_t* cand_item,
                         float* row_theta, void* stream);
int trk_score_filter_f16_excl(const void* user_split, const float* user_scale, const float* user_bias,
                              const float* user_norm, const void* item_hi_global, const float* item_stats,
                              const float* item_bias_padded, const float* block_bias_max, const float* block_bias_min,
                              const int32_t* item_perm, int64_t n_users, int64_t n_items, int32_t d_pad, int32_t k,
                              int32_t n_splits, int32_t item_id_offset, float* cand_score, int32_t* cand_item,
                              float* row_theta, const int32_t* excl_indptr, const int32_t* excl_pos, void* stream);
/* item_split / item_scale / item_bias hold the rows of THIS shard: global id g lives at row g - item_id_offset.
 * n_lists = n_splits, list_width = 16.  Row u of the result is written at out_score + u * out_row_stride and
 * out_item + u * out_row_stride (both may point into one [n_users, 2k] exchange buffer: stride 2k, out_item =
 * out_score + k).  out_flag[u] = 1 -> user u must be re-run through the exact kernel. */
int trk_rescore_topk_split(const void* user_split, const float* user_scale, const void* item_split,
                           const float* item_scale, const float* user_bias, const float* item_bias,
                           const int32_t* cand_item, const float* row_theta, const float* user_norm,
                           const float* item_stats, int64_t n_users, int64_t n_items_local, int32_t d_pad,
                           int32_t n_lists, int32_t list_width, int32_t k, int32_t item_id_offset, float* out_score,
                           int32_t* out_item, int64_t out_row_stride, int32_t* out_flag, void* stream);

/* Device-side routing of the flagged users (no host round trip):
 *   trk_select_flagged_rows  idx[0 .. min(count, capacity)) = rows with flags != 0 (any order), counters[0] = count
 *                            (counters: int32[4], zeroed by this call; count > capacity = overflow, the host layer
 *                            checks it at its next natural synchronisation and re-runs the whole batch exactly);
 *   trk_gather_operand_rows  sub_split / sub_scale / sub_bias [capacity, ...] = the selected rows of a split operand;
 *                            also sets the live counts of the two re-scoring tiers: counters[2] = count when
 *                            count <= small_capacity (else 0), counters[3] = min(count, capacity) otherwise (else 0);
 *   trk_score_topk_f16x3 + trk_topk_merge with n_users_live = &counters[2] over the first small_capacity rows and MANY
 *                            item splits (a handful of user blocks still fills the machine), and with n_users_live =
 *                            &counters[3] over all capacity rows and few splits: exactly one tier does work;
 *   trk_scatter_topk_rows    out[idx[i]] = sub[i] for i < min(count, capacity) (row i of sub_* at i * sub_row_stride). */
int trk_select_flagged_rows(const int32_t* flags, int64_t n, int32_t* idx, int32_t capacity, int32_t* counters,
                            void* stream);
int trk_gather_operand_rows(const int32_t* idx, int32_t* counters, int32_t capacity, int32_t small_capacity,
                            const void* split, const float* scale, const float* bias, int32_t d_pad, void* sub_split,
                            float* sub_scale, float* sub_bias, void* stream);
int trk_scatter_topk_rows(const int32_t* idx, const int32_t* counters, int32_t capacity, const float* sub_score,
                          const int32_t* sub_item, int64_t sub_row_stride, int32_t k, float* out_score,
                          int32_t* out_item, int64_t out_row_stride, void* stream);

/* Similar items with Euclidean similarity (EuclideanSimilarityPredictionGraph, tensorrec/prediction_graphs.py:84-100;
 * similar-items scores carry no biases, recommendation_graphs.py:124-137) on the fused top-k kernels above.  With
 * user bias -1/2 |q|^2 and item bias -1/2 |i|^2 their score q.i + ub + ib is -1/2 d^2(q, i), which ranks the items as
 * the reference's -sqrt(max(d^2, 1e-16)) does; the error bound of the filter covers the biases as for any model.
 *   trk_operand_half_sqnorm    out[r] = -1/2 sum_j (scale[r] (hi + lo)_j)^2 of a split operand [rows, 2 d_pad]
 *                              (fp32, fixed reduction order: deterministic).
 *   trk_topk_euclidean_finish  in place on k <= 32 (score, id) entries per row (row r at scores / items +
 *                              r * row_stride, e.g. a [n_rows, 2k] exchange-layout buffer with items = scores + k):
 *                              s = -sqrt(max(-2 s, 1e-16)) (sentinels stay -inf), then each row is re-sorted by
 *                              (score desc, id asc): distances the sqrt or the clamp makes equal are ordered by id, as
 *                              tf.nn.top_k orders them. */
int trk_operand_half_sqnorm(const void* split, const float* scale, int64_t rows, int32_t d_pad, float* out,
                            void* stream);
int trk_topk_euclidean_finish(float* scores, int32_t* items, int64_t row_stride, int64_t n_rows, int32_t k,
                              void* stream);

/* Wide form of the filter top-k: 32 < k <= trk_score_wide_max_k() (1024), same inputs as trk_score_filter_f16 (the
 * hi item operand in processing order, packed biases, block maxima, perm, statistics) except block_bias_min: the wide
 * form has no warm start.  Every (user, split) keeps its candidates in a list in global memory of
 * trk_score_wide_list_capacity(k) entries; a warp compacts a full list by a radix select of the k-th best approximate
 * score, keeps everything within the error bound of it (at most half the capacity) and raises its threshold.
 *   trk_score_wide_f16        list_score / list_item [n_users, n_splits, capacity] (scratch while the kernel runs; on
 *                             return entries [0, list_count) hold (approximate score, global item id)), list_count
 *                             [n_users, n_splits], row_theta [n_users, n_splits] = max(theta, best dropped score).
 *   trk_score_wide_f16_excl   the same plus the exclusion lists as processing positions (see
 *                             trk_score_filter_f16_excl).
 *   trk_select_wide_topk      per row: the candidate ids cand_item[row * cand_row_stride + l * list_width + e] for
 *                             the n_lists lists l and e < list_count[row * n_lists + l] (list_count NULL: every entry;
 *                             ids outside [item_id_offset, item_id_offset + n_items_local) and INT32_MAX are not
 *                             candidates) are re-scored with the arithmetic of trk_rescore_topk_split, sorted by
 *                             (score desc, id asc) and the first k written to out_score / out_item (row stride
 *                             out_row_stride; sentinels (-inf, INT32_MAX)).  out_flag (may be NULL: no certificate)
 *                             receives 1 for rows the certificate of trk_rescore_topk_split rejects (row_theta
 *                             [n_rows, n_lists], user_norm, item_stats are then required).  euclidean != 0: the
 *                             scores (-1/2 d^2) are mapped to -sqrt(max(d^2, 1e-16)) after the certificate and the
 *                             row is sorted again.  n_lists * list_width <= 16384. */
int trk_score_wide_max_k(void);
int trk_score_wide_list_capacity(int32_t k);
int trk_score_wide_f16(const void* user_split, const float* user_scale, const float* user_bias,
                       const float* user_norm, const void* item_hi_global, const float* item_stats,
                       const float* item_bias_padded, const float* block_bias_max, const int32_t* item_perm,
                       int64_t n_users, int64_t n_items, int32_t d_pad, int32_t k, int32_t n_splits,
                       int32_t item_id_offset, float* list_score, int32_t* list_item, int32_t* list_count,
                       float* row_theta, void* stream);
int trk_score_wide_f16_excl(const void* user_split, const float* user_scale, const float* user_bias,
                            const float* user_norm, const void* item_hi_global, const float* item_stats,
                            const float* item_bias_padded, const float* block_bias_max, const int32_t* item_perm,
                            int64_t n_users, int64_t n_items, int32_t d_pad, int32_t k, int32_t n_splits,
                            int32_t item_id_offset, float* list_score, int32_t* list_item, int32_t* list_count,
                            float* row_theta, const int32_t* excl_indptr, const int32_t* excl_pos, void* stream);
int trk_select_wide_topk(const void* user_split, const float* user_scale, const void* item_split,
                         const float* item_scale, const float* user_bias, const float* item_bias,
                         const int32_t* cand_item, int64_t cand_row_stride, int32_t n_lists, int32_t list_width,
                         const int32_t* list_count, const float* row_theta, const float* user_norm,
                         const float* item_stats, int64_t n_rows, int64_t n_items_local, int32_t d_pad, int32_t k,
                         int32_t item_id_offset, int32_t euclidean, float* out_score, int32_t* out_item,
                         int64_t out_row_stride, int32_t* out_flag, void* stream);

/* Tensor-core dense prediction with the same operands, writing the full fp32 matrix out[n_users, n_items]
 * (predict(); tensorrec/tensorrec.py:636-664).  HBM-write bound. */
int trk_score_dense_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                          const void* item_split, const float* item_meta, int64_t n_users, int64_t n_items,
                          int32_t d_pad, float* out, int64_t out_row_stride, void* stream);

/* Euclidean user x item models (EuclideanSimilarityPredictionGraph, tensorrec/prediction_graphs.py:84-100, then
 * bias_prediction_dense, recommendation_graphs.py:41) on the same tensor-core kernels: the epilogue turns each
 * accumulator into the final score
 *   p = acc * scale_u * scale_i,  d2 = (|u|^2 - 2 p) + |i|^2,  s = -sqrt(max(d2, 1e-16)) + user_bias[u] + item_bias[i]
 * (left to right, correctly rounded sqrt; exact for integer-valued representations), then compares / stores it as the
 * dot forms do.  The squared norms come from the split operands, as -1/2 |row|^2 written by trk_operand_half_sqnorm:
 *   user_half_sqnorm [n_users];
 *   item_half_sqnorm [n_items_padded256] (16-byte aligned), entries beyond n_items = 0 (any finite value).
 *   trk_score_dense_euclid_f16x3  the arguments of trk_score_dense_f16x3 plus the two norm arrays.
 *   trk_score_topk_euclid_f16x3   the arguments of trk_score_topk_f16x3_excl plus the two norm arrays; excl_indptr /
 *                                 excl_ids / excl_row_map may all be NULL (no exclusion).
 * Constraints: d_pad in {64, 128}; top-k: 1 <= k <= trk_score_topk_max_k(d_pad).  The top-k of a mixture of tastes is
 * one call per taste and trk_topk_merge with dedup, as for the dot form: every step after the sqrt is monotone. */
int trk_score_dense_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                 const void* item_split, const float* item_meta, int64_t n_users, int64_t n_items,
                                 int32_t d_pad, float* out, int64_t out_row_stride, const float* user_half_sqnorm,
                                 const float* item_half_sqnorm, void* stream);
int trk_score_topk_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                const void* item_split, const float* item_meta, int64_t n_users, int64_t n_items,
                                int32_t d_pad, int32_t k, int32_t n_splits, int32_t item_id_offset,
                                float* cand_score, int32_t* cand_item, const int32_t* n_users_live,
                                const int32_t* excl_indptr, const int32_t* excl_ids, const int32_t* excl_row_map,
                                const float* user_half_sqnorm, const float* item_half_sqnorm, void* stream);

/* Mixtures of tastes, with or without attention (collapse_mixture_of_tastes, tensorrec/recommendation_graphs.py:85-109,
 * then bias_prediction_dense, :41), dot / cosine prediction (cosine: operands pre-normalised by K1), on the same
 * tensor-core kernels.  Every user has n_ops operand rows: u_0 .. u_{T-1} and, with attention != 0, a_0 .. a_{T-1}
 * (n_ops = T or 2T), stacked as user_split [n_ops, n_users, 2 d_pad] (16-byte aligned) with user_scale
 * [n_ops, n_users]; every dot product is the 3-pass split product.  Per (user, item), left to right, each product and
 * sum rounded on its own:
 *   p_t = u_t . i;   no attention:  pred = max_t p_t;
 *   attention:  a_t = a_t . i,  m = max_t a_t,  e_t = expf(a_t - m),  s = sum_t e_t (taste order),
 *               pred = sum_t p_t * (e_t / s) (taste order);
 *   out = (pred + user_bias[u]) + item_bias[i]
 * (exact for integer-valued representations without attention, and with attention when every pair's weights are
 * one-hot).  user_bias [n_users] may be NULL; item_meta as for trk_score_dense_f16x3.
 *   trk_score_dense_tastes_f16x3  out[n_users, n_items] (row stride out_row_stride).
 *   trk_score_topk_tastes_f16x3   cand_score / cand_item [n_users, n_splits, k] as trk_score_topk_f16x3_excl;
 *                                 excl_indptr / excl_ids / excl_row_map may all be NULL (no exclusion).
 * Constraints: d_pad in {64, 128}; n_tastes >= 1 and 2 <= n_ops <= 64 (T <= 64 without attention, T <= 32 with it;
 * larger n_ops returns TRK_ERR_UNSUPPORTED); top-k: 1 <= k <= trk_score_topk_max_k(d_pad).  A user block holds
 * 2 * floor(64 / n_ops) users. */
int trk_score_dense_tastes_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                 int32_t n_tastes, int32_t attention, const void* item_split, const float* item_meta,
                                 int64_t n_users, int64_t n_items, int32_t d_pad, float* out, int64_t out_row_stride,
                                 void* stream);
int trk_score_topk_tastes_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                int32_t n_tastes, int32_t attention, const void* item_split, const float* item_meta,
                                int64_t n_users, int64_t n_items, int32_t d_pad, int32_t k, int32_t n_splits,
                                int32_t item_id_offset, float* cand_score, int32_t* cand_item,
                                const int32_t* excl_indptr, const int32_t* excl_ids, const int32_t* excl_row_map,
                                void* stream);

/* Mixtures of tastes with Euclidean prediction (EuclideanSimilarityPredictionGraph, tensorrec/prediction_graphs.py:84-100,
 * then collapse_mixture_of_tastes and bias_prediction_dense): every operand row x_j -- taste rows and attention rows
 * alike -- gives e_j = -sqrtf(max((|x_j|^2 - 2 p_j) + |i|^2, 1e-16)), p_j its 3-pass dot product with i, and the e_j
 * are collapsed as above (max over the tastes, or the softmax of the attention e_j weighting the taste e_j).  The
 * arguments of the _tastes_ twins plus the norms: user_half_sqnorm [n_ops, n_users] = -1/2 |x_j|^2 of every operand
 * row (trk_operand_half_sqnorm of each slice of the stacked operand) and item_half_sqnorm as for
 * trk_score_dense_euclid_f16x3 (16-byte aligned, padded to whole item tiles); NULL norms return TRK_ERR_ARG.
 *   trk_score_dense_tastes_euclid_f16x3       as trk_score_dense_tastes_f16x3.
 *   trk_score_topk_tastes_euclid_f16x3        as trk_score_topk_tastes_f16x3; attention != 0 (a Euclidean mixture of
 *                                             tastes without attention returns TRK_ERR_UNSUPPORTED: its top k is the
 *                                             merge of one trk_score_topk_euclid_f16x3 sweep per taste).
 *   trk_score_topk_wide_tastes_euclid_f16x3   as trk_score_topk_wide_tastes_f16x3; attention != 0 likewise
 *                                             (trk_score_topk_wide_euclid_f16x3 per taste).
 *   trk_score_count_tastes_euclid_f16x3       as trk_score_count_tastes_f16x3, attention or not. */
int trk_score_dense_tastes_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                        int32_t n_tastes, int32_t attention, const void* item_split,
                                        const float* item_meta, int64_t n_users, int64_t n_items, int32_t d_pad,
                                        float* out, int64_t out_row_stride, const float* user_half_sqnorm,
                                        const float* item_half_sqnorm, void* stream);
int trk_score_topk_tastes_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                       int32_t n_tastes, int32_t attention, const void* item_split,
                                       const float* item_meta, int64_t n_users, int64_t n_items, int32_t d_pad, int32_t k,
                                       int32_t n_splits, int32_t item_id_offset, float* cand_score, int32_t* cand_item,
                                       const int32_t* excl_indptr, const int32_t* excl_ids,
                                       const int32_t* excl_row_map, const float* user_half_sqnorm,
                                       const float* item_half_sqnorm, void* stream);
int trk_score_topk_wide_tastes_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                            int32_t n_tastes, int32_t attention, const void* item_split,
                                            const float* item_meta, int64_t n_users, int64_t n_items, int32_t d_pad,
                                            int32_t k, int32_t n_splits, int32_t item_id_offset, float* list_score,
                                            int32_t* list_item, int32_t* list_count, const int32_t* excl_indptr,
                                            const int32_t* excl_ids, const int32_t* excl_row_map,
                                            const float* user_half_sqnorm, const float* item_half_sqnorm,
                                            void* stream);
int trk_score_count_tastes_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                        int32_t n_tastes, int32_t attention, const void* item_split,
                                        const float* item_meta, int64_t n_users, int64_t n_items, int32_t d_pad,
                                        int32_t n_splits, int32_t item_id_offset, const int32_t* pair_indptr,
                                        const int32_t* pair_ids, float* pair_score, int32_t* pair_count,
                                        const int32_t* block_pairs, int32_t pass, const int32_t* excl_indptr,
                                        const int32_t* excl_ids, const int32_t* excl_row_map,
                                        const float* user_half_sqnorm, const float* item_half_sqnorm, void* stream);

/* Wide top-k of the Euclidean and attention forms on the exact kernel: 1 <= k <= 1024, every score final and exact
 * (the same epilogue as trk_score_topk_euclid_f16x3 / trk_score_topk_tastes_f16x3), so no certificate, re-scoring or
 * fallback.  Every (user, item split, column half) keeps a list in global memory of
 * trk_score_topk_wide_list_capacity(k) entries (0 for k outside [1, 1024]); a warp compacts a full list to exactly its
 * top k by (score desc, id asc).
 *   trk_score_topk_wide_euclid_f16x3  the arguments of trk_score_topk_euclid_f16x3 with cand_score / cand_item
 *                                     replaced by list_score / list_item [n_users, n_splits, 2, capacity] (scratch
 *                                     while the kernel runs; on return entries [0, list_count) hold (final score,
 *                                     global item id), unsorted) and list_count [n_users, n_splits, 2] (<= k).
 *   trk_score_topk_wide_tastes_f16x3  the same for trk_score_topk_tastes_f16x3; attention != 0 (a mixture of tastes
 *                                     without attention returns TRK_ERR_UNSUPPORTED: the wide filter serves it).
 *                                     Only the users own lists: [n_users, n_splits, 2, capacity].
 *   trk_select_topk_lists             per row: the n_lists lists of list_width entries (list l of row r at
 *                                     (r * n_lists + l) * list_width, list_count[r * n_lists + l] <= k entries) sorted
 *                                     by (score desc, id asc); the first k go to out_score / out_item (row stride
 *                                     out_row_stride), sentinels (-inf, INT32_MAX) where there are fewer.  For the
 *                                     lists above, n_lists = 2 n_splits and list_width = the capacity.
 *                                     n_lists * k <= 16384. */
int trk_score_topk_wide_list_capacity(int32_t k);
int trk_score_topk_wide_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                     const void* item_split, const float* item_meta, int64_t n_users, int64_t n_items,
                                     int32_t d_pad, int32_t k, int32_t n_splits, int32_t item_id_offset,
                                     float* list_score, int32_t* list_item, int32_t* list_count,
                                     const int32_t* n_users_live, const int32_t* excl_indptr, const int32_t* excl_ids,
                                     const int32_t* excl_row_map, const float* user_half_sqnorm,
                                     const float* item_half_sqnorm, void* stream);
int trk_score_topk_wide_tastes_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                     int32_t n_tastes, int32_t attention, const void* item_split,
                                     const float* item_meta, int64_t n_users, int64_t n_items, int32_t d_pad, int32_t k,
                                     int32_t n_splits, int32_t item_id_offset, float* list_score, int32_t* list_item,
                                     int32_t* list_count, const int32_t* excl_indptr, const int32_t* excl_ids,
                                     const int32_t* excl_row_map, void* stream);
int trk_select_topk_lists(const float* list_score, const int32_t* list_item, const int32_t* list_count,
                          int64_t n_rows, int32_t n_lists, int32_t list_width, int32_t k, float* out_score,
                          int32_t* out_item, int64_t out_row_stride, void* stream);

/* Counting mode of the exact kernel: the full rank of listed (user, item) pairs without the score matrix.  Every
 * score is the one trk_score_dense_{f16x3, euclid_f16x3, tastes_f16x3} writes for the same users at the same rows
 * (user row u of the call at accumulator row u mod 128, or u mod 2 floor(64 / n_ops) for a mixture of tastes): a
 * caller that splits its users into several calls cuts them at multiples of that block for the ranks to equal the
 * ranks of the dense scores bit for bit.  A column (s, id) outranks a pair (t, tid) when s > t, or s == t and
 * id < tid (ids global: local id + item_id_offset); -0.0 == +0.0.  Pairs of user row u: [pair_indptr[u],
 * pair_indptr[u + 1]) of pair_ids / pair_score / pair_count; block_pairs [ceil(n_users / block)] = the most pairs of a
 * row of each user block (the block above).
 *   pass = -1  capture: pair_ids = LOCAL item ids, ascending per row; pair_score[pair] = the pair's score (never
 *              masked by the exclusion lists).  pair_count is not read (may be NULL).
 *   pass >= 0  count: every row's pairs sorted by (score desc, id asc) -- pair_ids (LOCAL) and pair_score (from the
 *              capture) in that order; pass p adds to pair_count[pair] (int32, zeroed by the caller before pass 0)
 *              the number of columns outranking pair 32 p + j of its row, j < 32.  Columns listed in the row's
 *              exclusion list (excl_indptr / excl_ids / excl_row_map as for trk_score_topk_f16x3_excl, or all NULL)
 *              count as -inf; a pair never counts itself.  A row with n pairs needs passes 0 .. ceil(n / 32) - 1, and
 *              user blocks whose block_pairs <= 32 p are skipped.
 * After every pass: rank of a pair = 1 + pair_count (the rank among the row's non-excluded items plus the pair).  The
 * counts add up over item splits and over item shards (integer adds: deterministic).
 *   trk_score_count_f16x3         operands as trk_score_topk_f16x3 (dot / cosine).
 *   trk_score_count_euclid_f16x3  plus the two norm arrays of trk_score_topk_euclid_f16x3 (Euclidean similarity).
 *   trk_score_count_tastes_f16x3  operands as trk_score_topk_tastes_f16x3 (mixtures of tastes, attention or not).
 * Constraints: d_pad in {64, 128}; n_splits >= 1; pass >= -1. */
int trk_score_count_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                          const void* item_split, const float* item_meta, int64_t n_users, int64_t n_items,
                          int32_t d_pad, int32_t n_splits, int32_t item_id_offset, const int32_t* pair_indptr,
                          const int32_t* pair_ids, float* pair_score, int32_t* pair_count,
                          const int32_t* block_pairs, int32_t pass, const int32_t* excl_indptr,
                          const int32_t* excl_ids, const int32_t* excl_row_map, void* stream);
int trk_score_count_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                 const void* item_split, const float* item_meta, int64_t n_users, int64_t n_items,
                                 int32_t d_pad, int32_t n_splits, int32_t item_id_offset, const int32_t* pair_indptr,
                                 const int32_t* pair_ids, float* pair_score, int32_t* pair_count,
                                 const int32_t* block_pairs, int32_t pass, const int32_t* excl_indptr,
                                 const int32_t* excl_ids, const int32_t* excl_row_map, const float* user_half_sqnorm,
                                 const float* item_half_sqnorm, void* stream);
int trk_score_count_tastes_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                 int32_t n_tastes, int32_t attention, const void* item_split, const float* item_meta,
                                 int64_t n_users, int64_t n_items, int32_t d_pad, int32_t n_splits,
                                 int32_t item_id_offset, const int32_t* pair_indptr, const int32_t* pair_ids,
                                 float* pair_score, int32_t* pair_count, const int32_t* block_pairs, int32_t pass,
                                 const int32_t* excl_indptr, const int32_t* excl_ids, const int32_t* excl_row_map,
                                 void* stream);

/* Pairs mode of the exact kernel: the scores of listed (user, item) pairs, each bit for bit the score
 * trk_score_dense_{f16x3, euclid_f16x3, tastes_f16x3, tastes_euclid_f16x3} writes for the same users at the same rows
 * (user row u of the call at accumulator row u mod 128, or u mod 2 floor(64 / n_ops) for a mixture of tastes), from
 * item tiles gathered out of each user block's listed items (DESIGN.md §3.13):
 *   tile_items [n_tiles, 128]  the item of every slot of every gathered tile; item i sits at column i mod 128 (its
 *                              column in the dense sweep), -1 marks an empty slot;
 *   work [n_work, 3]           (user block, first tile, end tile) of every work item: the block's rows are multiplied
 *                              against the gathered tiles [first, end);
 *   pair_indptr [n_users + 1], pair_cols  the pairs of user row u as VIRTUAL columns tile * 128 + column, ascending per
 *                              row, every one inside a tile of a work item of u's block;
 *   slot_meta [n_tiles * 128, 2]  {scale, bias} of every slot (trk_pack_item_meta's entries gathered by tile_items);
 *   pair_score[pair]           the pair's score.
 *   trk_score_pairs_f16x3                operands as trk_score_count_f16x3 (dot / cosine).
 *   trk_score_pairs_euclid_f16x3         plus user_half_sqnorm and slot_half_sqnorm [n_tiles * 128], the item norms
 *                                        gathered as slot_meta (Euclidean similarity).
 *   trk_score_pairs_tastes_f16x3         operands as trk_score_count_tastes_f16x3 (mixtures of tastes).
 *   trk_score_pairs_tastes_euclid_f16x3  as trk_score_pairs_tastes_f16x3 plus the operand norms [n_ops, n_users] and
 *                                        slot_half_sqnorm (Euclidean mixtures of tastes, attention or not).
 * Constraints: d_pad in {64, 128}; 1 <= n_tiles <= 2^24; n_work >= 1; slot_meta and slot_half_sqnorm 16-byte aligned. */
int trk_score_pairs_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                          const void* item_split, const float* slot_meta, int64_t n_users, int64_t n_items,
                          int32_t d_pad, const int32_t* pair_indptr, const int32_t* pair_cols, float* pair_score,
                          const int32_t* tile_items, int32_t n_tiles, const int32_t* work, int32_t n_work,
                          void* stream);
int trk_score_pairs_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                 const void* item_split, const float* slot_meta, int64_t n_users, int64_t n_items,
                                 int32_t d_pad, const int32_t* pair_indptr, const int32_t* pair_cols,
                                 float* pair_score, const int32_t* tile_items, int32_t n_tiles, const int32_t* work,
                                 int32_t n_work, const float* user_half_sqnorm, const float* slot_half_sqnorm,
                                 void* stream);
int trk_score_pairs_tastes_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                 int32_t n_tastes, int32_t attention, const void* item_split, const float* slot_meta,
                                 int64_t n_users, int64_t n_items, int32_t d_pad, const int32_t* pair_indptr,
                                 const int32_t* pair_cols, float* pair_score, const int32_t* tile_items,
                                 int32_t n_tiles, const int32_t* work, int32_t n_work, void* stream);
int trk_score_pairs_tastes_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                        int32_t n_tastes, int32_t attention, const void* item_split,
                                        const float* slot_meta, int64_t n_users, int64_t n_items, int32_t d_pad,
                                        const int32_t* pair_indptr, const int32_t* pair_cols, float* pair_score,
                                        const int32_t* tile_items, int32_t n_tiles, const int32_t* work,
                                        int32_t n_work, const float* user_half_sqnorm, const float* slot_half_sqnorm,
                                        void* stream);

/* Merges n_lists candidate lists per user (each sorted by (score desc, id asc), k_in entries) into the global
 * top k_out per user, same order.  Lists are the n_splits of one GPU and/or the shards received from the other GPUs
 * (item-axis sharding; the exchange itself is one NCCL all-to-all done by the host layer, SURVEY 8e).
 * Entry j of list l of user u is read at cand_*[u * user_stride + l * list_stride + j]:
 *   one GPU, [n_users, n_lists, k_in]:                user_stride = n_lists * k_in, list_stride = k_in;
 *   exchange receive buffer [n_lists, n_users, 2k]:   user_stride = 2k, list_stride = n_users * 2k, cand_item = cand_score + k.
 * Row u of the result goes to out_*[u * out_row_stride ...].  n_users_live: see trk_score_topk_f16x3.
 * dedup != 0: the lists of a user may name the same item -- the per-TASTE top-k lists of a mixture-of-tastes model,
 * whose prediction is the maximum over the tastes (collapse_mixture_of_tastes, tensorrec/recommendation_graphs.py:107):
 * every item is emitted once, with its best score (k_out <= 32).  The top-k of max_t s_t(u, .) is contained in the union
 * of the per-taste top-k lists, so n_tastes fused top-k sweeps + this merge give the model's top-k without the
 * [n_users, n_items] matrix. */
int trk_topk_merge(const float* cand_score, const int32_t* cand_item, int64_t n_users, int32_t n_lists,
                   int32_t k_in, int32_t k_out, int64_t user_stride, int64_t list_stride, float* out_score,
                   int32_t* out_item, int64_t out_row_stride, const int32_t* n_users_live, int32_t dedup, void* stream);

/* De-duplicating merge of TWO lists per row for any 1 <= k <= 1024 (trk_score_wide_max_k): the top-k of a mixture of
 * tastes on the wide route folds the per-taste lists one at a time, R_t = R_{t-1} (+) L_t (DESIGN §3.6).  Entry j of
 * row u of list A is (a_score, a_item)[u * a_row_stride + j], of B and of the result likewise with their own strides
 * (a PackedTopK [n_rows, 2k] buffer: *_score = the row base, *_item = *_score + k, stride 2k).  Both lists are sorted
 * by (score desc, id asc) with real ids unique within a list, padded with sentinels (-inf, INT32_MAX); a row may be
 * all sentinels.  Row u of the result = the k best entries of A_u united with B_u, every real id once at the higher of
 * its scores (an id with equal scores in both lists keeps one copy), in the same order, padded with sentinels.
 * Sentinels are never entries.  The output must not overlap A or B.  Deterministic. */
int trk_topk_merge_dedup_pair(const float* a_score, const int32_t* a_item, int64_t a_row_stride, const float* b_score,
                              const int32_t* b_item, int64_t b_row_stride, int64_t n_rows, int32_t k, float* out_score,
                              int32_t* out_item, int64_t out_row_stride, void* stream);

/* ------------------------------------------------------------------------------------------------------
 * The sampled-rank training step (SURVEY 8 row f1): everything of one Adam step of
 * LinearRepresentationGraph x DotProductPredictionGraph x WMRBLossGraph / BalancedWMRBLossGraph that is not a
 * sparse x dense product (those are trk_csr_gather_reduce_f32 on the CSR of the features and of their transpose).
 *
 * trk_sample_items   replaces sample_items behind tf.py_func (tensorrec/util.py:12-21, tensorrec/tensorrec.py:298-302):
 *                    out[u, j] (int32 [n_users, n_sampled]) = item ids drawn for user u, with replacement (uniform) or
 *                    without (Floyd's algorithm: a uniformly random n_sampled-subset; n_sampled <= 4096), from the
 *                    counter-based Philox4x32-10 stream (seed, step, user, draw).  trk_sample_stream_u64 exposes that
 *                    stream on the host (tests reproduce a device sample from it).
 * trk_wmrb_step      forward and backward between the representations and the loss, one warp per user:
 *                      pred(u, i) = (sum_k user_repr[u, k] * item_repr[i, k] + user_bias[u]) + item_bias[i]
 *                                   (tensorrec/prediction_graphs.py:52-55, recommendation_graphs.py:44-57)
 *                      for every stored interaction n = (u, i, val) (CSR by user, reference COO order) with val > 0:
 *                        loss[n] = log(n_items / n_sampled * sum_j max(0, 1 - pred(u, i) + pred(u, samples[u, j]))
 *                                      [* val / item_weight_sum[i]]  + 1)     (tensorrec/loss_graphs.py:153-180, 190-227)
 *                      loss[n] = 0 for val <= 0; pred_serial[n] = pred(u, i) for every n;
 *                      gradients of sum_n loss[n]: d_user_repr [n_users, d] and d_user_bias [n_users] are written,
 *                      d_item_repr [n_items, d] and d_item_bias [n_items] are ADDED to with red.global.add (zero them
 *                      first; the order of the floating-point additions is not fixed, as in tf.gather's GPU gradient).
 *                    Representations are fp32 or bf16 (repr_is_bf16; BASELINE config #4 allows bf16), arithmetic and
 *                    gradients fp32.  coef [nnz] is scratch.  Constraints: d % 4 == 0, d <= 512, n_sampled <= 2048.
 *                    It is the one-taste dot shorthand of trk_wmrb_step_tastes (n_tastes = 1, attention = 0,
 *                    euclidean = 0), and checks its arguments as that does.
 * trk_wmrb_step_tastes
 *                    the general WMRB step, every form the fused path trains (DESIGN §3.10): n_tastes taste rows per user,
 *                    with n_tastes attention rows after them when attention = 1, stacked as planes [n_rows, n_users, d]
 *                    in user_rows (and d_user_rows, written); euclidean = 1 scores a pair -sqrt(max(|u - i|^2, 1e-16)),
 *                    0 scores it u . i (cosine: the caller passes L2-normalised rows).  The prediction collapses the
 *                    tastes' scores with max (ties split the gradient evenly, as tf.reduce_max) or, with attention, with
 *                    sum_t softmax_t(a_t) score_t, a_t = score of attention row t for an interaction and of taste row t
 *                    itself for a sampled item (tensorrec/tensorrec.py:367-372); then biases and loss as trk_wmrb_step.
 *                    d_item_repr receives one red.global.add per pair, summed over the operand rows.  Constraints:
 *                    d % 4 == 0 (pad with zero columns), d <= 512 for one taste and <= 128 for several, n_tastes <= 8
 *                    (<= 4 and >= 2 with attention), n_sampled <= 2048; others return TRK_ERR_UNSUPPORTED.
 * trk_serial_loss_step
 *                    the training step of the serial losses (DESIGN §3.11): loss_kind 0 is RMSELossGraph,
 *                    L = sqrt(mean_n (y_n - p_n)^2) (tensorrec/loss_graphs.py:53-59), 1 is SeparationLossGraph,
 *                    L = 1 - Phi(-(mu_Q - mu_P) / sqrt(v_Q + v_P)) over the predictions of P = {y > 0} and
 *                    Q = {y <= 0} (mean and biased variance, loss_graphs.py:75-98), over all nnz stored interactions
 *                    (explicit zeros and duplicates included).  Operands, forms and constraints as trk_wmrb_step_tastes,
 *                    without samples.  Three launches on `stream`: pred_serial [nnz] (as trk_wmrb_step_tastes computes
 *                    it); the statistics, which write the scalar loss [1] and a loss state into `workspace`
 *                    (trk_serial_loss_workspace_bytes(nnz) bytes, 8-byte aligned); then the gradients of L: d_user_rows
 *                    and d_user_bias written, d_item_repr and d_item_bias ADDED to (zero them first).  nnz == 0
 *                    launches no kernel: loss = NaN, d_user_rows = d_user_bias = 0, and pred_serial, inter_item,
 *                    inter_val and workspace may be null.  An empty group or L = 0 gives NaN, as the losses' own
 *                    gradients do.  nnz < 2^31.
 * trk_l2_normalize_rows_step_f32
 *                    row L2-normalisation N(x) = x rsqrt(max(|x|^2, 1e-12)), n_normalize (1 or 2) times, of raw rows
 *                    x [rows, d <= 512]: out (if non-null) receives N^n(x); grad (if non-null) holds d loss / d N^n(x) and
 *                    is replaced by d loss / d x (the Jacobian of each normalisation, tf.maximum's gradient rule).
 * trk_f32_to_bf16    round-to-nearest-even conversion of a representation for the bf16 form.
 * trk_adam_step_f32  tf.train.AdamOptimizer on (grad + l2 * w) (tensorrec/tensorrec.py:487-489):
 *                      m = b1 m + (1 - b1) g;  v = b2 v + (1 - b2) g^2;  w -= lr_t m / (sqrt(v) + epsilon),
 *                    lr_t = lr sqrt(1 - b2^t) / (1 - b1^t) formed by the caller.
 * trk_relu_layer_forward_f32
 *                    the hidden layer of ReLURepresentationGraph (DESIGN §3.14): out [rows, d] = relu(pre + bias) . w2 for
 *                    pre [rows, hidden] (the K1 product X . W1), bias [hidden], w2 [hidden, d], as 3xTF32 products on
 *                    the tensor cores (fp32-grade).  hidden % 8 == 0 and <= 2048, d % 4 == 0 and <= 512 (pad hidden with
 *                    zero W1 columns, bias and w2 rows, d with zero w2 columns); pre, bias, w2 and out 16-byte aligned.
 * trk_relu_layer_backward_f32
 *                    its gradients for d_out = d loss / d out [rows, d]: pre is REPLACED by d loss / d pre =
 *                    (d_out . w2^T) * [pre + bias > 0] (an exact 0 passes no gradient, tf.nn.relu's rule); d_bias
 *                    [hidden] and d_w2 [hidden, d] are written.  Deterministic: per-CTA partials in `workspace`
 *                    (trk_relu_layer_workspace_bytes(rows, hidden, d) bytes, 16-byte aligned), summed in a fixed order;
 *                    no atomics.  Constraints as the forward; d_out 16-byte aligned.
 * ---------------------------------------------------------------------------------------------------- */
int trk_sample_items(int64_t n_users, int64_t n_items, int32_t n_sampled, int32_t replace, uint64_t seed,
                     uint32_t step, int32_t* out, void* stream);
uint64_t trk_sample_stream_u64(uint64_t seed, uint32_t step, uint32_t user, uint32_t draw);
int trk_wmrb_step(const void* user_repr, const void* item_repr, int32_t repr_is_bf16, const float* user_bias,
                  const float* item_bias, const int32_t* inter_indptr, const int32_t* inter_item,
                  const float* inter_val, const float* item_weight_sum, const int32_t* samples, int64_t n_users,
                  int64_t n_items, int32_t d, int32_t n_sampled, float* loss, float* pred_serial, float* coef,
                  float* d_user_repr, float* d_user_bias, float* d_item_repr, float* d_item_bias, void* stream);
int trk_wmrb_step_tastes(const void* user_rows, const void* item_repr, int32_t repr_is_bf16, int32_t n_tastes,
                         int32_t attention, int32_t euclidean, const float* user_bias, const float* item_bias,
                         const int32_t* inter_indptr, const int32_t* inter_item, const float* inter_val,
                         const float* item_weight_sum, const int32_t* samples, int64_t n_users, int64_t n_items,
                         int32_t d, int32_t n_sampled, float* loss, float* pred_serial, float* coef, float* d_user_rows,
                         float* d_user_bias, float* d_item_repr, float* d_item_bias, void* stream);
size_t trk_serial_loss_workspace_bytes(int64_t nnz);
int trk_serial_loss_step(int32_t loss_kind, const void* user_rows, const void* item_repr, int32_t repr_is_bf16,
                         int32_t n_tastes, int32_t attention, int32_t euclidean, const float* user_bias,
                         const float* item_bias, const int32_t* inter_indptr, const int32_t* inter_item,
                         const float* inter_val, int64_t n_users, int64_t n_items, int32_t d, int64_t nnz, float* loss,
                         float* pred_serial, float* d_user_rows, float* d_user_bias, float* d_item_repr,
                         float* d_item_bias, void* workspace, size_t workspace_bytes, void* stream);
int trk_l2_normalize_rows_step_f32(const float* x, int64_t rows, int32_t d, int32_t n_normalize, float* out,
                                   float* grad, void* stream);
int trk_f32_to_bf16(const float* x, int64_t n, void* out, void* stream);
int trk_adam_step_f32(float* w, const float* grad, float* m, float* v, int64_t n, float lr_t, float beta1, float beta2,
                      float epsilon, float l2, void* stream);
size_t trk_relu_layer_workspace_bytes(int64_t rows, int32_t hidden, int32_t d);
int trk_relu_layer_forward_f32(const float* pre, const float* bias, const float* w2, int64_t rows, int32_t hidden,
                               int32_t d, float* out, void* stream);
int trk_relu_layer_backward_f32(float* pre, const float* bias, const float* w2, const float* d_out, int64_t rows,
                                int32_t hidden, int32_t d, float* d_bias, float* d_w2, void* workspace,
                                size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TENSORREC_B200_H_ */
