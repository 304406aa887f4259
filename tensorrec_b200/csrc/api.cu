// extern "C" entry points declared in include/tensorrec_b200.h (plain pointers and sizes, no torch types).
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace trk {

static thread_local char g_last_error[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
}

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return kSMsH100;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = kSMsH100;
    cached[dev] = n;
  }
  return cached[dev];
}

int capped_grid(int64_t blocks, int per_sm) {
  const int64_t cap = static_cast<int64_t>(sm_count()) * per_sm;
  return static_cast<int>(blocks < 1 ? 1 : (blocks < cap ? blocks : cap));
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn encode = nullptr;   // the library links no driver: the entry point is looked up at run time
  if (encode == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      encode = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  if (encode == nullptr) set_error("cuTensorMapEncodeTiled is not available from the CUDA driver");
  return encode;
}

int encode_tiled_3d(CUtensorMap* map, CUtensorMapDataType type, const void* base, uint64_t cols, uint64_t rows,
                    uint64_t planes, uint64_t row_bytes, uint64_t plane_bytes, uint32_t box_cols, uint32_t box_rows,
                    uint32_t box_planes, CUtensorMapL2promotion l2_promotion) {
  const EncodeTiledFn encode = encode_tiled_fn();
  if (encode == nullptr) return TRK_ERR_CUDA;
  const cuuint64_t dims[3] = {cols, rows, planes};
  const cuuint64_t strides[2] = {row_bytes, plane_bytes};
  const cuuint32_t box[3] = {box_cols, box_rows, box_planes};
  const cuuint32_t elem_strides[3] = {1, 1, 1};
  const CUresult r = encode(map, type, 3, const_cast<void*>(base), dims, strides, box, elem_strides,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, l2_promotion,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (planes=%llu rows=%llu cols=%llu)", static_cast<int>(r),
              static_cast<unsigned long long>(planes), static_cast<unsigned long long>(rows),
              static_cast<unsigned long long>(cols));
    return TRK_ERR_CUDA;
  }
  return TRK_OK;
}

int encode_tiled_2d(CUtensorMap* map, CUtensorMapDataType type, const void* base, uint64_t cols, uint64_t rows,
                    uint64_t row_bytes, uint32_t box_cols, uint32_t box_rows, CUtensorMapL2promotion l2_promotion) {
  const EncodeTiledFn encode = encode_tiled_fn();
  if (encode == nullptr) return TRK_ERR_CUDA;
  const cuuint64_t dims[2] = {cols, rows};
  const cuuint64_t strides[1] = {row_bytes};
  const cuuint32_t box[2] = {box_cols, box_rows};
  const cuuint32_t elem_strides[2] = {1, 1};
  const CUresult r = encode(map, type, 2, const_cast<void*>(base), dims, strides, box, elem_strides,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, l2_promotion,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (rows=%llu cols=%llu)", static_cast<int>(r),
              static_cast<unsigned long long>(rows), static_cast<unsigned long long>(cols));
    return TRK_ERR_CUDA;
  }
  return TRK_OK;
}

// implemented in the kernel translation units
int csr_gather_reduce(const int32_t*, const int32_t*, const float*, const float*, int64_t, int32_t, int32_t, int32_t,
                      float*, void*, int32_t, float*, float*, float*, cudaStream_t);
int split_rows(const float*, int64_t, int32_t, int32_t, float*, void*, int32_t, float*, cudaStream_t);
int csr_project_biases(const int32_t*, const int32_t*, const float*, const float*, int64_t, float*, cudaStream_t);
int pack_item_meta(const float*, const float*, int64_t, float*, int64_t, cudaStream_t);
int score_f32(const float*, const float*, const float*, const float*, const float*, float*, int64_t, int64_t, int32_t,
              int32_t, int32_t, cudaStream_t);
int l2_normalize_rows(float*, int64_t, int32_t, cudaStream_t);
size_t rank_full_workspace_bytes(int64_t, int64_t);
int rank_full(const float*, int32_t*, int64_t, int64_t, void*, size_t, cudaStream_t);
int order_from_ranks(const int32_t*, int64_t, int32_t*, cudaStream_t);
int score_topk_max_k(int32_t);
int topk_merge(const float*, const int32_t*, int64_t, int32_t, int32_t, int32_t, int64_t, int64_t, float*, int32_t*,
               int64_t, const int32_t*, int32_t, cudaStream_t);
int topk_merge_dedup_pair(const float*, const int32_t*, int64_t, const float*, const int32_t*, int64_t, int64_t,
                          int32_t, float*, int32_t*, int64_t, cudaStream_t);
int score_topk_wide_list_capacity(int32_t);
int select_topk_lists(const float*, const int32_t*, const int32_t*, int64_t, int32_t, int32_t, int32_t, float*,
                      int32_t*, int64_t, cudaStream_t);
int score_filter_max_k();
int score_filter_list_width();
int operand_stats(const void*, const float*, int64_t, int32_t, float*, float*, cudaStream_t);
int rescale_hi_global(const void*, const float*, const float*, const int32_t*, int64_t, int32_t, void*, cudaStream_t);
int pack_item_bias(const float*, const int32_t*, int64_t, float*, int64_t, float*, float*, float*, cudaStream_t);
int score_filter_f16(const void*, const float*, const float*, const float*, const void*, const float*, const float*,
                     const float*, const float*, const int32_t*, int64_t, int64_t, int32_t, int32_t, int32_t, int32_t,
                     float*, int32_t*, float*, const int32_t*, const int32_t*, cudaStream_t);
int exclusion_positions(const int32_t*, int64_t, int32_t*, const int32_t*, const int32_t*, int64_t, int64_t*,
                        cudaStream_t);
int rescore_topk(const void*, const float*, const void*, const float*, const float*, const float*, const int32_t*,
                 const float*, const float*, const float*, int64_t, int64_t, int32_t, int32_t, int32_t, int32_t, int32_t,
                 float*, int32_t*, int64_t, int32_t*, cudaStream_t);
int select_flagged_rows(const int32_t*, int64_t, int32_t*, int32_t, int32_t*, cudaStream_t);
int gather_operand_rows(const int32_t*, int32_t*, int32_t, int32_t, const void*, const float*, const float*, int32_t,
                        void*, float*, float*, cudaStream_t);
int scatter_topk_rows(const int32_t*, const int32_t*, int32_t, const float*, const int32_t*, int64_t, int32_t, float*,
                      int32_t*, int64_t, cudaStream_t);
int operand_half_sqnorm(const void*, const float*, int64_t, int32_t, float*, cudaStream_t);
int topk_euclidean_finish(float*, int32_t*, int64_t, int64_t, int32_t, cudaStream_t);
int score_wide_max_k();
int score_wide_list_capacity(int32_t);
int score_wide_f16(const void*, const float*, const float*, const float*, const void*, const float*, const float*,
                   const float*, const int32_t*, int64_t, int64_t, int32_t, int32_t, int32_t, int32_t, float*, int32_t*,
                   int32_t*, float*, const int32_t*, const int32_t*, cudaStream_t);
int select_wide_topk(const void*, const float*, const void*, const float*, const float*, const float*, const int32_t*,
                     int64_t, int32_t, int32_t, const int32_t*, const float*, const float*, const float*, int64_t,
                     int64_t, int32_t, int32_t, int32_t, int32_t, float*, int32_t*, int64_t, int32_t*, cudaStream_t);

int sample_items(int64_t, int64_t, int32_t, int32_t, uint64_t, uint32_t, int32_t*, cudaStream_t);
int wmrb_step_tastes(const char*, const void*, const void*, int32_t, int32_t, int32_t, int32_t, const float*,
                     const float*, const int32_t*, const int32_t*, const float*, const float*, const int32_t*, int64_t,
                     int64_t, int32_t, int32_t, float*, float*, float*, float*, float*, float*, float*, cudaStream_t);
size_t serial_loss_workspace_bytes(int64_t);
int serial_loss_step(int32_t, const void*, const void*, int32_t, int32_t, int32_t, int32_t, const float*, const float*,
                     const int32_t*, const int32_t*, const float*, int64_t, int64_t, int32_t, int64_t, float*, float*,
                     float*, float*, float*, float*, void*, size_t, cudaStream_t);
int l2_normalize_rows_step(const float*, int64_t, int32_t, int32_t, float*, float*, cudaStream_t);
int f32_to_bf16(const float*, int64_t, void*, cudaStream_t);
int adam_step(float*, const float*, float*, float*, int64_t, float, float, float, float, float, cudaStream_t);
uint64_t philox_u64_host(uint64_t, uint32_t, uint32_t, uint32_t);
size_t relu_layer_workspace_bytes(int64_t, int32_t, int32_t);
int relu_layer_forward(const float*, const float*, const float*, int64_t, int32_t, int32_t, float*, cudaStream_t);
int relu_layer_backward(float*, const float*, const float*, const float*, int64_t, int32_t, int32_t, float*, float*,
                        void*, size_t, cudaStream_t);

static inline cudaStream_t as_stream(void* s) { return static_cast<cudaStream_t>(s); }

}  // namespace trk

extern "C" {

int trk_version(void) { return 2000; }

const char* trk_last_error(void) { return trk::g_last_error; }

int trk_csr_gather_reduce_f32(const int32_t* indptr, const int32_t* col, const float* val, const float* weights,
                              int64_t rows, int32_t n_features, int32_t d, int32_t n_normalize, float* out_f32,
                              void* out_split, int32_t d_pad, float* out_scale, float* out_norm, float* stats,
                              void* stream) {
  return trk::csr_gather_reduce(indptr, col, val, weights, rows, n_features, d, n_normalize, out_f32, out_split,
                                d_pad, out_scale, out_norm, stats, trk::as_stream(stream));
}

int trk_split_f32_to_f16x2(const float* repr, int64_t rows, int32_t d, int32_t n_normalize, void* out_split,
                           int32_t d_pad, float* out_scale, void* stream) {
  TRK_CHECK_ARG(out_split != nullptr, "trk_split_f32_to_f16x2: null output");
  return trk::split_rows(repr, rows, d, n_normalize, nullptr, out_split, d_pad, out_scale, trk::as_stream(stream));
}

int trk_l2_normalize_rows_f32(float* x, int64_t rows, int32_t d, void* stream) {
  return trk::l2_normalize_rows(x, rows, d, trk::as_stream(stream));
}

int trk_csr_project_biases_f32(const int32_t* indptr, const int32_t* col, const float* val,
                               const float* feature_biases, int64_t rows, float* out, void* stream) {
  return trk::csr_project_biases(indptr, col, val, feature_biases, rows, out, trk::as_stream(stream));
}

int trk_score_f32(const float* user_repr, const float* item_repr, const float* user_bias, const float* item_bias,
                  float* out, int64_t n_users, int64_t n_items, int32_t d, int32_t n_tastes, int32_t mode,
                  void* stream) {
  return trk::score_f32(user_repr, nullptr, item_repr, user_bias, item_bias, out, n_users, n_items, d, n_tastes,
                        mode, trk::as_stream(stream));
}

int trk_score_attention_f32(const float* user_repr, const float* attention_repr, const float* item_repr,
                            const float* user_bias, const float* item_bias, float* out, int64_t n_users,
                            int64_t n_items, int32_t d, int32_t n_tastes, void* stream) {
  TRK_CHECK_ARG(attention_repr != nullptr, "trk_score_attention_f32: null attention representation");
  return trk::score_f32(user_repr, attention_repr, item_repr, user_bias, item_bias, out, n_users, n_items, d,
                        n_tastes, 0, trk::as_stream(stream));
}

size_t trk_rank_full_workspace_bytes(int64_t n_users, int64_t n_items) {
  return trk::rank_full_workspace_bytes(n_users, n_items);
}

int trk_rank_full(const float* scores, int32_t* ranks, int64_t n_users, int64_t n_items, void* workspace,
                  size_t workspace_bytes, void* stream) {
  return trk::rank_full(scores, ranks, n_users, n_items, workspace, workspace_bytes, trk::as_stream(stream));
}

int trk_order_from_ranks(const int32_t* ranks, int64_t n, int32_t* order, void* stream) {
  return trk::order_from_ranks(ranks, n, order, trk::as_stream(stream));
}

int trk_score_topk_max_k(int32_t d_pad) { return trk::score_topk_max_k(d_pad); }

int trk_pack_item_meta(const float* item_scale, const float* item_bias, int64_t n_items, float* item_meta,
                       int64_t n_items_padded, void* stream) {
  return trk::pack_item_meta(item_scale, item_bias, n_items, item_meta, n_items_padded, trk::as_stream(stream));
}

int trk_score_topk_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                         const void* item_split, const float* item_meta, int64_t n_users, int64_t n_items,
                         int32_t d_pad, int32_t k, int32_t n_splits, int32_t item_id_offset, float* cand_score,
                         int32_t* cand_item, const int32_t* n_users_live, void* stream) {
  return trk::score_tc({user_split, user_scale, user_bias, item_split, item_meta, n_users, n_items, d_pad, k, n_splits,
                        item_id_offset, cand_score, cand_item, n_users_live},
                       trk::as_stream(stream));
}

int trk_score_topk_f16x3_excl(const void* user_split, const float* user_scale, const float* user_bias,
                              const void* item_split, const float* item_meta, int64_t n_users, int64_t n_items,
                              int32_t d_pad, int32_t k, int32_t n_splits, int32_t item_id_offset, float* cand_score,
                              int32_t* cand_item, const int32_t* n_users_live, const int32_t* excl_indptr,
                              const int32_t* excl_ids, const int32_t* excl_row_map, void* stream) {
  TRK_CHECK_ARG(excl_indptr != nullptr && excl_ids != nullptr, "trk_score_topk_f16x3_excl: null exclusion list");
  return trk::score_tc({user_split, user_scale, user_bias, item_split, item_meta, n_users, n_items, d_pad, k, n_splits,
                        item_id_offset, cand_score, cand_item, n_users_live, excl_indptr, excl_ids, excl_row_map},
                       trk::as_stream(stream));
}

int trk_score_topk_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                const void* item_split, const float* item_meta, int64_t n_users, int64_t n_items,
                                int32_t d_pad, int32_t k, int32_t n_splits, int32_t item_id_offset, float* cand_score,
                                int32_t* cand_item, const int32_t* n_users_live, const int32_t* excl_indptr,
                                const int32_t* excl_ids, const int32_t* excl_row_map, const float* user_half_sqnorm,
                                const float* item_half_sqnorm, void* stream) {
  TRK_CHECK_ARG(user_half_sqnorm != nullptr && item_half_sqnorm != nullptr,
                "trk_score_topk_euclid_f16x3: null squared norms");
  return trk::score_tc({user_split, user_scale, user_bias, item_split, item_meta, n_users, n_items, d_pad, k, n_splits,
                        item_id_offset, cand_score, cand_item, n_users_live, excl_indptr, excl_ids, excl_row_map,
                        user_half_sqnorm, item_half_sqnorm},
                       trk::as_stream(stream));
}

int trk_score_dense_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                          const void* item_split, const float* item_meta, int64_t n_users, int64_t n_items,
                          int32_t d_pad, float* out, int64_t out_row_stride, void* stream) {
  trk::ScoreTcArgs a = {user_split, user_scale, user_bias, item_split, item_meta, n_users, n_items, d_pad};
  a.dense = true;
  a.dense_out = out;
  a.dense_stride = out_row_stride;
  return trk::score_tc(a, trk::as_stream(stream));
}

int trk_score_dense_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                 const void* item_split, const float* item_meta, int64_t n_users, int64_t n_items,
                                 int32_t d_pad, float* out, int64_t out_row_stride, const float* user_half_sqnorm,
                                 const float* item_half_sqnorm, void* stream) {
  TRK_CHECK_ARG(user_half_sqnorm != nullptr && item_half_sqnorm != nullptr,
                "trk_score_dense_euclid_f16x3: null squared norms");
  trk::ScoreTcArgs a = {user_split, user_scale, user_bias, item_split, item_meta, n_users, n_items, d_pad};
  a.user_half_sqnorm = user_half_sqnorm;
  a.item_half_sqnorm = item_half_sqnorm;
  a.dense = true;
  a.dense_out = out;
  a.dense_stride = out_row_stride;
  return trk::score_tc(a, trk::as_stream(stream));
}

int trk_score_dense_tastes_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                 int32_t n_tastes, int32_t attention, const void* item_split, const float* item_meta,
                                 int64_t n_users, int64_t n_items, int32_t d_pad, float* out, int64_t out_row_stride,
                                 void* stream) {
  TRK_CHECK_ARG(n_tastes >= 1, "score_tastes: n_tastes=%d < 1", n_tastes);
  trk::ScoreTcArgs a = {user_split, user_scale, user_bias, item_split, item_meta, n_users, n_items, d_pad};
  a.dense = true;
  a.dense_out = out;
  a.dense_stride = out_row_stride;
  a.n_tastes = n_tastes;
  a.attention = attention;
  return trk::score_tc(a, trk::as_stream(stream));
}

int trk_score_dense_tastes_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                        int32_t n_tastes, int32_t attention, const void* item_split,
                                        const float* item_meta, int64_t n_users, int64_t n_items, int32_t d_pad,
                                        float* out, int64_t out_row_stride, const float* user_half_sqnorm,
                                        const float* item_half_sqnorm, void* stream) {
  TRK_CHECK_ARG(n_tastes >= 1, "score_tastes: n_tastes=%d < 1", n_tastes);
  TRK_CHECK_ARG(user_half_sqnorm != nullptr && item_half_sqnorm != nullptr,
                "trk_score_dense_tastes_euclid_f16x3: null squared norms");
  trk::ScoreTcArgs a = {user_split, user_scale, user_bias, item_split, item_meta, n_users, n_items, d_pad};
  a.user_half_sqnorm = user_half_sqnorm;
  a.item_half_sqnorm = item_half_sqnorm;
  a.dense = true;
  a.dense_out = out;
  a.dense_stride = out_row_stride;
  a.n_tastes = n_tastes;
  a.attention = attention;
  return trk::score_tc(a, trk::as_stream(stream));
}

int trk_score_topk_tastes_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                int32_t n_tastes, int32_t attention, const void* item_split, const float* item_meta,
                                int64_t n_users, int64_t n_items, int32_t d_pad, int32_t k, int32_t n_splits,
                                int32_t item_id_offset, float* cand_score, int32_t* cand_item,
                                const int32_t* excl_indptr, const int32_t* excl_ids, const int32_t* excl_row_map,
                                void* stream) {
  TRK_CHECK_ARG(n_tastes >= 1, "score_tastes: n_tastes=%d < 1", n_tastes);
  trk::ScoreTcArgs a = {user_split, user_scale, user_bias, item_split, item_meta, n_users, n_items, d_pad, k, n_splits,
                        item_id_offset, cand_score, cand_item};
  a.excl_indptr = excl_indptr;
  a.excl_ids = excl_ids;
  a.excl_row_map = excl_row_map;
  a.n_tastes = n_tastes;
  a.attention = attention;
  return trk::score_tc(a, trk::as_stream(stream));
}

int trk_score_topk_tastes_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                       int32_t n_tastes, int32_t attention, const void* item_split,
                                       const float* item_meta, int64_t n_users, int64_t n_items, int32_t d_pad, int32_t k,
                                       int32_t n_splits, int32_t item_id_offset, float* cand_score, int32_t* cand_item,
                                       const int32_t* excl_indptr, const int32_t* excl_ids,
                                       const int32_t* excl_row_map, const float* user_half_sqnorm,
                                       const float* item_half_sqnorm, void* stream) {
  TRK_CHECK_ARG(n_tastes >= 1, "score_tastes: n_tastes=%d < 1", n_tastes);
  TRK_CHECK_ARG(user_half_sqnorm != nullptr && item_half_sqnorm != nullptr,
                "trk_score_topk_tastes_euclid_f16x3: null squared norms");
  trk::ScoreTcArgs a = {user_split, user_scale, user_bias, item_split, item_meta, n_users, n_items, d_pad, k, n_splits,
                        item_id_offset, cand_score, cand_item, nullptr, excl_indptr, excl_ids, excl_row_map,
                        user_half_sqnorm, item_half_sqnorm};
  a.n_tastes = n_tastes;
  a.attention = attention;
  return trk::score_tc(a, trk::as_stream(stream));
}

int trk_score_topk_wide_list_capacity(int32_t k) { return trk::score_topk_wide_list_capacity(k); }

int trk_score_topk_wide_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                     const void* item_split, const float* item_meta, int64_t n_users, int64_t n_items,
                                     int32_t d_pad, int32_t k, int32_t n_splits, int32_t item_id_offset,
                                     float* list_score, int32_t* list_item, int32_t* list_count,
                                     const int32_t* n_users_live, const int32_t* excl_indptr, const int32_t* excl_ids,
                                     const int32_t* excl_row_map, const float* user_half_sqnorm,
                                     const float* item_half_sqnorm, void* stream) {
  TRK_CHECK_ARG(user_half_sqnorm != nullptr && item_half_sqnorm != nullptr,
                "trk_score_topk_wide_euclid_f16x3: null squared norms");
  trk::ScoreTcArgs a = {user_split, user_scale, user_bias, item_split, item_meta, n_users, n_items, d_pad, k, n_splits,
                        item_id_offset, list_score, list_item, n_users_live, excl_indptr, excl_ids, excl_row_map,
                        user_half_sqnorm, item_half_sqnorm};
  a.wide = true;
  a.list_count = list_count;
  return trk::score_tc(a, trk::as_stream(stream));
}

int trk_score_topk_wide_tastes_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                     int32_t n_tastes, int32_t attention, const void* item_split,
                                     const float* item_meta, int64_t n_users, int64_t n_items, int32_t d_pad, int32_t k,
                                     int32_t n_splits, int32_t item_id_offset, float* list_score, int32_t* list_item,
                                     int32_t* list_count, const int32_t* excl_indptr, const int32_t* excl_ids,
                                     const int32_t* excl_row_map, void* stream) {
  TRK_CHECK_ARG(n_tastes >= 1, "score_tastes: n_tastes=%d < 1", n_tastes);
  trk::ScoreTcArgs a = {user_split, user_scale, user_bias, item_split, item_meta, n_users, n_items, d_pad, k, n_splits,
                        item_id_offset, list_score, list_item};
  a.excl_indptr = excl_indptr;
  a.excl_ids = excl_ids;
  a.excl_row_map = excl_row_map;
  a.n_tastes = n_tastes;
  a.attention = attention;
  a.wide = true;
  a.list_count = list_count;
  return trk::score_tc(a, trk::as_stream(stream));
}

int trk_score_topk_wide_tastes_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                            int32_t n_tastes, int32_t attention, const void* item_split,
                                            const float* item_meta, int64_t n_users, int64_t n_items, int32_t d_pad,
                                            int32_t k, int32_t n_splits, int32_t item_id_offset, float* list_score,
                                            int32_t* list_item, int32_t* list_count, const int32_t* excl_indptr,
                                            const int32_t* excl_ids, const int32_t* excl_row_map,
                                            const float* user_half_sqnorm, const float* item_half_sqnorm,
                                            void* stream) {
  TRK_CHECK_ARG(n_tastes >= 1, "score_tastes: n_tastes=%d < 1", n_tastes);
  TRK_CHECK_ARG(user_half_sqnorm != nullptr && item_half_sqnorm != nullptr,
                "trk_score_topk_wide_tastes_euclid_f16x3: null squared norms");
  trk::ScoreTcArgs a = {user_split, user_scale, user_bias, item_split, item_meta, n_users, n_items, d_pad, k, n_splits,
                        item_id_offset, list_score, list_item, nullptr, excl_indptr, excl_ids, excl_row_map,
                        user_half_sqnorm, item_half_sqnorm};
  a.n_tastes = n_tastes;
  a.attention = attention;
  a.wide = true;
  a.list_count = list_count;
  return trk::score_tc(a, trk::as_stream(stream));
}

namespace {

// the counting-mode fields of score_tc's arguments
void set_count(trk::ScoreTcArgs& a, const int32_t* pair_indptr, const int32_t* pair_ids, float* pair_score,
               int32_t* pair_count, const int32_t* block_pairs, int32_t pass, const int32_t* excl_indptr,
               const int32_t* excl_ids, const int32_t* excl_row_map) {
  a.count = true;
  a.pair_indptr = pair_indptr;
  a.pair_ids = pair_ids;
  a.pair_score = pair_score;
  a.pair_count = pair_count;
  a.block_pairs = block_pairs;
  a.pass = pass;
  a.excl_indptr = excl_indptr;
  a.excl_ids = excl_ids;
  a.excl_row_map = excl_row_map;
}

}  // namespace

int trk_score_count_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                          const void* item_split, const float* item_meta, int64_t n_users, int64_t n_items,
                          int32_t d_pad, int32_t n_splits, int32_t item_id_offset, const int32_t* pair_indptr,
                          const int32_t* pair_ids, float* pair_score, int32_t* pair_count,
                          const int32_t* block_pairs, int32_t pass, const int32_t* excl_indptr,
                          const int32_t* excl_ids, const int32_t* excl_row_map, void* stream) {
  trk::ScoreTcArgs a = {user_split, user_scale, user_bias, item_split, item_meta, n_users, n_items, d_pad, 0, n_splits,
                        item_id_offset};
  set_count(a, pair_indptr, pair_ids, pair_score, pair_count, block_pairs, pass, excl_indptr, excl_ids, excl_row_map);
  return trk::score_tc(a, trk::as_stream(stream));
}

int trk_score_count_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                 const void* item_split, const float* item_meta, int64_t n_users, int64_t n_items,
                                 int32_t d_pad, int32_t n_splits, int32_t item_id_offset, const int32_t* pair_indptr,
                                 const int32_t* pair_ids, float* pair_score, int32_t* pair_count,
                                 const int32_t* block_pairs, int32_t pass, const int32_t* excl_indptr,
                                 const int32_t* excl_ids, const int32_t* excl_row_map, const float* user_half_sqnorm,
                                 const float* item_half_sqnorm, void* stream) {
  TRK_CHECK_ARG(user_half_sqnorm != nullptr && item_half_sqnorm != nullptr,
                "trk_score_count_euclid_f16x3: null squared norms");
  trk::ScoreTcArgs a = {user_split, user_scale, user_bias, item_split, item_meta, n_users, n_items, d_pad, 0, n_splits,
                        item_id_offset};
  set_count(a, pair_indptr, pair_ids, pair_score, pair_count, block_pairs, pass, excl_indptr, excl_ids, excl_row_map);
  a.user_half_sqnorm = user_half_sqnorm;
  a.item_half_sqnorm = item_half_sqnorm;
  return trk::score_tc(a, trk::as_stream(stream));
}

int trk_score_count_tastes_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                 int32_t n_tastes, int32_t attention, const void* item_split, const float* item_meta,
                                 int64_t n_users, int64_t n_items, int32_t d_pad, int32_t n_splits,
                                 int32_t item_id_offset, const int32_t* pair_indptr, const int32_t* pair_ids,
                                 float* pair_score, int32_t* pair_count, const int32_t* block_pairs, int32_t pass,
                                 const int32_t* excl_indptr, const int32_t* excl_ids, const int32_t* excl_row_map,
                                 void* stream) {
  TRK_CHECK_ARG(n_tastes >= 1, "score_tastes: n_tastes=%d < 1", n_tastes);
  trk::ScoreTcArgs a = {user_split, user_scale, user_bias, item_split, item_meta, n_users, n_items, d_pad, 0, n_splits,
                        item_id_offset};
  set_count(a, pair_indptr, pair_ids, pair_score, pair_count, block_pairs, pass, excl_indptr, excl_ids, excl_row_map);
  a.n_tastes = n_tastes;
  a.attention = attention;
  return trk::score_tc(a, trk::as_stream(stream));
}

int trk_score_count_tastes_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                        int32_t n_tastes, int32_t attention, const void* item_split,
                                        const float* item_meta, int64_t n_users, int64_t n_items, int32_t d_pad,
                                        int32_t n_splits, int32_t item_id_offset, const int32_t* pair_indptr,
                                        const int32_t* pair_ids, float* pair_score, int32_t* pair_count,
                                        const int32_t* block_pairs, int32_t pass, const int32_t* excl_indptr,
                                        const int32_t* excl_ids, const int32_t* excl_row_map,
                                        const float* user_half_sqnorm, const float* item_half_sqnorm, void* stream) {
  TRK_CHECK_ARG(n_tastes >= 1, "score_tastes: n_tastes=%d < 1", n_tastes);
  TRK_CHECK_ARG(user_half_sqnorm != nullptr && item_half_sqnorm != nullptr,
                "trk_score_count_tastes_euclid_f16x3: null squared norms");
  trk::ScoreTcArgs a = {user_split, user_scale, user_bias, item_split, item_meta, n_users, n_items, d_pad, 0, n_splits,
                        item_id_offset};
  set_count(a, pair_indptr, pair_ids, pair_score, pair_count, block_pairs, pass, excl_indptr, excl_ids, excl_row_map);
  a.user_half_sqnorm = user_half_sqnorm;
  a.item_half_sqnorm = item_half_sqnorm;
  a.n_tastes = n_tastes;
  a.attention = attention;
  return trk::score_tc(a, trk::as_stream(stream));
}

namespace {

// the pairs-mode fields of score_tc's arguments
void set_pairs(trk::ScoreTcArgs& a, const int32_t* pair_indptr, const int32_t* pair_cols, float* pair_score,
               const int32_t* tile_items, int32_t n_tiles, const int32_t* work, int32_t n_work) {
  a.pairs = true;
  a.pair_indptr = pair_indptr;
  a.pair_ids = pair_cols;
  a.pair_score = pair_score;
  a.tile_items = tile_items;
  a.n_tiles = n_tiles;
  a.work = work;
  a.n_work = n_work;
}

}  // namespace

int trk_score_pairs_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                          const void* item_split, const float* slot_meta, int64_t n_users, int64_t n_items,
                          int32_t d_pad, const int32_t* pair_indptr, const int32_t* pair_cols, float* pair_score,
                          const int32_t* tile_items, int32_t n_tiles, const int32_t* work, int32_t n_work,
                          void* stream) {
  trk::ScoreTcArgs a = {user_split, user_scale, user_bias, item_split, slot_meta, n_users, n_items, d_pad};
  set_pairs(a, pair_indptr, pair_cols, pair_score, tile_items, n_tiles, work, n_work);
  return trk::score_tc(a, trk::as_stream(stream));
}

int trk_score_pairs_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                 const void* item_split, const float* slot_meta, int64_t n_users, int64_t n_items,
                                 int32_t d_pad, const int32_t* pair_indptr, const int32_t* pair_cols,
                                 float* pair_score, const int32_t* tile_items, int32_t n_tiles, const int32_t* work,
                                 int32_t n_work, const float* user_half_sqnorm, const float* slot_half_sqnorm,
                                 void* stream) {
  TRK_CHECK_ARG(user_half_sqnorm != nullptr && slot_half_sqnorm != nullptr,
                "trk_score_pairs_euclid_f16x3: null squared norms");
  trk::ScoreTcArgs a = {user_split, user_scale, user_bias, item_split, slot_meta, n_users, n_items, d_pad};
  set_pairs(a, pair_indptr, pair_cols, pair_score, tile_items, n_tiles, work, n_work);
  a.user_half_sqnorm = user_half_sqnorm;
  a.item_half_sqnorm = slot_half_sqnorm;
  return trk::score_tc(a, trk::as_stream(stream));
}

int trk_score_pairs_tastes_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                 int32_t n_tastes, int32_t attention, const void* item_split, const float* slot_meta,
                                 int64_t n_users, int64_t n_items, int32_t d_pad, const int32_t* pair_indptr,
                                 const int32_t* pair_cols, float* pair_score, const int32_t* tile_items,
                                 int32_t n_tiles, const int32_t* work, int32_t n_work, void* stream) {
  TRK_CHECK_ARG(n_tastes >= 1, "score_tastes: n_tastes=%d < 1", n_tastes);
  trk::ScoreTcArgs a = {user_split, user_scale, user_bias, item_split, slot_meta, n_users, n_items, d_pad};
  set_pairs(a, pair_indptr, pair_cols, pair_score, tile_items, n_tiles, work, n_work);
  a.n_tastes = n_tastes;
  a.attention = attention;
  return trk::score_tc(a, trk::as_stream(stream));
}

int trk_score_pairs_tastes_euclid_f16x3(const void* user_split, const float* user_scale, const float* user_bias,
                                        int32_t n_tastes, int32_t attention, const void* item_split,
                                        const float* slot_meta, int64_t n_users, int64_t n_items, int32_t d_pad,
                                        const int32_t* pair_indptr, const int32_t* pair_cols, float* pair_score,
                                        const int32_t* tile_items, int32_t n_tiles, const int32_t* work,
                                        int32_t n_work, const float* user_half_sqnorm, const float* slot_half_sqnorm,
                                        void* stream) {
  TRK_CHECK_ARG(n_tastes >= 1, "score_tastes: n_tastes=%d < 1", n_tastes);
  TRK_CHECK_ARG(user_half_sqnorm != nullptr && slot_half_sqnorm != nullptr,
                "trk_score_pairs_tastes_euclid_f16x3: null squared norms");
  trk::ScoreTcArgs a = {user_split, user_scale, user_bias, item_split, slot_meta, n_users, n_items, d_pad};
  set_pairs(a, pair_indptr, pair_cols, pair_score, tile_items, n_tiles, work, n_work);
  a.user_half_sqnorm = user_half_sqnorm;
  a.item_half_sqnorm = slot_half_sqnorm;
  a.n_tastes = n_tastes;
  a.attention = attention;
  return trk::score_tc(a, trk::as_stream(stream));
}

int trk_select_topk_lists(const float* list_score, const int32_t* list_item, const int32_t* list_count,
                          int64_t n_rows, int32_t n_lists, int32_t list_width, int32_t k, float* out_score,
                          int32_t* out_item, int64_t out_row_stride, void* stream) {
  return trk::select_topk_lists(list_score, list_item, list_count, n_rows, n_lists, list_width, k, out_score, out_item,
                                out_row_stride, trk::as_stream(stream));
}

int trk_topk_merge(const float* cand_score, const int32_t* cand_item, int64_t n_users, int32_t n_lists,
                   int32_t k_in, int32_t k_out, int64_t user_stride, int64_t list_stride, float* out_score,
                   int32_t* out_item, int64_t out_row_stride, const int32_t* n_users_live, int32_t dedup, void* stream) {
  return trk::topk_merge(cand_score, cand_item, n_users, n_lists, k_in, k_out, user_stride, list_stride, out_score,
                         out_item, out_row_stride, n_users_live, dedup, trk::as_stream(stream));
}

int trk_topk_merge_dedup_pair(const float* a_score, const int32_t* a_item, int64_t a_row_stride, const float* b_score,
                              const int32_t* b_item, int64_t b_row_stride, int64_t n_rows, int32_t k, float* out_score,
                              int32_t* out_item, int64_t out_row_stride, void* stream) {
  return trk::topk_merge_dedup_pair(a_score, a_item, a_row_stride, b_score, b_item, b_row_stride, n_rows, k, out_score,
                                    out_item, out_row_stride, trk::as_stream(stream));
}

int trk_score_filter_max_k(void) { return trk::score_filter_max_k(); }

int trk_score_filter_list_width(void) { return trk::score_filter_list_width(); }

int trk_operand_stats(const void* split, const float* scale, int64_t rows, int32_t d_pad, float* out_norm,
                      float* stats, void* stream) {
  return trk::operand_stats(split, scale, rows, d_pad, out_norm, stats, trk::as_stream(stream));
}

int trk_rescale_hi_global(const void* split, const float* scale, const float* stats, const int32_t* perm,
                          int64_t rows, int32_t d_pad, void* out_hi, void* stream) {
  return trk::rescale_hi_global(split, scale, stats, perm, rows, d_pad, out_hi, trk::as_stream(stream));
}

int trk_pack_item_bias(const float* item_bias, const int32_t* perm, int64_t n_items, float* out,
                       int64_t n_items_padded, float* stats, float* block_max, float* block_min, void* stream) {
  return trk::pack_item_bias(item_bias, perm, n_items, out, n_items_padded, stats, block_max, block_min,
                             trk::as_stream(stream));
}

int trk_score_filter_f16(const void* user_split, const float* user_scale, const float* user_bias,
                         const float* user_norm, const void* item_hi_global, const float* item_stats,
                         const float* item_bias_padded, const float* block_bias_max, const float* block_bias_min,
                         const int32_t* item_perm, int64_t n_users, int64_t n_items, int32_t d_pad, int32_t k,
                         int32_t n_splits, int32_t item_id_offset, float* cand_score, int32_t* cand_item,
                         float* row_theta, void* stream) {
  return trk::score_filter_f16(user_split, user_scale, user_bias, user_norm, item_hi_global, item_stats,
                               item_bias_padded, block_bias_max, block_bias_min, item_perm, n_users, n_items, d_pad, k,
                               n_splits, item_id_offset, cand_score, cand_item, row_theta, nullptr, nullptr,
                               trk::as_stream(stream));
}

int trk_exclusion_positions(const int32_t* item_perm, int64_t n_items, int32_t* inv_perm, const int32_t* excl_indptr,
                            const int32_t* excl_ids, int64_t n_rows, int64_t* out_keys, void* stream) {
  return trk::exclusion_positions(item_perm, n_items, inv_perm, excl_indptr, excl_ids, n_rows, out_keys,
                                  trk::as_stream(stream));
}

int trk_score_filter_f16_excl(const void* user_split, const float* user_scale, const float* user_bias,
                              const float* user_norm, const void* item_hi_global, const float* item_stats,
                              const float* item_bias_padded, const float* block_bias_max, const float* block_bias_min,
                              const int32_t* item_perm, int64_t n_users, int64_t n_items, int32_t d_pad, int32_t k,
                              int32_t n_splits, int32_t item_id_offset, float* cand_score, int32_t* cand_item,
                              float* row_theta, const int32_t* excl_indptr, const int32_t* excl_pos, void* stream) {
  TRK_CHECK_ARG(excl_indptr != nullptr && excl_pos != nullptr, "trk_score_filter_f16_excl: null exclusion list");
  return trk::score_filter_f16(user_split, user_scale, user_bias, user_norm, item_hi_global, item_stats,
                               item_bias_padded, block_bias_max, block_bias_min, item_perm, n_users, n_items, d_pad, k,
                               n_splits, item_id_offset, cand_score, cand_item, row_theta, excl_indptr, excl_pos,
                               trk::as_stream(stream));
}

int trk_rescore_topk_split(const void* user_split, const float* user_scale, const void* item_split,
                           const float* item_scale, const float* user_bias, const float* item_bias,
                           const int32_t* cand_item, const float* row_theta, const float* user_norm,
                           const float* item_stats, int64_t n_users, int64_t n_items_local, int32_t d_pad,
                           int32_t n_lists, int32_t list_width, int32_t k, int32_t item_id_offset, float* out_score,
                           int32_t* out_item, int64_t out_row_stride, int32_t* out_flag, void* stream) {
  return trk::rescore_topk(user_split, user_scale, item_split, item_scale, user_bias, item_bias, cand_item, row_theta,
                           user_norm, item_stats, n_users, n_items_local, d_pad, n_lists, list_width, k, item_id_offset,
                           out_score, out_item, out_row_stride, out_flag, trk::as_stream(stream));
}

int trk_select_flagged_rows(const int32_t* flags, int64_t n, int32_t* idx, int32_t capacity, int32_t* counters,
                            void* stream) {
  return trk::select_flagged_rows(flags, n, idx, capacity, counters, trk::as_stream(stream));
}

int trk_gather_operand_rows(const int32_t* idx, int32_t* counters, int32_t capacity, int32_t small_capacity,
                            const void* split, const float* scale, const float* bias, int32_t d_pad, void* sub_split,
                            float* sub_scale, float* sub_bias, void* stream) {
  return trk::gather_operand_rows(idx, counters, capacity, small_capacity, split, scale, bias, d_pad, sub_split,
                                  sub_scale, sub_bias, trk::as_stream(stream));
}

int trk_scatter_topk_rows(const int32_t* idx, const int32_t* counters, int32_t capacity, const float* sub_score,
                          const int32_t* sub_item, int64_t sub_row_stride, int32_t k, float* out_score,
                          int32_t* out_item, int64_t out_row_stride, void* stream) {
  return trk::scatter_topk_rows(idx, counters, capacity, sub_score, sub_item, sub_row_stride, k, out_score, out_item,
                                out_row_stride, trk::as_stream(stream));
}

int trk_operand_half_sqnorm(const void* split, const float* scale, int64_t rows, int32_t d_pad, float* out,
                            void* stream) {
  return trk::operand_half_sqnorm(split, scale, rows, d_pad, out, trk::as_stream(stream));
}

int trk_topk_euclidean_finish(float* scores, int32_t* items, int64_t row_stride, int64_t n_rows, int32_t k,
                              void* stream) {
  return trk::topk_euclidean_finish(scores, items, row_stride, n_rows, k, trk::as_stream(stream));
}

int trk_score_wide_max_k(void) { return trk::score_wide_max_k(); }

int trk_score_wide_list_capacity(int32_t k) { return trk::score_wide_list_capacity(k); }

int trk_score_wide_f16(const void* user_split, const float* user_scale, const float* user_bias,
                       const float* user_norm, const void* item_hi_global, const float* item_stats,
                       const float* item_bias_padded, const float* block_bias_max, const int32_t* item_perm,
                       int64_t n_users, int64_t n_items, int32_t d_pad, int32_t k, int32_t n_splits,
                       int32_t item_id_offset, float* list_score, int32_t* list_item, int32_t* list_count,
                       float* row_theta, void* stream) {
  return trk::score_wide_f16(user_split, user_scale, user_bias, user_norm, item_hi_global, item_stats,
                             item_bias_padded, block_bias_max, item_perm, n_users, n_items, d_pad, k, n_splits,
                             item_id_offset, list_score, list_item, list_count, row_theta, nullptr, nullptr,
                             trk::as_stream(stream));
}

int trk_score_wide_f16_excl(const void* user_split, const float* user_scale, const float* user_bias,
                            const float* user_norm, const void* item_hi_global, const float* item_stats,
                            const float* item_bias_padded, const float* block_bias_max, const int32_t* item_perm,
                            int64_t n_users, int64_t n_items, int32_t d_pad, int32_t k, int32_t n_splits,
                            int32_t item_id_offset, float* list_score, int32_t* list_item, int32_t* list_count,
                            float* row_theta, const int32_t* excl_indptr, const int32_t* excl_pos, void* stream) {
  TRK_CHECK_ARG(excl_indptr != nullptr && excl_pos != nullptr, "trk_score_wide_f16_excl: null exclusion list");
  return trk::score_wide_f16(user_split, user_scale, user_bias, user_norm, item_hi_global, item_stats,
                             item_bias_padded, block_bias_max, item_perm, n_users, n_items, d_pad, k, n_splits,
                             item_id_offset, list_score, list_item, list_count, row_theta, excl_indptr, excl_pos,
                             trk::as_stream(stream));
}

int trk_select_wide_topk(const void* user_split, const float* user_scale, const void* item_split,
                         const float* item_scale, const float* user_bias, const float* item_bias,
                         const int32_t* cand_item, int64_t cand_row_stride, int32_t n_lists, int32_t list_width,
                         const int32_t* list_count, const float* row_theta, const float* user_norm,
                         const float* item_stats, int64_t n_rows, int64_t n_items_local, int32_t d_pad, int32_t k,
                         int32_t item_id_offset, int32_t euclidean, float* out_score, int32_t* out_item,
                         int64_t out_row_stride, int32_t* out_flag, void* stream) {
  return trk::select_wide_topk(user_split, user_scale, item_split, item_scale, user_bias, item_bias, cand_item,
                               cand_row_stride, n_lists, list_width, list_count, row_theta, user_norm, item_stats,
                               n_rows, n_items_local, d_pad, k, item_id_offset, euclidean, out_score, out_item,
                               out_row_stride, out_flag, trk::as_stream(stream));
}

int trk_sample_items(int64_t n_users, int64_t n_items, int32_t n_sampled, int32_t replace, uint64_t seed,
                     uint32_t step, int32_t* out, void* stream) {
  return trk::sample_items(n_users, n_items, n_sampled, replace, seed, step, out, trk::as_stream(stream));
}

uint64_t trk_sample_stream_u64(uint64_t seed, uint32_t step, uint32_t user, uint32_t draw) {
  return trk::philox_u64_host(seed, step, user, draw);
}

int trk_wmrb_step(const void* user_repr, const void* item_repr, int32_t repr_is_bf16, const float* user_bias,
                  const float* item_bias, const int32_t* inter_indptr, const int32_t* inter_item,
                  const float* inter_val, const float* item_weight_sum, const int32_t* samples, int64_t n_users,
                  int64_t n_items, int32_t d, int32_t n_sampled, float* loss, float* pred_serial, float* coef,
                  float* d_user_repr, float* d_user_bias, float* d_item_repr, float* d_item_bias, void* stream) {
  // the one-taste dot form of trk_wmrb_step_tastes
  return trk::wmrb_step_tastes("wmrb_step", user_repr, item_repr, repr_is_bf16, 1, 0, 0, user_bias, item_bias,
                               inter_indptr, inter_item, inter_val, item_weight_sum, samples, n_users, n_items, d,
                               n_sampled, loss, pred_serial, coef, d_user_repr, d_user_bias, d_item_repr, d_item_bias,
                               trk::as_stream(stream));
}

int trk_wmrb_step_tastes(const void* user_rows, const void* item_repr, int32_t repr_is_bf16, int32_t n_tastes,
                         int32_t attention, int32_t euclidean, const float* user_bias, const float* item_bias,
                         const int32_t* inter_indptr, const int32_t* inter_item, const float* inter_val,
                         const float* item_weight_sum, const int32_t* samples, int64_t n_users, int64_t n_items,
                         int32_t d, int32_t n_sampled, float* loss, float* pred_serial, float* coef, float* d_user_rows,
                         float* d_user_bias, float* d_item_repr, float* d_item_bias, void* stream) {
  return trk::wmrb_step_tastes("wmrb_step_tastes", user_rows, item_repr, repr_is_bf16, n_tastes, attention, euclidean,
                               user_bias, item_bias, inter_indptr, inter_item, inter_val, item_weight_sum, samples,
                               n_users, n_items, d, n_sampled, loss, pred_serial, coef, d_user_rows, d_user_bias,
                               d_item_repr, d_item_bias, trk::as_stream(stream));
}

size_t trk_serial_loss_workspace_bytes(int64_t nnz) { return trk::serial_loss_workspace_bytes(nnz); }

int trk_serial_loss_step(int32_t loss_kind, const void* user_rows, const void* item_repr, int32_t repr_is_bf16,
                         int32_t n_tastes, int32_t attention, int32_t euclidean, const float* user_bias,
                         const float* item_bias, const int32_t* inter_indptr, const int32_t* inter_item,
                         const float* inter_val, int64_t n_users, int64_t n_items, int32_t d, int64_t nnz, float* loss,
                         float* pred_serial, float* d_user_rows, float* d_user_bias, float* d_item_repr,
                         float* d_item_bias, void* workspace, size_t workspace_bytes, void* stream) {
  return trk::serial_loss_step(loss_kind, user_rows, item_repr, repr_is_bf16, n_tastes, attention, euclidean, user_bias,
                               item_bias, inter_indptr, inter_item, inter_val, n_users, n_items, d, nnz, loss,
                               pred_serial, d_user_rows, d_user_bias, d_item_repr, d_item_bias, workspace,
                               workspace_bytes, trk::as_stream(stream));
}

int trk_l2_normalize_rows_step_f32(const float* x, int64_t rows, int32_t d, int32_t n_normalize, float* out,
                                   float* grad, void* stream) {
  return trk::l2_normalize_rows_step(x, rows, d, n_normalize, out, grad, trk::as_stream(stream));
}

int trk_f32_to_bf16(const float* x, int64_t n, void* out, void* stream) {
  return trk::f32_to_bf16(x, n, out, trk::as_stream(stream));
}

int trk_adam_step_f32(float* w, const float* grad, float* m, float* v, int64_t n, float lr_t, float beta1, float beta2,
                      float epsilon, float l2, void* stream) {
  return trk::adam_step(w, grad, m, v, n, lr_t, beta1, beta2, epsilon, l2, trk::as_stream(stream));
}

size_t trk_relu_layer_workspace_bytes(int64_t rows, int32_t hidden, int32_t d) {
  return trk::relu_layer_workspace_bytes(rows, hidden, d);
}

int trk_relu_layer_forward_f32(const float* pre, const float* bias, const float* w2, int64_t rows, int32_t hidden,
                               int32_t d, float* out, void* stream) {
  return trk::relu_layer_forward(pre, bias, w2, rows, hidden, d, out, trk::as_stream(stream));
}

int trk_relu_layer_backward_f32(float* pre, const float* bias, const float* w2, const float* d_out, int64_t rows,
                                int32_t hidden, int32_t d, float* d_bias, float* d_w2, void* workspace,
                                size_t workspace_bytes, void* stream) {
  return trk::relu_layer_backward(pre, bias, w2, d_out, rows, hidden, d, d_bias, d_w2, workspace, workspace_bytes,
                                  trk::as_stream(stream));
}

}  // extern "C"
