// Re-scoring, selection and certificate of the wide filter's survivors (score_wide_tc.cu): the k > 32 counterpart of
// rescore_topk_kernel (rescore_topk.cu).  One CTA per user row:
//   * every candidate is scored from the split operands with rescore_topk_kernel's arithmetic -- per lane a 4-element
//     FMA chain over hi + lo, a butterfly sum over the lanes (offsets 16, 8, 4, 2, 1: the tree of transpose_sum_16),
//     then fma(dot, scale_i * scale_u, user bias) + item bias -- so an item scores the same on both filter routes;
//   * the candidates are sorted by (score desc, id asc) with a bitonic sort of 64-bit keys in shared memory and the
//     first k are written (sentinels (-inf, INT32_MAX) fill what real candidates cannot);
//   * the row is certified with the rule of rescore_topk_kernel: max(theta, dropped) + m < the exact k-th best, and k
//     real candidates unless theta stayed -inf.
// With `euclidean` the survivors' scores -1/2 d^2 are mapped to -sqrt(max(d^2, 1e-16)) after the certificate (which is
// checked on the -1/2 d^2 scale, DESIGN §3.2) and sorted again: topk_euclidean_finish_kernel's job for k > 32.
#include "filter_tc.cuh"

namespace trk {

constexpr int kSelectThreads = 256;
constexpr int kSelectMaxSlots = 16384;   // candidates of one row (128 KB of keys in shared memory)

// ascending key = (score desc, id asc)
__device__ __forceinline__ uint64_t select_key(float s, int32_t id) {
  return (static_cast<uint64_t>(~wide_key(s)) << 32) | static_cast<uint32_t>(id);
}
__device__ __forceinline__ float select_key_score(uint64_t key) {
  return wide_unkey(~static_cast<uint32_t>(key >> 32));
}

// ascending bitonic sort of n (a power of two) keys in shared memory by the whole CTA; ends with a barrier
__device__ __forceinline__ void block_sort_keys(uint64_t* key, int n) {
#pragma unroll 1
  for (int size = 2; size <= n; size <<= 1) {
#pragma unroll 1
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int t = threadIdx.x; t < n / 2; t += blockDim.x) {
        const int i = 2 * t - (t & (stride - 1));   // lower index of the pair
        const int j = i + stride;
        const bool ascending = (i & size) == 0;
        const uint64_t a = key[i], b = key[j];
        if ((a > b) == ascending) {
          key[i] = b;
          key[j] = a;
        }
      }
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kSelectThreads)
select_wide_kernel(const __half* __restrict__ user_split, const float* __restrict__ user_scale,
                   const __half* __restrict__ item_split, const float* __restrict__ item_scale,
                   const float* __restrict__ user_bias, const float* __restrict__ item_bias,
                   const int32_t* __restrict__ cand_item, int64_t cand_row_stride, int n_lists, int list_width,
                   const int32_t* __restrict__ list_count, const float* __restrict__ row_theta,
                   const float* __restrict__ user_norm, const float* __restrict__ item_stats, int64_t n_items_local,
                   int d_pad, int k, int item_id_offset, int n_slots, int euclidean, float* __restrict__ out_score,
                   int32_t* __restrict__ out_item, int64_t out_stride, int32_t* __restrict__ out_flag) {
  extern __shared__ uint64_t keys[];
  const int64_t u = blockIdx.x;
  const int lane = threadIdx.x % 32, warp = threadIdx.x / 32, n_warps = blockDim.x / 32;
  const float kNegInf = -__int_as_float(0x7f800000);
  const int n_cand = n_lists * list_width;
  const int64_t row_halves = 2 * static_cast<int64_t>(d_pad);

  for (int t = threadIdx.x; t < n_slots; t += blockDim.x) {
    int32_t id = 0x7fffffff;
    if (t < n_cand) {
      const int l = t / list_width;
      if (list_count == nullptr || t - l * list_width < __ldg(list_count + u * n_lists + l)) {
        id = __ldg(cand_item + u * cand_row_stride + t);
        const int64_t local = static_cast<int64_t>(id) - item_id_offset;
        if (local < 0 || local >= n_items_local) id = 0x7fffffff;
      }
    }
    keys[t] = static_cast<uint32_t>(id);
  }
  __syncthreads();

  float uv[4];
  load_split4(user_split + u * row_halves, d_pad, lane, true, uv);
  const float su = __ldg(user_scale + u);
  const float ub = user_bias != nullptr ? __ldg(user_bias + u) : 0.0f;
  // warp w scores slots [4 w', 4 w' + 4) for w' = w, w + n_warps, ...: four independent row loads in flight
  for (int t0 = 4 * warp; t0 < n_slots; t0 += 4 * n_warps) {
    int32_t id[4];
    float part[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      id[q] = static_cast<int32_t>(static_cast<uint32_t>(keys[t0 + q]));
      const bool ok = id[q] != 0x7fffffff;   // warp-uniform
      float iv[4];
      load_split4(item_split + (ok ? static_cast<int64_t>(id[q]) - item_id_offset : 0) * row_halves, d_pad, lane, ok,
                  iv);
      float acc = 0.0f;
#pragma unroll
      for (int j = 0; j < 4; ++j) acc = fmaf(uv[j], iv[j], acc);
      part[q] = acc;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int q = 0; q < 4; ++q) part[q] += __shfl_xor_sync(0xffffffffu, part[q], o);
    }
    if (lane == 0) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float s = kNegInf;
        if (id[q] != 0x7fffffff) {
          const int64_t local = static_cast<int64_t>(id[q]) - item_id_offset;
          const float ib = item_bias != nullptr ? __ldg(item_bias + local) : 0.0f;
          s = fmaf(part[q], __ldg(item_scale + local) * su, ub) + ib;   // rescore_topk_kernel's bias arithmetic
        }
        keys[t0 + q] = select_key(s, id[q]);
      }
    }
  }
  block_sort_keys(keys, n_slots);

  if (out_flag != nullptr && threadIdx.x == 0) {
    float theta_max = kNegInf;
    for (int l = 0; l < n_lists; ++l) theta_max = fmaxf(theta_max, __ldg(row_theta + u * n_lists + l));
    const uint64_t kth = keys[k - 1];
    const bool have_k = static_cast<int32_t>(static_cast<uint32_t>(kth)) != 0x7fffffff;
    const float m = kMarginFactor * __ldg(user_norm + u) * __ldg(item_stats + 0) +
                    kBiasUlps * (fabsf(ub) + __ldg(item_stats + 2));
    bool valid = m < -kNegInf;   // an infinite (or NaN) margin certifies nothing
    if (theta_max > kNegInf) valid = valid && have_k && (theta_max + m < select_key_score(kth));
    out_flag[u] = valid ? 0 : 1;
  }
  if (euclidean) {
    for (int t = threadIdx.x; t < n_slots; t += blockDim.x) {
      const uint64_t key = keys[t];
      const int32_t id = static_cast<int32_t>(static_cast<uint32_t>(key));
      if (id != 0x7fffffff) keys[t] = select_key(-sqrtf(fmaxf(-2.0f * select_key_score(key), 1e-16f)), id);
    }
    block_sort_keys(keys, n_slots);
  }
  for (int j = threadIdx.x; j < k; j += blockDim.x) {
    const uint64_t key = keys[j];
    const int32_t id = static_cast<int32_t>(static_cast<uint32_t>(key));
    out_score[u * out_stride + j] = id != 0x7fffffff ? select_key_score(key) : kNegInf;
    out_item[u * out_stride + j] = id;
  }
}

// The exact kernel's wide mode (score_topk_tc.cu, DESIGN §3.8) leaves per row n_lists lists of FINAL scores, at most
// k entries each (list_count): select_lists_kernel sorts their union by (score desc, id asc) and writes the first k,
// sentinels (-inf, INT32_MAX) where there are fewer -- no re-scoring, no certificate.  Slot l * k + e holds entry e of
// list l.  One CTA per row.
__global__ void __launch_bounds__(kSelectThreads)
select_lists_kernel(const float* __restrict__ list_score, const int32_t* __restrict__ list_item,
                    const int32_t* __restrict__ list_count, int n_lists, int list_width, int k, int n_slots,
                    float* __restrict__ out_score, int32_t* __restrict__ out_item, int64_t out_stride) {
  extern __shared__ uint64_t keys[];
  const int64_t u = blockIdx.x;
  const float kNegInf = -__int_as_float(0x7f800000);
  for (int t = threadIdx.x; t < n_slots; t += blockDim.x) {
    uint64_t key = select_key(kNegInf, 0x7fffffff);
    const int l = t / k;
    if (l < n_lists && t - l * k < __ldg(list_count + u * n_lists + l)) {
      const int64_t at = (u * n_lists + l) * list_width + (t - l * k);
      key = select_key(__ldg(list_score + at), __ldg(list_item + at));
    }
    keys[t] = key;
  }
  block_sort_keys(keys, n_slots);
  for (int j = threadIdx.x; j < k; j += blockDim.x) {
    const uint64_t key = keys[j];
    const int32_t id = static_cast<int32_t>(static_cast<uint32_t>(key));
    out_score[u * out_stride + j] = id != 0x7fffffff ? select_key_score(key) : kNegInf;
    out_item[u * out_stride + j] = id;
  }
}

int select_topk_lists(const float* list_score, const int32_t* list_item, const int32_t* list_count, int64_t n_rows,
                      int32_t n_lists, int32_t list_width, int32_t k, float* out_score, int32_t* out_item,
                      int64_t out_row_stride, cudaStream_t stream) {
  TRK_CHECK_ARG(list_score && list_item && list_count, "select_topk_lists: null input");
  TRK_CHECK_ARG(out_score && out_item, "select_topk_lists: null output");
  TRK_CHECK_ARG(n_rows >= 0 && n_lists >= 1 && k >= 1 && list_width >= k, "select_topk_lists: bad sizes");
  TRK_CHECK_ARG(out_row_stride >= k, "select_topk_lists: out_row_stride < k");
  int n_slots = 64;
  while (n_slots < static_cast<int64_t>(n_lists) * k && n_slots <= kSelectMaxSlots) n_slots *= 2;
  TRK_CHECK_ARG(n_slots <= kSelectMaxSlots, "select_topk_lists: n_lists x k = %lld entries per row exceed %d",
                static_cast<long long>(n_lists) * k, kSelectMaxSlots);
  if (n_rows == 0) return TRK_OK;
  const size_t smem = static_cast<size_t>(n_slots) * sizeof(uint64_t);
  TRK_CHECK_CUDA(cudaFuncSetAttribute(select_lists_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      static_cast<int>(smem)));
  select_lists_kernel<<<static_cast<unsigned>(n_rows), kSelectThreads, smem, stream>>>(
      list_score, list_item, list_count, n_lists, list_width, k, n_slots, out_score, out_item, out_row_stride);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

int select_wide_topk(const void* user_split, const float* user_scale, const void* item_split, const float* item_scale,
                     const float* user_bias, const float* item_bias, const int32_t* cand_item, int64_t cand_row_stride,
                     int32_t n_lists, int32_t list_width, const int32_t* list_count, const float* row_theta,
                     const float* user_norm, const float* item_stats, int64_t n_rows, int64_t n_items_local,
                     int32_t d_pad, int32_t k, int32_t item_id_offset, int32_t euclidean, float* out_score,
                     int32_t* out_item, int64_t out_row_stride, int32_t* out_flag, cudaStream_t stream) {
  TRK_CHECK_ARG(user_split && user_scale && item_split && item_scale && cand_item, "select_wide_topk: null input");
  TRK_CHECK_ARG(out_score && out_item, "select_wide_topk: null output");
  TRK_CHECK_ARG(out_flag == nullptr || (row_theta && user_norm && item_stats),
                "select_wide_topk: the certificate needs row_theta, user_norm and item_stats");
  TRK_CHECK_ARG(n_rows >= 0 && n_items_local >= 0 && n_lists >= 1 && list_width >= 1 && k >= 1,
                "select_wide_topk: bad sizes");
  TRK_CHECK_ARG(cand_row_stride >= static_cast<int64_t>(n_lists) * list_width, "select_wide_topk: cand_row_stride");
  TRK_CHECK_ARG(d_pad == 64 || d_pad == 128, "select_wide_topk: d_pad=%d (64 or 128)", d_pad);
  TRK_CHECK_ARG(out_row_stride >= k, "select_wide_topk: out_row_stride < k");
  TRK_CHECK_ARG(reinterpret_cast<uintptr_t>(user_split) % 16 == 0 && reinterpret_cast<uintptr_t>(item_split) % 16 == 0,
                "select_wide_topk: operands must be 16-byte aligned");
  int n_slots = 64;
  while (n_slots < n_lists * list_width || n_slots < k) n_slots *= 2;
  TRK_CHECK_ARG(n_slots <= kSelectMaxSlots, "select_wide_topk: %d candidates per row exceed %d",
                n_lists * list_width, kSelectMaxSlots);
  if (n_rows == 0) return TRK_OK;
  const size_t smem = static_cast<size_t>(n_slots) * sizeof(uint64_t);
  TRK_CHECK_CUDA(cudaFuncSetAttribute(select_wide_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      static_cast<int>(smem)));
  select_wide_kernel<<<static_cast<unsigned>(n_rows), kSelectThreads, smem, stream>>>(
      static_cast<const __half*>(user_split), user_scale, static_cast<const __half*>(item_split), item_scale, user_bias,
      item_bias, cand_item, cand_row_stride, n_lists, list_width, list_count, row_theta, user_norm, item_stats,
      n_items_local, d_pad, k, item_id_offset, n_slots, euclidean, out_score, out_item, out_row_stride, out_flag);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

}  // namespace trk
