// Re-scoring and ranking of the survivors of the tensor-core filter (score_filter_tc.cu), and the device-side routing
// of the users whose bound could not be certified.
//
// For every user each surviving item is scored from the SPLIT operands K1 wrote (x * 2^e = hi + lo, 22 significant bits):
//     s = fma( sum_e (hi_u + lo_u)_e (hi_i + lo_i)_e , scale_u * scale_i , user bias ) + item bias
// i.e. the fp32 dot product of tf.matmul (tensorrec/prediction_graphs.py:49-50) on operands rounded to 22 bits, then
// + user bias, + item bias left to right (tensorrec/recommendation_graphs.py:41) -- the same operands and the same
// bias arithmetic as the exact tensor-core kernel (score_topk_tc.cu), <= 2^-21 |u||i| from the fp32 product and EXACT
// for integer-valued representations.  The k best are selected in tf.nn.top_k order (score descending, equal scores by
// lower item id, recommendation_graphs.py:81).  One warp per user: lanes split the components of the dot product
// (fixed xor-tree reduction -> deterministic), the running top-k lives one entry per lane.
//
// Verification: the filter excluded only items whose approximate score was <= theta (per list), so their score is
// <= theta + m.  If max theta + m is not strictly below the k-th best found here the row is flagged; flagged rows are
// compacted ON THE DEVICE (trk_select_flagged_rows), their operands gathered (trk_gather_operand_rows), scored by the
// exact 3-pass kernel with a device-side row count and scattered back (trk_scatter_topk_rows): no host round trip.
#include "common.cuh"

namespace trk {

constexpr float kRMarginFactor = 1.5f * 0.0009765625f;
constexpr float kRBiasUlps = 4.0f * 1.1920929e-7f;

// Sum over the 32 lanes of 16 values per lane, all 16 at once: at every halving step a lane keeps half of its values and
// hands the other half to its partner (8 + 4 + 2 + 1 shuffles), a last exchange completes the sum: 16 shuffles instead of
// 16 x 5.  Afterwards lanes 2c and 2c + 1 both hold the total of value c.  Fixed order: deterministic.
__device__ __forceinline__ float transpose_sum_16(float (&v)[16], int lane) {
#pragma unroll
  for (int half = 8, off = 16; half >= 1; half >>= 1, off >>= 1) {
    const bool upper = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < half; ++i) {
      const float send = upper ? v[i] : v[i + half];
      const float keep = upper ? v[i + half] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
  }
  return v[0] + __shfl_xor_sync(0xffffffffu, v[0], 1);
}

// One warp per user, 16 candidates (one filter list) at a time: the 16 item rows are requested together, the 16 dot
// products are reduced by one transposed reduction, the survivors are ordered by one 32-lane bitonic sort (even lanes:
// the new candidates, odd lanes: the best 16 of the lists before).
__global__ void __launch_bounds__(256)
rescore_topk_kernel(const __half* __restrict__ user_split, const float* __restrict__ user_scale,
                    const __half* __restrict__ item_split, const float* __restrict__ item_scale,
                    const float* __restrict__ user_bias, const float* __restrict__ item_bias,
                    const int32_t* __restrict__ cand_item, const float* __restrict__ row_theta,
                    const float* __restrict__ user_norm, const float* __restrict__ item_stats, int64_t n_users,
                    int64_t n_items_local, int d_pad, int n_lists, int list_width, int k, int item_id_offset,
                    float* __restrict__ out_score, int32_t* __restrict__ out_item, int64_t out_stride,
                    int32_t* __restrict__ out_flag) {
  const int lane = threadIdx.x % 32;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / 32;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * blockDim.x / 32;
  const float kNegInf = -__int_as_float(0x7f800000);
  const float max_item_norm = __ldg(item_stats + 0);
  const float max_item_bias = __ldg(item_stats + 2);
  const int n_cand = n_lists * list_width;
  const int64_t row_halves = 2 * static_cast<int64_t>(d_pad);

  for (int64_t u = warp; u < n_users; u += n_warps) {
    float uv[4];
    load_split4(user_split + u * row_halves, d_pad, lane, true, uv);
    const float su = __ldg(user_scale + u);
    const float ub = user_bias != nullptr ? __ldg(user_bias + u) : 0.0f;
    const int32_t* ci = cand_item + u * n_cand;
    float best_s = kNegInf;        // after a group: lanes 0..15 hold the best 16 so far, in order
    int32_t best_i = 0x7fffffff;
    int n_real = 0;

    for (int c0 = 0; c0 < n_cand; c0 += 16) {
      // lane l < 16 owns candidate c0 + l (id, validity, row index); every lane needs every id for the row loads
      int32_t my_id = (lane < 16 && c0 + lane < n_cand) ? __ldg(ci + c0 + lane) : 0x7fffffff;
      const int64_t my_local = static_cast<int64_t>(my_id) - item_id_offset;
      const bool my_ok = my_id != 0x7fffffff && my_local >= 0 && my_local < n_items_local;
      if (!my_ok) my_id = 0x7fffffff;
      n_real += __popc(__ballot_sync(0xffffffffu, my_ok));
      float part[16];
#pragma unroll
      for (int q = 0; q < 16; ++q) {
        const int32_t id = __shfl_sync(0xffffffffu, my_id, q);
        const bool ok = id != 0x7fffffff;                      // warp-uniform
        float iv[4];
        load_split4(item_split + (ok ? static_cast<int64_t>(id) - item_id_offset : 0) * row_halves, d_pad, lane, ok, iv);
        float acc = 0.0f;
#pragma unroll
        for (int j = 0; j < 4; ++j) acc = fmaf(uv[j], iv[j], acc);
        part[q] = acc;
      }
      const float dot = transpose_sum_16(part, lane);           // lanes 2c, 2c + 1: candidate c0 + c
      const int owner = lane >> 1;
      int32_t id = __shfl_sync(0xffffffffu, my_id, owner);
      float s = kNegInf;
      if ((lane & 1) == 0 && id != 0x7fffffff) {
        const int64_t local = static_cast<int64_t>(id) - item_id_offset;
        const float ib = item_bias != nullptr ? __ldg(item_bias + local) : 0.0f;
        s = fmaf(dot, __ldg(item_scale + local) * su, ub) + ib;   // the bias arithmetic of the exact kernel's epilogue
      } else {
        id = 0x7fffffff;
      }
      // odd lanes: the best 16 of the groups before (lane 2j + 1 takes entry j)
      const float prev_s = __shfl_sync(0xffffffffu, best_s, owner);
      const int32_t prev_i = __shfl_sync(0xffffffffu, best_i, owner);
      if ((lane & 1) != 0) {
        s = prev_s;
        id = prev_i;
      }
      warp_sort_desc(s, id, lane);
      best_s = s;
      best_i = id;
    }

    // verification of the filter's bound for this user
    float theta_max = kNegInf;
    for (int l = lane; l < n_lists; l += 32) theta_max = fmaxf(theta_max, __ldg(row_theta + u * n_lists + l));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) theta_max = fmaxf(theta_max, __shfl_xor_sync(0xffffffffu, theta_max, o));
    const float kth = __shfl_sync(0xffffffffu, best_s, k - 1);
    const float m = kRMarginFactor * __ldg(user_norm + u) * max_item_norm + kRBiasUlps * (fabsf(ub) + max_item_bias);
    bool valid = m < -kNegInf;   // an infinite (or NaN) margin certifies nothing
    if (theta_max > kNegInf) valid = valid && (n_real >= k) && (theta_max + m < kth);
    if (lane < k) {
      out_score[u * out_stride + lane] = best_s;
      out_item[u * out_stride + lane] = best_i;
    }
    if (lane == 0) out_flag[u] = valid ? 0 : 1;
  }
}

// ---------------------------------------------------------------------------------------------------------
// device-side routing of the flagged rows
// ---------------------------------------------------------------------------------------------------------
// idx[0 .. min(count, capacity)) = the flagged rows (any order: every row is processed independently downstream),
// counters[0] = count.  Warp-aggregated: one atomic per warp that holds a flagged row.
__global__ void select_flagged_rows_kernel(const int32_t* __restrict__ flags, int64_t n, int32_t* __restrict__ idx,
                                           int capacity, int32_t* __restrict__ counters) {
  const int lane = threadIdx.x % 32;
  for (int64_t base = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) - lane; base < n;
       base += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t i = base + lane;
    const bool f = i < n && flags[i] != 0;
    const unsigned ballot = __ballot_sync(0xffffffffu, f);
    if (ballot == 0) continue;
    int start = 0;
    if (lane == 0) start = atomicAdd(counters, __popc(ballot));
    start = __shfl_sync(0xffffffffu, start, 0);
    const int pos = start + __popc(ballot & ((1u << lane) - 1u));
    if (f && pos < capacity) idx[pos] = static_cast<int32_t>(i);
  }
}

// sub_*[i] = *[idx[i]] for i < min(count, capacity): split rows (2 d_pad halves), scale, bias.  Also publishes the live
// row counts of the two re-scoring tiers: counters[2] = count if it fits the small tier (few rows: the exact kernel is
// then launched with many item splits so that a handful of user blocks still fills the machine), else 0;
// counters[3] = min(count, capacity) if it does not, else 0.
__global__ void gather_operand_rows_kernel(const int32_t* __restrict__ idx, int32_t* __restrict__ counters,
                                           int capacity, int small_capacity, const uint4* __restrict__ split,
                                           const float* __restrict__ scale, const float* __restrict__ bias, int row_vec,
                                           uint4* __restrict__ sub_split, float* __restrict__ sub_scale,
                                           float* __restrict__ sub_bias) {
  const int n = min(counters[0], capacity);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    counters[2] = counters[0] <= small_capacity ? counters[0] : 0;
    counters[3] = counters[0] <= small_capacity ? 0 : n;
  }
  const int lane = threadIdx.x % 32;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / 32;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * blockDim.x / 32;
  for (int64_t i = warp; i < n; i += n_warps) {
    const int64_t src = idx[i];
    for (int v = lane; v < row_vec; v += 32) sub_split[i * row_vec + v] = split[src * row_vec + v];
    if (lane == 0) {
      sub_scale[i] = scale[src];
      if (bias != nullptr) sub_bias[i] = bias[src];
    }
  }
}

__global__ void scatter_topk_rows_kernel(const int32_t* __restrict__ idx, const int32_t* __restrict__ counters,
                                         int capacity, const float* __restrict__ sub_score,
                                         const int32_t* __restrict__ sub_item, int64_t sub_stride, int k,
                                         float* __restrict__ out_score, int32_t* __restrict__ out_item,
                                         int64_t out_stride) {
  const int n = min(counters[0], capacity);
  for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < static_cast<int64_t>(n) * k;
       t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t i = t / k;
    const int j = static_cast<int>(t % k);
    const int64_t dst = idx[i];
    out_score[dst * out_stride + j] = sub_score[i * sub_stride + j];
    out_item[dst * out_stride + j] = sub_item[i * sub_stride + j];
  }
}

// item biases in processing order (out[p] = bias[perm[p]]), padded to whole tiles with -inf (a padded column can
// never pass the filter); max |bias| -> stats[2]; block_max[b] = max bias of positions [128 b, 128 b + 128).
__global__ void pack_item_bias_kernel(const float* __restrict__ bias, const int32_t* __restrict__ perm, int64_t n,
                                      float* __restrict__ out, int64_t n_padded, float* __restrict__ stats,
                                      float* __restrict__ block_max, float* __restrict__ block_min) {
  // one warp per block of 128 positions
  const int lane = threadIdx.x % 32;
  const int64_t blk = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / 32;
  if (blk * 128 >= n_padded) return;
  const float kNegInf = -__int_as_float(0x7f800000);
  float vmax = kNegInf, vmin = -kNegInf, amax = 0.0f;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int64_t pos = blk * 128 + q * 32 + lane;
    float v = kNegInf;
    if (pos < n) {
      const int64_t src = perm != nullptr ? perm[pos] : pos;
      v = bias != nullptr ? bias[src] : 0.0f;
      amax = fmaxf(amax, fabsf(v));
    }
    if (pos < n_padded) out[pos] = v;
    vmax = fmaxf(vmax, v);
    vmin = fminf(vmin, v);     // a block that contains padding has minimum -inf: no lower bound can be drawn from it
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
    vmin = fminf(vmin, __shfl_xor_sync(0xffffffffu, vmin, o));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  }
  if (lane == 0) {
    if (block_max != nullptr) block_max[blk] = vmax;
    if (block_min != nullptr) block_min[blk] = vmin;
    if (stats != nullptr && amax > 0.0f) atomicMax(reinterpret_cast<int*>(stats + 2), __float_as_int(amax));
  }
}

int pack_item_bias(const float* bias, const int32_t* perm, int64_t n, float* out, int64_t n_padded, float* stats,
                   float* block_max, float* block_min, cudaStream_t stream) {
  TRK_CHECK_ARG(out && n >= 0 && n_padded >= n && n_padded % 128 == 0, "pack_item_bias: bad arguments");
  if (n_padded == 0) return TRK_OK;
  const int threads = 256;
  const int64_t n_blocks128 = n_padded / 128;
  pack_item_bias_kernel<<<static_cast<unsigned>(ceil_div(n_blocks128, threads / 32)), threads, 0, stream>>>(
      bias, perm, n, out, n_padded, stats, block_max, block_min);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

int rescore_topk(const void* user_split, const float* user_scale, const void* item_split, const float* item_scale,
                 const float* user_bias, const float* item_bias, const int32_t* cand_item, const float* row_theta,
                 const float* user_norm, const float* item_stats, int64_t n_users, int64_t n_items_local,
                 int32_t d_pad, int32_t n_lists, int32_t list_width, int32_t k, int32_t item_id_offset,
                 float* out_score, int32_t* out_item, int64_t out_row_stride, int32_t* out_flag, cudaStream_t stream) {
  TRK_CHECK_ARG(user_split && user_scale && item_split && item_scale && cand_item && row_theta && user_norm &&
                    item_stats,
                "rescore_topk: null input");
  TRK_CHECK_ARG(out_score && out_item && out_flag, "rescore_topk: null output");
  TRK_CHECK_ARG(n_users >= 0 && n_items_local >= 0 && n_lists >= 1 && list_width >= 1, "rescore_topk: bad sizes");
  TRK_CHECK_ARG(d_pad == 64 || d_pad == 128, "rescore_topk: d_pad=%d (64 or 128)", d_pad);
  TRK_CHECK_ARG(k >= 1 && k <= 16, "rescore_topk: k=%d outside [1, 16]", k);
  TRK_CHECK_ARG(list_width <= 16 || list_width % 16 == 0, "rescore_topk: list_width=%d", list_width);
  TRK_CHECK_ARG(out_row_stride >= k, "rescore_topk: out_row_stride=%lld < k", static_cast<long long>(out_row_stride));
  TRK_CHECK_ARG(reinterpret_cast<uintptr_t>(user_split) % 16 == 0 && reinterpret_cast<uintptr_t>(item_split) % 16 == 0,
                "rescore_topk: operands must be 16-byte aligned");
  if (n_users == 0) return TRK_OK;
  const int threads = 256;
  rescore_topk_kernel<<<capped_grid(ceil_div(n_users, threads / 32), 8), threads, 0, stream>>>(
      static_cast<const __half*>(user_split), user_scale, static_cast<const __half*>(item_split), item_scale, user_bias,
      item_bias, cand_item, row_theta, user_norm, item_stats, n_users, n_items_local, d_pad, n_lists, list_width, k,
      item_id_offset, out_score, out_item, out_row_stride, out_flag);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

int select_flagged_rows(const int32_t* flags, int64_t n, int32_t* idx, int32_t capacity, int32_t* counters,
                        cudaStream_t stream) {
  TRK_CHECK_ARG(flags && idx && counters && n >= 0 && capacity >= 1, "select_flagged_rows: bad arguments");
  TRK_CHECK_CUDA(cudaMemsetAsync(counters, 0, 4 * sizeof(int32_t), stream));
  if (n == 0) return TRK_OK;
  const int threads = 256;
  select_flagged_rows_kernel<<<capped_grid(ceil_div(n, threads), 8), threads, 0, stream>>>(
      flags, n, idx, capacity, counters);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

int gather_operand_rows(const int32_t* idx, int32_t* counters, int32_t capacity, int32_t small_capacity,
                        const void* split, const float* scale, const float* bias, int32_t d_pad, void* sub_split,
                        float* sub_scale, float* sub_bias, cudaStream_t stream) {
  TRK_CHECK_ARG(idx && counters && split && scale && sub_split && sub_scale && capacity >= 1 && d_pad >= 64 &&
                    d_pad % 64 == 0,
                "gather_operand_rows: bad arguments");
  TRK_CHECK_ARG(bias == nullptr || sub_bias != nullptr, "gather_operand_rows: bias without sub_bias");
  const int threads = 256;
  const int64_t blocks = ceil_div(static_cast<int64_t>(capacity), threads / 32);
  gather_operand_rows_kernel<<<capped_grid(blocks, 8), threads, 0, stream>>>(
      idx, counters, capacity, small_capacity, static_cast<const uint4*>(split), scale, bias, 2 * d_pad * 2 / 16,
      static_cast<uint4*>(sub_split), sub_scale, sub_bias);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

int scatter_topk_rows(const int32_t* idx, const int32_t* counters, int32_t capacity, const float* sub_score,
                      const int32_t* sub_item, int64_t sub_row_stride, int32_t k, float* out_score, int32_t* out_item,
                      int64_t out_row_stride, cudaStream_t stream) {
  TRK_CHECK_ARG(idx && counters && sub_score && sub_item && out_score && out_item && capacity >= 1 && k >= 1 &&
                    out_row_stride >= k && sub_row_stride >= k,
                "scatter_topk_rows: bad arguments");
  const int threads = 256;
  const int64_t blocks = ceil_div(static_cast<int64_t>(capacity) * k, threads);
  scatter_topk_rows_kernel<<<capped_grid(blocks, 8), threads, 0, stream>>>(
      idx, counters, capacity, sub_score, sub_item, sub_row_stride, k, out_score, out_item, out_row_stride);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

}  // namespace trk
