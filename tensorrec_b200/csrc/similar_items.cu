// Similar items on the fused top-k kernels (TensorRec.predict_similar_items_top_k).
//
// The queries are rows of the item operand itself and similar-items scores carry no biases (tensorrec/
// recommendation_graphs.py:124-137), so the dot and cosine forms are the fused top-k with both bias pointers NULL.
// Euclidean similarity (prediction_graphs.py:84-100, -sqrt(max(d^2, 1e-16))) is reduced to the same kernels:
//     q.i + (-1/2 |q|^2) + (-1/2 |i|^2) = -1/2 d^2(q, i)
// i.e. a per-query "user bias" and a per-item "item bias" of -1/2 |row|^2 (trk_operand_half_sqnorm).  -1/2 d^2 orders the
// items exactly as -sqrt(d^2) does; trk_topk_euclidean_finish maps the k survivors to the reference score and restores
// tf.nn.top_k order among entries that the sqrt (or the 1e-16 clamp) made equal.
#include "common.cuh"

namespace trk {

// out[r] = -1/2 sum_j (scale_r (hi + lo)_j)^2 from the split operand, so the norm sees the values the re-scoring dot
// product sees.  One warp per row; fixed per-lane order and xor-tree reduction: deterministic.
__global__ void operand_half_sqnorm_kernel(const __half* __restrict__ split, const float* __restrict__ scale,
                                           int64_t rows, int d_pad, float* __restrict__ out) {
  const int lane = threadIdx.x % 32;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / 32;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * blockDim.x / 32;
  for (int64_t r = warp; r < rows; r += n_warps) {
    const __half* hi = split + r * 2 * d_pad;
    const __half* lo = hi + d_pad;
    const float sc = __ldg(scale + r);
    float ss = 0.0f;
    for (int e = lane * 2; e < d_pad; e += 64) {
      const float2 h = __half22float2(*reinterpret_cast<const __half2*>(hi + e));
      const float2 l = __half22float2(*reinterpret_cast<const __half2*>(lo + e));
      const float x0 = sc * (h.x + l.x), x1 = sc * (h.y + l.y);   // power-of-two scale: exact
      ss = fmaf(x0, x0, ss);
      ss = fmaf(x1, x1, ss);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if (lane == 0) out[r] = -0.5f * ss;
  }
}

// In place on k <= 32 (score, id) entries per row: s = -1/2 d^2  ->  -sqrt(max(d^2, 1e-16)) (sentinels stay -inf:
// -2 * -inf = +inf), then the row is re-sorted into (score desc, id asc) order.  One warp per row, one entry per lane.
__global__ void topk_euclidean_finish_kernel(float* __restrict__ scores, int32_t* __restrict__ items, int64_t stride,
                                             int64_t n_rows, int k) {
  const int lane = threadIdx.x % 32;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / 32;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * blockDim.x / 32;
  for (int64_t r = warp; r < n_rows; r += n_warps) {
    float s = -__int_as_float(0x7f800000);
    int32_t id = 0x7fffffff;
    if (lane < k) {
      s = -sqrtf(fmaxf(-2.0f * scores[r * stride + lane], 1e-16f));
      id = items[r * stride + lane];
    }
    warp_sort_desc(s, id, lane);
    if (lane < k) {
      scores[r * stride + lane] = s;
      items[r * stride + lane] = id;
    }
  }
}

int operand_half_sqnorm(const void* split, const float* scale, int64_t rows, int32_t d_pad, float* out,
                        cudaStream_t stream) {
  TRK_CHECK_ARG(split && scale && out && rows >= 0 && d_pad >= 64 && d_pad % 64 == 0,
                "operand_half_sqnorm: bad arguments");
  if (rows == 0) return TRK_OK;
  const int threads = 256;
  operand_half_sqnorm_kernel<<<capped_grid(ceil_div(rows, threads / 32), 8), threads, 0, stream>>>(
      static_cast<const __half*>(split), scale, rows, d_pad, out);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

int topk_euclidean_finish(float* scores, int32_t* items, int64_t row_stride, int64_t n_rows, int32_t k,
                          cudaStream_t stream) {
  TRK_CHECK_ARG(scores && items && n_rows >= 0, "topk_euclidean_finish: bad arguments");
  TRK_CHECK_ARG(k >= 1 && k <= 32, "topk_euclidean_finish: k=%d outside [1, 32]", k);
  TRK_CHECK_ARG(row_stride >= k, "topk_euclidean_finish: row_stride=%lld < k", static_cast<long long>(row_stride));
  if (n_rows == 0) return TRK_OK;
  const int threads = 256;
  topk_euclidean_finish_kernel<<<capped_grid(ceil_div(n_rows, threads / 32), 8), threads, 0, stream>>>(
      scores, items, row_stride, n_rows, k);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

}  // namespace trk
