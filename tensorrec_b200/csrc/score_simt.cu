// K2 (exact fp32 on CUDA cores) -- dense prediction for every (user, item) pair, any shape.
//
// Reference semantics: DotProductPredictionGraph.connect_dense_prediction_graph = tf.matmul(u, i, transpose_b=True)
// (tensorrec/prediction_graphs.py:49-50); EuclideanSimilarityPredictionGraph dense (:84-100);
// collapse_mixture_of_tastes (tensorrec/recommendation_graphs.py:85-109: max over tastes :107, attention softmax
// :96-103); bias_prediction_dense (:41: pred + ub[:,None] + ib[None,:], left to right).
//
// This is the any-shape, bit-deterministic path (k ascending, one fp32 FMA chain per output) that backs the
// reference API at small sizes (tests, n_components not a multiple of 16, n_tastes > 1, attention).  The
// throughput path is the wgmma kernel in score_topk_tc.cu.
#include "common.cuh"

namespace trk {

constexpr int kTileM = 64, kTileN = 64, kTileK = 16;
constexpr int kSimtThreads = 256;  // 16 x 16 threads, 4 x 4 outputs each

// loads a kTile x kTileK slab of a row-major [rows, d] matrix into smem as [k][row] (+1 pad against conflicts)
__device__ __forceinline__ void load_slab(const float* __restrict__ src, int64_t rows, int d, int64_t row0, int k0,
                                          float (*dst)[kTileM + 1]) {
  for (int i = threadIdx.x; i < kTileM * kTileK; i += kSimtThreads) {
    const int r = i / kTileK, k = i % kTileK;
    const int64_t gr = row0 + r;
    const int gk = k0 + k;
    dst[k][r] = (gr < rows && gk < d) ? __ldg(src + gr * d + gk) : 0.0f;
  }
}

template <int MODE, bool ATTENTION>
__global__ void __launch_bounds__(kSimtThreads)
score_simt_kernel(const float* __restrict__ user_repr, const float* __restrict__ attention_repr,
                  const float* __restrict__ item_repr, const float* __restrict__ user_bias,
                  const float* __restrict__ item_bias, float* __restrict__ out, int64_t n_users, int64_t n_items,
                  int d, int n_tastes) {
  __shared__ float s_u[kTileK][kTileM + 1];
  __shared__ float s_a[ATTENTION ? kTileK : 1][kTileM + 1];
  __shared__ float s_i[kTileK][kTileN + 1];

  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int64_t u0 = static_cast<int64_t>(blockIdx.y) * kTileM;
  const int64_t i0 = static_cast<int64_t>(blockIdx.x) * kTileN;

  float result[4][4];
  // attention: online softmax state per output
  float run_max[4][4], run_sum[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      result[a][b] = ATTENTION ? 0.0f : -__int_as_float(0x7f800000);
      run_max[a][b] = -__int_as_float(0x7f800000);
      run_sum[a][b] = 0.0f;
    }

  for (int t = 0; t < n_tastes; ++t) {
    const float* u_t = user_repr + static_cast<int64_t>(t) * n_users * d;
    const float* a_t = ATTENTION ? attention_repr + static_cast<int64_t>(t) * n_users * d : nullptr;
    float acc[4][4], att[4][4], ru[4], ri[4];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      ru[a] = 0.0f;
      ri[a] = 0.0f;
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        acc[a][b] = 0.0f;
        att[a][b] = 0.0f;
      }
    }
    for (int k0 = 0; k0 < d; k0 += kTileK) {
      __syncthreads();
      load_slab(u_t, n_users, d, u0, k0, s_u);
      if constexpr (ATTENTION) load_slab(a_t, n_users, d, u0, k0, s_a);
      load_slab(item_repr, n_items, d, i0, k0, s_i);
      __syncthreads();
#pragma unroll
      for (int k = 0; k < kTileK; ++k) {
        float uv[4], iv[4], av[4];
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          uv[a] = s_u[k][ty * 4 + a];
          iv[a] = s_i[k][tx * 4 + a];
          if constexpr (ATTENTION) av[a] = s_a[k][ty * 4 + a];
        }
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          if constexpr (MODE == 1) {
            ru[a] = fmaf(uv[a], uv[a], ru[a]);
            ri[a] = fmaf(iv[a], iv[a], ri[a]);
          }
#pragma unroll
          for (int b = 0; b < 4; ++b) {
            acc[a][b] = fmaf(uv[a], iv[b], acc[a][b]);
            if constexpr (ATTENTION) att[a][b] = fmaf(av[a], iv[b], att[a][b]);
          }
        }
      }
    }
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        float p = acc[a][b];
        if constexpr (MODE == 1) {  // -sqrt(max(r_user - 2 u.i + r_item, 1e-16))  (prediction_graphs.py:90-100)
          const float dist = fmaxf((ru[a] - 2.0f * p) + ri[b], 1e-16f);
          p = -sqrtf(dist);
        }
        if constexpr (ATTENTION) {  // sum_t softmax_t(att) * pred, evaluated as an online softmax over tastes
          const float m_new = fmaxf(run_max[a][b], att[a][b]);
          const float corr = expf(run_max[a][b] - m_new);
          const float w = expf(att[a][b] - m_new);
          run_sum[a][b] = run_sum[a][b] * corr + w;
          result[a][b] = result[a][b] * corr + w * p;
          run_max[a][b] = m_new;
        } else {
          result[a][b] = fmaxf(result[a][b], p);  // recommendation_graphs.py:107
        }
      }
  }

#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const int64_t u = u0 + ty * 4 + a;
    if (u >= n_users) continue;
    const float ub = user_bias != nullptr ? __ldg(user_bias + u) : 0.0f;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int64_t i = i0 + tx * 4 + b;
      if (i >= n_items) continue;
      float s = result[a][b];
      if constexpr (ATTENTION) s = s / run_sum[a][b];
      if (user_bias != nullptr) s = s + ub;                      // (pred + ub) + ib, left to right
      if (item_bias != nullptr) s = s + __ldg(item_bias + i);
      out[u * n_items + i] = s;
    }
  }
}

__global__ void l2_normalize_rows_kernel(float* __restrict__ x, int64_t rows, int d) {
  const int lane = threadIdx.x % 32;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / 32;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * blockDim.x / 32;
  for (int64_t r = warp; r < rows; r += n_warps) {
    float ss = 0.0f;
    for (int k = lane; k < d; k += 32) {
      const float v = x[r * d + k];
      ss = fmaf(v, v, ss);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float inv = 1.0f / sqrtf(fmaxf(ss, 1e-12f));
    for (int k = lane; k < d; k += 32) x[r * d + k] *= inv;
  }
}

int score_f32(const float* user_repr, const float* attention_repr, const float* item_repr,
              const float* user_bias, const float* item_bias, float* out, int64_t n_users, int64_t n_items,
              int32_t d, int32_t n_tastes, int32_t mode, cudaStream_t stream) {
  TRK_CHECK_ARG(user_repr && item_repr && out, "score_f32: null pointer");
  TRK_CHECK_ARG(n_users >= 0 && n_items >= 0 && d >= 1 && n_tastes >= 1, "score_f32: bad sizes");
  TRK_CHECK_ARG(mode == 0 || mode == 1, "score_f32: mode must be 0 (dot) or 1 (euclidean)");
  TRK_CHECK_ARG(!(attention_repr && mode != 0), "score_f32: attention is only defined for the dot product path");
  if (n_users == 0 || n_items == 0) return TRK_OK;
  const int64_t gy = ceil_div(n_users, kTileM), gx = ceil_div(n_items, kTileN);
  TRK_CHECK_ARG(gy <= 65535, "score_f32: n_users=%lld exceeds one launch; block the user axis",
                static_cast<long long>(n_users));
  const dim3 grid(static_cast<unsigned>(gx), static_cast<unsigned>(gy));
  if (attention_repr != nullptr) {
    score_simt_kernel<0, true><<<grid, kSimtThreads, 0, stream>>>(user_repr, attention_repr, item_repr, user_bias,
                                                                 item_bias, out, n_users, n_items, d, n_tastes);
  } else if (mode == 0) {
    score_simt_kernel<0, false><<<grid, kSimtThreads, 0, stream>>>(user_repr, nullptr, item_repr, user_bias,
                                                                  item_bias, out, n_users, n_items, d, n_tastes);
  } else {
    score_simt_kernel<1, false><<<grid, kSimtThreads, 0, stream>>>(user_repr, nullptr, item_repr, user_bias,
                                                                  item_bias, out, n_users, n_items, d, n_tastes);
  }
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

int l2_normalize_rows(float* x, int64_t rows, int32_t d, cudaStream_t stream) {
  TRK_CHECK_ARG(x && rows >= 0 && d >= 1, "l2_normalize_rows: bad arguments");
  if (rows == 0) return TRK_OK;
  const int threads = 256;
  l2_normalize_rows_kernel<<<capped_grid(ceil_div(rows, threads / 32), 8), threads, 0, stream>>>(x, rows, d);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

}  // namespace trk
