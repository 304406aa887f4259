// The sampled-rank training step (SURVEY 8 row f1; BASELINE config "WMRBLossGraph sampled-rank training step"):
//
//   sample_items_kernel   tensorrec/util.py:12-21 (np.random.choice per user behind tf.py_func, tensorrec.py:298-302):
//                         n_sampled item ids per user, with or without replacement, from a counter-based Philox4x32-10
//                         stream (seed, step, user, draw) -- no [n_users, n_items] temporary, no host round trip;
//   wmrb_step_kernel      forward AND backward of everything between the representations and the loss, one warp per user:
//                           serial predictions       DotProductPredictionGraph.connect_serial_prediction_graph
//                                                    (tensorrec/prediction_graphs.py:52-55: gather, multiply, reduce_sum)
//                           + biases                 bias_prediction_serial (tensorrec/recommendation_graphs.py:44-57)
//                           of the user's interactions and of its sampled items (densify_sampled_item_predictions,
//                           recommendation_graphs.py:60-70, is the [user, sample] indexing here),
//                           loss                     WMRBLossGraph.weighted_margin_rank_batch (tensorrec/loss_graphs.py:
//                                                    153-180) / BalancedWMRBLossGraph (:190-227):
//                                                    log(1 + n_items / n_sampled * sum_s max(0, 1 - positive + sample_s) [* w]),
//                           backward                 d loss / d (user row, user bias) accumulated in registers and written
//                                                    once per user; d loss / d (item rows, item biases) added with
//                                                    red.global.add (the scatter-add of tf.gather's gradient);
//   adam_step_kernel      tf.train.AdamOptimizer.minimize(basic_loss + alpha * sum l2_loss(w)) (tensorrec.py:487-489):
//                         L2 term, moment updates and the parameter step in one pass over every weight.
//
// The sparse x dense products on either side (representations forward, weight gradients backward) are K1
// (csr_gather.cu) on the CSR of the features / of their transpose.  HBM-bound: the step gathers one item row per
// (user, interaction or sample) pair, twice (the second time from L2).
#include <cuda_bf16.h>

#include "common.cuh"

namespace trk {

// ---------------------------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al., SC'11): counter-based, every (seed, step, user, draw) has its own 128-bit block
// ---------------------------------------------------------------------------------------------------------
__host__ __device__ inline void philox_round(uint32_t (&c)[4], uint32_t (&k)[2]) {
  const uint64_t p0 = static_cast<uint64_t>(0xD2511F53u) * c[0];
  const uint64_t p1 = static_cast<uint64_t>(0xCD9E8D57u) * c[2];
  const uint32_t n0 = static_cast<uint32_t>(p1 >> 32) ^ c[1] ^ k[0];
  const uint32_t n1 = static_cast<uint32_t>(p1);
  const uint32_t n2 = static_cast<uint32_t>(p0 >> 32) ^ c[3] ^ k[1];
  const uint32_t n3 = static_cast<uint32_t>(p0);
  c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
  k[0] += 0x9E3779B9u;
  k[1] += 0xBB67AE85u;
}
__host__ __device__ inline uint64_t philox_u64(uint64_t seed, uint32_t step, uint32_t user, uint32_t draw) {
  uint32_t c[4] = {user, draw, step, 0x7452656bu};
  uint32_t k[2] = {static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32)};
#pragma unroll
  for (int r = 0; r < 10; ++r) philox_round(c, k);
  return (static_cast<uint64_t>(c[0]) << 32) | c[1];
}
// uniform integer in [0, n): the high 64 bits of r * n (bias < n / 2^64)
__device__ __forceinline__ uint32_t bounded(uint64_t r, uint32_t n) {
  return static_cast<uint32_t>(__umul64hi(r, static_cast<uint64_t>(n)));
}

constexpr int kSampleWarps = 8;

// One warp per user.  With replacement: draw j = bounded(philox(user, j), n_items).  Without: Robert Floyd's algorithm --
// for j = n_items - S .. n_items - 1: t = uniform[0, j]; take t unless it was already taken, then take j -- which yields
// every S-subset with equal probability using S draws and an S-entry list (the membership test is a warp-parallel scan
// of that list: O(S^2 / 32) per user).
template <bool kReplace>
__global__ void __launch_bounds__(kSampleWarps * 32)
sample_items_kernel(int64_t n_users, uint32_t n_items, int n_sampled, uint64_t seed, uint32_t step,
                    int32_t* __restrict__ out) {
  extern __shared__ int32_t s_chosen[];
  const int lane = threadIdx.x % 32, wib = threadIdx.x / 32;
  int32_t* chosen = s_chosen + wib * n_sampled;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * kSampleWarps;
  for (int64_t u = static_cast<int64_t>(blockIdx.x) * kSampleWarps + wib; u < n_users; u += n_warps) {
    int32_t* row = out + u * n_sampled;
    if (kReplace) {
      for (int j = lane; j < n_sampled; j += 32)
        row[j] = static_cast<int32_t>(bounded(philox_u64(seed, step, static_cast<uint32_t>(u), j), n_items));
    } else {
      // the S Philox blocks are independent: lanes draw them in parallel (t_jj uniform in [0, n_items - S + jj]) ...
      for (int jj = lane; jj < n_sampled; jj += 32) {
        const uint32_t j = n_items - static_cast<uint32_t>(n_sampled) + jj;
        chosen[jj] = static_cast<int32_t>(bounded(philox_u64(seed, step, static_cast<uint32_t>(u), jj), j + 1));
      }
      __syncwarp();
      // ... only the "already taken?" test is sequential: entry jj is compared with the final entries [0, jj)
      for (int jj = 1; jj < n_sampled; ++jj) {
        const int32_t t = chosen[jj];
        bool found = false;
        for (int q = lane; q < jj; q += 32) found |= chosen[q] == t;
        if (__any_sync(0xffffffffu, found)) {
          if (lane == 0) chosen[jj] = static_cast<int32_t>(n_items - static_cast<uint32_t>(n_sampled) + jj);
          __syncwarp();
        }
      }
      for (int j = lane; j < n_sampled; j += 32) row[j] = chosen[j];
      __syncwarp();
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// representation rows: fp32 or bf16 storage, fp32 arithmetic
// ---------------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ void load4(const T* __restrict__ p, float (&x)[4]);
template <>
__device__ __forceinline__ void load4<float>(const float* __restrict__ p, float (&x)[4]) {
  const float4 v = __ldg(reinterpret_cast<const float4*>(p));
  x[0] = v.x; x[1] = v.y; x[2] = v.z; x[3] = v.w;
}
template <>
__device__ __forceinline__ void load4<__nv_bfloat16>(const __nv_bfloat16* __restrict__ p, float (&x)[4]) {
  const uint2 v = __ldg(reinterpret_cast<const uint2*>(p));
  const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v.x));
  const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v.y));
  x[0] = a.x; x[1] = a.y; x[2] = b.x; x[3] = b.y;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

struct WmrbParams {
  const void* user_repr;        // [n_users, d]
  const void* item_repr;        // [n_items, d]
  const float* user_bias;       // [n_users] or null (biased = False)
  const float* item_bias;       // [n_items] or null
  const int32_t* inter_indptr;  // interactions as CSR by user, entries in the reference's COO order
  const int32_t* inter_item;
  const float* inter_val;
  const float* item_weight_sum; // BalancedWMRB: sum of the positive interaction values per item, else null
  const int32_t* samples;       // [n_users, n_sampled]
  int64_t n_users;
  int32_t n_items;
  int32_t d;
  int32_t n_sampled;
  float rank_scale;             // n_items / n_sampled (float32, as tf.cast(...) / tf.cast(...))
  float* loss;                  // [nnz]: log(sampled margin rank + 1) of the positive interactions, 0 elsewhere
  float* pred_serial;           // [nnz]: the serial prediction of every interaction
  float* coef;                  // [nnz] scratch: d(sum of losses) / d(prediction of the interaction)
  float* d_user_repr;           // [n_users, d]
  float* d_user_bias;           // [n_users] or null
  float* d_item_repr;           // [n_items, d], zeroed by the caller: added to with red.global.add
  float* d_item_bias;           // [n_items] or null, zeroed by the caller
};

constexpr int kWmrbWarps = 4;

// CH: 128-column chunks per row (d <= 128 * CH, d a multiple of 4): lane l holds elements [4 (l + 32 c), +4) of chunk c.
template <typename T, int CH>
__global__ void __launch_bounds__(kWmrbWarps * 32)
wmrb_step_kernel(const WmrbParams p) {
  extern __shared__ float s_wmrb[];
  const int lane = threadIdx.x % 32, wib = threadIdx.x / 32;
  float* sp = s_wmrb + wib * 2 * p.n_sampled;   // sample predictions of this warp's user
  float* gs = sp + p.n_sampled;                 // d(sum of losses) / d(sample prediction)
  const T* user_repr = static_cast<const T*>(p.user_repr);
  const T* item_repr = static_cast<const T*>(p.item_repr);
  const int d = p.d, S = p.n_sampled;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * kWmrbWarps;

  for (int64_t u = static_cast<int64_t>(blockIdx.x) * kWmrbWarps + wib; u < p.n_users; u += n_warps) {
    float uv[CH][4];
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int e = 4 * (lane + 32 * c);
      if (e < d) load4<T>(user_repr + u * d + e, uv[c]);
      else uv[c][0] = uv[c][1] = uv[c][2] = uv[c][3] = 0.0f;
    }
    const float ub = p.user_bias != nullptr ? __ldg(p.user_bias + u) : 0.0f;
    const int32_t* srow = p.samples + u * S;
    const int a = __ldg(p.inter_indptr + u), b = __ldg(p.inter_indptr + u + 1);

    // prediction of (this user, item id): (sum_k u_k i_k + user bias) + item bias -- the order of
    // bias_prediction_serial; the k-sum is a per-lane FMA chain + xor tree (deterministic)
    auto predict4 = [&](const int32_t (&ids)[4], int n_valid, float (&out)[4]) {
      float part[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        part[q] = 0.0f;
        if (q < n_valid) {
#pragma unroll
          for (int c = 0; c < CH; ++c) {
            const int e = 4 * (lane + 32 * c);
            if (e < d) {
              float iv[4];
              load4<T>(item_repr + static_cast<int64_t>(ids[q]) * d + e, iv);
#pragma unroll
              for (int w = 0; w < 4; ++w) part[q] = fmaf(uv[c][w], iv[w], part[q]);
            }
          }
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float dot = warp_sum(part[q]);
        float s = dot;
        if (q < n_valid) {
          if (p.user_bias != nullptr) s = s + ub;
          if (p.item_bias != nullptr) s = s + __ldg(p.item_bias + ids[q]);
        }
        out[q] = s;
      }
    };

    // ---- forward 1: the sampled items ----
    for (int j0 = 0; j0 < S; j0 += 4) {
      int32_t ids[4];
      const int nv = min(4, S - j0);
#pragma unroll
      for (int q = 0; q < 4; ++q) ids[q] = q < nv ? __ldg(srow + j0 + q) : 0;
      float s[4];
      predict4(ids, nv, s);
      if (lane < nv) {
        sp[j0 + lane] = s[lane == 0 ? 0 : lane == 1 ? 1 : lane == 2 ? 2 : 3];
        gs[j0 + lane] = 0.0f;
      }
    }
    __syncwarp();

    // ---- forward 2 + loss: the user's interactions ----
    for (int n0 = a; n0 < b; n0 += 4) {
      int32_t ids[4];
      const int nv = min(4, b - n0);
#pragma unroll
      for (int q = 0; q < 4; ++q) ids[q] = q < nv ? __ldg(p.inter_item + n0 + q) : 0;
      float pr[4];
      predict4(ids, nv, pr);
      for (int q = 0; q < nv; ++q) {      // warp-uniform
        const float val = __ldg(p.inter_val + n0 + q);
        float loss = 0.0f, coef = 0.0f;
        if (val > 0.0f) {                 // loss_graphs.py:155 positive_interaction_mask
          const float base = 1.0f - pr[q];
          float sum = 0.0f;
          for (int j = lane; j < S; j += 32) sum += fmaxf(base + sp[j], 0.0f);       // :171-174
          sum = warp_sum(sum);
          float smr = p.rank_scale * sum, w = p.rank_scale;                          // :177
          if (p.item_weight_sum != nullptr) {                                        // :221-223, left to right
            const float gsum = __ldg(p.item_weight_sum + ids[q]);
            smr = smr * val / gsum;
            w = w * val / gsum;
          }
          loss = logf(smr + 1.0f);                                                   // :179
          const float dsum = w / (smr + 1.0f);      // d loss / d sum
          int active = 0;
          for (int j = lane; j < S; j += 32) {
            if (base + sp[j] >= 0.0f) {             // tf.maximum passes the gradient to its first argument on ties
              gs[j] += dsum;
              active += 1;
            }
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) active += __shfl_xor_sync(0xffffffffu, active, o);
          coef = -dsum * static_cast<float>(active);
        }
        if (lane == 0) {
          p.loss[n0 + q] = loss;
          p.pred_serial[n0 + q] = pr[q];
          p.coef[n0 + q] = coef;
        }
      }
    }
    __syncwarp();

    // ---- backward: d/d user row in registers, d/d item rows by red.global.add ----
    float du[CH][4];
#pragma unroll
    for (int c = 0; c < CH; ++c) du[c][0] = du[c][1] = du[c][2] = du[c][3] = 0.0f;
    float dub = 0.0f;
    // four pairs at a time: the item rows of all of them are requested before the first FMA (they were read by the
    // forward pass a moment ago: L1 / L2 hits); a pair whose coefficient is zero (inactive hinge) contributes exact
    // zeros and is skipped (warp-uniform)
    auto backward4 = [&](const int32_t (&ids)[4], const float (&g)[4]) {
      float iv[4][CH][4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (g[q] == 0.0f) continue;
#pragma unroll
        for (int c = 0; c < CH; ++c) {
          const int e = 4 * (lane + 32 * c);
          if (e < d) load4<T>(item_repr + static_cast<int64_t>(ids[q]) * d + e, iv[q][c]);
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (g[q] == 0.0f) continue;
        dub += g[q];
#pragma unroll
        for (int c = 0; c < CH; ++c) {
          const int e = 4 * (lane + 32 * c);
          if (e < d) {
#pragma unroll
            for (int w = 0; w < 4; ++w) du[c][w] = fmaf(g[q], iv[q][c][w], du[c][w]);
            red_add_v4(p.d_item_repr + static_cast<int64_t>(ids[q]) * d + e, g[q] * uv[c][0], g[q] * uv[c][1],
                       g[q] * uv[c][2], g[q] * uv[c][3]);
          }
        }
        if (lane == 0 && p.d_item_bias != nullptr) atomicAdd(p.d_item_bias + ids[q], g[q]);
      }
    };
    for (int j0 = 0; j0 < S; j0 += 4) {
      int32_t ids[4];
      float g[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const bool ok = j0 + q < S;
        ids[q] = ok ? __ldg(srow + j0 + q) : 0;
        g[q] = ok ? gs[j0 + q] : 0.0f;
      }
      backward4(ids, g);
    }
    for (int n0 = a; n0 < b; n0 += 4) {
      int32_t ids[4];
      float g[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const bool ok = n0 + q < b;
        ids[q] = ok ? __ldg(p.inter_item + n0 + q) : 0;
        // coef was written by lane 0 of this warp: that lane reads it back and broadcasts
        const float mine = (ok && lane == 0) ? p.coef[n0 + q] : 0.0f;
        g[q] = __shfl_sync(0xffffffffu, mine, 0);
      }
      backward4(ids, g);
    }
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int e = 4 * (lane + 32 * c);
      if (e < d)
        *reinterpret_cast<float4*>(p.d_user_repr + u * d + e) = make_float4(du[c][0], du[c][1], du[c][2], du[c][3]);
    }
    if (lane == 0 && p.d_user_bias != nullptr) p.d_user_bias[u] = dub;
    __syncwarp();
  }
}

__global__ void f32_to_bf16_kernel(const float* __restrict__ x, int64_t n, __nv_bfloat16* __restrict__ out) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    out[i] = __float2bfloat16_rn(x[i]);
}

// Adam as TensorFlow's ApplyAdam kernel evaluates it, in float32 (lr_t = lr sqrt(1 - b2^t) / (1 - b1^t) is formed by the
// host, with the running float32 powers of the betas):
//   g = grad + l2 * w;  m += (g - m) (1 - b1);  v += (g g - v) (1 - b2);  w -= (m lr_t) / (sqrt(v) + eps)
__global__ void adam_step_kernel(float* __restrict__ w, const float* __restrict__ grad, float* __restrict__ m,
                                 float* __restrict__ v, int64_t n, float lr_t, float b1, float b2, float eps, float l2) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float wi = w[i];
    const float g = grad[i] + l2 * wi;
    float mi = m[i], vi = v[i];
    mi = mi + (g - mi) * (1.0f - b1);
    vi = vi + (g * g - vi) * (1.0f - b2);
    m[i] = mi;
    v[i] = vi;
    w[i] = wi - (mi * lr_t) / (sqrtf(vi) + eps);
  }
}

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
int sample_items(int64_t n_users, int64_t n_items, int32_t n_sampled, int32_t replace, uint64_t seed, uint32_t step,
                 int32_t* out, cudaStream_t stream) {
  TRK_CHECK_ARG(out && n_users >= 0 && n_items >= 1 && n_items < (1ll << 31) && n_sampled >= 1,
                "sample_items: bad arguments");
  TRK_CHECK_ARG(n_users < (1ll << 32), "sample_items: n_users exceeds the counter width");
  TRK_CHECK_ARG(replace || n_sampled <= n_items, "sample_items: cannot take a larger sample than population when replace=False");
  if (!replace && n_sampled > 4096) {
    set_error("sample_items: n_sampled=%d without replacement exceeds 4096", n_sampled);
    return TRK_ERR_UNSUPPORTED;
  }
  if (n_users == 0) return TRK_OK;
  const int grid = capped_grid(ceil_div(n_users, kSampleWarps), 8);
  if (replace) {
    sample_items_kernel<true><<<grid, kSampleWarps * 32, 0, stream>>>(n_users, static_cast<uint32_t>(n_items), n_sampled,
                                                                      seed, step, out);
  } else {
    const size_t smem = static_cast<size_t>(kSampleWarps) * n_sampled * sizeof(int32_t);
    if (smem > 48 * 1024)
      TRK_CHECK_CUDA(cudaFuncSetAttribute(sample_items_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          static_cast<int>(smem)));
    sample_items_kernel<false><<<grid, kSampleWarps * 32, smem, stream>>>(n_users, static_cast<uint32_t>(n_items),
                                                                          n_sampled, seed, step, out);
  }
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

template <typename T>
static int launch_wmrb(const WmrbParams& p, cudaStream_t stream) {
  const int ch = static_cast<int>(ceil_div(p.d, 128));
  const size_t smem = static_cast<size_t>(kWmrbWarps) * 2 * p.n_sampled * sizeof(float);
  const int grid = capped_grid(ceil_div(p.n_users, kWmrbWarps), 16);
#define TRK_WMRB_LAUNCH(CH)                                                                                   \
  do {                                                                                                        \
    if (smem > 48 * 1024)                                                                                     \
      TRK_CHECK_CUDA(cudaFuncSetAttribute(wmrb_step_kernel<T, CH>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                          static_cast<int>(smem)));                                           \
    wmrb_step_kernel<T, CH><<<grid, kWmrbWarps * 32, smem, stream>>>(p);                                      \
  } while (0)
  if (ch == 1) TRK_WMRB_LAUNCH(1);
  else if (ch == 2) TRK_WMRB_LAUNCH(2);
  else TRK_WMRB_LAUNCH(4);
#undef TRK_WMRB_LAUNCH
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

int wmrb_step(const void* user_repr, const void* item_repr, int32_t repr_is_bf16, const float* user_bias,
              const float* item_bias, const int32_t* inter_indptr, const int32_t* inter_item, const float* inter_val,
              const float* item_weight_sum, const int32_t* samples, int64_t n_users, int64_t n_items, int32_t d,
              int32_t n_sampled, float* loss, float* pred_serial, float* coef, float* d_user_repr, float* d_user_bias,
              float* d_item_repr, float* d_item_bias, cudaStream_t stream) {
  TRK_CHECK_ARG(user_repr && item_repr && inter_indptr && samples, "wmrb_step: null input");
  TRK_CHECK_ARG(loss && pred_serial && coef && d_user_repr && d_item_repr, "wmrb_step: null output");
  TRK_CHECK_ARG((user_bias == nullptr) == (item_bias == nullptr), "wmrb_step: biases must be given together");
  TRK_CHECK_ARG((user_bias == nullptr) == (d_user_bias == nullptr) && (item_bias == nullptr) == (d_item_bias == nullptr),
                "wmrb_step: bias gradients must match the biases");
  TRK_CHECK_ARG(n_users >= 0 && n_items >= 1 && n_items < (1ll << 31) && n_sampled >= 1, "wmrb_step: bad sizes");
  if (d < 4 || d % 4 != 0 || d > 512 || n_sampled > 2048) {
    set_error("wmrb_step: n_components=%d (multiple of 4, <= 512) / n_sampled=%d (<= 2048) outside the fused kernel", d,
              n_sampled);
    return TRK_ERR_UNSUPPORTED;
  }
  TRK_CHECK_ARG(reinterpret_cast<uintptr_t>(user_repr) % 16 == 0 && reinterpret_cast<uintptr_t>(item_repr) % 16 == 0 &&
                    reinterpret_cast<uintptr_t>(d_user_repr) % 16 == 0 && reinterpret_cast<uintptr_t>(d_item_repr) % 16 == 0,
                "wmrb_step: rows must be 16-byte aligned");
  if (n_users == 0) return TRK_OK;
  WmrbParams p;
  p.user_repr = user_repr;
  p.item_repr = item_repr;
  p.user_bias = user_bias;
  p.item_bias = item_bias;
  p.inter_indptr = inter_indptr;
  p.inter_item = inter_item;
  p.inter_val = inter_val;
  p.item_weight_sum = item_weight_sum;
  p.samples = samples;
  p.n_users = n_users;
  p.n_items = static_cast<int32_t>(n_items);
  p.d = d;
  p.n_sampled = n_sampled;
  p.rank_scale = static_cast<float>(n_items) / static_cast<float>(n_sampled);
  p.loss = loss;
  p.pred_serial = pred_serial;
  p.coef = coef;
  p.d_user_repr = d_user_repr;
  p.d_user_bias = d_user_bias;
  p.d_item_repr = d_item_repr;
  p.d_item_bias = d_item_bias;
  return repr_is_bf16 ? launch_wmrb<__nv_bfloat16>(p, stream) : launch_wmrb<float>(p, stream);
}

int f32_to_bf16(const float* x, int64_t n, void* out, cudaStream_t stream) {
  TRK_CHECK_ARG(x && out && n >= 0, "f32_to_bf16: bad arguments");
  if (n == 0) return TRK_OK;
  f32_to_bf16_kernel<<<capped_grid(ceil_div(n, 256), 16), 256, 0, stream>>>(
      x, n, static_cast<__nv_bfloat16*>(out));
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

int adam_step(float* w, const float* grad, float* m, float* v, int64_t n, float lr_t, float beta1, float beta2,
              float epsilon, float l2, cudaStream_t stream) {
  TRK_CHECK_ARG(w && grad && m && v && n >= 0, "adam_step: bad arguments");
  if (n == 0) return TRK_OK;
  adam_step_kernel<<<capped_grid(ceil_div(n, 256), 16), 256, 0, stream>>>(w, grad, m, v, n, lr_t, beta1, beta2, epsilon,
                                                                         l2);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

// the sampler's stream on the host: lets tests (and the oracle) reproduce a device sample exactly
uint64_t philox_u64_host(uint64_t seed, uint32_t step, uint32_t user, uint32_t draw) {
  return philox_u64(seed, step, user, draw);
}

}  // namespace trk
