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
//                         The same kernel, templated on the pair form, the collapse and the taste count, trains cosine,
//                         Euclidean, mixture-of-tastes and attention models (trk_wmrb_step_tastes; DESIGN §3.10), with
//                         l2_normalize_rows_step_kernel normalising operands forward and backward;
//   serial losses         RMSELossGraph / SeparationLossGraph (loss_graphs.py:53-59, 75-98; trk_serial_loss_step,
//                         DESIGN §3.11): the same kernel's forward mode, serial_stats_kernel + serial_finish_kernel
//                         (the loss and the state its gradient needs), then the kernel's backward mode;
//   adam_step_kernel      tf.train.AdamOptimizer.minimize(basic_loss + alpha * sum l2_loss(w)) (tensorrec.py:487-489):
//                         L2 term, moment updates and the parameter step in one pass over every weight.
//
// The sparse x dense products on either side (representations forward, weight gradients backward) are K1
// (csr_gather.cu) on the CSR of the features / of their transpose.  HBM-bound: the step gathers one item row per
// (user, interaction or sample) pair, twice (the second time from L2).
#include <cuda_bf16.h>

#include <algorithm>
#include <type_traits>

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
  const void* serial_state;     // serial backward: the SerialLossState serial_finish_kernel wrote
  int32_t serial_loss;          // serial backward: kSerialRmse | kSerialSeparation
};

constexpr int kWmrbWarps = 4;

// What one launch of wmrb_step_kernel does: the fused WMRB step (forward, loss and backward in one pass), or one half
// of a serial-loss step (trk_serial_loss_step; DESIGN §3.11), whose global statistics need a launch in between:
//   kModeSerialForward   writes pred_serial of every interaction and nothing else;
//   kModeSerialBackward  reads pred_serial back, forms d loss / d prediction from the loss state, and runs the backward.
constexpr int kModeWmrb = 0, kModeSerialForward = 1, kModeSerialBackward = 2;
constexpr int kSerialRmse = 0, kSerialSeparation = 1;

// The gradient of a serial loss with respect to one prediction p of value y is g = a_k + b_k (p - mu_k), k the group of
// y (0: y > 0, 1: y <= 0) for Separation; RMSE has g = b_0 (p - y).
struct SerialLossState {
  float a[2], b[2], mu[2];
};

__device__ __forceinline__ float serial_grad(const WmrbParams& p, int n) {
  const SerialLossState* st = static_cast<const SerialLossState*>(p.serial_state);
  const float pr = p.pred_serial[n], y = __ldg(p.inter_val + n);
  if (p.serial_loss == kSerialRmse) return (pr - y) * st->b[0];
  const int k = y > 0.0f ? 0 : 1;
  return st->a[k] + st->b[k] * (pr - st->mu[k]);
}

// The forms of the step (trk_wmrb_step_tastes; trk_wmrb_step is the dot / single-taste form):
//   pair      the scalar function of a pair's operand rows, evaluated as a "row form" f per (pair, operand row):
//             kPairDot     f = u . i, score f (cosine: the same on rows the caller has L2-normalised);
//             kPairEuclid  f = sum_k (u_k - i_k)^2, score -sqrt(max(f, 1e-16)) (prediction_graphs.py:102-117);
//   collapse  over the tastes (recommendation_graphs.py:85-109): one taste; max_t score_t; or
//             sum_t softmax_t(a_t) score_t with a_t the score of the attention row -- of the user row itself for the
//             sampled items (tensorrec.py:367-372).
constexpr int kPairDot = 0, kPairEuclid = 1;
constexpr int kCollapseSingle = 0, kCollapseMax = 1, kCollapseAttention = 2;
constexpr float kEuclidEps = 1e-16f;

template <int kPair>
__device__ __forceinline__ float pair_score(float f) {
  if constexpr (kPair == kPairEuclid) return -sqrtf(fmaxf(f, kEuclidEps));
  else return f;
}

// the max collapse: max_t score_t
template <int kPair, int NT, int NF>
__device__ __forceinline__ float max_score(const float (&f)[NF]) {
  float m = pair_score<kPair>(f[0]);
#pragma unroll
  for (int t = 1; t < NT; ++t) m = fmaxf(m, pair_score<kPair>(f[t]));
  return m;
}

// the attention collapse: the scores s_t, the softmax weights w_t of the attention scores a_t (a sample's are its own
// scores) and the prediction sum_t w_t s_t
template <int kPair, int NT, bool kSample, int NF>
__device__ __forceinline__ float softmax_collapse(const float (&f)[NF], float (&s)[NT], float (&w)[NT]) {
  float a[NT];
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    s[t] = pair_score<kPair>(f[t]);
    a[t] = kSample ? s[t] : pair_score<kPair>(f[NT + t]);
  }
  float m = a[0];
#pragma unroll
  for (int t = 1; t < NT; ++t) m = fmaxf(m, a[t]);
  float z = 0.0f;
#pragma unroll
  for (int t = 0; t < NT; ++t) z += expf(a[t] - m);
  float pred = 0.0f;
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    w[t] = expf(a[t] - m) / z;
    pred += w[t] * s[t];
  }
  return pred;
}

// the prediction (without biases) of one pair from its row forms f[0, NT) (tastes) and f[NT, 2 NT) (attention rows of
// an interaction; a sample has none)
template <int kPair, int kCollapse, int NT, bool kSample, int NF>
__device__ __forceinline__ float collapse_tastes(const float (&f)[NF]) {
  if constexpr (kCollapse == kCollapseSingle) {
    return pair_score<kPair>(f[0]);
  } else if constexpr (kCollapse == kCollapseMax) {
    return max_score<kPair, NT>(f);
  } else {
    float s[NT], w[NT];
    return softmax_collapse<kPair, NT, kSample>(f, s, w);
  }
}

// c[r] = the coefficient of operand row r in the gradient of one pair whose prediction has gradient g:
//   dot:    d u_r = c_r i,        d i += c_r u_r         (c_r = g d pred / d f_r)
//   euclid: d u_r = c_r (i - u_r), d i += c_r (u_r - i)  (c_r = g d pred / d score_r / sqrt(f_r); 0 below the clamp,
//                                                        where tf.maximum passes no gradient to f)
// The max collapse splits g evenly among tied tastes (tf.reduce_max's gradient).
template <int kPair, int kCollapse, int NT, bool kSample, int NF>
__device__ __forceinline__ void taste_coefs(const float (&f)[NF], float g, float (&c)[NF]) {
  float ds[NF];
  if constexpr (kCollapse == kCollapseSingle) {
    ds[0] = g;
  } else if constexpr (kCollapse == kCollapseMax) {
    const float m = max_score<kPair, NT>(f);
    float n_max = 0.0f;
#pragma unroll
    for (int t = 0; t < NT; ++t) n_max += pair_score<kPair>(f[t]) == m ? 1.0f : 0.0f;
    const float share = g / n_max;
#pragma unroll
    for (int t = 0; t < NT; ++t) ds[t] = pair_score<kPair>(f[t]) == m ? share : 0.0f;
  } else {
    float s[NT], w[NT];
    const float pred = softmax_collapse<kPair, NT, kSample>(f, s, w);
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      const float da = g * w[t] * (s[t] - pred);    // d pred / d a_t = w_t (s_t - pred)
      ds[t] = g * w[t];
      if constexpr (kSample) ds[t] += da;           // a_t is s_t itself
      else ds[NT + t] = da;
    }
  }
#pragma unroll
  for (int r = 0; r < NF; ++r) {
    if constexpr (kPair == kPairEuclid) c[r] = f[r] >= kEuclidEps ? ds[r] / sqrtf(f[r]) : 0.0f;
    else c[r] = ds[r];
  }
}

// CH: 128-column chunks per row (d <= 128 * CH, d a multiple of 4): lane l holds elements [4 (l + 32 c), +4) of chunk c.
// NT tastes; the user operand is NR = NT (or 2 NT with attention: the attention rows follow the taste rows) planes
// [n_users, d], plane r at user_repr + r * n_users * d, and so is d_user_repr.  The dot / single-taste form (kPlain) is
// the step of trk_wmrb_step; the other forms recompute a pair's row forms in the backward pass (from the item row
// gathered there anyway) instead of keeping NT values per sample.  kMode selects the WMRB step or one half of a serial
// step; the serial modes touch neither the samples nor shared memory.
template <typename T, int CH, int kPair = kPairDot, int kCollapse = kCollapseSingle, int NT = 1, int kMode = kModeWmrb>
__global__ void __launch_bounds__(kWmrbWarps * 32)
wmrb_step_kernel(const WmrbParams p) {
  constexpr bool kPlain = kPair == kPairDot && kCollapse == kCollapseSingle;
  constexpr int NR = kCollapse == kCollapseAttention ? 2 * NT : NT;
  extern __shared__ float s_wmrb[];
  const int lane = threadIdx.x % 32, wib = threadIdx.x / 32;
  float* sp = s_wmrb + wib * 2 * p.n_sampled;   // sample predictions of this warp's user
  float* gs = sp + p.n_sampled;                 // d(sum of losses) / d(sample prediction)
  const T* user_repr = static_cast<const T*>(p.user_repr);
  const T* item_repr = static_cast<const T*>(p.item_repr);
  const int d = p.d, S = p.n_sampled;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * kWmrbWarps;
  const int64_t plane = p.n_users * d;

  for (int64_t u = static_cast<int64_t>(blockIdx.x) * kWmrbWarps + wib; u < p.n_users; u += n_warps) {
    float uv[NR][CH][4];
#pragma unroll
    for (int r = 0; r < NR; ++r) {
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const int e = 4 * (lane + 32 * c);
        if (e < d) load4<T>(user_repr + r * plane + u * d + e, uv[r][c]);
        else uv[r][c][0] = uv[r][c][1] = uv[r][c][2] = uv[r][c][3] = 0.0f;
      }
    }
    const float ub = p.user_bias != nullptr ? __ldg(p.user_bias + u) : 0.0f;
    const int32_t* srow = p.samples + u * S;
    const int a = __ldg(p.inter_indptr + u), b = __ldg(p.inter_indptr + u + 1);

    // row forms of (this user's first NU operand rows, one 4-element chunk c of an item row): a per-lane FMA chain, then
    // an xor tree (deterministic: the backward pass recomputes exactly the values of the forward pass)
    auto row_part = [&](auto nu, int c, const float (&iv)[4], float (&part)[decltype(nu)::value]) {
      constexpr int NU = decltype(nu)::value;
#pragma unroll
      for (int r = 0; r < NU; ++r)
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          if constexpr (kPair == kPairEuclid) {
            const float diff = uv[r][c][w] - iv[w];
            part[r] = fmaf(diff, diff, part[r]);
          } else {
            part[r] = fmaf(uv[r][c][w], iv[w], part[r]);
          }
        }
    };

    // prediction of (this user, item id): (collapse of the pair's scores + user bias) + item bias -- the order of
    // bias_prediction_serial.  nu: the operand rows the pair uses (NT for a sample, NR for an interaction)
    auto predict4 = [&](auto nu, const int32_t (&ids)[4], int n_valid, float (&out)[4]) {
      constexpr int NU = decltype(nu)::value;
      float part[4][NU];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
#pragma unroll
        for (int r = 0; r < NU; ++r) part[q][r] = 0.0f;
        if (q < n_valid) {
#pragma unroll
          for (int c = 0; c < CH; ++c) {
            const int e = 4 * (lane + 32 * c);
            if (e < d) {
              float iv[4];
              load4<T>(item_repr + static_cast<int64_t>(ids[q]) * d + e, iv);
              row_part(nu, c, iv, part[q]);
            }
          }
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float f[NU];
#pragma unroll
        for (int r = 0; r < NU; ++r) f[r] = warp_sum(part[q][r]);
        float s = collapse_tastes<kPair, kCollapse, NT, NU == NT && NR != NT>(f);
        if (q < n_valid) {
          if (p.user_bias != nullptr) s = s + ub;
          if (p.item_bias != nullptr) s = s + __ldg(p.item_bias + ids[q]);
        }
        out[q] = s;
      }
    };
    using SampleRows = std::integral_constant<int, NT>;
    using PairRows = std::integral_constant<int, NR>;

    // ---- forward 1: the sampled items ----
    if constexpr (kMode == kModeWmrb) {
      for (int j0 = 0; j0 < S; j0 += 4) {
        int32_t ids[4];
        const int nv = min(4, S - j0);
#pragma unroll
        for (int q = 0; q < 4; ++q) ids[q] = q < nv ? __ldg(srow + j0 + q) : 0;
        float s[4];
        predict4(SampleRows{}, ids, nv, s);
        if (lane < nv) {
          sp[j0 + lane] = s[lane == 0 ? 0 : lane == 1 ? 1 : lane == 2 ? 2 : 3];
          gs[j0 + lane] = 0.0f;
        }
      }
      __syncwarp();
    }

    // ---- forward 2 + loss: the user's interactions ----
    if constexpr (kMode != kModeSerialBackward) {
      for (int n0 = a; n0 < b; n0 += 4) {
        int32_t ids[4];
        const int nv = min(4, b - n0);
#pragma unroll
        for (int q = 0; q < 4; ++q) ids[q] = q < nv ? __ldg(p.inter_item + n0 + q) : 0;
        float pr[4];
        predict4(PairRows{}, ids, nv, pr);
        if constexpr (kMode == kModeSerialForward) {
          float mine = pr[0];               // lane q stores pr[q]: selects, not a local-memory array
#pragma unroll
          for (int q = 1; q < 4; ++q) mine = lane == q ? pr[q] : mine;
          if (lane < nv) p.pred_serial[n0 + lane] = mine;
        } else {
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
      }
      __syncwarp();
    }

    // ---- backward: d/d user rows in registers, d/d item rows by red.global.add ----
    if constexpr (kMode != kModeSerialForward) {
      float du[NR][CH][4];
#pragma unroll
      for (int r = 0; r < NR; ++r)
#pragma unroll
        for (int c = 0; c < CH; ++c) du[r][c][0] = du[r][c][1] = du[r][c][2] = du[r][c][3] = 0.0f;
      float dub = 0.0f;
      float csum[NR];                   // euclid: sum over the pairs of c_r, the coefficient of -u_r in d u_r
#pragma unroll
      for (int r = 0; r < NR; ++r) csum[r] = 0.0f;
      // four pairs at a time: the item rows of all of them are requested before the first FMA (they were read by the
      // forward pass a moment ago: L1 / L2 hits); a pair whose coefficient is zero (inactive hinge) contributes exact
      // zeros and is skipped (warp-uniform).  Each pair's item gradient, summed over the operand rows, is one red.add.
      auto backward4 = [&](auto nu, const int32_t (&ids)[4], const float (&g)[4]) {
        constexpr int NU = decltype(nu)::value;
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
          float cr[NU];
          if constexpr (kPlain) {
            cr[0] = g[q];
          } else {
            float part[NU];
#pragma unroll
            for (int r = 0; r < NU; ++r) part[r] = 0.0f;
#pragma unroll
            for (int c = 0; c < CH; ++c)
              if (4 * (lane + 32 * c) < d) row_part(nu, c, iv[q][c], part);
            float f[NU];
#pragma unroll
            for (int r = 0; r < NU; ++r) f[r] = warp_sum(part[r]);
            taste_coefs<kPair, kCollapse, NT, NU == NT && NR != NT>(f, g[q], cr);
          }
          float cs = 0.0f;
#pragma unroll
          for (int r = 0; r < NU; ++r) cs += cr[r];
#pragma unroll
          for (int c = 0; c < CH; ++c) {
            const int e = 4 * (lane + 32 * c);
            if (e < d) {
#pragma unroll
              for (int r = 0; r < NU; ++r)
#pragma unroll
                for (int w = 0; w < 4; ++w) du[r][c][w] = fmaf(cr[r], iv[q][c][w], du[r][c][w]);
              float gi[4];
#pragma unroll
              for (int w = 0; w < 4; ++w) {
                if constexpr (kPair == kPairEuclid) gi[w] = -cs * iv[q][c][w];
                else gi[w] = cr[0] * uv[0][c][w];
#pragma unroll
                for (int r = kPair == kPairEuclid ? 0 : 1; r < NU; ++r) gi[w] = fmaf(cr[r], uv[r][c][w], gi[w]);
              }
              red_add_v4(p.d_item_repr + static_cast<int64_t>(ids[q]) * d + e, gi[0], gi[1], gi[2], gi[3]);
            }
          }
          if constexpr (kPair == kPairEuclid) {
#pragma unroll
            for (int r = 0; r < NU; ++r) csum[r] += cr[r];
          }
          if (lane == 0 && p.d_item_bias != nullptr) atomicAdd(p.d_item_bias + ids[q], g[q]);
        }
      };
      if constexpr (kMode == kModeWmrb) {
        for (int j0 = 0; j0 < S; j0 += 4) {
          int32_t ids[4];
          float g[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const bool ok = j0 + q < S;
            ids[q] = ok ? __ldg(srow + j0 + q) : 0;
            g[q] = ok ? gs[j0 + q] : 0.0f;
          }
          backward4(SampleRows{}, ids, g);
        }
      }
      for (int n0 = a; n0 < b; n0 += 4) {
        int32_t ids[4];
        float g[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const bool ok = n0 + q < b;
          ids[q] = ok ? __ldg(p.inter_item + n0 + q) : 0;
          if constexpr (kMode == kModeSerialBackward) {
            g[q] = ok ? serial_grad(p, n0 + q) : 0.0f;    // every lane reads the same words: warp-uniform
          } else {
            // coef was written by lane 0 of this warp: that lane reads it back and broadcasts
            const float mine = (ok && lane == 0) ? p.coef[n0 + q] : 0.0f;
            g[q] = __shfl_sync(0xffffffffu, mine, 0);
          }
        }
        backward4(PairRows{}, ids, g);
      }
#pragma unroll
      for (int r = 0; r < NR; ++r) {
#pragma unroll
        for (int c = 0; c < CH; ++c) {
          const int e = 4 * (lane + 32 * c);
          if (e < d) {
            if constexpr (kPair == kPairEuclid) {
#pragma unroll
              for (int w = 0; w < 4; ++w) du[r][c][w] = fmaf(-csum[r], uv[r][c][w], du[r][c][w]);
            }
            *reinterpret_cast<float4*>(p.d_user_repr + r * plane + u * d + e) =
                make_float4(du[r][c][0], du[r][c][1], du[r][c][2], du[r][c][3]);
          }
        }
      }
      if (lane == 0 && p.d_user_bias != nullptr) p.d_user_bias[u] = dub;
    }
    __syncwarp();
  }
}

// The statistics of a serial loss over the nnz predictions, between the forward and the backward launch:
// serial_stats_kernel (a grid fixed by serial_stats_grid) writes one SerialMoments per block, serial_finish_kernel (one
// block) merges exactly that many in a fixed order and writes the loss and the SerialLossState.  Double throughout:
//   RMSE        group 0 holds the count and the sum of (y - p)^2 (in m2);
//   Separation  per group (0: y > 0, 1: y <= 0) the count, mean and sum of squared deviations, merged pairwise (Chan et
//               al.), so the biased variance m2 / n does not cancel.
struct SerialMoments {
  double n[2], mean[2], m2[2];
};
constexpr int kStatsThreads = 256;
constexpr int kStatsMaxBlocks = 1024;
constexpr int kStatsPerThread = 8;

__device__ __forceinline__ void merge_moments(double& n, double& mean, double& m2, double nb, double meanb,
                                              double m2b) {
  if (nb == 0.0) return;
  if (n == 0.0) {
    n = nb; mean = meanb; m2 = m2b;
    return;
  }
  const double nn = n + nb, delta = meanb - mean;
  mean += delta * (nb / nn);
  m2 += m2b + delta * delta * (n * nb / nn);
  n = nn;
}

// Welford's update of one group's moments by x
__device__ __forceinline__ void welford(double& n, double& mean, double& m2, double x) {
  n += 1.0;
  const double delta = x - mean;
  mean += delta / n;
  m2 = fma(delta, x - mean, m2);
}

// merges b into m: RMSE adds the counts and the sums, Separation merges each group's moments
template <int kLoss>
__device__ __forceinline__ void merge(SerialMoments& m, const SerialMoments& b) {
  for (int k = 0; k < 2; ++k) {
    if constexpr (kLoss == kSerialRmse) {
      m.n[k] += b.n[k];
      m.m2[k] += b.m2[k];
    } else {
      merge_moments(m.n[k], m.mean[k], m.m2[k], b.n[k], b.mean[k], b.m2[k]);
    }
  }
}

// merges s[0, kStatsThreads) into s[0] in a fixed tree order (every thread of the block calls it)
template <int kLoss>
__device__ __forceinline__ void block_merge(SerialMoments* s) {
  const int t = threadIdx.x;
  for (int half = kStatsThreads / 2; half > 0; half /= 2) {
    __syncthreads();
    if (t < half) merge<kLoss>(s[t], s[t + half]);
  }
  __syncthreads();
}

template <int kLoss>
__global__ void __launch_bounds__(kStatsThreads)
serial_stats_kernel(const float* __restrict__ pred, const float* __restrict__ val, int64_t nnz,
                    SerialMoments* __restrict__ partial) {
  __shared__ SerialMoments s[kStatsThreads];
  SerialMoments m = {};
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * kStatsThreads + threadIdx.x; i < nnz;
       i += static_cast<int64_t>(gridDim.x) * kStatsThreads) {
    const float p = pred[i], y = val[i];
    if constexpr (kLoss == kSerialRmse) {
      const double e = static_cast<double>(y) - static_cast<double>(p);
      m.n[0] += 1.0;
      m.m2[0] = fma(e, e, m.m2[0]);
    } else if (y > 0.0f) {
      welford(m.n[0], m.mean[0], m.m2[0], p);
    } else {
      welford(m.n[1], m.mean[1], m.m2[1], p);
    }
  }
  s[threadIdx.x] = m;
  block_merge<kLoss>(s);
  if (threadIdx.x == 0) partial[blockIdx.x] = s[0];
}

template <int kLoss>
__global__ void __launch_bounds__(kStatsThreads)
serial_finish_kernel(const SerialMoments* __restrict__ partial, int n_partial, float* __restrict__ loss,
                     SerialLossState* __restrict__ state) {
  __shared__ SerialMoments s[kStatsThreads];
  SerialMoments m = {};
  for (int j = threadIdx.x; j < n_partial; j += kStatsThreads) merge<kLoss>(m, partial[j]);
  s[threadIdx.x] = m;
  block_merge<kLoss>(s);
  if (threadIdx.x != 0) return;
  SerialLossState st = {};
  double l;
  if constexpr (kLoss == kSerialRmse) {
    // L = sqrt(sum (y - p)^2 / N), dL / dp_n = (p_n - y_n) / (N L)
    const double n = s[0].n[0];
    l = sqrt(s[0].m2[0] / n);
    st.b[0] = static_cast<float>(1.0 / (n * l));
  } else {
    // L = 1 - Phi(-loc / sigma), loc = mu_Q - mu_P, sigma = sqrt(v_Q + v_P), with phi the normal density at -loc / sigma:
    //   n in P: dL / dp_n = -(phi / (sigma |P|)) (1 + loc (p_n - mu_P) / sigma^2)
    //   n in Q: dL / dp_n =  (phi / (sigma |Q|)) (1 - loc (p_n - mu_Q) / sigma^2)
    const double np = s[0].n[0], nq = s[0].n[1];
    const double mp = np > 0.0 ? s[0].mean[0] : nan(""), mq = nq > 0.0 ? s[0].mean[1] : nan("");
    const double loc = mq - mp, var = s[0].m2[1] / nq + s[0].m2[0] / np, sigma = sqrt(var);
    const double z = -loc / sigma;
    l = 1.0 - 0.5 * (1.0 + erf(z * 0.70710678118654752440));
    const double phi = exp(-0.5 * z * z) * 0.39894228040143267794;
    const double ap = -phi / (sigma * np), aq = phi / (sigma * nq);
    st.a[0] = static_cast<float>(ap);
    st.b[0] = static_cast<float>(ap * loc / var);
    st.mu[0] = static_cast<float>(mp);
    st.a[1] = static_cast<float>(aq);
    st.b[1] = static_cast<float>(-aq * loc / var);
    st.mu[1] = static_cast<float>(mq);
  }
  *state = st;
  *loss = static_cast<float>(l);
}

// Row L2-normalisation of an operand of the step, forward and backward, from its raw rows x (K1's output, d <= 512):
//   N(x) = x rsqrt(max(|x|^2, 1e-12))    (tf.nn.l2_normalize; representation_graphs.py:53-58, prediction_graphs.py:67-72)
// applied n_normalize (1 or 2) times.  out (if non-null) receives N^n(x).  grad (if non-null) holds d loss / d N^n(x) and
// is replaced by d loss / d x: through each normalisation, from the last, g <- s g - [|v|^2 >= 1e-12] s^3 (v . g) v with
// v that normalisation's input and s its rsqrt (below the clamp tf.maximum passes nothing to |v|^2: g <- s g).
// One warp per row; lane l holds elements l + 32 k.
constexpr int kNormWarps = 8;
__global__ void __launch_bounds__(kNormWarps * 32)
l2_normalize_rows_step_kernel(const float* __restrict__ x, int64_t rows, int d, int n_normalize, float* __restrict__ out,
                              float* __restrict__ grad) {
  constexpr int K = 16;
  const int lane = threadIdx.x % 32;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * kNormWarps;
  for (int64_t row = static_cast<int64_t>(blockIdx.x) * kNormWarps + threadIdx.x / 32; row < rows; row += n_warps) {
    float v[K];
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] = lane + 32 * k < d ? x[row * d + lane + 32 * k] : 0.0f;
    float scale[2];
    bool clamped[2];
    float y[K];
#pragma unroll
    for (int k = 0; k < K; ++k) y[k] = v[k];
    for (int n = 0; n < n_normalize; ++n) {
      float ss = 0.0f;
#pragma unroll
      for (int k = 0; k < K; ++k) ss = fmaf(y[k], y[k], ss);
      ss = warp_sum(ss);
      scale[n] = 1.0f / sqrtf(fmaxf(ss, 1e-12f));
      clamped[n] = ss < 1e-12f;
#pragma unroll
      for (int k = 0; k < K; ++k) y[k] *= scale[n];
    }
    if (out != nullptr) {
#pragma unroll
      for (int k = 0; k < K; ++k)
        if (lane + 32 * k < d) out[row * d + lane + 32 * k] = y[k];
    }
    if (grad != nullptr) {
      float g[K];
#pragma unroll
      for (int k = 0; k < K; ++k) g[k] = lane + 32 * k < d ? grad[row * d + lane + 32 * k] : 0.0f;
      for (int n = n_normalize - 1; n >= 0; --n) {
        // the input of normalisation n: x, or N(x) for the second one
        float in[K];
#pragma unroll
        for (int k = 0; k < K; ++k) in[k] = n == 0 ? v[k] : v[k] * scale[0];
        float vg = 0.0f;
#pragma unroll
        for (int k = 0; k < K; ++k) vg = fmaf(in[k], g[k], vg);
        vg = warp_sum(vg);
        const float s = scale[n];
        const float t = clamped[n] ? 0.0f : s * s * s * vg;
#pragma unroll
        for (int k = 0; k < K; ++k) g[k] = s * g[k] - t * in[k];
      }
#pragma unroll
      for (int k = 0; k < K; ++k)
        if (lane + 32 * k < d) grad[row * d + lane + 32 * k] = g[k];
    }
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

template <typename T, int kPair, int kCollapse, int NT, int kMode>
static int launch_wmrb(const WmrbParams& p, cudaStream_t stream) {
  const int ch = static_cast<int>(ceil_div(p.d, 128));
  // the serial modes keep nothing per sample
  const size_t smem = kMode == kModeWmrb ? static_cast<size_t>(kWmrbWarps) * 2 * p.n_sampled * sizeof(float) : 0;
  const int grid = capped_grid(ceil_div(p.n_users, kWmrbWarps), 16);
#define TRK_WMRB_LAUNCH(CH)                                                                                             \
  do {                                                                                                                  \
    auto* kernel = wmrb_step_kernel<T, CH, kPair, kCollapse, NT, kMode>;                                                \
    if (smem > 48 * 1024)                                                                                               \
      TRK_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem))); \
    kernel<<<grid, kWmrbWarps * 32, smem, stream>>>(p);                                                                 \
  } while (0)
  if constexpr (NT == 1) {
    if (ch == 1) TRK_WMRB_LAUNCH(1);
    else if (ch == 2) TRK_WMRB_LAUNCH(2);
    else TRK_WMRB_LAUNCH(4);
  } else {
    TRK_WMRB_LAUNCH(1);    // mixtures of tastes: d <= 128
  }
#undef TRK_WMRB_LAUNCH
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

// the instantiation of (pair form, n_tastes, attention); the caller has checked the limits
template <typename T, int kPair, int kMode>
static int launch_wmrb_form(const WmrbParams& p, int n_tastes, bool attention, cudaStream_t stream) {
  if (n_tastes == 1) return launch_wmrb<T, kPair, kCollapseSingle, 1, kMode>(p, stream);
  if (attention) {
    switch (n_tastes) {
      case 2: return launch_wmrb<T, kPair, kCollapseAttention, 2, kMode>(p, stream);
      case 3: return launch_wmrb<T, kPair, kCollapseAttention, 3, kMode>(p, stream);
      default: return launch_wmrb<T, kPair, kCollapseAttention, 4, kMode>(p, stream);
    }
  }
  switch (n_tastes) {
    case 2: return launch_wmrb<T, kPair, kCollapseMax, 2, kMode>(p, stream);
    case 3: return launch_wmrb<T, kPair, kCollapseMax, 3, kMode>(p, stream);
    case 4: return launch_wmrb<T, kPair, kCollapseMax, 4, kMode>(p, stream);
    case 5: return launch_wmrb<T, kPair, kCollapseMax, 5, kMode>(p, stream);
    case 6: return launch_wmrb<T, kPair, kCollapseMax, 6, kMode>(p, stream);
    case 7: return launch_wmrb<T, kPair, kCollapseMax, 7, kMode>(p, stream);
    default: return launch_wmrb<T, kPair, kCollapseMax, 8, kMode>(p, stream);
  }
}

// one launch of the step in mode kMode for the storage type and the form
template <int kMode>
static int launch_step(const WmrbParams& p, bool bf16, bool euclidean, int n_tastes, bool attention,
                       cudaStream_t stream) {
  if (bf16)
    return euclidean ? launch_wmrb_form<__nv_bfloat16, kPairEuclid, kMode>(p, n_tastes, attention, stream)
                     : launch_wmrb_form<__nv_bfloat16, kPairDot, kMode>(p, n_tastes, attention, stream);
  return euclidean ? launch_wmrb_form<float, kPairEuclid, kMode>(p, n_tastes, attention, stream)
                   : launch_wmrb_form<float, kPairDot, kMode>(p, n_tastes, attention, stream);
}

// The checks of the operands and the form that the WMRB and the serial step share, after each entry point has checked
// its own buffers and sizes; `who` (the entry point) prefixes every message.  n_sampled is 0 for the serial step,
// which samples nothing.  The form limits return TRK_ERR_UNSUPPORTED, everything else TRK_ERR_ARG.
static int check_step(const char* who, const void* user_rows, const void* item_repr, int32_t n_tastes,
                      int32_t attention, int32_t euclidean, const float* user_bias, const float* item_bias,
                      int64_t n_users, int64_t n_items, int32_t d, int32_t n_sampled, const float* d_user_rows,
                      const float* d_user_bias, const float* d_item_repr, const float* d_item_bias) {
  TRK_CHECK_ARG((user_bias == nullptr) == (item_bias == nullptr), "%s: biases must be given together", who);
  TRK_CHECK_ARG((user_bias == nullptr) == (d_user_bias == nullptr) && (item_bias == nullptr) == (d_item_bias == nullptr),
                "%s: bias gradients must match the biases", who);
  TRK_CHECK_ARG((attention == 0 || attention == 1) && (euclidean == 0 || euclidean == 1),
                "%s: attention and euclidean are flags", who);
  TRK_CHECK_ARG(n_users >= 0 && n_items >= 1 && n_items < (1ll << 31) && n_tastes >= 1, "%s: bad sizes", who);
  const int max_d = n_tastes == 1 ? 512 : 128;
  const int max_tastes = attention ? 4 : 8;
  if (d < 4 || d % 4 != 0 || d > max_d || n_sampled > 2048 || n_tastes > max_tastes || (attention && n_tastes == 1)) {
    set_error("%s: n_components=%d (multiple of 4, <= 512 for one taste, <= 128 for several) / n_tastes=%d (<= 8, <= 4 "
              "with attention, attention needs >= 2) / n_sampled=%d (<= 2048) outside the fused kernel", who, d,
              n_tastes, n_sampled);
    return TRK_ERR_UNSUPPORTED;
  }
  TRK_CHECK_ARG(reinterpret_cast<uintptr_t>(user_rows) % 16 == 0 && reinterpret_cast<uintptr_t>(item_repr) % 16 == 0 &&
                    reinterpret_cast<uintptr_t>(d_user_rows) % 16 == 0 && reinterpret_cast<uintptr_t>(d_item_repr) % 16 == 0,
                "%s: rows must be 16-byte aligned", who);
  return TRK_OK;
}

// the WmrbParams fields of every mode; the WMRB step adds its samples and loss outputs, the serial step its loss state
static WmrbParams step_params(const void* user_rows, const void* item_repr, const float* user_bias,
                              const float* item_bias, const int32_t* inter_indptr, const int32_t* inter_item,
                              const float* inter_val, int64_t n_users, int64_t n_items, int32_t d, float* pred_serial,
                              float* d_user_rows, float* d_user_bias, float* d_item_repr, float* d_item_bias) {
  WmrbParams p = {};
  p.user_repr = user_rows;
  p.item_repr = item_repr;
  p.user_bias = user_bias;
  p.item_bias = item_bias;
  p.inter_indptr = inter_indptr;
  p.inter_item = inter_item;
  p.inter_val = inter_val;
  p.n_users = n_users;
  p.n_items = static_cast<int32_t>(n_items);
  p.d = d;
  p.pred_serial = pred_serial;
  p.d_user_repr = d_user_rows;
  p.d_user_bias = d_user_bias;
  p.d_item_repr = d_item_repr;
  p.d_item_bias = d_item_bias;
  return p;
}

// trk_wmrb_step_tastes, and trk_wmrb_step as its one-taste dot form (who = the entry point, for the messages)
int wmrb_step_tastes(const char* who, const void* user_rows, const void* item_repr, int32_t repr_is_bf16,
                     int32_t n_tastes, int32_t attention, int32_t euclidean, const float* user_bias,
                     const float* item_bias, const int32_t* inter_indptr, const int32_t* inter_item,
                     const float* inter_val, const float* item_weight_sum, const int32_t* samples, int64_t n_users,
                     int64_t n_items, int32_t d, int32_t n_sampled, float* loss, float* pred_serial, float* coef,
                     float* d_user_rows, float* d_user_bias, float* d_item_repr, float* d_item_bias,
                     cudaStream_t stream) {
  TRK_CHECK_ARG(user_rows && item_repr && inter_indptr && samples, "%s: null input", who);
  TRK_CHECK_ARG(loss && pred_serial && coef && d_user_rows && d_item_repr, "%s: null output", who);
  TRK_CHECK_ARG(n_sampled >= 1, "%s: bad sizes", who);
  const int rc = check_step(who, user_rows, item_repr, n_tastes, attention, euclidean, user_bias, item_bias, n_users,
                            n_items, d, n_sampled, d_user_rows, d_user_bias, d_item_repr, d_item_bias);
  if (rc != TRK_OK) return rc;
  if (n_users == 0) return TRK_OK;
  WmrbParams p = step_params(user_rows, item_repr, user_bias, item_bias, inter_indptr, inter_item, inter_val, n_users,
                             n_items, d, pred_serial, d_user_rows, d_user_bias, d_item_repr, d_item_bias);
  p.item_weight_sum = item_weight_sum;
  p.samples = samples;
  p.n_sampled = n_sampled;
  p.rank_scale = static_cast<float>(n_items) / static_cast<float>(n_sampled);
  p.loss = loss;
  p.coef = coef;
  return launch_step<kModeWmrb>(p, repr_is_bf16 != 0, euclidean != 0, n_tastes, attention != 0, stream);
}

// The statistics grid of nnz predictions: fixed by nnz alone, so the workspace size and the finish kernel's partial
// count both come from here.
static int serial_stats_grid(int64_t nnz) {
  return static_cast<int>(std::min<int64_t>(ceil_div(nnz, int64_t{kStatsThreads} * kStatsPerThread), kStatsMaxBlocks));
}
static constexpr size_t kSerialStateBytes = 64;     // SerialLossState, then the partials at an 8-byte boundary
static_assert(sizeof(SerialLossState) <= kSerialStateBytes, "loss state outgrows its slot");

size_t serial_loss_workspace_bytes(int64_t nnz) {
  return kSerialStateBytes + static_cast<size_t>(serial_stats_grid(std::max<int64_t>(nnz, 0))) * sizeof(SerialMoments);
}

template <int kLoss>
static int launch_serial_stats(const float* pred, const float* val, int64_t nnz, void* workspace, float* loss,
                               cudaStream_t stream) {
  const int grid = serial_stats_grid(nnz);
  auto* state = static_cast<SerialLossState*>(workspace);
  auto* partial = reinterpret_cast<SerialMoments*>(static_cast<char*>(workspace) + kSerialStateBytes);
  serial_stats_kernel<kLoss><<<grid, kStatsThreads, 0, stream>>>(pred, val, nnz, partial);
  TRK_CHECK_LAUNCH();
  serial_finish_kernel<kLoss><<<1, kStatsThreads, 0, stream>>>(partial, grid, loss, state);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

int serial_loss_step(int32_t loss_kind, const void* user_rows, const void* item_repr, int32_t repr_is_bf16,
                     int32_t n_tastes, int32_t attention, int32_t euclidean, const float* user_bias,
                     const float* item_bias, const int32_t* inter_indptr, const int32_t* inter_item,
                     const float* inter_val, int64_t n_users, int64_t n_items, int32_t d, int64_t nnz, float* loss,
                     float* pred_serial, float* d_user_rows, float* d_user_bias, float* d_item_repr,
                     float* d_item_bias, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  TRK_CHECK_ARG(loss_kind == kSerialRmse || loss_kind == kSerialSeparation, "serial_loss_step: unknown loss %d",
                loss_kind);
  TRK_CHECK_ARG(nnz >= 0 && nnz < (1ll << 31) && (nnz == 0 || n_users >= 1), "serial_loss_step: bad sizes");
  TRK_CHECK_ARG(item_repr && d_item_repr && loss && inter_indptr,
                "serial_loss_step: null item operand, loss or indptr");
  TRK_CHECK_ARG(n_users == 0 || (user_rows && d_user_rows), "serial_loss_step: null user operand");
  TRK_CHECK_ARG(nnz == 0 || (inter_item && inter_val && pred_serial && workspace),
                "serial_loss_step: null interaction, prediction or workspace buffer");
  TRK_CHECK_ARG(workspace_bytes >= serial_loss_workspace_bytes(nnz) && reinterpret_cast<uintptr_t>(workspace) % 8 == 0,
                "serial_loss_step: workspace of %zu bytes (8-byte aligned) below the %zu needed", workspace_bytes,
                serial_loss_workspace_bytes(nnz));
  int rc = check_step("serial_loss_step", user_rows, item_repr, n_tastes, attention, euclidean, user_bias, item_bias,
                      n_users, n_items, d, 0, d_user_rows, d_user_bias, d_item_repr, d_item_bias);
  if (rc != TRK_OK) return rc;
  if (nnz == 0) {
    // no interaction: the mean of nothing is NaN and no prediction reaches a representation (launches nothing)
    TRK_CHECK_CUDA(cudaMemsetAsync(loss, 0xFF, sizeof(float), stream));        // all ones: a quiet NaN
    const int64_t n_rows = attention ? 2 * n_tastes : n_tastes;
    if (n_users > 0) {
      TRK_CHECK_CUDA(cudaMemsetAsync(d_user_rows, 0, static_cast<size_t>(n_rows * n_users * d) * sizeof(float),
                                     stream));
      if (d_user_bias)
        TRK_CHECK_CUDA(cudaMemsetAsync(d_user_bias, 0, static_cast<size_t>(n_users) * sizeof(float), stream));
    }
    return TRK_OK;
  }
  WmrbParams p = step_params(user_rows, item_repr, user_bias, item_bias, inter_indptr, inter_item, inter_val, n_users,
                             n_items, d, pred_serial, d_user_rows, d_user_bias, d_item_repr, d_item_bias);
  p.serial_state = workspace;
  p.serial_loss = loss_kind;
  const bool bf16 = repr_is_bf16 != 0, euclid = euclidean != 0, att = attention != 0;
  rc = launch_step<kModeSerialForward>(p, bf16, euclid, n_tastes, att, stream);
  if (rc != TRK_OK) return rc;
  rc = loss_kind == kSerialRmse ? launch_serial_stats<kSerialRmse>(pred_serial, inter_val, nnz, workspace, loss, stream)
                                : launch_serial_stats<kSerialSeparation>(pred_serial, inter_val, nnz, workspace, loss,
                                                                        stream);
  if (rc != TRK_OK) return rc;
  return launch_step<kModeSerialBackward>(p, bf16, euclid, n_tastes, att, stream);
}

int l2_normalize_rows_step(const float* x, int64_t rows, int32_t d, int32_t n_normalize, float* out, float* grad,
                           cudaStream_t stream) {
  TRK_CHECK_ARG(x && rows >= 0 && d >= 1 && (out || grad), "l2_normalize_rows_step: bad arguments");
  if (d > 512 || n_normalize < 1 || n_normalize > 2) {
    set_error("l2_normalize_rows_step: d=%d (<= 512) / n_normalize=%d (1 or 2) outside the kernel", d, n_normalize);
    return TRK_ERR_UNSUPPORTED;
  }
  if (rows == 0) return TRK_OK;
  l2_normalize_rows_step_kernel<<<capped_grid(ceil_div(rows, kNormWarps), 16), kNormWarps * 32, 0, stream>>>(
      x, rows, d, n_normalize, out, grad);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
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
