// Merge of per-(user, list) top-k candidate lists into the global per-user top-k.
//
// Lists come from the n_splits item ranges of one GPU and/or from the item shards of the other GPUs (exchanged by
// one NCCL all-to-all in the host layer: list l of user u sits at cand + u * user_stride + l * list_stride, which
// covers both the [U, L, k] layout of one GPU and the [L, U_slice, 2k] receive buffer of the exchange).  Every list is ordered by (score descending, item id ascending) -- the
// order tf.nn.top_k gives the reference (tensorrec/recommendation_graphs.py:81) -- and padded with
// (-inf, INT32_MAX).  One warp per user performs an n_lists-way merge: lane l holds the heads of lists l, l+32, ...;
// each round is a warp arg-best over the heads.  Integer/float compares only: deterministic.
// dedup: lists may name the same item (the per-taste lists of a mixture-of-tastes model: the score of an item is its
// MAXIMUM over the tastes, tensorrec/recommendation_graphs.py:107): an id that was already emitted -- with a score that is
// at least as high, the rounds go downwards -- is skipped.
#include "common.cuh"

namespace trk {

constexpr int kMergeMaxListsPerLane = 8;  // n_lists <= 256

__device__ __forceinline__ bool cand_better(float s, int32_t i, float bs, int32_t bi) {
  return s > bs || (s == bs && i < bi);
}

__global__ void __launch_bounds__(256)
topk_merge_kernel(const float* __restrict__ cand_score, const int32_t* __restrict__ cand_item, int64_t n_users,
                  int n_lists, int k_in, int k_out, int64_t user_stride, int64_t list_stride,
                  float* __restrict__ out_score, int32_t* __restrict__ out_item, int64_t out_stride,
                  const int32_t* __restrict__ n_users_live, int dedup) {
  if (n_users_live != nullptr) n_users = min(n_users, static_cast<int64_t>(*n_users_live));
  const int lane = threadIdx.x % 32;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / 32;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * blockDim.x / 32;
  const float kNegInf = -__int_as_float(0x7f800000);
  for (int64_t u = warp; u < n_users; u += n_warps) {
    const float* cs = cand_score + u * user_stride;
    const int32_t* ci = cand_item + u * user_stride;
    int pos[kMergeMaxListsPerLane];
#pragma unroll
    for (int j = 0; j < kMergeMaxListsPerLane; ++j) pos[j] = 0;
    int emitted = 0;
    int32_t mine = 0x7fffffff;     // dedup: lane r remembers the id emitted at position r
    const int max_rounds = dedup ? n_lists * k_in : k_out;
    for (int round = 0; round < max_rounds && emitted < k_out; ++round) {
      float bs = kNegInf;
      int32_t bi = 0x7fffffff;
      int bj = -1;
#pragma unroll
      for (int j = 0; j < kMergeMaxListsPerLane; ++j) {
        const int l = lane + 32 * j;
        if (l < n_lists && pos[j] < k_in) {
          const float s = cs[l * list_stride + pos[j]];
          const int32_t i = ci[l * list_stride + pos[j]];
          if (cand_better(s, i, bs, bi)) {
            bs = s;
            bi = i;
            bj = j;
          }
        }
      }
      float ws = bs;
      int32_t wi = bi;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float os = __shfl_xor_sync(0xffffffffu, ws, o);
        const int32_t oi = __shfl_xor_sync(0xffffffffu, wi, o);
        if (cand_better(os, oi, ws, wi)) {
          ws = os;
          wi = oi;
        }
      }
      // real candidates have unique ids; the owner of the winner advances its list head
      if (bj >= 0 && wi != 0x7fffffff && bs == ws && bi == wi) {
#pragma unroll
        for (int j = 0; j < kMergeMaxListsPerLane; ++j)
          if (j == bj) pos[j] += 1;
      }
      if (wi == 0x7fffffff) break;        // every list is exhausted (warp-uniform)
      if (dedup && __any_sync(0xffffffffu, mine == wi)) continue;
      if (lane == emitted) mine = wi;
      if (lane == 0) {
        out_score[u * out_stride + emitted] = ws;
        out_item[u * out_stride + emitted] = wi;
      }
      emitted += 1;
    }
    for (int r = emitted + lane; r < k_out; r += 32) {    // fewer candidates than k_out: sentinels
      out_score[u * out_stride + r] = kNegInf;
      out_item[u * out_stride + r] = 0x7fffffff;
    }
  }
}

int topk_merge(const float* cand_score, const int32_t* cand_item, int64_t n_users, int32_t n_lists, int32_t k_in,
               int32_t k_out, int64_t user_stride, int64_t list_stride, float* out_score, int32_t* out_item,
               int64_t out_row_stride, const int32_t* n_users_live, int32_t dedup, cudaStream_t stream) {
  TRK_CHECK_ARG(cand_score && cand_item && out_score && out_item, "topk_merge: null pointer");
  TRK_CHECK_ARG(n_users >= 0 && n_lists >= 1 && k_in >= 1 && k_out >= 1, "topk_merge: bad sizes");
  TRK_CHECK_ARG(user_stride >= 1 && list_stride >= 1 && out_row_stride >= k_out, "topk_merge: bad strides");
  TRK_CHECK_ARG(!dedup || k_out <= 32, "topk_merge: dedup needs k_out <= 32");
  TRK_CHECK_ARG(n_lists <= 32 * kMergeMaxListsPerLane, "topk_merge: n_lists=%d exceeds %d", n_lists,
                32 * kMergeMaxListsPerLane);
  if (n_users == 0) return TRK_OK;
  const int threads = 256;
  topk_merge_kernel<<<capped_grid(ceil_div(n_users, threads / 32), 8), threads, 0, stream>>>(
      cand_score, cand_item, n_users, n_lists, k_in, k_out, user_stride, list_stride, out_score, out_item,
      out_row_stride, n_users_live, dedup);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

}  // namespace trk
