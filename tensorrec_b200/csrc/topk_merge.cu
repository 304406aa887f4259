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

// De-duplicating merge of two sorted lists per row for any k <= kPairMaxK (DESIGN §3.6): the fold of the per-taste
// top-k lists of a mixture-of-tastes model on the wide route, where k is too large for topk_merge_kernel's one id per
// lane.  One CTA per row, both lists in shared memory:
//   1. A's real ids go into an open-addressing table of A positions (ids are unique within a list, so what a probe
//      finds does not depend on the order of the insertions);
//   2. every real id of B is looked up; of a duplicate pair the copy with the lower score is dropped, A's on a tie;
//   3. the survivor flags of A and B are scanned into exclusive prefix counts;
//   4. a survivor lands at (survivors of its own list before it) + (survivors of the other list ordered before it):
//      the second term is a binary search of the other list for the first entry not before it, then a prefix count.
//      Survivors have distinct ids, hence a strict order, so the positions are a permutation of [0, survivors);
//   5. positions below k are written and the slots from the survivor count on get the sentinel.
// Integer and float compares only: the result does not depend on thread scheduling.
constexpr int kPairThreads = 256;
constexpr int kPairMaxK = 1024;

// exclusive prefix sum of v[0, n) in place, v[n] = the total, by the whole CTA; ends with a barrier
__device__ __forceinline__ void block_exclusive_scan(int* v, int n, int* warp_total) {
  const int lane = threadIdx.x % 32, warp = threadIdx.x / 32;
  const int per = (n + blockDim.x - 1) / blockDim.x;
  const int lo = min(n, static_cast<int>(threadIdx.x) * per), hi = min(n, lo + per);
  int sum = 0;
  for (int i = lo; i < hi; ++i) sum += v[i];
  int incl = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) warp_total[warp] = incl;
  __syncthreads();
  int run = incl - sum;
  for (int w = 0; w < warp; ++w) run += warp_total[w];
  for (int i = lo; i < hi; ++i) {
    const int x = v[i];
    v[i] = run;
    run += x;
  }
  if (threadIdx.x == blockDim.x - 1) v[n] = run;
  __syncthreads();
}

// first position j of the sorted list (s, id)[0, n) whose entry is not ordered before (xs, xi)
__device__ __forceinline__ int count_before(const float* s, const int32_t* id, int n, float xs, int32_t xi) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) / 2;
    if (cand_better(s[mid], id[mid], xs, xi)) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ uint32_t pair_hash(int32_t id, int table_bits) {
  return (static_cast<uint32_t>(id) * 0x9e3779b1u) >> (32 - table_bits);
}

__global__ void __launch_bounds__(kPairThreads)
topk_merge_dedup_pair_kernel(const float* __restrict__ a_score, const int32_t* __restrict__ a_item, int64_t a_stride,
                             const float* __restrict__ b_score, const int32_t* __restrict__ b_item, int64_t b_stride,
                             int k, int table_bits, float* __restrict__ out_score, int32_t* __restrict__ out_item,
                             int64_t out_stride) {
  extern __shared__ int32_t pair_smem[];
  __shared__ int warp_total[kPairThreads / 32];
  float* as = reinterpret_cast<float*>(pair_smem);
  int32_t* ai = pair_smem + k;
  float* bs = reinterpret_cast<float*>(pair_smem + 2 * k);
  int32_t* bi = pair_smem + 3 * k;
  int* pa = pair_smem + 4 * k;        // A's survivor flags, then their exclusive prefix counts ([k + 1])
  int* pb = pa + k + 1;               // the same for B
  int* table = pb + k + 1;            // A position per slot, -1 = empty ([1 << table_bits])
  const int table_size = 1 << table_bits;
  const uint32_t mask = table_size - 1;
  const int64_t u = blockIdx.x;
  const float kNegInf = -__int_as_float(0x7f800000);

  for (int t = threadIdx.x; t < k; t += blockDim.x) {
    as[t] = __ldg(a_score + u * a_stride + t);
    ai[t] = __ldg(a_item + u * a_stride + t);
    bs[t] = __ldg(b_score + u * b_stride + t);
    bi[t] = __ldg(b_item + u * b_stride + t);
    pa[t] = ai[t] != 0x7fffffff ? 1 : 0;
  }
  for (int t = threadIdx.x; t < table_size; t += blockDim.x) table[t] = -1;
  __syncthreads();
  for (int i = threadIdx.x; i < k; i += blockDim.x) {
    if (ai[i] == 0x7fffffff) continue;
    uint32_t h = pair_hash(ai[i], table_bits);
    while (atomicCAS(table + h, -1, i) != -1) h = (h + 1) & mask;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < k; j += blockDim.x) {
    const int32_t id = bi[j];
    int keep = id != 0x7fffffff ? 1 : 0;
    if (keep) {
      for (uint32_t h = pair_hash(id, table_bits);; h = (h + 1) & mask) {
        const int i = table[h];
        if (i < 0) break;
        if (ai[i] == id) {        // the only copy of this id in A: exactly one thread writes pa[i]
          if (bs[j] > as[i]) pa[i] = 0;
          else keep = 0;
          break;
        }
      }
    }
    pb[j] = keep;
  }
  __syncthreads();
  block_exclusive_scan(pa, k, warp_total);
  block_exclusive_scan(pb, k, warp_total);

  for (int t = threadIdx.x; t < 2 * k; t += blockDim.x) {
    const bool from_a = t < k;
    const int j = from_a ? t : t - k;
    const int* own = from_a ? pa : pb;
    if (own[j + 1] == own[j]) continue;       // dropped duplicate or sentinel
    const float s = from_a ? as[j] : bs[j];
    const int32_t id = from_a ? ai[j] : bi[j];
    const int other = from_a ? pb[count_before(bs, bi, k, s, id)] : pa[count_before(as, ai, k, s, id)];
    const int pos = own[j] + other;
    if (pos < k) {
      out_score[u * out_stride + pos] = s;
      out_item[u * out_stride + pos] = id;
    }
  }
  for (int r = pa[k] + pb[k] + threadIdx.x; r < k; r += blockDim.x) {
    out_score[u * out_stride + r] = kNegInf;
    out_item[u * out_stride + r] = 0x7fffffff;
  }
}

int topk_merge_dedup_pair(const float* a_score, const int32_t* a_item, int64_t a_row_stride, const float* b_score,
                          const int32_t* b_item, int64_t b_row_stride, int64_t n_rows, int32_t k, float* out_score,
                          int32_t* out_item, int64_t out_row_stride, cudaStream_t stream) {
  TRK_CHECK_ARG(a_score && a_item && b_score && b_item && out_score && out_item, "topk_merge_dedup_pair: null pointer");
  TRK_CHECK_ARG(n_rows >= 0 && n_rows <= 0x7fffffff, "topk_merge_dedup_pair: n_rows=%lld",
                static_cast<long long>(n_rows));
  TRK_CHECK_ARG(k >= 1 && k <= kPairMaxK, "topk_merge_dedup_pair: k=%d outside [1, %d]", k, kPairMaxK);
  TRK_CHECK_ARG(a_row_stride >= k && b_row_stride >= k && out_row_stride >= k, "topk_merge_dedup_pair: bad strides");
  if (n_rows == 0) return TRK_OK;
  int table_bits = 6;
  while ((1 << table_bits) < 2 * k) ++table_bits;        // load factor <= 1/2
  const size_t smem = (4 * static_cast<size_t>(k) + 2 * (k + 1) + (size_t{1} << table_bits)) * sizeof(int32_t);
  topk_merge_dedup_pair_kernel<<<static_cast<unsigned>(n_rows), kPairThreads, smem, stream>>>(
      a_score, a_item, a_row_stride, b_score, b_item, b_row_stride, k, table_bits, out_score, out_item,
      out_row_stride);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

}  // namespace trk
