// K3 (full) -- rank_predictions (tensorrec/recommendation_graphs.py:73-82).
//
// The reference ranks by a double full sort: order = top_k(pred, k=n).indices (descending, equal values by
// lower index first), ranks = top_k(-order, k=n).indices + 1 (the inverse permutation).  In closed form
//     rank[u,i] = 1 + #{j : s[u,j] > s[u,i]} + #{j < i : s[u,j] == s[u,i]}                    (int32)
// Each score becomes the 64-bit key (descending-order bits of the float) << 32 | index; keys of a row are unique,
// ascending key order IS the reference's order, so no stable sort is needed:
//   pass 1: every chunk of up to kChunk keys of a row is bitonic-sorted by one block: 256 threads x KPT keys each in
//           REGISTERS -- exchange distances below KPT are compile-time register swaps, distances inside a warp are
//           shuffles, only the largest distances (<= 6 of the 78 stages at 4096 keys) go through shared memory;
//   pass 2 (rows longer than one chunk): sorted runs are merged pairwise (merge path: every block produces one tile
//           of kChunk outputs from the two input windows it locates by binary search), log2(#chunks) passes that
//           ping-pong between two workspace buffers; the last pass scatters ranks instead of keys.
// Integer compares only -> exact and run-to-run deterministic.
#include "common.cuh"

namespace trk {

constexpr int kChunk = 4096;          // keys per sorted chunk
constexpr int kSortThreads = 256;
constexpr uint64_t kPadKey = ~0ull;   // sorts behind every real key

__device__ __forceinline__ uint64_t rank_key(float s, uint32_t idx) {
  s = s + 0.0f;  // -0.0 -> +0.0: the reference compares values, where the two are equal
  const uint32_t b = __float_as_uint(s);
  const uint32_t asc = (b & 0x80000000u) ? ~b : (b | 0x80000000u);  // monotone float -> uint
  return (static_cast<uint64_t>(~asc) << 32) | idx;                  // descending score, ascending index
}

__device__ __forceinline__ void cmp_swap(uint64_t& a, uint64_t& b, bool ascending) {
  const bool sw = (a > b) == ascending;
  const uint64_t lo = sw ? b : a, hi = sw ? a : b;
  a = lo;
  b = hi;
}

// One in-register stage: exchange distance J < KPT (compile time, so every register index is static).
template <int KPT, int J>
__device__ __forceinline__ void bitonic_stage_regs(uint64_t (&key)[KPT], int k, int tid) {
#pragma unroll
  for (int r = 0; r < KPT; ++r) {
    if ((r & J) == 0) {
      const bool ascending = ((tid * KPT + r) & k) == 0;
      cmp_swap(key[r], key[r | J], ascending);
    }
  }
}

// Ascending bitonic sort of kSortThreads * KPT keys held blocked in registers (element e = tid * KPT + r).
// The (k, j) stage loops stay ROLLED: the fully unrolled network (78 stages x 16 keys at 4096) is ~30k instructions,
// overflows the instruction cache and ran 3x slower than the shared-memory version it replaces.  Only the register
// slot loops are unrolled; the in-register stages dispatch on j to one of log2(KPT) specialised bodies.
template <int KPT>
__device__ __forceinline__ void block_bitonic_sort(uint64_t (&key)[KPT], uint64_t* s_keys) {
  constexpr int N = kSortThreads * KPT;
  constexpr int kLogN = N == 256 ? 8 : N == 512 ? 9 : N == 1024 ? 10 : N == 2048 ? 11 : 12;
  static_assert((1 << kLogN) == N, "block_bitonic_sort: unsupported size");
  const int tid = threadIdx.x;
#pragma unroll 1
  for (int lk = 1; lk <= kLogN; ++lk) {
    const int k = 1 << lk;
#pragma unroll 1
    for (int lj = lk - 1; lj >= 0; --lj) {
      const int j = 1 << lj;
      if (j < KPT) {
        // partner inside this thread's registers
        if (KPT > 1 && j == 1) bitonic_stage_regs<KPT, 1 % (KPT > 1 ? KPT : 2)>(key, k, tid);
        if (KPT > 2 && j == 2) bitonic_stage_regs<KPT, 2 % (KPT > 2 ? KPT : 3)>(key, k, tid);
        if (KPT > 4 && j == 4) bitonic_stage_regs<KPT, 4 % (KPT > 4 ? KPT : 5)>(key, k, tid);
        if (KPT > 8 && j == 8) bitonic_stage_regs<KPT, 8 % (KPT > 8 ? KPT : 9)>(key, k, tid);
      } else {
        const int m = j / KPT;                            // partner thread = tid ^ m, same register slot
        const bool lower = (tid & m) == 0;
        const bool ascending = ((tid * KPT) & k) == 0;    // k >= 2 KPT here: the bit comes from tid alone
        const bool keep_min = lower == ascending;
        if (m < 32) {
          // partner in another lane of the warp
#pragma unroll
          for (int r = 0; r < KPT; ++r) {
            const uint32_t olo = __shfl_xor_sync(0xffffffffu, static_cast<uint32_t>(key[r]), m);
            const uint32_t ohi = __shfl_xor_sync(0xffffffffu, static_cast<uint32_t>(key[r] >> 32), m);
            const uint64_t other = (static_cast<uint64_t>(ohi) << 32) | olo;
            key[r] = keep_min ? (other < key[r] ? other : key[r]) : (other > key[r] ? other : key[r]);
          }
        } else {
          // partner in another warp: through shared memory
          __syncthreads();
#pragma unroll
          for (int r = 0; r < KPT; ++r) s_keys[tid * KPT + r] = key[r];
          __syncthreads();
#pragma unroll
          for (int r = 0; r < KPT; ++r) {
            const uint64_t other = s_keys[(tid ^ m) * KPT + r];
            key[r] = keep_min ? (other < key[r] ? other : key[r]) : (other > key[r] ? other : key[r]);
          }
        }
      }
    }
  }
}

// grid = (chunks per row, rows).  Single-chunk rows are ranked directly.
template <int KPT>
__global__ void __launch_bounds__(kSortThreads)
rank_chunk_sort_kernel(const float* __restrict__ scores, int32_t* __restrict__ ranks, uint64_t* __restrict__ sorted,
                       int64_t n_items, int n_chunks) {
  __shared__ uint64_t s_keys[kSortThreads * KPT];
  const int64_t row = blockIdx.y;
  const int chunk = blockIdx.x;
  const int64_t base = static_cast<int64_t>(chunk) * kChunk;
  const float* srow = scores + row * n_items;
  const int tid = threadIdx.x;
  uint64_t key[KPT];
#pragma unroll
  for (int r = 0; r < KPT; ++r) {
    const int64_t i = base + tid * KPT + r;
    key[r] = i < n_items ? rank_key(__ldg(srow + i), static_cast<uint32_t>(i)) : kPadKey;
  }
  block_bitonic_sort<KPT>(key, s_keys);
  if (n_chunks == 1) {
    int32_t* rrow = ranks + row * n_items;
#pragma unroll
    for (int r = 0; r < KPT; ++r)
      if (key[r] != kPadKey) rrow[static_cast<uint32_t>(key[r])] = tid * KPT + r + 1;
  } else {
    uint64_t* dst = sorted + (row * n_chunks + chunk) * kChunk + tid * KPT;   // multi-chunk rows use KPT = 16
#pragma unroll
    for (int r = 0; r < KPT; ++r) dst[r] = key[r];
  }
}

// One merge pass over a row of n_chunks sorted runs of `run` keys (the last run may be shorter): runs 2p and 2p+1
// merge into one run of 2 * run keys.  Block (tile, row) produces outputs [tile * kChunk, +kChunk) of the row.
// final_pass: the outputs are in their final order -> write rank = position + 1 at the key's item index.
constexpr int kMergePer = kChunk / kSortThreads;   // 16 outputs per thread

__device__ __forceinline__ int64_t merge_path(const uint64_t* __restrict__ A, int64_t len_a,
                                              const uint64_t* __restrict__ B, int64_t len_b, int64_t diag) {
  int64_t lo = diag > len_b ? diag - len_b : 0, hi = diag < len_a ? diag : len_a;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (A[mid] < B[diag - 1 - mid]) lo = mid + 1; else hi = mid;   // keys are unique
  }
  return lo;
}

__global__ void __launch_bounds__(kSortThreads)
rank_merge_pass_kernel(const uint64_t* __restrict__ src, uint64_t* __restrict__ dst, int32_t* __restrict__ ranks,
                       int64_t n_items, int n_chunks, int64_t run, int final_pass) {
  __shared__ uint64_t s_in[kChunk];
  __shared__ int64_t s_split[2];
  const int64_t row = blockIdx.y;
  const int64_t row_len = static_cast<int64_t>(n_chunks) * kChunk;
  const uint64_t* row_src = src + row * row_len;
  const int64_t out0 = static_cast<int64_t>(blockIdx.x) * kChunk;   // first output position of this tile in the row
  const int64_t pair_base = (out0 / (2 * run)) * (2 * run);
  const int64_t len_a = row_len - pair_base < run ? row_len - pair_base : run;
  const int64_t rest = row_len - pair_base - len_a;
  const int64_t len_b = rest < run ? rest : run;
  const uint64_t* A = row_src + pair_base;
  const uint64_t* B = A + len_a;
  const int64_t d0 = out0 - pair_base;
  const int64_t d1 = d0 + kChunk < len_a + len_b ? d0 + kChunk : len_a + len_b;
  if (threadIdx.x < 2) s_split[threadIdx.x] = merge_path(A, len_a, B, len_b, threadIdx.x == 0 ? d0 : d1);
  __syncthreads();
  const int64_t a0 = s_split[0], a1 = s_split[1];
  const int64_t b0 = d0 - a0, b1 = d1 - a1;
  const int na = static_cast<int>(a1 - a0), nb = static_cast<int>(b1 - b0);
  for (int t = threadIdx.x; t < na; t += kSortThreads) s_in[t] = A[a0 + t];
  for (int t = threadIdx.x; t < nb; t += kSortThreads) s_in[na + t] = B[b0 + t];
  __syncthreads();
  const uint64_t* sa = s_in;
  const uint64_t* sb = s_in + na;
  // this thread's window of the tile: outputs [dt, dt + kMergePer)
  const int n_out = na + nb;
  const int dt = threadIdx.x * kMergePer < n_out ? threadIdx.x * kMergePer : n_out;
  int lo = dt > nb ? dt - nb : 0, hi = dt < na ? dt : na;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (sa[mid] < sb[dt - 1 - mid]) lo = mid + 1; else hi = mid;
  }
  int i = lo, j = dt - lo;
  int32_t* rrow = ranks + row * n_items;
  uint64_t* drow = dst + row * row_len + out0;
#pragma unroll
  for (int r = 0; r < kMergePer; ++r) {
    const int o = dt + r;
    if (o < n_out) {
      const bool take_a = j >= nb || (i < na && sa[i] < sb[j]);
      const uint64_t key = take_a ? sa[i] : sb[j];
      i += take_a ? 1 : 0;
      j += take_a ? 0 : 1;
      if (final_pass) {
        if (key != kPadKey) rrow[static_cast<uint32_t>(key)] = static_cast<int32_t>(out0 + o + 1);
      } else {
        drow[o] = key;
      }
    }
  }
}

static int next_pow2(int64_t n) {
  int p = 2;
  while (p < n) p <<= 1;
  return p;
}

size_t rank_full_workspace_bytes(int64_t n_users, int64_t n_items) {
  if (n_items <= kChunk || n_users <= 0) return 0;
  const int64_t n_chunks = ceil_div(n_items, kChunk);
  // two key buffers: the merge passes ping-pong between them
  return 2 * static_cast<size_t>(n_users) * static_cast<size_t>(n_chunks) * kChunk * sizeof(uint64_t);
}

int rank_full(const float* scores, int32_t* ranks, int64_t n_users, int64_t n_items, void* workspace,
              size_t workspace_bytes, cudaStream_t stream) {
  TRK_CHECK_ARG(scores && ranks, "rank_full: null pointer");
  TRK_CHECK_ARG(n_users >= 0 && n_items >= 0, "rank_full: negative size");
  TRK_CHECK_ARG(n_items < (1ll << 31), "rank_full: n_items must fit int32 (the reference returns int32 ranks)");
  if (n_users == 0 || n_items == 0) return TRK_OK;
  const int64_t n_chunks = ceil_div(n_items, kChunk);
  TRK_CHECK_ARG(n_chunks <= 65535 && n_users <= 2147483647ll, "rank_full: shape exceeds one launch");
  const size_t need = rank_full_workspace_bytes(n_users, n_items);
  TRK_CHECK_ARG(workspace_bytes >= need && (need == 0 || workspace != nullptr),
                "rank_full: workspace too small (%zu < %zu)", workspace_bytes, need);
  const int sort_n = n_chunks == 1 ? next_pow2(n_items) : kChunk;
  const int kpt = sort_n <= kSortThreads ? 1 : sort_n / kSortThreads;   // 1, 2, 4, 8 or 16 keys per thread
  uint64_t* ws0 = static_cast<uint64_t*>(workspace);
  uint64_t* ws1 = ws0 ? ws0 + static_cast<size_t>(n_users) * n_chunks * kChunk : nullptr;
  // rows go on grid.y (<= 65535 per launch)
  for (int64_t r0 = 0; r0 < n_users; r0 += 65535) {
    const int64_t nr = n_users - r0 < 65535 ? n_users - r0 : 65535;
    const dim3 grid(static_cast<unsigned>(n_chunks), static_cast<unsigned>(nr));
    const float* sc = scores + r0 * n_items;
    int32_t* rk = ranks + r0 * n_items;
    uint64_t* a = ws0 ? ws0 + r0 * n_chunks * kChunk : nullptr;
    uint64_t* b = ws1 ? ws1 + r0 * n_chunks * kChunk : nullptr;
    const int nc = static_cast<int>(n_chunks);
    switch (kpt) {
      case 1: rank_chunk_sort_kernel<1><<<grid, kSortThreads, 0, stream>>>(sc, rk, a, n_items, nc); break;
      case 2: rank_chunk_sort_kernel<2><<<grid, kSortThreads, 0, stream>>>(sc, rk, a, n_items, nc); break;
      case 4: rank_chunk_sort_kernel<4><<<grid, kSortThreads, 0, stream>>>(sc, rk, a, n_items, nc); break;
      case 8: rank_chunk_sort_kernel<8><<<grid, kSortThreads, 0, stream>>>(sc, rk, a, n_items, nc); break;
      default: rank_chunk_sort_kernel<16><<<grid, kSortThreads, 0, stream>>>(sc, rk, a, n_items, nc); break;
    }
    TRK_CHECK_LAUNCH();
    for (int64_t run = kChunk; run < n_chunks * kChunk; run *= 2) {
      const int final_pass = 2 * run >= n_chunks * kChunk ? 1 : 0;
      rank_merge_pass_kernel<<<grid, kSortThreads, 0, stream>>>(a, b, rk, n_items, nc, run, final_pass);
      TRK_CHECK_LAUNCH();
      uint64_t* t = a;
      a = b;
      b = t;
    }
  }
  return TRK_OK;
}

// order[rank - 1] = index: the permutation that lists one row's items by reference rank (the inverse of rank_full's
// output for that row).  With the item biases as the row this is the stable descending sort the filter kernel's
// processing order needs (tf.nn.top_k order: value descending, lower index first on ties).
__global__ void order_from_ranks_kernel(const int32_t* __restrict__ ranks, int64_t n, int32_t* __restrict__ order) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    order[ranks[i] - 1] = static_cast<int32_t>(i);
}

int order_from_ranks(const int32_t* ranks, int64_t n, int32_t* order, cudaStream_t stream) {
  TRK_CHECK_ARG(ranks && order && n >= 0 && n < (1ll << 31), "order_from_ranks: bad arguments");
  if (n == 0) return TRK_OK;
  order_from_ranks_kernel<<<capped_grid(ceil_div(n, 256), 8), 256, 0, stream>>>(ranks, n, order);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

}  // namespace trk
