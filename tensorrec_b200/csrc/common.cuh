// Shared helpers for the sm_90a kernels: error plumbing for the C ABI and thin inline-PTX wrappers for
// mbarrier / TMA / wgmma / clusters (CUDA 12.9; PTX names as in the PTX ISA, no CUTLASS dependency).
#pragma once

#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/tensorrec_b200.h"

namespace trk {

void set_error(const char* fmt, ...);

#define TRK_CHECK_ARG(cond, ...)      \
  do {                                \
    if (!(cond)) {                    \
      ::trk::set_error(__VA_ARGS__);  \
      return TRK_ERR_ARG;             \
    }                                 \
  } while (0)

#define TRK_CHECK_CUDA(expr)                                                                       \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      ::trk::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return TRK_ERR_CUDA;                                                                         \
    }                                                                                              \
  } while (0)

#define TRK_CHECK_LAUNCH()                                                                       \
  do {                                                                                           \
    cudaError_t _e = cudaGetLastError();                                                         \
    if (_e != cudaSuccess) {                                                                     \
      ::trk::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
      return TRK_ERR_CUDA;                                                                       \
    }                                                                                            \
  } while (0)

// Number of SMs of the current device (cached per device id).
int sm_count();

// Grid of a grid-stride launch: `blocks` CTAs, at most per_sm x sm_count(), at least 1.
int capped_grid(int64_t blocks, int per_sm);

// Encodes a 2-D row-major tensor map with the 128-byte swizzle: `rows` rows of `cols` elements of `type`, row_bytes
// apart, loaded / stored in boxes of box_cols x box_rows.
int encode_tiled_2d(CUtensorMap* map, CUtensorMapDataType type, const void* base, uint64_t cols, uint64_t rows,
                    uint64_t row_bytes, uint32_t box_cols, uint32_t box_rows, CUtensorMapL2promotion l2_promotion);

// Encodes a 3-D tensor map with the 128-byte swizzle: `planes` planes of `rows` rows of `cols` elements, rows
// row_bytes apart and planes plane_bytes apart, loaded in boxes of box_cols x box_rows x box_planes.  A box lands in
// shared memory as box_planes x box_rows consecutive rows (plane-major), swizzled as a 2-D box of that many rows.
int encode_tiled_3d(CUtensorMap* map, CUtensorMapDataType type, const void* base, uint64_t cols, uint64_t rows,
                    uint64_t planes, uint64_t row_bytes, uint64_t plane_bytes, uint32_t box_cols, uint32_t box_rows,
                    uint32_t box_planes, CUtensorMapL2promotion l2_promotion);

// Host arguments of score_tc (score_topk_tc.cu), which validates them and launches the exact tensor-core kernel behind
// every trk_score_{topk,dense,count}* entry point.  The fields up to item_half_sqnorm are the arguments of
// trk_score_topk_euclid_f16x3, in its order.  The score form follows from the fields that are set: n_tastes != 0 is a
// mixture of tastes (attention != 0: with attention), the two norms are Euclidean similarity, neither is dot / cosine.
struct ScoreTcArgs {
  const void* user_split = nullptr;
  const float* user_scale = nullptr;
  const float* user_bias = nullptr;   // may be null
  const void* item_split = nullptr;
  const float* item_meta = nullptr;
  int64_t n_users = 0;
  int64_t n_items = 0;
  int32_t d_pad = 0;
  int32_t k = 0;                      // top-k mode: k, n_splits .. n_users_live and the exclusion lists
  int32_t n_splits = 0;
  int32_t item_id_offset = 0;
  float* cand_score = nullptr;
  int32_t* cand_item = nullptr;
  const int32_t* n_users_live = nullptr;
  const int32_t* excl_indptr = nullptr;
  const int32_t* excl_ids = nullptr;
  const int32_t* excl_row_map = nullptr;
  const float* user_half_sqnorm = nullptr;
  const float* item_half_sqnorm = nullptr;
  bool dense = false;                 // dense mode: the score matrix to dense_out instead of top-k candidates
  bool wide = false;                  // wide mode: cand_score / cand_item are the lists [n_users, n_splits, 2, cap]
  int32_t* list_count = nullptr;      // wide mode: [n_users, n_splits, 2] entries of each list
  float* dense_out = nullptr;
  int64_t dense_stride = 0;
  int32_t n_tastes = 0;
  int32_t attention = 0;
  bool count = false;                 // counting mode (TcCount): the listed pairs' scores (pass -1) or counts (pass >= 0)
  const int32_t* pair_indptr = nullptr;
  const int32_t* pair_ids = nullptr;
  float* pair_score = nullptr;
  int32_t* pair_count = nullptr;
  const int32_t* block_pairs = nullptr;
  int32_t pass = 0;
  bool pairs = false;                 // pairs mode: the listed pairs' scores over gathered item tiles (pair_indptr,
  const int32_t* tile_items = nullptr;   // pair_ids = virtual columns, pair_score; item_meta / item_half_sqnorm per slot)
  int32_t n_tiles = 0;
  const int32_t* work = nullptr;
  int32_t n_work = 0;
};
int score_tc(const ScoreTcArgs& a, cudaStream_t stream);

constexpr int kWarp = 32;
constexpr int kSMsH100 = 132;

// Tile geometry of the two tensor-core kernels (score_topk_tc.cu, score_filter_tc.cu): a producer warpgroup streams
// 128-row operand tiles of 64 fp16 (one 128-byte swizzle row) per k-block, two consumer warpgroups issue wgmma.
constexpr int kBlockM = 128;          // user tile
constexpr int kBlockN = 128;          // item tile
constexpr int kKBlock = 64;           // fp16 per 128-byte swizzle row
constexpr int kMmaK = 16;
constexpr int kTcThreads = 384;
constexpr int kConsumerThreads = 128; // per consumer warpgroup
constexpr uint32_t kATileBytes = kBlockM * kKBlock * 2;   // 16 KB
constexpr uint32_t kBTileBytes = kBlockN * kKBlock * 2;   // 16 KB
constexpr int kMaxStages = 10;
constexpr uint32_t kSmemLimit = 232448;   // 227 KB opt-in limit per CTA on sm_90
constexpr uint32_t kSmemAlignSlack = 1024;   // dynamic shared memory requested beyond the layout: see smem_base_1024

__host__ __device__ constexpr int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
__host__ __device__ constexpr int64_t round_up(int64_t a, int64_t b) { return ceil_div(a, b) * b; }

// ---------------------------------------------------------------------------------------------------------
// device-side PTX wrappers
// ---------------------------------------------------------------------------------------------------------
#ifdef __CUDACC__

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// The dynamic shared memory rounded up to 1024 bytes: 128B-swizzled tiles need a 1024-byte aligned base.
__device__ __forceinline__ uint8_t* smem_base_1024() {
  extern __shared__ uint8_t smem_raw[];
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---- mbarrier ------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t arrive_count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(arrive_count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---- TMA -----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// 2-D tiled load: box -> smem, completion counted in bytes on `bar`.  c0 = innermost coordinate.
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int32_t c0,
                                            int32_t c1, uint64_t cache_hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
        "l"(cache_hint)
      : "memory");
}
// 3-D tiled load (see encode_tiled_3d), completion counted in bytes on `bar`.  c0 = innermost coordinate.
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int32_t c0,
                                            int32_t c1, int32_t c2, uint64_t cache_hint) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4, %5}], [%2], %6;"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
        "r"(c2), "l"(cache_hint)
      : "memory");
}
// 1-D bulk copy global -> shared (16-byte aligned, size a multiple of 16), completion counted in bytes on `bar`
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(gmem_src)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// L2 cache-hint policies (same encodings CUTLASS uses for TMA::CacheHintSm90)
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;

// ---- wgmma (warpgroup MMA, sm_90a) -------------------------------------------------------------------------
// Shared-memory matrix descriptor for a K-major operand tile stored as rows of 128 bytes with the 128-byte swizzle
// (what a TMA box of 64 fp16 x rows with CU_TENSOR_MAP_SWIZZLE_128B produces):
//   start address >> 4 in bits [0,14); leading byte offset (ignored for swizzled K-major) = 1 in [16,30);
//   stride byte offset = 8 rows * 128 B = 1024 B (>> 4 = 64) in [32,46); layout type SWIZZLE_128B = 1 in [62,64).
// The tile base must be 1024-byte aligned; advancing 16 fp16 (32 bytes) along K inside the swizzle atom is +2 in the
// address field, advancing 64 rows is +512.
__device__ __forceinline__ uint64_t wgmma_desc_k_major_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kPending>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory");
}
// Register accumulators of wgmma.m64nNk16 with fp32 D: thread t of the warpgroup (warp w = t / 32, lane l) holds
// d[i] = D[16 w + l / 4 + 8 ((i / 2) % 2)][8 (i / 4) + 2 (l % 4) + i % 2].
__device__ __forceinline__ int wgmma_acc_row(int wg_thread, int i) {
  return 16 * (wg_thread / 32) + (wg_thread % 32) / 4 + 8 * ((i / 2) % 2);
}
__device__ __forceinline__ int wgmma_acc_col(int wg_thread, int i) { return 8 * (i / 4) + 2 * (wg_thread % 4) + i % 2; }
// D (+)= A[64 x 16, smem desc] * B[N x 16, smem desc]^T, fp16 inputs, fp32 accumulate, both operands K-major;
// issued by the whole warpgroup.
__device__ __forceinline__ void wgmma_m64n64k16_f16(float (&d)[32], uint64_t desc_a, uint64_t desc_b,
                                                    uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_m64n128k16_f16(float (&d)[64], uint64_t desc_a, uint64_t desc_b,
                                                     uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

// ---- thread-block clusters: TMA multicast ------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// 2-D tiled load delivered to EVERY CTA of `cta_mask`: the box lands at the same shared-memory offset in each of them
// and its bytes are counted on the mbarrier at the same offset in each of them (one L2 read feeds all CTAs).
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int32_t c0,
                                                      int32_t c1, uint16_t cta_mask, uint64_t cache_hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5, %6;"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
        "h"(cta_mask), "l"(cache_hint)
      : "memory");
}
// arrive on the barrier at the same shared-memory offset in CTA `rank` of the cluster (the own CTA included), with the
// default semantics (release at CTA scope).  That is all that handing back a ring slot needs: the slot's readers are
// wgmma that have completed before the arrival, and nothing the arriving thread wrote is read by the other side.  A
// .release.cluster arrive would put a GPU-scope memory barrier (MEMBAR.ALL.GPU) in front of every arrival on sm_90.
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(rank));
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
// wait on a barrier that other CTAs of the cluster arrive on (mbar_arrive_cluster), with cluster-scope acquire
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{\n\t"
        ".reg .pred P;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, P;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  }
}

__device__ __forceinline__ void named_barrier_sync(uint32_t id, uint32_t threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// Exclusion lists (top-k of the items a user has not seen): CSR rows of ascending int32 values (item ids or processing
// positions).  Index of the first value >= x in v[lo, hi), hi if there is none.
__device__ __forceinline__ int excl_lower_bound(const int32_t* v, int lo, int hi, int32_t x) {
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(v + mid) < x)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo;
}
// The first value >= x of CSR row `row`, INT32_MAX if there is none.
__device__ __forceinline__ int32_t excl_next_at(const int32_t* indptr, const int32_t* v, int64_t row, int32_t x) {
  const int hi = __ldg(indptr + row + 1);
  const int i = excl_lower_bound(v, __ldg(indptr + row), hi, x);
  return i < hi ? __ldg(v + i) : 0x7fffffff;
}

// tf.nn.top_k order of two (score, id) entries: score descending, lower id first on ties
__device__ __forceinline__ bool r_before(float xs, int32_t xi, float ys, int32_t yi) {
  return xs > ys || (xs == ys && xi < yi);
}

// bitonic sort of one (score, id) entry per lane into (score desc, id asc) order; sentinels (-inf, INT32_MAX) go last
__device__ __forceinline__ void warp_sort_desc(float& s, int32_t& id, int lane) {
#pragma unroll
  for (int size = 2; size <= 32; size <<= 1) {
#pragma unroll
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      const float os = __shfl_xor_sync(0xffffffffu, s, stride);
      const int32_t oi = __shfl_xor_sync(0xffffffffu, id, stride);
      const bool lower = (lane & stride) == 0;
      const bool descending = (lane & size) == 0;
      const bool other_first = r_before(os, oi, s, id);
      const bool take_other = (lower == descending) ? other_first : !other_first;
      if (take_other) {
        s = os;
        id = oi;
      }
    }
  }
}

// order-preserving keys of the wide form's selections: a > b  <=>  key(a) > key(b) for non-NaN floats
__device__ __forceinline__ uint32_t wide_key(float s) {
  const uint32_t u = __float_as_uint(s);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float wide_unkey(uint32_t key) {
  return __uint_as_float((key & 0x80000000u) ? (key & 0x7fffffffu) : ~key);
}

// The key of the rank-th largest (1-based) real entry (id != INT32_MAX) of the list ls / li [0, n) in global memory;
// the list holds at least `rank` real entries.  4 passes of 8 bits; `hist` = 256 words of the warp's shared-memory
// scratch.  Called warp-uniformly.  (The compactions of the wide filter, score_wide_tc.cu, and of the exact kernel's
// wide mode, score_topk_tc.cu.)
__device__ __forceinline__ uint32_t wide_select(const float* ls, const int32_t* li, int n, int rank, uint32_t* hist,
                                                int lane) {
  uint32_t prefix = 0, mask = 0;
#pragma unroll 1
  for (int shift = 24; shift >= 0; shift -= 8) {
#pragma unroll
    for (int j = 0; j < 8; ++j) hist[8 * lane + j] = 0u;
    __syncwarp();
    for (int i = lane; i < n; i += 32) {
      const uint32_t key = wide_key(ls[i]);
      if (li[i] != 0x7fffffff && (key & mask) == prefix) atomicAdd(hist + ((key >> shift) & 255u), 1u);
    }
    __syncwarp();
    uint32_t c8[8], local = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      c8[j] = hist[8 * lane + j];
      local += c8[j];
    }
    uint32_t incl = local;   // entries in the bins of lanes >= lane
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_down_sync(0xffffffffu, incl, o);
      if (lane + o < 32) incl += t;
    }
    const uint32_t above = incl - local;
    const uint32_t r = static_cast<uint32_t>(rank);
    const int src = __ffs(__ballot_sync(0xffffffffu, above < r && r <= incl)) - 1;
    int bin = 0;
    uint32_t rest = 0, acc = above;
    bool found = false;
#pragma unroll
    for (int j = 7; j >= 0; --j) {
      if (!found && acc + c8[j] >= r) {
        bin = 8 * lane + j;
        rest = r - acc;
        found = true;
      }
      acc += c8[j];
    }
    bin = __shfl_sync(0xffffffffu, bin, src);
    rank = static_cast<int>(__shfl_sync(0xffffffffu, rest, src));
    prefix |= static_cast<uint32_t>(bin) << shift;
    mask |= 255u << shift;
    __syncwarp();   // every lane has read the histogram before the next pass clears it
  }
  return prefix;
}

// four consecutive elements of a split row (hi | lo halves, d_pad apart) as fp32 values hi + lo; zeros past d_pad
__device__ __forceinline__ void load_split4(const __half* __restrict__ row, int d_pad, int lane, bool ok, float (&x)[4]) {
  const int e = lane * 4;
  if (ok && e < d_pad) {
    const uint2 h = __ldg(reinterpret_cast<const uint2*>(row + e));
    const uint2 l = __ldg(reinterpret_cast<const uint2*>(row + d_pad + e));
    const float2 h0 = __half22float2(*reinterpret_cast<const __half2*>(&h.x));
    const float2 h1 = __half22float2(*reinterpret_cast<const __half2*>(&h.y));
    const float2 l0 = __half22float2(*reinterpret_cast<const __half2*>(&l.x));
    const float2 l1 = __half22float2(*reinterpret_cast<const __half2*>(&l.y));
    x[0] = h0.x + l0.x;
    x[1] = h0.y + l0.y;
    x[2] = h1.x + l1.x;
    x[3] = h1.y + l1.y;
  } else {
    x[0] = x[1] = x[2] = x[3] = 0.0f;
  }
}

#endif  // __CUDACC__

}  // namespace trk
