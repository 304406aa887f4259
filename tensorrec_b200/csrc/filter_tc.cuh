// Pieces of the one-pass tensor-core filter (DESIGN §2-3) shared by its narrow form (score_filter_tc.cu, a
// 32-entry candidate buffer per row in shared memory, k <= 12) and its wide form (score_wide_tc.cu, a candidate list
// per row in global memory, k <= 1024):
//   * the sweep skeleton: the parameters both forms read, the shared-memory layout and barriers, the TMA producer warp,
//     the consumers' work-unit decode, row constants, user-block load and B-slot release, and the host launcher (stage
//     count, launch form, tensor maps).  None of it depends on how a form stores its candidates;
//   * the error-bound constants, the warpgroup's tile MMA (m64n128k16 row halves for the narrow form, m64n64k16 column
//     halves for the wide form), the register fast path on the wgmma fragments and the per-warp staging of a flagged
//     chunk, with the exclusion cursor.
// Each form keeps its own kernel body: its tile epilogue, compaction and output.
#pragma once

#include <stdlib.h>

#include "common.cuh"

namespace trk {

constexpr uint32_t kWarpStageBytes = 32 * 32 * 4u;   // 32 rows x 32 fp32 per consumer warp
constexpr uint32_t kAccStageBytes = 4 * kWarpStageBytes;   // per warpgroup
constexpr float kMarginFactor = 1.5f * 0.0009765625f;   // 1.5 * 2^-10
constexpr float kBiasUlps = 4.0f * 1.1920929e-7f;        // 4 ulp(1): rounding of (dot + ub) + ib
constexpr float kThetaMargins = 2.25f;                   // theta = a_k - 2.25 m  (> 2 m is what the proof needs)
constexpr int kGiveUpOverflows = 8;   // a row whose compactions overflow this often is handed to the exact kernel

// Inputs of the admission path that are the same for the whole kernel.
struct AdmitCtx {
  const float* bias;     // item biases in processing order, padded with -inf
  const int32_t* perm;   // processing position -> local item index, or null = identity
  int32_t id_offset;
  int32_t n_items;
  int32_t k;
};

// theta -> tau: the admission test runs on v = acc + bias / c; a few ulps of slack (extra survivors are harmless, a
// missed one is not)
template <class Row>
__device__ __forceinline__ void set_tau(Row& r) {
  const float t = (r.theta - r.ubias) * r.inv_c;
  r.tau = t - 8.0f * 1.1920929e-7f * fabsf(t) - 1e-30f;
}

// ---- the sweep skeleton ---------------------------------------------------------------------------------------------
// A work unit is 256 user rows (two 128-row blocks, one per consumer warpgroup) x an item split.  Warp 0 streams the
// split's 128-item tiles with TMA into a ring of tile slots; consumer warpgroup g (warps 4+4g..7+4g) loads user block g
// once per unit and runs the form's epilogue on every tile, so every B tile fetched from L2 feeds two warpgroups.
// Template parameters of both kernels: kNKB = k-blocks of 64 per row (d_pad / 64); kCluster = 1, or 2 = clusters of two
// CTAs on two different user pairs over the SAME item tiles, each CTA fetching half of every tile and TMA-multicasting it
// into both (the L2 -> SM stream of the item operand is halved); kExclude = mask each row's exclusion list
// (excl_indptr / excl_pos) out of the candidate universe, see excl_mask_chunk.

// The inputs and shapes both forms read (FilterParams / WideParams hold one, plus their candidate storage).
struct SweepParams {
  const float* user_scale;
  const float* user_bias;      // may be null
  const float* user_norm;      // |u|_2 per user
  const float* item_bias;      // [padded items] in PROCESSING order (see item_perm), padding = -inf
  const float* block_bias_max; // max item bias of every block of 128 processing positions (-inf for all-padding)
  const int32_t* item_perm;    // processing position -> local item index (items sorted by bias), or null = identity
  const float* item_stats;     // device: [0] = max_j |i_j|_2, [1] = global item scale (2^-E), [2] = max_j |bias_j|
  int64_t n_users;
  int64_t n_items;
  int32_t n_stages;            // B ring in k-block tiles
  int32_t k;
  int32_t n_splits;
  int32_t tiles_per_split;
  int32_t n_tiles;
  int32_t n_user_pairs;        // ceil(n_users / 256)
  int32_t item_id_offset;
  float* row_theta;            // [n_users, n_splits] max(theta, drop_max), certified by the form's rescore kernel
  // exclusion lists (kExclude instantiations only): row u's excluded items as PROCESSING positions, ascending, at
  // excl_pos[excl_indptr[u] .. excl_indptr[u + 1])
  const int32_t* excl_indptr;
  const int32_t* excl_pos;
};

// Shared memory: user blocks 0 and 1 (n_kblocks tiles each), the B ring, `extra_bytes` of the form's own at extra_off,
// the consumer warps' staging tiles and the barriers.
struct SweepLayout {
  uint32_t a_off, b_off, extra_off, acc_off, bar_off, total;
};
__host__ __device__ inline SweepLayout sweep_layout(int n_kblocks, int n_stages, uint32_t extra_bytes) {
  SweepLayout L;
  L.a_off = 0;
  L.b_off = L.a_off + 2u * static_cast<uint32_t>(n_kblocks) * kATileBytes;
  L.extra_off = L.b_off + static_cast<uint32_t>(n_stages) * kBTileBytes;
  L.acc_off = L.extra_off + extra_bytes;
  L.bar_off = L.acc_off + 2u * kAccStageBytes;
  L.total = L.bar_off + 512u;
  return L;
}
// The B ring is organised in TILE slots of n_kblocks k-blocks (16 KB each): one full / one empty barrier per item tile.
// barriers (uint64): [0..1] a_full (per user block) [2 .. 2+T) b_full [2+T .. 2+2T) b_empty, T = n_stages / n_kblocks
// tile slots.  b_empty counts the 8 consumer warps of every CTA that received the tile.
// The item biases are NOT staged: the hot loop needs only the block maximum (one cached global load per tile,
// prefetched a tile ahead) and the rare admission path reads the few biases it needs through L2.

// What every thread of the CTA knows about the sweep after sweep_prologue.
struct SweepCta {
  uint8_t* smem;
  SweepLayout L;
  int n_slots;                  // B tile slots
  uint64_t* a_full;             // [user block]
  uint64_t* b_full;             // [slot]
  uint64_t* b_empty;            // [slot]
  uint32_t crank;               // rank in the cluster
  int n_groups;                 // groups of kCluster user pairs
  int64_t n_work, w_first, w_step;   // work units, this CTA's first one and its stride
};

// Tensor-map prefetch, barrier init and (kCluster = 2) the cluster sync after which the peer's barriers exist.
template <int kNKB, int kCluster>
__device__ __forceinline__ SweepCta sweep_prologue(const SweepParams& p, uint32_t extra_bytes,
                                                   const CUtensorMap* map_users, const CUtensorMap* map_items) {
  SweepCta cta;
  cta.smem = smem_base_1024();
  cta.L = sweep_layout(kNKB, p.n_stages, extra_bytes);
  cta.n_slots = p.n_stages / kNKB;
  uint64_t* bars = reinterpret_cast<uint64_t*>(cta.smem + cta.L.bar_off);
  cta.a_full = bars + 0;
  cta.b_full = bars + 2;
  cta.b_empty = bars + 2 + cta.n_slots;

  const int warp = threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  // work unit = (group of kCluster user pairs, item split); CTA `crank` of the cluster takes pair kCluster * g + crank
  cta.crank = kCluster == 2 ? cluster_ctarank() : 0u;
  cta.n_groups = (p.n_user_pairs + kCluster - 1) / kCluster;
  cta.n_work = static_cast<int64_t>(cta.n_groups) * p.n_splits;
  cta.w_first = blockIdx.x / kCluster;
  cta.w_step = gridDim.x / kCluster;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(map_items);
    tma_prefetch_desc(map_users);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < 2; ++i) mbar_init(cta.a_full + i, 1);
    for (int i = 0; i < cta.n_slots; ++i) {
      mbar_init(cta.b_full + i, 1);
      mbar_init(cta.b_empty + i, 8 * kCluster);   // the consumer warps of all CTAs that received the tile
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (kCluster == 2) cluster_sync_all();   // the peer's barriers exist before anything is multicast to them
  return cta;
}

// Register budget: the producer warpgroup (one issuing warp) needs few, the consumers hold the accumulators, a staged
// row and the admission state per thread (40 x 128 + 232 x 256 = 64,512 of the 65,536 registers).  Returns whether
// `warp` is in the producer warpgroup.
__device__ __forceinline__ bool sweep_split_registers(int warp) {
  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    return true;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
  return false;
}

// Work unit w as a consumer thread of warpgroup `group` that owns block row `row` sees it (the producer passes 0, 0
// and reads the tile range only).
struct SweepUnit {
  int sp, t0, t1;               // item split, its tiles [t0, t1)
  int64_t ublock_row0;          // first row of the warpgroup's user block
  int64_t u;                    // the thread's user row
  bool u_ok;                    // u < n_users
};
template <int kCluster>
__device__ __forceinline__ SweepUnit sweep_unit(const SweepParams& p, const SweepCta& cta, int64_t w, int group,
                                                int row) {
  SweepUnit wu;
  const int up = static_cast<int>(w % cta.n_groups) * kCluster + static_cast<int>(cta.crank);
  wu.sp = static_cast<int>(w / cta.n_groups);
  wu.t0 = wu.sp * p.tiles_per_split;
  wu.t1 = min(wu.t0 + p.tiles_per_split, p.n_tiles);
  wu.ublock_row0 = (static_cast<int64_t>(up) * 2 + group) * kBlockM;
  wu.u = wu.ublock_row0 + row;
  wu.u_ok = wu.u < p.n_users;
  return wu;
}

__device__ __forceinline__ void sweep_ring_advance(int& ts, uint32_t& ts_phase, int n_slots) {
  if (++ts == n_slots) {
    ts = 0;
    ts_phase ^= 1;
  }
}

// Warp 0: every tile of every work unit of this CTA into the ring, warp-uniform control flow, one elected lane issues.
// (TRK_FILTER_CYCLES builds: `empty_wait`, if given, accumulates the clocks spent waiting for a free slot.)
template <int kNKB, int kCluster>
__device__ __forceinline__ void sweep_producer(const SweepParams& p, const SweepCta& cta,
                                               const CUtensorMap* map_items
#ifdef TRK_FILTER_CYCLES
                                               , unsigned long long* empty_wait = nullptr
#endif
) {
  constexpr uint32_t kSlotBytes = kNKB * kBTileBytes;
  constexpr uint16_t kClusterMask = (1u << kCluster) - 1u;
  uint8_t* const ring = cta.smem + cta.L.b_off;
  int ts = 0;
  uint32_t ts_phase = 0;
  for (int64_t w = cta.w_first; w < cta.n_work; w += cta.w_step) {
    const SweepUnit wu = sweep_unit<kCluster>(p, cta, w, 0, 0);
    for (int t = wu.t0; t < wu.t1; ++t) {
#ifdef TRK_FILTER_CYCLES
      const long long c0 = clock64();
#endif
      if (kCluster == 2)
        mbar_wait_cluster(cta.b_empty + ts, ts_phase ^ 1);
      else
        mbar_wait(cta.b_empty + ts, ts_phase ^ 1);
#ifdef TRK_FILTER_CYCLES
      if (empty_wait != nullptr) *empty_wait += clock64() - c0;
#endif
      if (elect_one()) {
        mbar_arrive_expect_tx(cta.b_full + ts, kSlotBytes);
#pragma unroll
        for (int kb = 0; kb < kNKB; ++kb) {
          if (kCluster == 2)   // this CTA's half of the tile rows (box = 64 rows), delivered to both CTAs
            tma_load_2d_multicast(ring + ts * kSlotBytes + kb * kBTileBytes + cta.crank * (kBTileBytes / 2), map_items,
                                  cta.b_full + ts, kb * kKBlock,
                                  t * kBlockN + static_cast<int>(cta.crank) * (kBlockN / 2), kClusterMask, kEvictLast);
          else
            tma_load_2d(ring + ts * kSlotBytes + kb * kBTileBytes, map_items, cta.b_full + ts, kb * kKBlock,
                        t * kBlockN, kEvictLast);
        }
      }
      __syncwarp();
      sweep_ring_advance(ts, ts_phase, cta.n_slots);
    }
  }
}

// The row constants of the unit's user row (fields m3, ubias, c, inv_c of the form's row state): the margin 2.25 m,
// the user bias, c = user scale x global item scale (powers of two: exact) and 1 / c.  Returns the exclusion cursor
// (kExclude): the first excluded processing position of the row in the unit's tiles, INT32_MAX if none.
template <bool kExclude, class Row>
__device__ __forceinline__ int32_t sweep_row_start(Row& r, const SweepParams& p, const SweepUnit& wu,
                                                   float max_item_norm, float item_scale, float max_item_bias) {
  const float su = wu.u_ok ? __ldg(p.user_scale + wu.u) : 1.0f;
  const float ubias = (wu.u_ok && p.user_bias != nullptr) ? __ldg(p.user_bias + wu.u) : 0.0f;
  const float unorm = wu.u_ok ? __ldg(p.user_norm + wu.u) : 0.0f;
  r.ubias = ubias;
  r.c = su * item_scale;
  r.inv_c = 1.0f / r.c;
  // error bound of one approximate score: operand rounding + the fp32 rounding of the two bias adds
  r.m3 = kThetaMargins * (kMarginFactor * unorm * max_item_norm + kBiasUlps * (fabsf(ubias) + max_item_bias));
  int32_t excl_next = 0x7fffffff;
  if constexpr (kExclude) {
    if (wu.u_ok && wu.t1 > wu.t0) excl_next = excl_next_at(p.excl_indptr, p.excl_pos, wu.u, wu.t0 * kBlockN);
  }
  return excl_next;
}

// The warpgroup's user block (hi half, fp16; rows past n_users arrive as zeros) goes to shared memory.  Every wgmma of
// the previous unit has completed in all four warps once they pass the named barrier.  Called by the whole warpgroup.
template <int kNKB>
__device__ __forceinline__ void sweep_load_user_block(const SweepCta& cta, const CUtensorMap* map_users,
                                                      const SweepUnit& wu, int group, int warp, int lane,
                                                      uint32_t& witer) {
  if (wu.t1 > wu.t0) {
    named_barrier_sync(1 + group, kConsumerThreads);
    if (warp % 4 == 0 && lane == 0) {
      mbar_arrive_expect_tx(cta.a_full + group, kNKB * kATileBytes);
#pragma unroll
      for (int kb = 0; kb < kNKB; ++kb)
        tma_load_2d(cta.smem + cta.L.a_off + (group * kNKB + kb) * kATileBytes, map_users, cta.a_full + group,
                    kb * kKBlock, static_cast<int32_t>(wu.ublock_row0), kEvictFirst);
    }
    mbar_wait(cta.a_full + group, witer & 1);
    ++witer;
  }
}

// After the warp's last MMAs of a tile: release B slot ts in every CTA that received it.  Called warp-uniformly.
template <int kCluster>
__device__ __forceinline__ void sweep_release_slot(const SweepCta& cta, int ts, int lane) {
  __syncwarp();
  if (lane == 0) {
    if (kCluster == 2) {
#pragma unroll
      for (uint32_t r = 0; r < kCluster; ++r) mbar_arrive_cluster(cta.b_empty + ts, r);
    } else {
      mbar_arrive(cta.b_empty + ts);
    }
  }
}

// Every excluded or dropped item has an approximate score <= max(theta, drop_max); a NaN (inf - inf with infinite
// biases) must not read as "nothing was excluded": +inf makes the certificate fail and the row goes through the exact
// kernel.
template <class Row>
__device__ __forceinline__ void sweep_store_theta(const SweepParams& p, int64_t list, const Row& r) {
  const bool th_nan = r.theta != r.theta || r.drop_max != r.drop_max;
  p.row_theta[list] = th_nan ? __int_as_float(0x7f800000) : fmaxf(r.theta, r.drop_max);
}

__device__ __forceinline__ float ldg_nc_f32(const float* p) {
  float v;
  asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ int32_t ldg_nc_s32(const int32_t* p) {
  int32_t v;
  asm volatile("ld.global.nc.s32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}

// maximum of 16 columns; g[q] = maximum of columns [4q, 4q + 4) (the slow path looks only into the groups that pass)
__device__ __forceinline__ float acc_max_16(const uint32_t* acc, float (&g)[4]) {
#pragma unroll
  for (int q = 0; q < 4; ++q)
    g[q] = fmaxf(fmaxf(__uint_as_float(acc[4 * q]), __uint_as_float(acc[4 * q + 1])),
                 fmaxf(__uint_as_float(acc[4 * q + 2]), __uint_as_float(acc[4 * q + 3])));
  return fmaxf(fmaxf(g[0], g[1]), fmaxf(g[2], g[3]));
}

// Bit mask of the columns of acc[0, 16) whose admission bound passes.  g[q] = maximum of columns [4q, 4q + 4) from the
// hot loop: only a group whose maximum passes is looked into (x -> x + bmax is monotonic), so the usual single hit
// costs 4 + 4 compares instead of 16; independent compares, OR'ed pairwise (a serial `mask |= ...` chain put ~80 cycles
// of dependent latency into every slow-path entry).
__device__ __forceinline__ uint32_t pass_mask_16(const uint32_t* acc, const float (&g)[4], float bmax_scaled,
                                                 float tau) {
  uint32_t mask = 0;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    if (g[q] + bmax_scaled > tau) {
      const uint32_t b0 = (__uint_as_float(acc[4 * q + 0]) + bmax_scaled > tau) ? (1u << (4 * q + 0)) : 0u;
      const uint32_t b1 = (__uint_as_float(acc[4 * q + 1]) + bmax_scaled > tau) ? (1u << (4 * q + 1)) : 0u;
      const uint32_t b2 = (__uint_as_float(acc[4 * q + 2]) + bmax_scaled > tau) ? (1u << (4 * q + 2)) : 0u;
      const uint32_t b3 = (__uint_as_float(acc[4 * q + 3]) + bmax_scaled > tau) ? (1u << (4 * q + 3)) : 0u;
      mask |= (b0 | b1) | (b2 | b3);
    }
  }
  return mask;
}

// ---- a consumer warp's 32 rows: fragments, fast path, staging ------------------------------------------------------
// The warpgroup computes a tile's 128 x 128 accumulator as two row halves (filter_mma_rows): in row half rh, lane l of
// warp w holds the 128 columns of block rows 64 rh + 16 w + l / 4 + 8 s, s = 0, 1 (wgmma_acc_row).  Lane L of the warp
// OWNS (keeps the admission state of) block row 16 w + L % 16 + 64 (L / 16): lane 16 rh + 8 s + g owns the row that
// the lanes of quad g hold as class s in row half rh.  Its staged row is row L of the warp's 32 x 32 staging tile.
__device__ __forceinline__ int filter_owned_row(int warp_in_group, int lane) {
  return 16 * warp_in_group + (lane & 15) + 64 * (lane >> 4);
}

// Each lane's copies of a per-row value x of its two fragment rows of row half rh: f[s] = x of the owner lane
// 16 rh + 8 s + l / 4.  The fast path needs the rows' tau (taken after the row half's MMAs and again after every slow
// path, whose compactions raise it) and their bias bound bmax / c (c is the row's user scale).
__device__ __forceinline__ void frag_rows(float x, int rh, int lane, float (&f)[2]) {
  f[0] = __shfl_sync(0xffffffffu, x, 16 * rh + (lane >> 2));
  f[1] = __shfl_sync(0xffffffffu, x, 16 * rh + 8 + (lane >> 2));
}

// Fast path of columns [32 c, 32 c + 32) of a row half: does one of the lane's two fragment rows pass its bound on the
// 8 columns the lane holds of it (registers 16 c + 4 j + 2 s + {0, 1}, j < 4)?  bf / tf: frag_rows of the rows' bias
// bound and tau.  Rounding is monotonic, so fl(max_i m_i + b) = max_i fl(m_i + b): a warp vote on this flag is the
// vote on the 32-column row maxima.
template <int c>
__device__ __forceinline__ bool chunk_frag_pass(const float (&acc)[64], const float (&bf)[2], const float (&tf)[2]) {
  bool pass = false;
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    const int i = 16 * c + 2 * s;
    const float m = fmaxf(fmaxf(fmaxf(acc[i], acc[i + 1]), fmaxf(acc[i + 4], acc[i + 5])),
                          fmaxf(fmaxf(acc[i + 8], acc[i + 9]), fmaxf(acc[i + 12], acc[i + 13])));
    pass = pass || m + bf[s] > tf[s];
  }
  return pass;
}

// The staging tile of a warp: row r at r * 128 bytes, column x at word x ^ stage_swizzle(r % 8), an XOR of bits 2..4
// that keeps 2- and 4-word groups together.  Stores (st.shared.v2: one quad-row of 8 columns per lane pair) and the
// owner's row loads (ld.shared.v4) are both free of bank conflicts.  One store instruction writes, for a fixed
// column block j and class s, the tile rows 16 rh + 8 s + g of all 8 quads g; a half-warp of it covers quads 0..3 or
// 4..7, whose swizzles 8 (g % 4) (+ 4), XOR'ed with the common 8 j, send its 16 column pairs to 16 different bank
// pairs.  A quarter-warp of loads reads 8 rows whose swizzles 4 * {0..7} differ, so its 16-byte groups land in 8
// different bank quads.
__device__ __forceinline__ uint32_t stage_swizzle(int g) { return 4u * static_cast<uint32_t>(((g & 3) << 1) | (g >> 2)); }
__device__ __forceinline__ void f_sts32(uint32_t addr, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}

// Writes columns [32 c, 32 c + 32) of the warp's 16 fragment rows of row half rh to rows 16 rh .. 16 rh + 15 of its
// staging tile (base `stage`): afterwards each owner lane 16 rh + i finds its row's 32 raw accumulators with
// load_staged_row; the rows of the other half keep what they held.  Called warp-uniformly.
template <int c>
__device__ __forceinline__ void stage_warp_chunk(const float (&acc)[64], int rh, uint32_t stage, int lane) {
  __syncwarp();   // every lane has read its row of the previous staged chunk
  const int g = lane >> 2;
  const uint32_t col0 = 2u * static_cast<uint32_t>(lane & 3) ^ stage_swizzle(g);
  const uint32_t row_g = stage + 2048u * static_cast<uint32_t>(rh) + 128u * g;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t a = row_g + 4u * (col0 ^ (8u * j));
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const int i = 16 * c + 4 * j + 2 * s;   // class s: tile row 16 rh + 8 s + g
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a + 1024u * s), "f"(acc[i]), "f"(acc[i + 1]) : "memory");
    }
  }
  __syncwarp();
}
// the 32 staged raw accumulators of the lane's own row, in column order
__device__ __forceinline__ void load_staged_row(uint32_t stage, int lane, uint32_t (&v)[32]) {
  const uint32_t row = stage + 128u * lane, sw = stage_swizzle(lane & 7);
#pragma unroll
  for (uint32_t q = 0; q < 8; ++q)
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v[4 * q]), "=r"(v[4 * q + 1]), "=r"(v[4 * q + 2]), "=r"(v[4 * q + 3])
                 : "r"(row + 4u * ((4u * q) ^ sw))
                 : "memory");
}

// Exclusion (kExclude): every consumer lane keeps ONE register, `next` = the first excluded processing position of its
// row at or after the chunk being filtered (INT32_MAX: none left).  When it falls inside the staged chunk [base,
// base + 32) -- rare, divergent -- this writes -inf over the lane's own staged raw accumulators of every listed
// position of the chunk (only this lane reads that staged row: no synchronisation) and returns the new `next`, the
// first listed position past the chunk.  A -inf accumulator never passes the admission bound (-inf + x > tau is false even for tau = -inf), and it is the
// neutral element of the warm start's group maxima, so an excluded item neither becomes a candidate nor sets a threshold.
// (inline: one definition for every translation unit that includes this header)
inline __device__ __noinline__ int32_t excl_mask_chunk(const int32_t* indptr, const int32_t* pos, int64_t u,
                                                       int32_t base, uint32_t stage, int lane) {
  const uint32_t row = stage + 128u * lane, sw = stage_swizzle(lane & 7);
  const int hi = __ldg(indptr + u + 1);
  int i = excl_lower_bound(pos, __ldg(indptr + u), hi, base);
  int32_t e = i < hi ? __ldg(pos + i) : 0x7fffffff;
  while (e < base + 32) {
    f_sts32(row + 4u * (static_cast<uint32_t>(e - base) ^ sw), -__int_as_float(0x7f800000));
    ++i;
    e = i < hi ? __ldg(pos + i) : 0x7fffffff;
  }
  return e;
}

// Row half rh of the tile in B slot `b_slot`: block rows [64 rh, 64 rh + 64) x all 128 items, fp16 hi x hi, fp32
// accumulate.  One N = 128 chain reads every user element once per tile, where two 64-column halves read it twice; with
// the admission epilogue replaced by a maximum over the accumulators, that made the sweep 4 % faster (DESIGN §5).
template <int kNKB>
__device__ __forceinline__ void filter_mma_rows(float (&acc)[64], uint32_t a_base, uint32_t b_slot, int rh) {
  wgmma_fence();
#pragma unroll
  for (int kb = 0; kb < kNKB; ++kb) {
#pragma unroll
    for (int ks = 0; ks < kKBlock / kMmaK; ++ks) {
      const uint64_t db = wgmma_desc_k_major_sw128(b_slot + kb * kBTileBytes) + 2u * ks;
      const uint64_t da = wgmma_desc_k_major_sw128(a_base + kb * kATileBytes) + 2u * ks +
                          static_cast<uint32_t>(rh) * ((kATileBytes / 2) >> 4);   // rows 64..127: +8 KB
      wgmma_m64n128k16_f16(acc, da, db, static_cast<uint32_t>(kb > 0 || ks > 0));
    }
  }
  wgmma_commit();
  wgmma_wait<0>();
}

// ---- the wide form (score_wide_tc.cu): the tile in two 64-column halves --------------------------------------------
// Its slow path runs far more often than the narrow form's (no warm start, k up to 1024), and a flagged 32-column
// chunk of a half covers all 32 rows of the warp rather than the 16 of a row half: there, the 64-row halves made the
// k = 100 sweep 39 % slower (DESIGN §5).  acc0 / acc1 hold block rows 16 w + l / 4 (+ 8) and 64 + the same: lane L
// owns the row of class q = L / 8, quad g = L % 8, where class 0/1 = acc0 row +0 / +8 and class 2/3 = acc1 row +0 / +8
// (filter_owned_row).

// Maximum of the raw accumulators of columns [32 c, 32 c + 32) of the half, for the row this lane owns.  Each lane
// reduces the 8 columns it holds of each of its 4 rows; a reduce-scatter through the quad (2 + 1 shuffles) leaves lane
// l with the full maximum of class l % 4 of quad l / 4, and one more shuffle brings it to the owner.  fmaxf is exact,
// so this is the maximum the staged row would give.
template <int c>
__device__ __forceinline__ float chunk_row_max(const float (&acc0)[32], const float (&acc1)[32], int lane) {
  float m[4];
#pragma unroll
  for (int s = 0; s < 2; ++s) {   // registers 16 c + 4 j + 2 s + {0, 1}, j < 4: row +8 s, 8 columns
    const int i = 16 * c + 2 * s;
    m[s] = fmaxf(fmaxf(fmaxf(acc0[i], acc0[i + 1]), fmaxf(acc0[i + 4], acc0[i + 5])),
                 fmaxf(fmaxf(acc0[i + 8], acc0[i + 9]), fmaxf(acc0[i + 12], acc0[i + 13])));
    m[2 + s] = fmaxf(fmaxf(fmaxf(acc1[i], acc1[i + 1]), fmaxf(acc1[i + 4], acc1[i + 5])),
                     fmaxf(fmaxf(acc1[i + 8], acc1[i + 9]), fmaxf(acc1[i + 12], acc1[i + 13])));
  }
  const bool b0 = (lane & 1) != 0, b1 = (lane & 2) != 0;
  // step 1 (lane ^ 1): keep the classes with bit 0 = b0, send the other two
  const float k0 = fmaxf(b0 ? m[1] : m[0], __shfl_xor_sync(0xffffffffu, b0 ? m[0] : m[1], 1));   // class b0
  const float k1 = fmaxf(b0 ? m[3] : m[2], __shfl_xor_sync(0xffffffffu, b0 ? m[2] : m[3], 1));   // class 2 + b0
  // step 2 (lane ^ 2): keep class b0 + 2 b1 = lane % 4
  const float r = fmaxf(b1 ? k1 : k0, __shfl_xor_sync(0xffffffffu, b1 ? k0 : k1, 2));
  return __shfl_sync(0xffffffffu, r, 4 * (lane & 7) + (lane >> 3));   // owner 8 q + g <- lane 4 g + q
}

// Writes columns [32 c, 32 c + 32) of the warp's four fragment rows of the 128 x 64 half to its staging tile (base
// `stage`): afterwards lane L finds its row's 32 raw accumulators with load_staged_row.  Called warp-uniformly.
template <int c>
__device__ __forceinline__ void stage_warp_chunk(const float (&acc0)[32], const float (&acc1)[32], uint32_t stage,
                                                 int lane) {
  __syncwarp();   // every lane has read its row of the previous staged chunk
  const int g = lane >> 2;
  const uint32_t col0 = 2u * static_cast<uint32_t>(lane & 3) ^ stage_swizzle(g);
  const uint32_t row_g = stage + 128u * g;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t a = row_g + 4u * (col0 ^ (8u * j));
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const int i = 16 * c + 4 * j + 2 * s;   // rows of class s (acc0) and 2 + s (acc1): tile rows 8 s + g, 16 + 8 s + g
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a + 1024u * s), "f"(acc0[i]), "f"(acc0[i + 1]) : "memory");
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a + 1024u * (2 + s)), "f"(acc1[i]), "f"(acc1[i + 1])
                   : "memory");
    }
  }
  __syncwarp();
}

// 128 user rows x 64 items (column half `h` of the tile in B slot `b_slot`), fp16 hi x hi, fp32 accumulate
template <int kNKB>
__device__ __forceinline__ void filter_mma_half(float (&acc0)[32], float (&acc1)[32], uint32_t a_base, uint32_t b_slot,
                                                int h) {
  wgmma_fence();
#pragma unroll
  for (int kb = 0; kb < kNKB; ++kb) {
#pragma unroll
    for (int ks = 0; ks < kKBlock / kMmaK; ++ks) {
      const uint64_t db = wgmma_desc_k_major_sw128(b_slot + kb * kBTileBytes + h * (kBTileBytes / 2)) + 2u * ks;
      const uint64_t da = wgmma_desc_k_major_sw128(a_base + kb * kATileBytes) + 2u * ks;
      const uint32_t accumulate = static_cast<uint32_t>(kb > 0 || ks > 0);
      wgmma_m64n64k16_f16(acc0, da, db, accumulate);
      wgmma_m64n64k16_f16(acc1, da + ((kATileBytes / 2) >> 4), db, accumulate);   // rows 64..127: +8 KB
    }
  }
  wgmma_commit();
  wgmma_wait<0>();
}

// ---- host: the launcher of both forms -------------------------------------------------------------------------------
// Checks the arguments both C entry points take (messages prefixed with `name`), fills p.sweep, picks the stage count
// and the launch form, encodes the two tensor maps and launches Kernel<d_pad / 64, cluster, exclusion>::fn.  The
// caller has checked and filled its own part of p; `extra_bytes` is its shared memory (sweep_layout).
//
// Launch form: clusters of two CTAs sharing every item tile through TMA multicast (default when the device can keep
// (almost) all SMs busy with 2-CTA clusters), else independent CTAs.  TRK_FILTER_CLUSTER=1|2 forces one.
template <template <int, int, bool> class Kernel, class P>
int launch_sweep(const char* name, P p, uint32_t extra_bytes, const void* user_split, const float* user_scale,
                 const float* user_bias, const float* user_norm, const void* item_hi, const float* item_stats,
                 const float* item_bias, const float* block_bias_max, const int32_t* item_perm, int64_t n_users,
                 int64_t n_items, int32_t d_pad, int32_t k, int32_t n_splits, int32_t item_id_offset,
                 float* row_theta, const int32_t* excl_indptr, const int32_t* excl_pos, cudaStream_t stream) {
  TRK_CHECK_ARG(user_split && user_scale && user_norm && item_hi && item_stats && item_bias && block_bias_max,
                "%s: null input", name);
  TRK_CHECK_ARG((excl_indptr == nullptr) == (excl_pos == nullptr), "%s: excl_indptr and excl_pos go together", name);
  TRK_CHECK_ARG(n_users >= 1 && n_items >= 1 && n_splits >= 1, "%s: empty shape", name);
  TRK_CHECK_ARG(n_users < (1ll << 31) && n_items < (1ll << 31) - 512, "%s: shape exceeds int32 indexing", name);
  if (d_pad != 64 && d_pad != 128) {
    set_error("%s: d_pad=%d not supported (64 or 128)", name, d_pad);
    return TRK_ERR_UNSUPPORTED;
  }
  TRK_CHECK_ARG(reinterpret_cast<uintptr_t>(user_split) % 16 == 0 && reinterpret_cast<uintptr_t>(item_hi) % 16 == 0,
                "%s: operands must be 16-byte aligned", name);

  SweepParams& s = p.sweep;
  s.user_scale = user_scale;
  s.user_bias = user_bias;
  s.user_norm = user_norm;
  s.item_bias = item_bias;
  s.block_bias_max = block_bias_max;
  s.item_perm = item_perm;
  s.item_stats = item_stats;
  s.n_users = n_users;
  s.n_items = n_items;
  s.k = k;
  s.n_tiles = static_cast<int32_t>(ceil_div(n_items, kBlockN));
  s.n_splits = n_splits;
  s.tiles_per_split = static_cast<int32_t>(ceil_div(s.n_tiles, n_splits));
  s.n_user_pairs = static_cast<int32_t>(ceil_div(n_users, 2 * kBlockM));
  s.item_id_offset = item_id_offset;
  s.row_theta = row_theta;
  s.excl_indptr = excl_indptr;
  s.excl_pos = excl_pos;
  const int n_kblocks = d_pad / kKBlock;
  s.n_stages = 0;
  for (int st = kMaxStages; st >= 2; --st)
    if (st % n_kblocks == 0 && sweep_layout(n_kblocks, st, extra_bytes).total + kSmemAlignSlack <= kSmemLimit) {
      s.n_stages = st;
      break;
    }
  TRK_CHECK_ARG(s.n_stages >= 2 * n_kblocks, "%s: shared memory budget exceeded", name);
  const uint32_t smem_bytes = sweep_layout(n_kblocks, s.n_stages, extra_bytes).total + kSmemAlignSlack;

  const bool excl = excl_indptr != nullptr;
  using KernelFn = void (*)(CUtensorMap, CUtensorMap, P);
  const KernelFn kernel2 = excl ? (n_kblocks == 2 ? Kernel<2, 2, true>::fn : Kernel<1, 2, true>::fn)
                                : (n_kblocks == 2 ? Kernel<2, 2, false>::fn : Kernel<1, 2, false>::fn);
  const KernelFn kernel1 = excl ? (n_kblocks == 2 ? Kernel<2, 1, true>::fn : Kernel<1, 1, true>::fn)
                                : (n_kblocks == 2 ? Kernel<2, 1, false>::fn : Kernel<1, 1, false>::fn);
  int cluster = 2;
  const char* env = getenv("TRK_FILTER_CLUSTER");
  if (env != nullptr && (atoi(env) == 1 || atoi(env) == 2)) cluster = atoi(env);
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  int max_clusters = 0;
  if (cluster == 2) {
    TRK_CHECK_CUDA(cudaFuncSetAttribute(kernel2, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    cfg.gridDim = dim3(2);
    cfg.blockDim = dim3(kTcThreads);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.stream = stream;
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    // the answer depends on (device, kernel, shared memory) only: asked once per device and kernel (one table per
    // form, indexed by n_kblocks x exclusion)
    static int cached_clusters[64][4];
    static bool cached_valid[64][4];
    int device = 0;
    TRK_CHECK_CUDA(cudaGetDevice(&device));
    const int variant = (n_kblocks == 2 ? 1 : 0) + (excl ? 2 : 0);
    if (device >= 0 && device < 64 && cached_valid[device][variant]) {
      max_clusters = cached_clusters[device][variant];
    } else {
      if (cudaOccupancyMaxActiveClusters(&max_clusters, kernel2, &cfg) != cudaSuccess) {
        (void)cudaGetLastError();
        max_clusters = 0;
      }
      if (device >= 0 && device < 64) {
        cached_clusters[device][variant] = max_clusters;
        cached_valid[device][variant] = true;
      }
    }
    if (max_clusters * 2 < sm_count() - 8 && env == nullptr) cluster = 1;   // too many SMs would sit idle
    if (max_clusters < 1) cluster = 1;
  }
  // fp16 operands, boxes of one k-block: the items [n_items, d_pad] (each CTA of a cluster fetches half of a tile) and
  // the hi half of the split user rows [n_users, 2 d_pad]
  CUtensorMap map_users, map_items;
  int rc = encode_tiled_2d(&map_items, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, item_hi, d_pad, n_items, 2 * d_pad, kKBlock,
                           kBlockN / cluster, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (rc != TRK_OK) return rc;
  rc = encode_tiled_2d(&map_users, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, user_split, d_pad, n_users, 4 * d_pad, kKBlock,
                       kBlockM, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (rc != TRK_OK) return rc;
  if (cluster == 2) {
    const int64_t n_work = ceil_div(static_cast<int64_t>(s.n_user_pairs), 2) * n_splits;
    const int n_clusters = static_cast<int>(n_work < max_clusters ? n_work : max_clusters);
    cfg.gridDim = dim3(static_cast<unsigned>(2 * n_clusters));
    TRK_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kernel2, map_users, map_items, p));
  } else {
    TRK_CHECK_CUDA(cudaFuncSetAttribute(kernel1, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    const int grid = capped_grid(static_cast<int64_t>(s.n_user_pairs) * n_splits, 1);
    kernel1<<<grid, kTcThreads, smem_bytes, stream>>>(map_users, map_items, p);
  }
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

}  // namespace trk
