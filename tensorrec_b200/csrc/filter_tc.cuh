// Pieces of the one-pass tensor-core filter (DESIGN §2-3) shared by its narrow form (score_filter_tc.cu, a
// 32-entry candidate buffer per row in shared memory, k <= 12) and its wide form (score_wide_tc.cu, a candidate list
// per row in global memory, k <= 1024): the error-bound constants, the warpgroup's tile MMA (m64n128k16 row halves for
// the narrow form, m64n64k16 column halves for the wide form), the register fast path on the wgmma fragments and the
// per-warp staging of a flagged chunk, with the exclusion cursor.
#pragma once

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
__device__ __forceinline__ float acc_max_16(const uint32_t* acc) {
  float g[4];
  return acc_max_16(acc, g);
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

// order-preserving keys of the wide form's selections: a > b  <=>  key(a) > key(b) for non-NaN floats
__device__ __forceinline__ uint32_t wide_key(float s) {
  const uint32_t u = __float_as_uint(s);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float wide_unkey(uint32_t key) {
  return __uint_as_float((key & 0x80000000u) ? (key & 0x7fffffffu) : ~key);
}

}  // namespace trk
