// Wide form of the one-pass tensor-core filter (score_filter_tc.cu, DESIGN §3.3): the same warp-specialised CTA, the
// same fp16 "hi" operands in descending-bias order, the same register fast path on the wgmma fragments and the same
// per-warp staging of flagged chunks -- but every user row keeps its candidates in a list in GLOBAL memory, so k is not
// bounded by a 32-entry shared-memory buffer: 32 < k <= kWideMaxK.
//
// Per (row, item split) the list holds up to `cap` = 2 keep entries, keep = k + max(k / 2, 32) rounded up to 32.  The
// owner lane appends (raw accumulator, processing position) on the rare admission path; when a row's list could not
// take a chunk's new entries the whole warp compacts it:
//   1. raw entries are resolved to (approximate score, item id) -- their bias and permutation lookups are independent
//      loads spread over the lanes;
//   2. the k-th best approximate score a_k is found by a radix select on order-preserving uint keys (4 passes of 8
//      bits, a 256-bin histogram in the warp's staging tile, which is free once the staged chunk is in registers);
//   3. every entry >= a_k - 2.25 m is kept, at most `keep`: if more pass, the (keep + 1)-th best is selected too, only
//      the entries above it are kept and it is remembered in drop_max;
//   4. theta (and tau) rise as in the narrow form; after kGiveUpOverflows overflowing compactions the row stops
//      admitting and is marked uncertifiable.
// Kept entries are not sorted: select_wide_kernel (rescore_wide.cu) re-scores, sorts and certifies them.
//
// Warm start: none.  The sweep starts at theta = -inf and the first compaction sets the threshold.  That costs every
// row `cap` appends at the start of each work unit -- a handful of tiles out of the ~8K of a 1M-item sweep -- and keeps
// the certificate argument of §3 word for word: theta only ever comes from admitted (eligible) items.
#include <stdlib.h>

#include "filter_tc.cuh"

namespace trk {

constexpr int kWideMaxK = 1024;

__host__ __device__ inline int wide_keep(int k) { return static_cast<int>(round_up(k + (k / 2 > 32 ? k / 2 : 32), 32)); }

struct WideParams {
  const float* user_scale;
  const float* user_bias;      // may be null
  const float* user_norm;      // |u|_2 per user
  const float* item_bias;      // [padded items] in processing order, padding = -inf
  const float* block_bias_max; // max item bias of every block of 128 processing positions
  const int32_t* item_perm;    // processing position -> local item index, or null = identity
  const float* item_stats;     // [0] = max_j |i_j|_2, [1] = global item scale, [2] = max_j |bias_j|
  int64_t n_users;
  int64_t n_items;
  int32_t n_stages;
  int32_t k;
  int32_t keep;                // entries a compaction keeps at most
  int32_t cap;                 // list capacity per (row, split): 2 keep
  int32_t n_splits;
  int32_t tiles_per_split;
  int32_t n_tiles;
  int32_t n_user_pairs;
  int32_t item_id_offset;
  float* list_score;           // [n_users, n_splits, cap] approximate scores
  int32_t* list_item;          // [n_users, n_splits, cap] global item ids
  int32_t* list_count;         // [n_users, n_splits] entries of each list (<= keep at the end)
  float* row_theta;            // [n_users, n_splits] max(theta, drop_max) (certified by select_wide_kernel)
  const int32_t* excl_indptr;  // exclusion lists as processing positions (kExclude), see score_filter_tc.cu
  const int32_t* excl_pos;
};

struct WideLayout {
  uint32_t a_off, b_off, acc_off, bar_off, total;
};
__host__ __device__ inline WideLayout wide_layout(int n_kblocks, int n_stages) {
  WideLayout L;
  L.a_off = 0;
  L.b_off = L.a_off + 2u * static_cast<uint32_t>(n_kblocks) * kATileBytes;
  L.acc_off = L.b_off + static_cast<uint32_t>(n_stages) * kBTileBytes;
  L.bar_off = L.acc_off + 2u * kAccStageBytes;
  L.total = L.bar_off + 512u;
  return L;
}

// Admission state of the row a consumer lane owns (filter_owned_row); the list itself is in global memory.
struct WideRow {
  float* ls;        // the row's list for this split: scores (raw accumulators for entries >= n_res) ...
  int32_t* li;      // ... and item ids (processing positions for entries >= n_res)
  int cnt, n_res, n_ovf;
  float tau, theta, drop_max;
  float m3, ubias, c, inv_c;
};

// The key of the rank-th largest (1-based) real entry (id != INT32_MAX) of ls[0, n); the warp holds at least `rank`
// real entries.  4 passes of 8 bits; `hist` = 256 words of the warp's staging tile.  Called warp-uniformly.
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

// Warp-cooperative compaction of lane `src`'s list (steps 1-4 above).  Called warp-uniformly.
__device__ __forceinline__ void wide_compact(int src, int lane, WideRow& r, const AdmitCtx& ctx, int keep,
                                             uint32_t* hist) {
  const float kNegInf = -__int_as_float(0x7f800000);
  const int n = __shfl_sync(0xffffffffu, r.cnt, src);
  const int n_res = __shfl_sync(0xffffffffu, r.n_res, src);
  float* ls = reinterpret_cast<float*>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(r.ls), src));
  int32_t* li = reinterpret_cast<int32_t*>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(r.li), src));
  const float cs = __shfl_sync(0xffffffffu, r.c, src);
  const float ubs = __shfl_sync(0xffffffffu, r.ubias, src);
  const float m3s = __shfl_sync(0xffffffffu, r.m3, src);
  __syncwarp();   // the owner's appends are visible to every lane
  // 1. resolve the raw entries (a padded column of the last tile resolves to (-inf, INT32_MAX): not real)
  int n_real = 0;
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    bool real = false;
    if (i < n) {
      int32_t id = li[i];
      if (i >= n_res) {
        const int32_t pos = id;
        const float b = ldg_nc_f32(ctx.bias + pos);
        const int32_t pm = (ctx.perm != nullptr && pos < ctx.n_items) ? ldg_nc_s32(ctx.perm + pos) : pos;
        id = pos < ctx.n_items ? ctx.id_offset + pm : 0x7fffffff;
        ls[i] = fmaf(ls[i], cs, ubs) + b;   // approximate score: (acc * c + user bias) + item bias
        li[i] = id;
      }
      real = id != 0x7fffffff;
    }
    n_real += __popc(__ballot_sync(0xffffffffu, real));
  }
  __syncwarp();
  // 2. the k-th best, the floor, and how many entries reach it
  const bool have_k = n_real >= ctx.k;
  float floor_s = kNegInf;
  if (have_k) floor_s = wide_unkey(wide_select(ls, li, n, ctx.k, hist, lane)) - m3s;
  int n_ge = 0;
  for (int i = lane; i < n; i += 32) n_ge += (li[i] != 0x7fffffff && ls[i] >= floor_s) ? 1 : 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) n_ge += __shfl_xor_sync(0xffffffffu, n_ge, o);
  // 3. more than `keep` within the bound of the k-th best: keep only those above the (keep + 1)-th best
  const bool ovf = n_ge > keep;
  const float cut = ovf ? wide_unkey(wide_select(ls, li, n, keep + 1, hist, lane)) : kNegInf;
  int n_keep = 0;
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    float s = kNegInf;
    int32_t id = 0x7fffffff;
    if (i < n) {
      s = ls[i];
      id = li[i];
    }
    const bool kp = id != 0x7fffffff && s >= floor_s && (!ovf || s > cut);
    const unsigned b = __ballot_sync(0xffffffffu, kp);   // every lane has read its entry of this round
    if (kp) {
      const int dst = n_keep + __popc(b & ((1u << lane) - 1u));   // <= i: never an entry not yet read
      ls[dst] = s;
      li[dst] = id;
    }
    n_keep += __popc(b);
    __syncwarp();
  }
  // 4. thresholds
  if (lane == src) {
    r.cnt = n_keep;
    r.n_res = n_keep;
    if (ovf) {
      r.drop_max = fmaxf(r.drop_max, cut);
      r.n_ovf += 1;
    }
    if (have_k) {
      r.theta = fmaxf(r.theta, floor_s);   // every item left out so far is <= the largest theta ever set
      set_tau(r);
    }
    if (r.n_ovf >= kGiveUpOverflows) {
      r.tau = __int_as_float(0x7f800000);
      r.drop_max = __int_as_float(0x7f800000);
    }
  }
  __syncwarp();
}

__device__ __forceinline__ void wide_compact_rows(unsigned rows, int lane, WideRow& r, const AdmitCtx& ctx, int keep,
                                                  uint32_t* hist) {
  while (rows != 0u) {
    const int src = __ffs(rows) - 1;
    rows &= rows - 1u;
    wide_compact(src, lane, r, ctx, keep, hist);
  }
}

// 32 staged columns of the lane's row (positions [pos_base, pos_base + 32)): the lanes whose bound passes append the
// passing columns raw; rows whose list could not take them are compacted first (cap - keep >= 32).  Warp-uniform.
__device__ __forceinline__ void wide_32(const uint32_t* v, int32_t pos_base, float bmax_scaled, int lane, WideRow& r,
                                        const AdmitCtx& ctx, int keep, int cap, uint32_t* hist) {
  float g0[4], g1[4];
  const float a0 = acc_max_16(v, g0), a1 = acc_max_16(v + 16, g1);
  uint32_t mask = 0;
  if (a0 + bmax_scaled > r.tau) mask = pass_mask_16(v, g0, bmax_scaled, r.tau);
  if (a1 + bmax_scaled > r.tau) mask |= pass_mask_16(v + 16, g1, bmax_scaled, r.tau) << 16;
  const unsigned need = __ballot_sync(0xffffffffu, r.cnt + __popc(mask) > cap);
  if (need != 0u) wide_compact_rows(need, lane, r, ctx, keep, hist);
  if (mask != 0u && r.n_ovf < kGiveUpOverflows) {   // (a row that has just given up appends nothing more)
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      if ((mask >> j) & 1u) {
        const int e = r.cnt + __popc(mask & ((1u << j) - 1u));
        r.ls[e] = __uint_as_float(v[j]);
        r.li[e] = pos_base + j;
      }
    }
    r.cnt += __popc(mask);
  }
}

// filter_chunk of the narrow form with wide_32 as its slow path (amax = chunk_row_max<kC>)
template <int kC, bool kExclude>
__device__ __forceinline__ void wide_chunk(const float (&acc0)[32], const float (&acc1)[32], float amax, int32_t base,
                                           float bmax_scaled, uint32_t stage, int lane, int64_t u, const WideParams& p,
                                           int32_t& excl_next, WideRow& r, const AdmitCtx& ctx, uint32_t* hist) {
  bool flag = amax + bmax_scaled > r.tau;
  if constexpr (kExclude) flag = flag || excl_next < base + 32;
  if (!__any_sync(0xffffffffu, flag)) return;
  stage_warp_chunk<kC>(acc0, acc1, stage, lane);
  if constexpr (kExclude) {
    if (excl_next < base + 32) excl_next = excl_mask_chunk(p.excl_indptr, p.excl_pos, u, base, stage, lane);
  }
  uint32_t v[32];
  load_staged_row(stage, lane, v);
  __syncwarp();   // the staging tile doubles as the compaction's histogram
  wide_32(v, base, bmax_scaled, lane, r, ctx, p.keep, p.cap, hist);
}

// Template parameters as score_filter_kernel's.
template <int kNKB, int kCluster, bool kExclude>
__global__ void __launch_bounds__(kTcThreads, 1)
score_wide_kernel(const __grid_constant__ CUtensorMap map_users, const __grid_constant__ CUtensorMap map_items,
                  const WideParams p) {
  uint8_t* smem = smem_base_1024();
  const WideLayout L = wide_layout(kNKB, p.n_stages);
  const int n_slots = p.n_stages / kNKB;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.bar_off);
  uint64_t* a_full = bars + 0;
  uint64_t* b_full = bars + 2;
  uint64_t* b_empty = bars + 2 + n_slots;
  constexpr uint32_t kSlotBytes = kNKB * kBTileBytes;

  const int warp = threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  const uint32_t crank = kCluster == 2 ? cluster_ctarank() : 0u;
  const int n_groups = (p.n_user_pairs + kCluster - 1) / kCluster;
  const int64_t n_work = static_cast<int64_t>(n_groups) * p.n_splits;
  const int64_t w_first = blockIdx.x / kCluster, w_step = gridDim.x / kCluster;
  constexpr uint16_t kClusterMask = (1u << kCluster) - 1u;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&map_items);
    tma_prefetch_desc(&map_users);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < 2; ++i) mbar_init(a_full + i, 1);
    for (int i = 0; i < n_slots; ++i) {
      mbar_init(b_full + i, 1);
      mbar_init(b_empty + i, 8 * kCluster);
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (kCluster == 2) cluster_sync_all();

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    // ===================================== TMA producer ======================================
    if (warp == 0) {
      int ts = 0;
      uint32_t ts_phase = 0;
      for (int64_t w = w_first; w < n_work; w += w_step) {
        const int sp = static_cast<int>(w / n_groups);
        const int t0 = sp * p.tiles_per_split;
        const int t1 = min(t0 + p.tiles_per_split, p.n_tiles);
        for (int t = t0; t < t1; ++t) {
          if (kCluster == 2)
            mbar_wait_cluster(b_empty + ts, ts_phase ^ 1);
          else
            mbar_wait(b_empty + ts, ts_phase ^ 1);
          if (elect_one()) {
            mbar_arrive_expect_tx(b_full + ts, kSlotBytes);
#pragma unroll
            for (int kb = 0; kb < kNKB; ++kb) {
              if (kCluster == 2)
                tma_load_2d_multicast(smem + L.b_off + ts * kSlotBytes + kb * kBTileBytes + crank * (kBTileBytes / 2),
                                      &map_items, b_full + ts, kb * kKBlock,
                                      t * kBlockN + static_cast<int>(crank) * (kBlockN / 2), kClusterMask, kEvictLast);
              else
                tma_load_2d(smem + L.b_off + ts * kSlotBytes + kb * kBTileBytes, &map_items, b_full + ts,
                            kb * kKBlock, t * kBlockN, kEvictLast);
            }
          }
          __syncwarp();
          if (++ts == n_slots) {
            ts = 0;
            ts_phase ^= 1;
          }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
    // ================================ consumers: wgmma + admission ================================
    const int group = warp / 4 - 1;
    const int row = filter_owned_row(warp % 4, lane);
    const float kNegInf = -__int_as_float(0x7f800000);
    const uint32_t stage = smem_u32(smem + L.acc_off) + static_cast<uint32_t>(warp - 4) * kWarpStageBytes;
    uint32_t* hist = reinterpret_cast<uint32_t*>(smem + L.acc_off + static_cast<uint32_t>(warp - 4) * kWarpStageBytes);
    const uint32_t a_base = smem_u32(smem + L.a_off) + group * kNKB * kATileBytes;
    const uint32_t b_base = smem_u32(smem + L.b_off);
    const float max_item_norm = __ldg(p.item_stats + 0);
    const float item_scale = fmaxf(__ldg(p.item_stats + 1), 1e-38f);
    const float max_item_bias = __ldg(p.item_stats + 2);
    const AdmitCtx ctx = {p.item_bias, p.item_perm, p.item_id_offset, static_cast<int32_t>(p.n_items), p.k};
    int ts = 0;
    uint32_t ts_phase = 0, witer = 0;
    float acc0[32], acc1[32];

    for (int64_t w = w_first; w < n_work; w += w_step) {
      const int up = static_cast<int>(w % n_groups) * kCluster + static_cast<int>(crank);
      const int sp = static_cast<int>(w / n_groups);
      const int t0 = sp * p.tiles_per_split;
      const int t1 = min(t0 + p.tiles_per_split, p.n_tiles);
      const int64_t ublock_row0 = (static_cast<int64_t>(up) * 2 + group) * kBlockM;
      const int64_t u = ublock_row0 + row;
      const bool u_ok = u < p.n_users;
      const float su = u_ok ? __ldg(p.user_scale + u) : 1.0f;
      const float ubias = (u_ok && p.user_bias != nullptr) ? __ldg(p.user_bias + u) : 0.0f;
      const float unorm = u_ok ? __ldg(p.user_norm + u) : 0.0f;
      const int64_t list = u_ok ? (u * p.n_splits + sp) : 0;
      WideRow rs;
      rs.ls = p.list_score + list * p.cap;
      rs.li = p.list_item + list * p.cap;
      rs.cnt = rs.n_res = rs.n_ovf = 0;
      rs.theta = rs.drop_max = kNegInf;
      rs.tau = u_ok ? kNegInf : __int_as_float(0x7f800000);   // rows past n_users admit nothing (they have no list)
      rs.ubias = ubias;
      rs.c = su * item_scale;
      rs.inv_c = 1.0f / rs.c;
      rs.m3 = kThetaMargins * (kMarginFactor * unorm * max_item_norm + kBiasUlps * (fabsf(ubias) + max_item_bias));
      int32_t excl_next = 0x7fffffff;
      if constexpr (kExclude) {
        if (u_ok && t1 > t0) excl_next = excl_next_at(p.excl_indptr, p.excl_pos, u, t0 * kBlockN);
      }

      if (t1 > t0) {
        named_barrier_sync(1 + group, kConsumerThreads);
        if (warp % 4 == 0 && lane == 0) {
          mbar_arrive_expect_tx(a_full + group, kNKB * kATileBytes);
#pragma unroll
          for (int kb = 0; kb < kNKB; ++kb)
            tma_load_2d(smem + L.a_off + (group * kNKB + kb) * kATileBytes, &map_users, a_full + group, kb * kKBlock,
                        static_cast<int32_t>(ublock_row0), kEvictFirst);
        }
        mbar_wait(a_full + group, witer & 1);
        ++witer;
      }

      float bmax_next = t1 > t0 ? __ldg(p.block_bias_max + t0) : 0.0f;
      for (int t = t0; t < t1; ++t) {
        const float bmax_scaled = bmax_next * rs.inv_c;
        if (t + 1 < t1) bmax_next = __ldg(p.block_bias_max + t + 1);
        mbar_wait(b_full + ts, ts_phase);
        const uint32_t b_slot = b_base + ts * kSlotBytes;
        const int32_t pos0 = t * kBlockN;
#pragma unroll 1
        for (int h = 0; h < 2; ++h) {
          filter_mma_half<kNKB>(acc0, acc1, a_base, b_slot, h);
          if (h == 1) {
            __syncwarp();
            if (lane == 0) {
              if (kCluster == 2) {
#pragma unroll
                for (uint32_t r = 0; r < kCluster; ++r) mbar_arrive_cluster(b_empty + ts, r);
              } else {
                mbar_arrive(b_empty + ts);
              }
            }
          }
          const float amax0 = chunk_row_max<0>(acc0, acc1, lane), amax1 = chunk_row_max<1>(acc0, acc1, lane);
          wide_chunk<0, kExclude>(acc0, acc1, amax0, pos0 + h * 64, bmax_scaled, stage, lane, u, p, excl_next, rs, ctx,
                                  hist);
          wide_chunk<1, kExclude>(acc0, acc1, amax1, pos0 + h * 64 + 32, bmax_scaled, stage, lane, u, p, excl_next, rs,
                                  ctx, hist);
        }
        if (++ts == n_slots) {
          ts = 0;
          ts_phase ^= 1;
        }
      }

      // end of the item range: one last compaction of every row (resolves the raw entries, count <= keep)
      wide_compact_rows(__ballot_sync(0xffffffffu, u_ok), lane, rs, ctx, p.keep, hist);
      if (u_ok) {
        p.list_count[list] = rs.cnt;
        const bool th_nan = rs.theta != rs.theta || rs.drop_max != rs.drop_max;
        p.row_theta[list] = th_nan ? __int_as_float(0x7f800000) : fmaxf(rs.theta, rs.drop_max);
      }
      __syncwarp();
    }
  }

  __syncthreads();
  if (kCluster == 2) cluster_sync_all();
}

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
int score_wide_max_k() { return kWideMaxK; }
int score_wide_list_capacity(int32_t k) { return 2 * wide_keep(k); }

int score_wide_f16(const void* user_split, const float* user_scale, const float* user_bias, const float* user_norm,
                   const void* item_hi, const float* item_stats, const float* item_bias, const float* block_bias_max,
                   const int32_t* item_perm, int64_t n_users, int64_t n_items, int32_t d_pad, int32_t k,
                   int32_t n_splits, int32_t item_id_offset, float* list_score, int32_t* list_item,
                   int32_t* list_count, float* row_theta, const int32_t* excl_indptr, const int32_t* excl_pos,
                   cudaStream_t stream) {
  TRK_CHECK_ARG(user_split && user_scale && user_norm && item_hi && item_stats && item_bias && block_bias_max,
                "score_wide: null input");
  TRK_CHECK_ARG((excl_indptr == nullptr) == (excl_pos == nullptr), "score_wide: excl_indptr and excl_pos go together");
  TRK_CHECK_ARG(list_score && list_item && list_count && row_theta, "score_wide: null output");
  TRK_CHECK_ARG(n_users >= 1 && n_items >= 1 && n_splits >= 1, "score_wide: empty shape");
  TRK_CHECK_ARG(n_users < (1ll << 31) && n_items < (1ll << 31) - 512, "score_wide: shape exceeds int32 indexing");
  if (d_pad != 64 && d_pad != 128) {
    set_error("score_wide: d_pad=%d not supported (64 or 128)", d_pad);
    return TRK_ERR_UNSUPPORTED;
  }
  if (k < 1 || k > kWideMaxK) {
    set_error("score_wide: k=%d outside [1, %d]", k, kWideMaxK);
    return TRK_ERR_UNSUPPORTED;
  }
  TRK_CHECK_ARG(reinterpret_cast<uintptr_t>(user_split) % 16 == 0 && reinterpret_cast<uintptr_t>(item_hi) % 16 == 0,
                "score_wide: operands must be 16-byte aligned");

  WideParams p;
  p.user_scale = user_scale;
  p.user_bias = user_bias;
  p.user_norm = user_norm;
  p.item_bias = item_bias;
  p.block_bias_max = block_bias_max;
  p.item_perm = item_perm;
  p.item_stats = item_stats;
  p.n_users = n_users;
  p.n_items = n_items;
  p.k = k;
  p.keep = wide_keep(k);
  p.cap = 2 * p.keep;
  p.n_tiles = static_cast<int32_t>(ceil_div(n_items, kBlockN));
  p.n_splits = n_splits;
  p.tiles_per_split = static_cast<int32_t>(ceil_div(p.n_tiles, n_splits));
  p.n_user_pairs = static_cast<int32_t>(ceil_div(n_users, 2 * kBlockM));
  p.item_id_offset = item_id_offset;
  p.list_score = list_score;
  p.list_item = list_item;
  p.list_count = list_count;
  p.row_theta = row_theta;
  p.excl_indptr = excl_indptr;
  p.excl_pos = excl_pos;
  const bool excl = excl_indptr != nullptr;
  const int n_kblocks = d_pad / kKBlock;
  p.n_stages = 0;
  for (int s = kMaxStages; s >= 2; --s)
    if (s % n_kblocks == 0 && wide_layout(n_kblocks, s).total + kSmemAlignSlack <= kSmemLimit) {
      p.n_stages = s;
      break;
    }
  TRK_CHECK_ARG(p.n_stages >= 2 * n_kblocks, "score_wide: shared memory budget exceeded");
  const uint32_t smem_bytes = wide_layout(n_kblocks, p.n_stages).total + kSmemAlignSlack;

  // launch form as score_filter_f16: 2-CTA clusters sharing every item tile when the device can keep (almost) all SMs
  // busy with them, else independent CTAs; TRK_FILTER_CLUSTER=1|2 forces one
  int cluster = 2;
  const char* env = getenv("TRK_FILTER_CLUSTER");
  if (env != nullptr && (atoi(env) == 1 || atoi(env) == 2)) cluster = atoi(env);
  auto kernel2 = excl ? (n_kblocks == 2 ? score_wide_kernel<2, 2, true> : score_wide_kernel<1, 2, true>)
                      : (n_kblocks == 2 ? score_wide_kernel<2, 2, false> : score_wide_kernel<1, 2, false>);
  auto kernel1 = excl ? (n_kblocks == 2 ? score_wide_kernel<2, 1, true> : score_wide_kernel<1, 1, true>)
                      : (n_kblocks == 2 ? score_wide_kernel<2, 1, false> : score_wide_kernel<1, 1, false>);
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
    if (cudaOccupancyMaxActiveClusters(&max_clusters, kernel2, &cfg) != cudaSuccess) {
      (void)cudaGetLastError();
      max_clusters = 0;
    }
    if (max_clusters * 2 < sm_count() - 8 && env == nullptr) cluster = 1;
    if (max_clusters < 1) cluster = 1;
  }
  CUtensorMap map_users, map_items;
  int rc = encode_tiled_2d(&map_items, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, item_hi, d_pad, n_items, 2 * d_pad, kKBlock,
                           kBlockN / cluster, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (rc != TRK_OK) return rc;
  rc = encode_tiled_2d(&map_users, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, user_split, d_pad, n_users, 4 * d_pad, kKBlock,
                       kBlockM, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (rc != TRK_OK) return rc;
  if (cluster == 2) {
    const int64_t n_work = ceil_div(static_cast<int64_t>(p.n_user_pairs), 2) * n_splits;
    const int n_clusters = static_cast<int>(n_work < max_clusters ? n_work : max_clusters);
    cfg.gridDim = dim3(static_cast<unsigned>(2 * n_clusters));
    TRK_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kernel2, map_users, map_items, p));
  } else {
    TRK_CHECK_CUDA(cudaFuncSetAttribute(kernel1, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    const int grid = capped_grid(static_cast<int64_t>(p.n_user_pairs) * n_splits, 1);
    kernel1<<<grid, kTcThreads, smem_bytes, stream>>>(map_users, map_items, p);
  }
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

}  // namespace trk
