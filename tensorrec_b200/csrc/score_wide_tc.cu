// Wide form of the one-pass tensor-core filter (score_filter_tc.cu, DESIGN §3.3): the same sweep skeleton
// (filter_tc.cuh), the same fp16 "hi" operands in descending-bias order, the same register fast path on the wgmma
// fragments and the same per-warp staging of flagged chunks -- but every user row keeps its candidates in a list in
// GLOBAL memory, so k is not bounded by a 32-entry shared-memory buffer: 32 < k <= kWideMaxK.
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
#include "filter_tc.cuh"

namespace trk {

constexpr int kWideMaxK = 1024;

__host__ __device__ inline int wide_keep(int k) { return static_cast<int>(round_up(k + (k / 2 > 32 ? k / 2 : 32), 32)); }

struct WideParams {
  SweepParams sweep;
  int32_t keep;                // entries a compaction keeps at most
  int32_t cap;                 // list capacity per (row, split): 2 keep
  float* list_score;           // [n_users, n_splits, cap] approximate scores
  int32_t* list_item;          // [n_users, n_splits, cap] global item ids
  int32_t* list_count;         // [n_users, n_splits] entries of each list (<= keep at the end)
};

// Admission state of the row a consumer lane owns (filter_owned_row); the list itself is in global memory.
struct WideRow {
  float* ls;        // the row's list for this split: scores (raw accumulators for entries >= n_res) ...
  int32_t* li;      // ... and item ids (processing positions for entries >= n_res)
  int cnt, n_res, n_ovf;
  float tau, theta, drop_max;
  float m3, ubias, c, inv_c;
};

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
    if (excl_next < base + 32) excl_next = excl_mask_chunk(p.sweep.excl_indptr, p.sweep.excl_pos, u, base, stage, lane);
  }
  uint32_t v[32];
  load_staged_row(stage, lane, v);
  __syncwarp();   // the staging tile doubles as the compaction's histogram
  wide_32(v, base, bmax_scaled, lane, r, ctx, p.keep, p.cap, hist);
}

// Template parameters: see the sweep skeleton (filter_tc.cuh).
template <int kNKB, int kCluster, bool kExclude>
__global__ void __launch_bounds__(kTcThreads, 1)
score_wide_kernel(const __grid_constant__ CUtensorMap map_users, const __grid_constant__ CUtensorMap map_items,
                  const WideParams p) {
  const SweepParams& sweep = p.sweep;
  const SweepCta cta = sweep_prologue<kNKB, kCluster>(sweep, 0u, &map_users, &map_items);
  const int warp = threadIdx.x / 32;
  const int lane = threadIdx.x % 32;

  if (sweep_split_registers(warp)) {
    if (warp == 0) sweep_producer<kNKB, kCluster>(sweep, cta, &map_items);
  } else {
    // ================================ consumers: wgmma + admission ================================
    const int group = warp / 4 - 1;
    const int row = filter_owned_row(warp % 4, lane);
    const float kNegInf = -__int_as_float(0x7f800000);
    const uint32_t stage = smem_u32(cta.smem + cta.L.acc_off) + static_cast<uint32_t>(warp - 4) * kWarpStageBytes;
    uint32_t* hist =
        reinterpret_cast<uint32_t*>(cta.smem + cta.L.acc_off + static_cast<uint32_t>(warp - 4) * kWarpStageBytes);
    const uint32_t a_base = smem_u32(cta.smem + cta.L.a_off) + group * kNKB * kATileBytes;
    const uint32_t b_base = smem_u32(cta.smem + cta.L.b_off);
    const float max_item_norm = __ldg(sweep.item_stats + 0);
    const float item_scale = fmaxf(__ldg(sweep.item_stats + 1), 1e-38f);
    const float max_item_bias = __ldg(sweep.item_stats + 2);
    const AdmitCtx ctx = {sweep.item_bias, sweep.item_perm, sweep.item_id_offset, static_cast<int32_t>(sweep.n_items),
                          sweep.k};
    int ts = 0;
    uint32_t ts_phase = 0, witer = 0;
    float acc0[32], acc1[32];

    for (int64_t w = cta.w_first; w < cta.n_work; w += cta.w_step) {
      const SweepUnit wu = sweep_unit<kCluster>(sweep, cta, w, group, row);
      const int64_t u = wu.u;
      const int64_t list = wu.u_ok ? (u * sweep.n_splits + wu.sp) : 0;
      WideRow rs;
      rs.ls = p.list_score + list * p.cap;
      rs.li = p.list_item + list * p.cap;
      rs.cnt = rs.n_res = rs.n_ovf = 0;
      rs.theta = rs.drop_max = kNegInf;
      rs.tau = wu.u_ok ? kNegInf : __int_as_float(0x7f800000);   // rows past n_users admit nothing (they have no list)
      int32_t excl_next = sweep_row_start<kExclude>(rs, sweep, wu, max_item_norm, item_scale, max_item_bias);
      sweep_load_user_block<kNKB>(cta, &map_users, wu, group, warp, lane, witer);

      float bmax_next = wu.t1 > wu.t0 ? __ldg(sweep.block_bias_max + wu.t0) : 0.0f;
      for (int t = wu.t0; t < wu.t1; ++t) {
        const float bmax_scaled = bmax_next * rs.inv_c;
        if (t + 1 < wu.t1) bmax_next = __ldg(sweep.block_bias_max + t + 1);
        mbar_wait(cta.b_full + ts, ts_phase);
        const uint32_t b_slot = b_base + ts * (kNKB * kBTileBytes);
        const int32_t pos0 = t * kBlockN;
#pragma unroll 1
        for (int h = 0; h < 2; ++h) {
          filter_mma_half<kNKB>(acc0, acc1, a_base, b_slot, h);
          if (h == 1) sweep_release_slot<kCluster>(cta, ts, lane);
          const float amax0 = chunk_row_max<0>(acc0, acc1, lane), amax1 = chunk_row_max<1>(acc0, acc1, lane);
          wide_chunk<0, kExclude>(acc0, acc1, amax0, pos0 + h * 64, bmax_scaled, stage, lane, u, p, excl_next, rs, ctx,
                                  hist);
          wide_chunk<1, kExclude>(acc0, acc1, amax1, pos0 + h * 64 + 32, bmax_scaled, stage, lane, u, p, excl_next, rs,
                                  ctx, hist);
        }
        sweep_ring_advance(ts, ts_phase, cta.n_slots);
      }

      // end of the item range: one last compaction of every row (resolves the raw entries, count <= keep)
      wide_compact_rows(__ballot_sync(0xffffffffu, wu.u_ok), lane, rs, ctx, p.keep, hist);
      if (wu.u_ok) {
        p.list_count[list] = rs.cnt;
        sweep_store_theta(sweep, list, rs);
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

template <int kNKB, int kCluster, bool kExclude>
struct WideKernel {
  static constexpr auto fn = score_wide_kernel<kNKB, kCluster, kExclude>;
};

int score_wide_f16(const void* user_split, const float* user_scale, const float* user_bias, const float* user_norm,
                   const void* item_hi, const float* item_stats, const float* item_bias, const float* block_bias_max,
                   const int32_t* item_perm, int64_t n_users, int64_t n_items, int32_t d_pad, int32_t k,
                   int32_t n_splits, int32_t item_id_offset, float* list_score, int32_t* list_item,
                   int32_t* list_count, float* row_theta, const int32_t* excl_indptr, const int32_t* excl_pos,
                   cudaStream_t stream) {
  TRK_CHECK_ARG(list_score && list_item && list_count && row_theta, "score_wide: null output");
  if (k < 1 || k > kWideMaxK) {
    set_error("score_wide: k=%d outside [1, %d]", k, kWideMaxK);
    return TRK_ERR_UNSUPPORTED;
  }

  WideParams p;
  p.keep = wide_keep(k);
  p.cap = 2 * p.keep;
  p.list_score = list_score;
  p.list_item = list_item;
  p.list_count = list_count;
  return launch_sweep<WideKernel>("score_wide", p, 0u, user_split, user_scale, user_bias, user_norm, item_hi,
                                  item_stats, item_bias, block_bias_max, item_perm, n_users, n_items, d_pad, k,
                                  n_splits, item_id_offset, row_theta, excl_indptr, excl_pos, stream);
}

}  // namespace trk
