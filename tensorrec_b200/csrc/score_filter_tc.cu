// K2+K3 fused, filter form: ONE wgmma pass over the fp16 "hi" halves produces approximate scores with a proven
// error bound; per user row the kernel keeps every item that could still belong to the top-k (approximate score
// within the bound of the running k-th best).  The few survivors are re-scored exactly in fp32 and ranked by
// rescore_topk_kernel (rescore_topk.cu), which also verifies the bound and flags rows for the exact 3-pass kernel
// (score_topk_tc.cu) if it does not hold.  Same reference chain as score_topk_tc.cu: tf.matmul
// (tensorrec/prediction_graphs.py:49-50), bias_prediction_dense (tensorrec/recommendation_graphs.py:41),
// rank_predictions (:73-82) restricted to rank <= k.
//
// The CTA runs the sweep skeleton of filter_tc.cuh (256 user rows x a sweep over 128-item tiles).  Consumer warpgroup
// g computes each tile's 128 x 128 accumulator of user block g in two 64-row halves with m64n128k16 wgmma into
// registers.  Each consumer warp owns the 32 user rows whose accumulator fragments it
// holds (lane l: row 16 w + l % 16 + 64 (l / 16) of the block), so the admission test of a 32-column chunk is a
// register reduction in every lane and one warp vote; only a chunk in which some row passes goes through the warp's
// own shared-memory staging tile, where the admission code runs one lane per user row.  The two warpgroups issue their
// wgmma independently and share the tensor pipe (DESIGN §2).
//
// Why: the exact split-product kernel issues 3 tensor passes and its per-row sorted-list inserts serialise a warp.
// Here
//   * tensor work is 1 pass (2*U*I*d flops = the algorithmic count);
//   * items are processed in descending-bias order (host side), so within a 128-item block the biases are almost equal
//     and the admission test v_j = acc_j + bias_j / c > tau (c = user scale x GLOBAL item scale, both powers of two)
//     is bounded by max_j acc_j + blockmax / c: the hot loop is an FMNMX tree over the raw accumulators in the wgmma
//     fragments, two adds and one warp vote per 32 columns of 16 rows;
//   * a passing column is APPENDED raw (accumulator, position) to the row's 32-entry buffer in shared memory; when
//     some row's buffer passes half full the whole warp compacts it cooperatively: one entry per lane, raw entries
//     resolved to (approximate score, item id), a 15-step bitonic sort through shuffles, keep everything >= (k-th best
//     - 2.25m), tighten the threshold.
//
// Error bound.  hi = fp16(x * 2^e) has relative error <= 2^-11 per element (absolute 2^-25 below the fp16 normal
// range), so |approx - exact| <= (2^-10 + 2^-22) |u|.|i| <= m := kMarginFactor * |u|_2 * max_j |i_j|_2 with
// kMarginFactor = 1.5 * 2^-10 (covers the fp32 accumulation of the tensor core and the flush of tiny elements).
// Every item ever excluded had approx <= theta_final, hence exact <= theta_final + m, and theta = a_k - 2.25m keeps
// theta + m strictly below the exact k-th best of the survivors (which is >= a_k - m).  rescore_topk_kernel checks
// exactly that inequality.
#include <stdlib.h>

#include "filter_tc.cuh"

namespace trk {

constexpr int kBufEntries = 32;      // candidate buffer per (row, epilogue group)
constexpr int kKeepMax = 16;         // entries kept by a compaction (>= k + slack); also the per-group output width
constexpr int kFilterMaxK = 12;

constexpr uint32_t kBufBytes = 2u * kBlockM * kBufEntries * 8u;   // 64 KB of candidate buffers, after the B ring

struct FilterParams {
  SweepParams sweep;
  const float* block_bias_min; // min item bias of every block (-inf as soon as the block holds padding); may be null
  int32_t tile_end_trigger;    // rows holding more entries than this are compacted at the END of a tile
  float* cand_score;           // [n_users, n_splits, kKeepMax] approximate scores (sentinel -inf)
  int32_t* cand_item;          // [n_users, n_splits, kKeepMax] global ids (sentinel INT32_MAX)
};

// Cycle accounting, compiled only with -DTRK_FILTER_CYCLES (scripts/filter_cycles.py builds such a library; the
// shipped one has none of it).  Lane 0 of every consumer warp sums clock64() deltas per category in registers, the
// producer warp its waits for a free B slot; each warp adds its sums to g_filter_cycles when it leaves the kernel and
// trk_debug_filter_cycles copies them out.  kCycRowHalves holds the whole admission epilogue of the row halves, of
// which kCycSlow is the staged path and kCycCompactMid the compactions inside it.
#ifdef TRK_FILTER_CYCLES
enum FilterCycle {
  kCycBFull, kCycMma, kCycRowHalves, kCycSlow, kCycCompactMid, kCycCompactTileEnd, kCycCompactFinal, kCycOutput,
  kCycRelease, kCycUnitStart, kCycWarm, kCycConsumer, kCycConsumerWarps, kCycProducerEmpty, kCycProducer,
  kCycProducerWarps, kNumCycles
};
__device__ unsigned long long g_filter_cycles[kNumCycles];
#define TRK_CYC_START(t) const long long t = clock64()
#define TRK_CYC_ADD(sum, t) (sum) += static_cast<unsigned long long>(clock64() - (t))
#else
#define TRK_CYC_START(t)
#define TRK_CYC_ADD(sum, t)
#endif

__device__ __forceinline__ void f_sts64(uint32_t addr, float s, int32_t id) {
  asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(__float_as_uint(s)), "r"(id) : "memory");
}
__device__ __forceinline__ void f_lds64(uint32_t addr, float* s, int32_t* id) {
  uint32_t a, b;
  asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(a), "=r"(b) : "r"(addr) : "memory");
  *s = __uint_as_float(a);
  *id = static_cast<int32_t>(b);
}

// Admission state of the user row a consumer lane owns (filter_owned_row).  Only ever passed to __forceinline__
// functions, so that it stays in registers.
struct RowState {
  uint32_t buf;     // shared-memory address of the row's candidate buffer (kBufEntries entries of 8 bytes)
  int cnt;          // entries in the buffer
  int n_res;        // entries [0, n_res) are resolved (approximate score, item id), [n_res, cnt) raw
  int n_ovf;        // compactions that overflowed, see compact_finish
  float tau;        // admission threshold on v = acc + bias / c
  float theta;      // admission threshold on the approximate score
  float drop_max;   // best score a compaction dropped
  // row constants: the margin 2.25 m, the user bias, c = user scale x global item scale (a power of two) and 1 / c
  float m3, ubias, c, inv_c;
#ifdef TRK_FILTER_CYCLES
  unsigned long long cyc_slow, cyc_compact_mid;
#endif
};


// Warp-cooperative compaction of the candidate buffer of lane `src`'s row: one entry per lane, bitonic sort by
// (score desc, id asc), keep everything >= k-th best - 2.25m (at most kKeepMax), tighten that row's thresholds.
// Entries [n_res, cnt) of the buffer are RAW -- (accumulator value, processing position) exactly as the hot loop
// found them; they are turned into (approximate score, item id) here, where the bias and permutation lookups of all
// of them are independent loads issued by different lanes (one L2 latency per compaction, not one per admission).
//
// Split in two so that the lookups of the NEXT row to compact are in flight while THIS row is sorted: the rows of a warp
// overflow in bursts (their thresholds rise in step), a compaction is ~250 instructions, an L2 round trip ~700 cycles.
struct RowFetch {
  float s;        // raw accumulator (lanes >= n_res) or resolved approximate score
  int32_t id;     // processing position (raw) or item id (resolved)
  float bias;     // bias of the raw entry's position           } requested by compact_fetch,
  int32_t perm;   // original item index of that position       } first used by compact_finish
  int n, n_res;
  uint32_t addr;
};
__device__ __forceinline__ RowFetch compact_fetch(const RowState& r, int lane, int src, const AdmitCtx& ctx) {
  RowFetch f;
  f.n = __shfl_sync(0xffffffffu, r.cnt, src);
  f.n_res = __shfl_sync(0xffffffffu, r.n_res, src);
  f.addr = __shfl_sync(0xffffffffu, r.buf, src);
  f.s = -__int_as_float(0x7f800000);
  f.id = 0x7fffffff;
  f.bias = 0.0f;
  f.perm = 0;
  if (lane < f.n) {
    f_lds64(f.addr + lane * 8, &f.s, &f.id);
    if (lane >= f.n_res) {
      f.bias = ldg_nc_f32(ctx.bias + f.id);
      // (a padded column of the last tile can be appended -- its bias is -inf, it never survives -- and has no perm entry)
      f.perm = (ctx.perm != nullptr && f.id < ctx.n_items) ? ldg_nc_s32(ctx.perm + f.id) : f.id;
    }
  }
  return f;
}
// n_ovf counts the compactions of this lane's row that found more than kKeepMax entries within the bound of the k-th
// best.  Once in a while that is harmless (the surplus is remembered in drop_max).  A row where it keeps happening holds
// massive near-ties (all-equal scores in the limit: EVERY column passes, every chunk takes the slow path and the sweep of
// 1M x 1M took 43 s instead of 0.2): after kGiveUpOverflows of them the row stops admitting (tau = +inf) and is marked
// uncertifiable (drop_max = +inf), i.e. it goes through the exact kernel -- where a tie-heavy row belongs anyway.
__device__ __forceinline__ void compact_finish(const RowFetch& f, int lane, int src, RowState& r, const AdmitCtx& ctx) {
  const float kNegInf = -__int_as_float(0x7f800000);
  const int k = ctx.k;
  const int n = f.n;
  const uint32_t addr = f.addr;
  const float m3s = __shfl_sync(0xffffffffu, r.m3, src);
  const float cs = __shfl_sync(0xffffffffu, r.c, src);
  const float ubs = __shfl_sync(0xffffffffu, r.ubias, src);
  float s = f.s;
  int32_t id = f.id;
  if (lane < n && lane >= f.n_res) {
    const int32_t pos = id;
    id = pos < ctx.n_items ? ctx.id_offset + f.perm : 0x7fffffff;
    s = fmaf(s, cs, ubs) + f.bias;   // approximate score: (acc * c + user bias) + item bias
  }
  warp_sort_desc(s, id, lane);
  // lanes now hold the entries in (score desc, id asc) order, sentinels last
  const float kth = __shfl_sync(0xffffffffu, s, k - 1);
  const bool have_k = n >= k;
  const float floor_s = have_k ? kth - m3s : kNegInf;
  const unsigned keep = __ballot_sync(0xffffffffu, lane < n && s >= floor_s);
  int n_keep = __popc(keep);
  const bool ovf = n_keep > kKeepMax;
  n_keep = ovf ? kKeepMax : n_keep;
  // more than kKeepMax entries crowd within the bound of the k-th best: the surplus is dropped and the best dropped
  // score is remembered -- it only matters if it is still close to the k-th best at the END of the sweep (the
  // verification in rescore_topk_kernel compares max(theta, drop_max) + m with the exact k-th best)
  const float first_dropped = __shfl_sync(0xffffffffu, s, kKeepMax & 31);
  if (lane < n_keep) f_sts64(addr + lane * 8, s, id);
  if (lane == src) {
    r.cnt = n_keep;
    r.n_res = n_keep;
    if (ovf) {
      r.drop_max = fmaxf(r.drop_max, first_dropped);
      r.n_ovf += 1;
    }
    if (have_k) {
      r.theta = floor_s;
      set_tau(r);
    }
    if (r.n_ovf >= kGiveUpOverflows) {
      r.tau = __int_as_float(0x7f800000);
      r.drop_max = __int_as_float(0x7f800000);
    }
  }
  __syncwarp();
}
// compacts every row of `rows` (bit = lane), the lookups of the next row in flight while the current one is sorted
__device__ __forceinline__ void compact_rows(unsigned rows, int lane, RowState& r, const AdmitCtx& ctx) {
  if (rows == 0u) return;
  int src = __ffs(rows) - 1;
  rows &= rows - 1;
  RowFetch cur = compact_fetch(r, lane, src, ctx);
  while (true) {
    const int nxt = rows != 0u ? __ffs(rows) - 1 : -1;
    rows &= rows - 1;     // (0 stays 0)
    RowFetch ahead = cur;
    if (nxt >= 0) ahead = compact_fetch(r, lane, nxt, ctx);
    compact_finish(cur, lane, src, r, ctx);
    if (nxt < 0) break;
    cur = ahead;
    src = nxt;
  }
}

// 16 columns of one user row per lane.  The admission test is v_j = acc_j + bias_j / c > tau.  Items are processed in
// bias-sorted order, so the biases of one 128-item block differ by ~1e-4 of their range and v_j <= max_j acc_j +
// bmax_block / c is a tight upper bound: the fast path (chunk_frag_pass in the kernel) is an FMNMX reduction of the raw
// accumulators plus ONE add (no per-score bias load, no per-score FFMA) and one vote; only when some lane's bound
// passes is the chunk staged and are the exact v_j formed.  The hitting lanes then append their survivors (approximate
// score + original item id) and rows whose buffer passed half full are compacted by the whole warp.

// slow path of 16 columns: the lanes whose bound passed append every column that passes the same bound as a raw
// (accumulator, position) entry -- a superset of the exact test acc_j + bias_j / c > tau, since bias_j <= block max and
// rounding is monotonic; no memory is read here.  A row is compacted (by the whole warp) only when its buffer could not
// take the new entries: ~4 compactions per user at 1M items instead of 9 with a "more than half full" trigger.
// Called warp-uniformly.
__device__ __forceinline__ void admit_16(const uint32_t* acc, bool hit, int32_t pos_base, float bmax_scaled, int lane,
                                         RowState& r, const AdmitCtx& ctx) {
  uint32_t pass = 0;
  if (hit) {
#pragma unroll
    for (int j = 0; j < 16; ++j) pass |= (__uint_as_float(acc[j]) + bmax_scaled > r.tau) ? (1u << j) : 0u;
  }
  __syncwarp();   // earlier appends of every lane are visible to the lanes that may now compact its row
  const unsigned need = __ballot_sync(0xffffffffu, r.cnt + __popc(pass) > kBufEntries);
  TRK_CYC_START(c0);
  compact_rows(need, lane, r, ctx);
  TRK_CYC_ADD(r.cyc_compact_mid, c0);
  if (pass != 0 && r.n_ovf < kGiveUpOverflows) {   // (a row that has just given up appends nothing more)   // cnt + popc(pass) <= kBufEntries holds here (a compaction leaves at most kKeepMax = 16)
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      if ((pass >> j) & 1u) {
        f_sts64(r.buf + r.cnt * 8, __uint_as_float(acc[j]), pos_base + j);
        r.cnt += 1;
      }
    }
  }
}

// Appends the columns of `mask` (a 16-column half, its maximum `amax` known from the hot loop).  One passing column -- the
// normal case -- IS the maximum of its half (x -> x + bmax is monotonic, so the largest accumulator passes whenever any
// does): one store, no search through the registers.  Several: every slot is addressed by a prefix popcount, the
// stores are independent.
__device__ __forceinline__ void append_16(const uint32_t* acc, uint32_t mask, float amax, int32_t pos_base,
                                          RowState& r) {
  if ((mask & (mask - 1u)) == 0u) {
    f_sts64(r.buf + r.cnt * 8, amax, pos_base + __ffs(mask) - 1);
    r.cnt += 1;
  } else {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      if ((mask >> j) & 1u)
        f_sts64(r.buf + (r.cnt + __popc(mask & ((1u << j) - 1u))) * 8, __uint_as_float(acc[j]), pos_base + j);
    }
    r.cnt += __popc(mask);
  }
}

// 32 columns of a staged row behind ONE vote (the two 16-column maxima are independent chains).  Runs only on a chunk
// that the register fast path flagged, i.e. when some row of the warp passes its bound (32 rows share the instruction
// stream; the vote here is the same predicate, so it passes too unless only an exclusion flagged the chunk): the
// hitting lanes form the pass masks, ONE ballot tells whether every row's buffer can take its new entries -- the common
// case: the hitting lanes append, nobody else does anything -- and only otherwise the chunk goes through the two-step
// path (compact the rows that need it, append 16 columns at a time so that the 32-entry buffer cannot overflow between
// compactions).  Only the lanes with `own` set (the owners of the staged rows) test their row; the others take part in
// the votes and compactions only.
__device__ __forceinline__ void filter_32(const uint32_t* acc, bool own, int32_t pos_base, float bmax_scaled, int lane,
                                          RowState& r, const AdmitCtx& ctx) {
  float g0[4], g1[4];
  const float a0 = acc_max_16(acc, g0), a1 = acc_max_16(acc + 16, g1);
  const bool h0 = own && a0 + bmax_scaled > r.tau, h1 = own && a1 + bmax_scaled > r.tau;
  if (__any_sync(0xffffffffu, h0 || h1)) {
    uint32_t lo = 0, hi = 0;
    if (h0) lo = pass_mask_16(acc, g0, bmax_scaled, r.tau);
    if (h1) hi = pass_mask_16(acc + 16, g1, bmax_scaled, r.tau);
    if (__ballot_sync(0xffffffffu, r.cnt + __popc(lo) + __popc(hi) > kBufEntries) == 0u) {
      if (lo != 0u) append_16(acc, lo, a0, pos_base, r);
      if (hi != 0u) append_16(acc + 16, hi, a1, pos_base + 16, r);
    } else {
      admit_16(acc, h0, pos_base, bmax_scaled, lane, r, ctx);
      admit_16(acc + 16, h1, pos_base + 16, bmax_scaled, lane, r, ctx);
    }
  }
}

// ---- first tile of a work unit: a threshold to start from -----------------------------------------------------------
// With tau = -inf every column of the first tile is admitted: 128 appends and 8 warp-cooperative compactions per row,
// 32 rows of a warp one after the other -- a cost per work unit that weighs most on short sweeps (item shards).
// Instead every thread first reduces its row of the first accumulator to 16 group maxima (8 columns each), sorts them
// in registers and takes the k-th largest, A: k DIFFERENT columns have acc >= A, their biases are >= the block
// minimum, so the k-th best approximate score of the tile is >= fma(A, c, ub) + bmin and theta may start 2.25 m below
// that.  The tile is then filtered as usual: ~1.5 k admissions per row instead of 128, no compaction.  The cost of the
// admission path is proportional to the number of 32-column chunks in which ANY of a warp's 32 rows passes its bound,
// and the early tiles are few chunks whatever they admit.
__device__ __forceinline__ float acc_max_8(const uint32_t* acc) {
  return fmaxf(fmaxf(fmaxf(__uint_as_float(acc[0]), __uint_as_float(acc[1])),
                     fmaxf(__uint_as_float(acc[2]), __uint_as_float(acc[3]))),
               fmaxf(fmaxf(__uint_as_float(acc[4]), __uint_as_float(acc[5])),
                     fmaxf(__uint_as_float(acc[6]), __uint_as_float(acc[7]))));
}
// bitonic network on 16 registers, descending; every index is a compile-time constant after unrolling
__device__ __forceinline__ void sort16_desc(float (&g)[16]) {
#pragma unroll
  for (int size = 2; size <= 16; size <<= 1) {
#pragma unroll
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int j = i ^ stride;
        if (j > i) {
          const bool desc = (i & size) == 0;
          const float hi = fmaxf(g[i], g[j]), lo = fminf(g[i], g[j]);
          g[i] = desc ? hi : lo;
          g[j] = desc ? lo : hi;
        }
      }
    }
  }
}


// Columns [32 kC, 32 kC + 32) of row half rh in acc, processing positions [base, base + 32); bf / tf = frag_rows of
// the row half's bias bounds and tau.  Fast path: every lane tests the maxima of the 8 columns it holds of its two rows
// (and, kExclude, the owners of the row half whether their next excluded position lies in the chunk); one vote, no
// shuffles.  Most chunks stop here with no shared-memory traffic.  Otherwise the warp stages the chunk, masks excluded
// positions, and the owner lanes of the row half run filter_32 on their rows from registers.  Called warp-uniformly.
template <int kC, bool kExclude>
__device__ __forceinline__ void filter_chunk(const float (&acc)[64], int rh, int32_t base, float bmax_scaled,
                                             const float (&bf)[2], float (&tf)[2], uint32_t stage, int lane, int64_t u,
                                             const SweepParams& p, int32_t& excl_next, RowState& r,
                                             const AdmitCtx& ctx) {
  const bool own = (lane >> 4) == rh;
  bool flag = chunk_frag_pass<kC>(acc, bf, tf);   // == the h0 || h1 of filter_32 over the quad
  if constexpr (kExclude) flag = flag || (own && excl_next < base + 32);
  if (!__any_sync(0xffffffffu, flag)) return;
  TRK_CYC_START(c0);
  stage_warp_chunk<kC>(acc, rh, stage, lane);
  if constexpr (kExclude) {
    if (own && excl_next < base + 32) excl_next = excl_mask_chunk(p.excl_indptr, p.excl_pos, u, base, stage, lane);
  }
  uint32_t v[32];
  load_staged_row(stage, lane, v);
  filter_32(v, own, base, bmax_scaled, lane, r, ctx);
  frag_rows(r.tau, rh, lane, tf);
  TRK_CYC_ADD(r.cyc_slow, c0);
}

// The four chunks of row half rh, processing positions [pos0, pos0 + 128): every row's columns in ascending order, and
// a chunk's test sees the tau the chunks before it left.  Only a slow path changes tau, so while no chunk has taken
// one the four tests are independent: ONE vote on all four of them first (four independent FMNMX trees instead of four
// vote-and-branch steps in a row) ends the usual row half, in which no row passes, with exactly the decision of the
// four chunk votes.  Otherwise the chunks run one after the other as before.  (The exclusion code runs only on row
// halves where some owner's next excluded position lies, whose chunks are staged anyway.)  Called warp-uniformly.
template <bool kExclude>
__device__ __forceinline__ void filter_row_half(const float (&acc)[64], int rh, int32_t pos0, float bmax_scaled,
                                                uint32_t stage, int lane, int64_t u, const SweepParams& p,
                                                int32_t& excl_next, RowState& r, const AdmitCtx& ctx) {
  float bf[2], tf[2];
  frag_rows(bmax_scaled, rh, lane, bf);
  frag_rows(r.tau, rh, lane, tf);
  if constexpr (!kExclude) {
    const bool any = chunk_frag_pass<0>(acc, bf, tf) | chunk_frag_pass<1>(acc, bf, tf) |
                     chunk_frag_pass<2>(acc, bf, tf) | chunk_frag_pass<3>(acc, bf, tf);
    if (!__any_sync(0xffffffffu, any)) return;
  }
  filter_chunk<0, kExclude>(acc, rh, pos0, bmax_scaled, bf, tf, stage, lane, u, p, excl_next, r, ctx);
  filter_chunk<1, kExclude>(acc, rh, pos0 + 32, bmax_scaled, bf, tf, stage, lane, u, p, excl_next, r, ctx);
  filter_chunk<2, kExclude>(acc, rh, pos0 + 64, bmax_scaled, bf, tf, stage, lane, u, p, excl_next, r, ctx);
  filter_chunk<3, kExclude>(acc, rh, pos0 + 96, bmax_scaled, bf, tf, stage, lane, u, p, excl_next, r, ctx);
}

// Warm start: the 8-column group maxima g[4 kC + q] of columns [32 kC, 32 kC + 32) of the lane's row, for the owner
// lanes of row half rh; excluded positions are masked with the pre-pass cursor `pre_next`.  Called warp-uniformly.
template <int kC, bool kExclude>
__device__ __forceinline__ void warm_chunk(const float (&acc)[64], int rh, int32_t pos0, uint32_t stage, int lane,
                                           int64_t u, const SweepParams& p, int32_t& pre_next, float (&g)[16]) {
  const bool own = (lane >> 4) == rh;
  stage_warp_chunk<kC>(acc, rh, stage, lane);
  if constexpr (kExclude) {
    if (own && pre_next < pos0 + 32 * kC + 32)
      pre_next = excl_mask_chunk(p.excl_indptr, p.excl_pos, u, pos0 + 32 * kC, stage, lane);
  }
  uint32_t v[32];
  load_staged_row(stage, lane, v);
#pragma unroll
  for (int q = 0; q < 4; ++q)
    if (own) g[4 * kC + q] = acc_max_8(v + 8 * q);
}


// Template parameters: see the sweep skeleton (filter_tc.cuh).
template <int kNKB, int kCluster, bool kExclude = false>
__global__ void __launch_bounds__(kTcThreads, 1)
score_filter_kernel(const __grid_constant__ CUtensorMap map_users, const __grid_constant__ CUtensorMap map_items,
                    const FilterParams p) {
  const SweepParams& sweep = p.sweep;
  const SweepCta cta = sweep_prologue<kNKB, kCluster>(sweep, kBufBytes, &map_users, &map_items);
  const int warp = threadIdx.x / 32;
  const int lane = threadIdx.x % 32;

#ifdef TRK_FILTER_CYCLES
  unsigned long long cyc[kNumCycles] = {};
  TRK_CYC_START(c_all);
#endif
  if (sweep_split_registers(warp)) {
#ifdef TRK_FILTER_CYCLES
    if (warp == 0) {
      sweep_producer<kNKB, kCluster>(sweep, cta, &map_items, &cyc[kCycProducerEmpty]);
      TRK_CYC_ADD(cyc[kCycProducer], c_all);
      cyc[kCycProducerWarps] = 1;
    }
#else
    if (warp == 0) sweep_producer<kNKB, kCluster>(sweep, cta, &map_items);
#endif
  } else {
    // ================================ consumers: wgmma + admission ================================
    const int group = warp / 4 - 1;
    const int row = filter_owned_row(warp % 4, lane);   // row inside the user block
    const float kNegInf = -__int_as_float(0x7f800000);
    const uint32_t buf_row_addr =   // group g owns user block g of the pair
        smem_u32(cta.smem + cta.L.extra_off) + static_cast<uint32_t>((group * kBlockM + row) * kBufEntries * 8);
    const uint32_t stage = smem_u32(cta.smem + cta.L.acc_off) + static_cast<uint32_t>(warp - 4) * kWarpStageBytes;
    const uint32_t a_base = smem_u32(cta.smem + cta.L.a_off) + group * kNKB * kATileBytes;
    const uint32_t b_base = smem_u32(cta.smem + cta.L.b_off);
    const float max_item_norm = __ldg(sweep.item_stats + 0);
    const float item_scale = fmaxf(__ldg(sweep.item_stats + 1), 1e-38f);
    const float max_item_bias = __ldg(sweep.item_stats + 2);
    const AdmitCtx ctx = {sweep.item_bias, sweep.item_perm, sweep.item_id_offset, static_cast<int32_t>(sweep.n_items),
                          sweep.k};
    int ts = 0;
    uint32_t ts_phase = 0, witer = 0;
    float acc[64];

    for (int64_t w = cta.w_first; w < cta.n_work; w += cta.w_step) {
      const SweepUnit wu = sweep_unit<kCluster>(sweep, cta, w, group, row);
      const int64_t u = wu.u;
      TRK_CYC_START(c_unit);
      RowState rs;
      rs.buf = buf_row_addr;
      rs.cnt = rs.n_res = rs.n_ovf = 0;
      rs.tau = rs.theta = rs.drop_max = kNegInf;
#ifdef TRK_FILTER_CYCLES
      rs.cyc_slow = rs.cyc_compact_mid = 0;
#endif
      int32_t excl_next = sweep_row_start<kExclude>(rs, sweep, wu, max_item_norm, item_scale, max_item_bias);
      sweep_load_user_block<kNKB>(cta, &map_users, wu, group, warp, lane, witer);
      TRK_CYC_ADD(cyc[kCycUnitStart], c_unit);

      float bmax_next = wu.t1 > wu.t0 ? __ldg(sweep.block_bias_max + wu.t0) : 0.0f;
      for (int t = wu.t0; t < wu.t1; ++t) {
        const float bmax_scaled = bmax_next * rs.inv_c;
        if (t + 1 < wu.t1) bmax_next = __ldg(sweep.block_bias_max + t + 1);   // in flight while this tile is filtered
        TRK_CYC_START(c_full);
        mbar_wait(cta.b_full + ts, ts_phase);
        TRK_CYC_ADD(cyc[kCycBFull], c_full);
        const uint32_t b_slot = b_base + ts * (kNKB * kBTileBytes);
        const int32_t pos0 = t * kBlockN;
        TRK_CYC_START(c_warm);
        if (t == wu.t0 && p.block_bias_min != nullptr) {
          const float bmin = __ldg(p.block_bias_min + wu.t0);   // the same for the whole CTA: warp-uniform branch
          if (bmin > kNegInf) {
            float g[16];
            // the tile is filtered again below: the pre-pass masks with a copy of the cursor
            int32_t pre_next = excl_next;
#pragma unroll
            for (int rh = 0; rh < 2; ++rh) {   // each lane's row is in one row half: its 16 groups come from that one
              filter_mma_rows<kNKB>(acc, a_base, b_slot, rh);
              warm_chunk<0, kExclude>(acc, rh, pos0, stage, lane, u, sweep, pre_next, g);
              warm_chunk<1, kExclude>(acc, rh, pos0, stage, lane, u, sweep, pre_next, g);
              warm_chunk<2, kExclude>(acc, rh, pos0, stage, lane, u, sweep, pre_next, g);
              warm_chunk<3, kExclude>(acc, rh, pos0, stage, lane, u, sweep, pre_next, g);
            }
            sort16_desc(g);
            float a_k = g[0];
#pragma unroll
            for (int i = 1; i < 16; ++i) a_k = (i < sweep.k) ? g[i] : a_k;   // g[k - 1]: the k-th largest group maximum
            const float th0 = (fmaf(a_k, rs.c, rs.ubias) + bmin) - rs.m3;
            if (th0 == th0) {   // not NaN (infinite biases / margins): otherwise the sweep starts from -inf as before
              rs.theta = th0;
              set_tau(rs);
            }
          }
        }
        TRK_CYC_ADD(cyc[kCycWarm], c_warm);
        // Unrolled: each row half gets its own copy of the MMA issue, the fast path and the slot release, with rh a
        // constant (frag_rows' source lanes, the owner test, the A-descriptor offset).  Measured on an H100 80GB HBM3 at
        // 700 W against the rolled loop (DESIGN §5): 1M x 1M sweep 435-437 -> 417-418 ms; the 125K-item shard, where
        // the duplicated slow path runs more often, 68.3 -> 70.0 ms.
#pragma unroll
        for (int rh = 0; rh < 2; ++rh) {
          TRK_CYC_START(c_mma);
          filter_mma_rows<kNKB>(acc, a_base, b_slot, rh);
          TRK_CYC_ADD(cyc[kCycMma], c_mma);
          TRK_CYC_START(c_rel);
          if (rh == 1) sweep_release_slot<kCluster>(cta, ts, lane);   // the tile's last MMAs of this warp are complete
          TRK_CYC_ADD(cyc[kCycRelease], c_rel);
          TRK_CYC_START(c_rh);
          // kExclude: one vote per row half.  Only a row half in which some owner's next excluded position lies runs
          // the exclusion test of every chunk; every other one (all of them with empty lists) runs the exclusion-free
          // code, which decides exactly as the exclusion test would there.
          bool excl_rh = false;
          if constexpr (kExclude) excl_rh = __any_sync(0xffffffffu, (lane >> 4) == rh && excl_next < pos0 + kBlockN);
          if (excl_rh)
            filter_row_half<kExclude>(acc, rh, pos0, bmax_scaled, stage, lane, u, sweep, excl_next, rs, ctx);
          else
            filter_row_half<false>(acc, rh, pos0, bmax_scaled, stage, lane, u, sweep, excl_next, rs, ctx);
          TRK_CYC_ADD(cyc[kCycRowHalves], c_rh);
        }
        sweep_ring_advance(ts, ts_phase, cta.n_slots);
        // A compaction waits one L2 round trip for the biases / item ids of its new entries -- during which, in the
        // middle of a tile, the warp's 32 rows stand still.  So rows whose buffer is filling up are compacted HERE, at
        // the end of the tile, where the round trip overlaps the other warpgroup's MMAs.  The mid-tile path remains for
        // a row that overflows inside a tile.  (Measured on an H100 80GB HBM3 at 400 W, against a build without this
        // pass: 1M-item sweep 1570 -> 1560 ms, 125K-item shard 186.0 -> 183.6 ms.)
        {
          TRK_CYC_START(c_te);
          const unsigned early = __ballot_sync(0xffffffffu, rs.cnt > p.tile_end_trigger);
          compact_rows(early, lane, rs, ctx);
          TRK_CYC_ADD(cyc[kCycCompactTileEnd], c_te);
        }
      }

      // end of the item range: final compaction of every row of this warp, then emit the survivors
      TRK_CYC_START(c_fin);
      compact_rows(0xffffffffu, lane, rs, ctx);
      TRK_CYC_ADD(cyc[kCycCompactFinal], c_fin);
      TRK_CYC_START(c_out);
      if (wu.u_ok) {
        const int64_t base = u * sweep.n_splits + wu.sp;
        float* os = p.cand_score + base * kKeepMax;
        int32_t* oi = p.cand_item + base * kKeepMax;
        for (int e = 0; e < kKeepMax; ++e) {
          float s = kNegInf;
          int32_t id = 0x7fffffff;
          if (e < rs.cnt) f_lds64(rs.buf + e * 8, &s, &id);
          os[e] = s;
          oi[e] = id;
        }
        sweep_store_theta(sweep, base, rs);
      }
      __syncwarp();
      TRK_CYC_ADD(cyc[kCycOutput], c_out);
#ifdef TRK_FILTER_CYCLES
      cyc[kCycSlow] += rs.cyc_slow;
      cyc[kCycCompactMid] += rs.cyc_compact_mid;
#endif
    }
#ifdef TRK_FILTER_CYCLES
    TRK_CYC_ADD(cyc[kCycConsumer], c_all);
    cyc[kCycConsumerWarps] = 1;
#endif
  }

#ifdef TRK_FILTER_CYCLES
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < kNumCycles; ++i)
      if (cyc[i] != 0) atomicAdd(g_filter_cycles + i, cyc[i]);
  }
#endif
  __syncthreads();
  if (kCluster == 2) cluster_sync_all();   // no CTA leaves while its peer may still multicast into it or arrive on it
}

// ---------------------------------------------------------------------------------------------------------
// operand preparation: row norms + global statistics, and the globally scaled "hi" item operand
// ---------------------------------------------------------------------------------------------------------
// stats[0] = max row norm, stats[1] = max row scale (2^-e of the largest row); both via atomicMax on the float bits
// (non-negative floats order like their bit patterns) -> order independent, deterministic.  stats must be zeroed.
__global__ void operand_stats_kernel(const __half* __restrict__ split, const float* __restrict__ scale, int64_t rows,
                                     int d_pad, float* __restrict__ out_norm, float* __restrict__ stats) {
  const int lane = threadIdx.x % 32;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / 32;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * blockDim.x / 32;
  float local_max_norm = 0.0f, local_max_scale = 0.0f;
  for (int64_t r = warp; r < rows; r += n_warps) {
    const __half* hi = split + r * 2 * d_pad;
    const __half* lo = hi + d_pad;
    float ss = 0.0f;
    for (int e = lane * 2; e < d_pad; e += 64) {
      const float2 h = __half22float2(*reinterpret_cast<const __half2*>(hi + e));
      const float2 l = __half22float2(*reinterpret_cast<const __half2*>(lo + e));
      const float x0 = h.x + l.x, x1 = h.y + l.y;
      ss = fmaf(x0, x0, ss);
      ss = fmaf(x1, x1, ss);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float sc = scale[r];
    // the norm is used as an UPPER bound: inflate by 2^-9 to cover the 22-bit operand and the reduction rounding
    const float norm = sqrtf(ss) * sc * 1.002f;
    if (lane == 0) {
      if (out_norm != nullptr) out_norm[r] = norm;
      local_max_norm = fmaxf(local_max_norm, norm);
      if (ss > 0.0f) local_max_scale = fmaxf(local_max_scale, sc);   // all-zero rows carry the neutral scale 1
    }
  }
  if (lane == 0 && stats != nullptr) {
    atomicMax(reinterpret_cast<int*>(stats + 0), __float_as_int(local_max_norm));
    atomicMax(reinterpret_cast<int*>(stats + 1), __float_as_int(local_max_scale));
  }
}

// hi_global[r, :] = hi[r, :] * (scale_r / max_scale): an exact power-of-two rescale (values of small rows may fall
// into the fp16 subnormal range -- that loss is inside the filter's error bound).
__global__ void rescale_hi_global_kernel(const __half* __restrict__ split, const float* __restrict__ scale,
                                         const float* __restrict__ stats, const int32_t* __restrict__ perm,
                                         int64_t rows, int d_pad, __half* __restrict__ out_hi) {
  const float inv_max = 1.0f / fmaxf(stats[1], 1e-38f);
  const int64_t n_vec = rows * (d_pad / 8);
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n_vec;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / (d_pad / 8);                     // output row = processing position
    const int e = static_cast<int>(i % (d_pad / 8)) * 8;
    const int64_t src = perm != nullptr ? perm[r] : r;     // the item placed at that position
    const float f = scale[src] * inv_max;   // power of two <= 1
    uint4 raw = *reinterpret_cast<const uint4*>(split + src * 2 * d_pad + e);
    __half2* h = reinterpret_cast<__half2*>(&raw);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float2 v = __half22float2(h[q]);
      h[q] = __floats2half2_rn(v.x * f, v.y * f);
    }
    *reinterpret_cast<uint4*>(out_hi + r * d_pad + e) = raw;
  }
}

// Exclusion lists in processing order.  inv[perm[p]] = p, then one warp per list row writes, for every excluded local
// id of the row, the key (row << 32) | position.  Sorting the keys ascending orders every row's positions (the rows are
// already contiguous, so the row pointer is unchanged): the low 32 bits of the sorted keys are the filter's excl_pos.
__global__ void invert_perm_kernel(const int32_t* __restrict__ perm, int64_t n, int32_t* __restrict__ inv) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    inv[perm[i]] = static_cast<int32_t>(i);
}
__global__ void exclusion_keys_kernel(const int32_t* __restrict__ indptr, const int32_t* __restrict__ ids,
                                      const int32_t* __restrict__ inv, int64_t rows, int64_t* __restrict__ keys) {
  const int lane = threadIdx.x % 32;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / 32;
  const int64_t n_warps = static_cast<int64_t>(gridDim.x) * blockDim.x / 32;
  for (int64_t r = warp; r < rows; r += n_warps) {
    const int e1 = indptr[r + 1];
    for (int e = indptr[r] + lane; e < e1; e += 32) {
      const int32_t pos = inv != nullptr ? inv[ids[e]] : ids[e];
      keys[e] = static_cast<int64_t>(static_cast<uint64_t>(r) << 32 | static_cast<uint32_t>(pos));
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
#ifdef TRK_FILTER_CYCLES
// Copies the cycle sums of every filter launch since the last call (categories in FilterCycle order) to `out` and
// zeroes them.  Returns the number of categories.
extern "C" int trk_debug_filter_cycles(unsigned long long* out, int n) {
  if (out == nullptr || n < kNumCycles) return -kNumCycles;
  if (cudaDeviceSynchronize() != cudaSuccess) return 0;
  if (cudaMemcpyFromSymbol(out, g_filter_cycles, sizeof(g_filter_cycles)) != cudaSuccess) return 0;
  const unsigned long long zero[kNumCycles] = {};
  if (cudaMemcpyToSymbol(g_filter_cycles, zero, sizeof(zero)) != cudaSuccess) return 0;
  return kNumCycles;
}
#endif

int score_filter_max_k() { return kFilterMaxK; }
int score_filter_list_width() { return kKeepMax; }

int operand_stats(const void* split, const float* scale, int64_t rows, int32_t d_pad, float* out_norm, float* stats,
                  cudaStream_t stream) {
  TRK_CHECK_ARG(split && scale && rows >= 0 && d_pad >= 64 && d_pad % 64 == 0, "operand_stats: bad arguments");
  if (rows == 0) return TRK_OK;
  const int threads = 256;
  operand_stats_kernel<<<capped_grid(ceil_div(rows, threads / 32), 8), threads, 0, stream>>>(
      static_cast<const __half*>(split), scale, rows, d_pad, out_norm, stats);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

int rescale_hi_global(const void* split, const float* scale, const float* stats, const int32_t* perm, int64_t rows,
                      int32_t d_pad, void* out_hi, cudaStream_t stream) {
  TRK_CHECK_ARG(split && scale && stats && out_hi && rows >= 0 && d_pad >= 64 && d_pad % 64 == 0,
                "rescale_hi_global: bad arguments");
  if (rows == 0) return TRK_OK;
  const int threads = 256;
  rescale_hi_global_kernel<<<capped_grid(ceil_div(rows * (d_pad / 8), threads), 16), threads, 0, stream>>>(
      static_cast<const __half*>(split), scale, stats, perm, rows, d_pad, static_cast<__half*>(out_hi));
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

int exclusion_positions(const int32_t* item_perm, int64_t n_items, int32_t* inv_perm, const int32_t* excl_indptr,
                        const int32_t* excl_ids, int64_t n_rows, int64_t* out_keys, cudaStream_t stream) {
  TRK_CHECK_ARG(excl_indptr && excl_ids && out_keys && n_rows >= 0 && n_items >= 0, "exclusion_positions: bad arguments");
  TRK_CHECK_ARG(item_perm == nullptr || inv_perm != nullptr, "exclusion_positions: item_perm needs inv_perm");
  if (item_perm != nullptr && n_items > 0) {
    invert_perm_kernel<<<capped_grid(ceil_div(n_items, 256), 16), 256, 0, stream>>>(item_perm, n_items, inv_perm);
    TRK_CHECK_LAUNCH();
  }
  if (n_rows == 0) return TRK_OK;
  exclusion_keys_kernel<<<capped_grid(ceil_div(n_rows, 256 / 32), 16), 256, 0, stream>>>(
      excl_indptr, excl_ids, item_perm != nullptr ? inv_perm : nullptr, n_rows, out_keys);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

// (the kernel of one instantiation, for launch_sweep)
template <int kNKB, int kCluster, bool kExclude>
struct FilterKernel {
  static constexpr auto fn = score_filter_kernel<kNKB, kCluster, kExclude>;
};

int score_filter_f16(const void* user_split, const float* user_scale, const float* user_bias,
                     const float* user_norm, const void* item_hi, const float* item_stats, const float* item_bias,
                     const float* block_bias_max, const float* block_bias_min, const int32_t* item_perm,
                     int64_t n_users, int64_t n_items, int32_t d_pad, int32_t k, int32_t n_splits,
                     int32_t item_id_offset, float* cand_score, int32_t* cand_item, float* row_theta,
                     const int32_t* excl_indptr, const int32_t* excl_pos, cudaStream_t stream) {
  TRK_CHECK_ARG(cand_score && cand_item && row_theta, "score_filter: null output");
  if (k < 1 || k > kFilterMaxK) {
    set_error("score_filter: k=%d outside [1, %d]", k, kFilterMaxK);
    return TRK_ERR_UNSUPPORTED;
  }
  TRK_CHECK_ARG(reinterpret_cast<uintptr_t>(item_bias) % 16 == 0, "score_filter: operands must be 16-byte aligned");

  FilterParams p;
  p.block_bias_min = block_bias_min;
  // Tile-end compaction trigger.  TRK_FILTER_TILE_END_TRIGGER (probe knob) sets it; kBufEntries or more turns the
  // tile-end pass off (no buffer holds more than kBufEntries entries).
  p.tile_end_trigger = 26;
  {
    const char* env = getenv("TRK_FILTER_TILE_END_TRIGGER");
    if (env != nullptr) p.tile_end_trigger = atoi(env) < kBufEntries ? atoi(env) : kBufEntries;
    if (p.tile_end_trigger < kKeepMax + 2) p.tile_end_trigger = kKeepMax + 2;   // (a compaction leaves up to kKeepMax)
  }
  p.cand_score = cand_score;
  p.cand_item = cand_item;
  return launch_sweep<FilterKernel>("score_filter", p, kBufBytes, user_split, user_scale, user_bias, user_norm, item_hi,
                                    item_stats, item_bias, block_bias_max, item_perm, n_users, n_items, d_pad, k,
                                    n_splits, item_id_offset, row_theta, excl_indptr, excl_pos, stream);
}

}  // namespace trk
