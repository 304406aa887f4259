// K2 + K3 fused on Hopper tensor cores (wgmma): user x item scores and the per-user top-k (or the dense score matrix),
// without the [n_users, n_items] matrix ever reaching HBM in the top-k form.
//
// Reference chain replaced: tf.matmul(user_repr, item_repr, transpose_b=True) (tensorrec/prediction_graphs.py:49-50,
// and :64-65 -> recommendation_graphs.py:121 for cosine, operands pre-normalised by K1), bias_prediction_dense
// (tensorrec/recommendation_graphs.py:41) and rank_predictions (:73-82) restricted to rank <= k.
//
// Arithmetic: operands are the split-fp16 rows written by K1 (hi | lo, per-row power-of-two scale).  Per 64-wide
// k-block three groups of wgmma accumulate hi.hi + lo.hi + hi.lo into ONE fp32 register accumulator, i.e. an
// fp32-grade dot product (the dropped lo.lo term is < 2^-22 relative) that is exact for integer-valued
// representations -- which is what makes rank parity with the reference testable bit for bit.
//
// CTA = 384 threads (three warpgroups), one CTA per SM, persistent over work items (user block of 128 rows, item split):
//   warp 0        TMA producer: the A block (all k-blocks, resident for the whole sweep) then a ring of B k-block
//                 tiles [128 items x 64 fp16, 128B-swizzled] over the item range;
//   warpgroups 1, 2  consumers: warpgroup g owns user rows [64 g, 64 g + 64) of the block and computes, per item tile,
//                 their 64 x 128 scores with m64n128k16 wgmma into registers.  The accumulator goes through a small
//                 shared-memory staging tile (32 columns per half at a time) so that the epilogue runs one thread per
//                 (user row, column half): score = acc * scale_u * scale_i + bias_u + bias_i, compare against that
//                 list's current k-th best, rare insert into the sorted list in shared memory.  The two half-lists of
//                 a row are merged at the end of the item range.  Items are visited in ascending id order and the
//                 compare is strict, so equal scores keep the lower item id first -- tf.nn.top_k's order.
//
// Score forms (ScoreForm, one template parameter; DESIGN.md §3.7): dot / cosine as above, Euclidean similarity (§3.4),
// and mixtures of tastes collapsed by a max or by attention (§3.5), of dot products or of Euclidean similarities
// (§3.12).  Modes (TcMode): the dense matrix, the top-k above
// (k <= 32), or the wide top-k (k <= 1024, DESIGN.md §3.8), where every (row, column half) keeps its list in global
// memory and a warp compacts a full list to its exact top k, or the counting mode (DESIGN.md §3.9), which captures the
// scores of listed (user, item) pairs and counts the columns that outrank each of them, or the pairs mode (DESIGN.md
// §3.13), which captures the scores of listed pairs from item tiles gathered out of each user block's own listed items.
// score_tc is the one host entry point behind every trk_score_{topk,dense,count,pairs}* function: it validates the
// arguments and launches one of the 68 instantiations.
#include "common.cuh"

namespace trk {

constexpr int kWgRows = 64;           // user rows per consumer warpgroup
constexpr int kStageStride = 33;      // fp32 per staged row (32 columns + 1: conflict-free row reads)
constexpr uint32_t kAccStageBytes = 2u * kWgRows * kStageStride * 4u;   // per warpgroup: 2 halves x 64 rows x 32 cols
constexpr int kMaxK = 32;
constexpr int kExactWideMaxK = 1024;   // wide mode

// What the kernel makes of the scores: the dense matrix, a sorted top-k list per (row, column half) in shared memory
// (k <= kMaxK), or an unsorted list per (row, column half) in global memory (k <= kExactWideMaxK).
enum TcMode { kModeDense, kModeTopk, kModeWide, kModeCount, kModePairs };

// Wide mode: a list keeps at most k entries between compactions and holds exact_wide_cap(k) = 2 keep, keep = k rounded
// up to 32, so a compacted list always has room for one whole chunk of 32 columns (DESIGN.md §3.8).
__host__ __device__ constexpr int exact_wide_keep(int k) { return static_cast<int>(round_up(k, 32)); }
__host__ __device__ constexpr int exact_wide_cap(int k) { return 2 * exact_wide_keep(k); }
constexpr uint32_t kWideScratchBytes = 8u * 256u * 4u;   // wide mode: a 256-bin histogram per consumer warp

struct TcParams {
  const float* user_scale;
  const float* user_bias;   // may be null
  const float2* item_meta;  // [tiles*128] {scale, bias}; padding {0, -inf}
  int64_t n_users;
  int64_t n_items;
  int32_t n_kblocks;        // d_pad / 64  (hi half); the operand has 2*n_kblocks k-blocks
  int32_t n_stages;
  int32_t k;                // top-k mode
  int32_t n_splits;
  int32_t tiles_per_split;
  int32_t n_tiles;          // ceil(n_items / 128)
  int32_t n_user_blocks;
  int32_t item_id_offset;
  float* cand_score;        // top-k mode outputs
  int32_t* cand_item;
  float* dense_out;         // dense mode output
  int64_t dense_stride;
  int32_t tma_store;        // dense mode: 1 = rows are 16-byte aligned, the epilogue stores through TMA
  const int32_t* n_users_live;  // device, may be null: only the first *n_users_live user rows hold work (rows flagged
                                // by the filter's certificate, counted on the device) -- later user blocks are skipped
};

// Exclusion lists (kExclude instantiations, top-k mode only): the excluded LOCAL item ids of list row r, ascending, at
// ids[indptr[r] .. indptr[r + 1]); user row u reads list row row_map[u] (null = u).  A kernel parameter of its own:
// TcParams keeps its size, so the instantiations without exclusion compile exactly as before.
struct TcExcl {
  const int32_t* indptr;
  const int32_t* ids;
  const int32_t* row_map;
};

// The score form of an instantiation: what the epilogue makes of a (user, item) tile's accumulators.
enum ScoreForm {
  kFormDot,               // dot / cosine (score_chunk)
  kFormEuclid,            // Euclidean similarity (score_chunk_euclid, TcEuclid)
  kFormTastesMax,         // pred = max_t u_t . i        (recommendation_graphs.py:107; collapse_chunk, TcTastes)
  kFormTastesAttention,   // pred = sum_t softmax_t(a_t . i) u_t . i   (:96-103)
  kFormTastesEuclidMax,        // pred = max_t e(u_t, i),  e(x, i) = -|x - i|   (DESIGN.md §3.12)
  kFormTastesEuclidAttention,  // pred = sum_t softmax_t(e(a_t, i)) e(u_t, i)
};
__host__ __device__ constexpr bool is_tastes_euclid(ScoreForm f) {
  return f == kFormTastesEuclidMax || f == kFormTastesEuclidAttention;
}
__host__ __device__ constexpr bool is_tastes(ScoreForm f) {
  return f == kFormTastesMax || f == kFormTastesAttention || is_tastes_euclid(f);
}
// the forms that read item norms (TcEuclid)
__host__ __device__ constexpr bool is_euclid(ScoreForm f) { return f == kFormEuclid || is_tastes_euclid(f); }

// Euclidean similarity (kFormEuclid and the Euclidean tastes forms): -1/2 |row|^2 of every user operand row -- [n_users],
// or [n_ops, n_users] for a mixture of tastes -- and of every item column, as operand_half_sqnorm_kernel
// (similar_items.cu) computes them from the split operands -- the norms see exactly the values the dot product sees.
// The epilogue reads item norms for whole 128-column tiles, so item_half_sqnorm holds n_items_padded256 entries, 0
// beyond n_items (finite: the meta's -inf bias still gives those columns -inf).  Also a kernel parameter of its own,
// for the same reason as TcExcl.
struct TcEuclid {
  const float* user_half_sqnorm;
  const float* item_half_sqnorm;
};

// Mixtures of tastes (the tastes forms): every user has n_ops operand rows -- u_0 .. u_{T-1} and, with attention,
// a_0 .. a_{T-1} -- stacked as [n_ops, n_users, 2 d_pad] with scales [n_ops, n_users].  A consumer warpgroup's 64
// accumulator rows hold per_wg = 64 / n_ops users x n_ops operands (row j * per_wg + q = operand j of user q; rows at
// or beyond n_ops * per_wg are never loaded nor read), so a user block is 2 per_wg users and all operands of a (user,
// item) pair come out of one tile's MMAs.  Also a kernel parameter of its own, for the same reason as TcExcl.
struct TcTastes {
  int32_t n_ops;
  int32_t n_tastes;
  int32_t per_wg;
};

// Wide mode (kModeWide): the lists live in global memory, [n_users, n_splits, 2, exact_wide_cap(k)] scores and ids
// (list (u, split, column half)) plus [n_users, n_splits, 2] counts.  A kernel parameter of its own, for the same reason
// as TcExcl.
struct TcWide {
  int32_t* list_count;
};

// Counting mode (kModeCount, DESIGN.md §3.9): listed (user row, item) pairs, the pairs of user row u at
// [indptr[u], indptr[u + 1]).  pass < 0 (capture): ids = LOCAL item ids ascending per row, and the final unmasked score
// of every pair goes to score[pair].  pass >= 0 (count): the row's pairs sorted by (score desc, id asc) -- ids and
// score in that order -- and pass p adds to count[pair] how many columns outrank pair 32 p + j of the row (j < 32).
// block_pairs [n_user_blocks]: the most pairs of a row of the block; user blocks with at most 32 max(p, 0) are
// skipped.  A kernel parameter of its own, for the same reason as TcExcl.
// The pairs mode (kModePairs, DESIGN.md §3.13) is a capture (pass = -1) over gathered item tiles: ids are VIRTUAL
// columns tile * 128 + c, ascending per row; tile_items [tiles, 128] = the item of every slot (-1: empty, a zero row);
// work [n_work, 3] = (user block, first tile, end tile) of every work item; item_split = the item operand rows the
// producer gathers.  TcParams.item_meta and TcEuclid.item_half_sqnorm hold one entry per slot.  (The fields follow
// `pass`, so the counting mode's instantiations see the layout they always had.)
struct TcCount {
  const int32_t* indptr;
  const int32_t* ids;
  float* score;
  int32_t* count;
  const int32_t* block_pairs;
  int32_t pass;
  int32_t n_work;
  const int32_t* tile_items;
  const int32_t* work;
  const uint8_t* item_split;
};
constexpr int kCountTargets = 32;   // targets of a row per counting pass

// shared-memory carve-up (offsets from a 1024-byte aligned base); the list region holds the top-k lists, the dense
// mode's TMA store tiles or the wide mode's histograms
struct SmemLayout {
  uint32_t a_off, b_off, list_score_off, list_item_off, acc_off, bar_off, total;
};
constexpr uint32_t kStoreTileBytes = 32 * 32 * 4;   // one warp's 32 rows x 32 columns of fp32 scores
__host__ __device__ inline SmemLayout make_layout(int n_kblocks, int n_stages, int k, bool dense_staging = false,
                                                  bool wide = false) {
  SmemLayout L;
  L.a_off = 0;
  L.b_off = L.a_off + 2u * n_kblocks * kATileBytes;
  L.list_score_off = L.b_off + static_cast<uint32_t>(n_stages) * kBTileBytes;
  L.list_item_off = L.list_score_off + (dense_staging ? 16u * kStoreTileBytes
                                                      : wide ? kWideScratchBytes : 2u * k * kBlockM * 4u);
  L.acc_off = L.list_item_off + (dense_staging ? 0u : 2u * k * kBlockM * 4u);
  L.bar_off = L.acc_off + 2u * kAccStageBytes;
  L.total = L.bar_off + 512u;
  return L;
}

// barrier block (uint64 each): [0] a_full, [1] a_empty, [2 .. 2+S) b_full, [2+S .. 2+2S) b_empty.
// Both consumer warpgroups read every stage: the empty barriers count the 8 consumer warps.

__device__ __noinline__ float list_insert(float s, int32_t id, float* ls, int32_t* li, int k) {
  // ls/li point at this row's column of the [k][128] arrays.  Entries are sorted by (score desc, id asc) and the
  // new id is larger than every id already stored, so it goes behind all entries with score >= s.
  // Returns the row's new k-th best score (the insertion threshold).
  int j = k - 1;
  while (j > 0 && ls[(j - 1) * kBlockM] < s) {
    ls[j * kBlockM] = ls[(j - 1) * kBlockM];
    li[j * kBlockM] = li[(j - 1) * kBlockM];
    --j;
  }
  ls[j * kBlockM] = s;
  li[j * kBlockM] = id;
  return ls[(k - 1) * kBlockM];
}

// 16-byte read-only global load ({scale, bias} of two item columns; the 1 KB of a tile stays in L1)
__device__ __forceinline__ float4 ldg128(const float2* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// Scores one 32-column chunk held in r[] (raw accumulators in, final scores out) and returns the chunk maximum.
// Branch-free: the 16 loads and 96 FP ops of a chunk pipeline freely; the rare insert path is taken per chunk.
__device__ __forceinline__ float score_chunk(uint32_t (&r)[32], const float2* meta, float su, float ubias) {
  float cmax = -__int_as_float(0x7f800000);
#pragma unroll
  for (int j = 0; j < 32; j += 2) {
    const float4 m = ldg128(meta + j);   // {scale_j, bias_j, scale_j+1, bias_j+1}
    const float s0 = fmaf(__uint_as_float(r[j]), m.x * su, ubias) + m.y;       // (acc*scales + ub) + ib
    const float s1 = fmaf(__uint_as_float(r[j + 1]), m.z * su, ubias) + m.w;
    r[j] = __float_as_uint(s0);
    r[j + 1] = __float_as_uint(s1);
    cmax = fmaxf(cmax, fmaxf(s0, s1));
  }
  return cmax;
}

// The Euclidean form of score_chunk: EuclideanSimilarityPredictionGraph dense (prediction_graphs.py:84-100) then
// bias_prediction_dense (recommendation_graphs.py:41), every step in the reference's order:
//   p = acc * (scale_u * scale_i)  (powers of two: exact),  d2 = (|u|^2 - 2 p) + |i|^2,
//   s = (-sqrt(max(d2, 1e-16)) + ub) + ib
// with |row|^2 = -2 * (-1/2 |row|^2) (exact) and a correctly rounded sqrtf.  A missing bias is 0 here, and s <= -1e-8
// is never zero, so adding it changes nothing.  usq = |u|^2 of the row, ihsq = the chunk's -1/2 |i|^2 (16-byte aligned).
__device__ __forceinline__ float score_chunk_euclid(uint32_t (&r)[32], const float2* meta, const float* ihsq, float su,
                                                    float usq, float ubias) {
  float cmax = -__int_as_float(0x7f800000);
#pragma unroll
  for (int j = 0; j < 32; j += 4) {
    const float4 h = __ldg(reinterpret_cast<const float4*>(ihsq + j));
    const float hq[4] = {h.x, h.y, h.z, h.w};
#pragma unroll
    for (int q = 0; q < 4; q += 2) {
      const float4 m = ldg128(meta + j + q);   // {scale_j, bias_j, scale_j+1, bias_j+1}
      const float p0 = __uint_as_float(r[j + q]) * (m.x * su);
      const float p1 = __uint_as_float(r[j + q + 1]) * (m.z * su);
      const float d0 = (usq - 2.0f * p0) + -2.0f * hq[q];
      const float d1 = (usq - 2.0f * p1) + -2.0f * hq[q + 1];
      const float s0 = (-sqrtf(fmaxf(d0, 1e-16f)) + ubias) + m.y;
      const float s1 = (-sqrtf(fmaxf(d1, 1e-16f)) + ubias) + m.w;
      r[j + q] = __float_as_uint(s0);
      r[j + q + 1] = __float_as_uint(s1);
      cmax = fmaxf(cmax, fmaxf(s0, s1));
    }
  }
  return cmax;
}

// The taste collapse of one staged chunk: columns [32 c, 32 c + 32) of both 64-column halves of the tile,
// in the warpgroup's staging tile (stage = acc_stage, rows as in TcTastes).  Every (column half, user, column) element
// is collapsed by one thread -- all 128 of the warpgroup share the work, lane = column -- and its final score replaces
// operand row 0 of its user; the element reads and writes only its own user's rows in its own column.  Reference
// order (collapse_mixture_of_tastes, recommendation_graphs.py:85-109, then bias_prediction_dense, :41), every
// product and sum rounded on its own (no contraction):
//   p_j = acc_j * (scale_i * scale_j)  (powers of two: exact);
//   max:        pred = max_t p_t;
//   attention:  m = max_t a_t,  e_t = expf(a_t - m),  s = sum_t e_t,  pred = sum_t p_t * (e_t / s)  (taste order);
//   score = (pred + ub) + ib.
// With attention, e_t is parked in a_t's staging row between the two passes.  The Euclidean tastes forms (DESIGN.md
// §3.12) give every operand row -- taste rows and attention rows alike, as the reference feeds both through the
// prediction graph -- its similarity e_j = -sqrt(max(d2_j, 1e-16)), d2_j = (|x_j|^2 - 2 p_j) + |i|^2.  With attention
// the e_j replace the staged accumulators first and are collapsed as above (operand_value then reads them as they
// are); the max form takes pred = -sqrt(max(min_t d2_t, 1e-16)), the same value with one root instead of T.
template <ScoreForm kForm>
__device__ __forceinline__ float operand_value(float staged, float scales) {
  if constexpr (is_tastes_euclid(kForm)) return staged;
  else return __fmul_rn(staged, scales);
}

template <ScoreForm kForm>
__device__ __forceinline__ void collapse_chunk(float* stage, int wt, int c, const float2* meta, const float* ihsq,
                                               const TcParams& p, const TcEuclid& ev, const TcTastes z, int64_t u0) {
  const int lane = wt % 32;
  const int n_tastes = z.n_tastes;
  for (int e = wt / 32; e < 2 * z.per_wg; e += kConsumerThreads / 32) {   // warp-uniform: one (half, user) per warp
    const int h = e / z.per_wg;
    const int q = e - h * z.per_wg;
    const int64_t u = u0 + q;
    const bool u_ok = u < p.n_users;
    const float2 m = meta[h * 64 + c * 32 + lane];
    float* col = stage + (h * kWgRows + q) * kStageStride + lane;   // operand j at col[j * per_wg * kStageStride]
    const int64_t op_stride = z.per_wg * kStageStride;
    float pred;
    if constexpr (is_tastes_euclid(kForm)) {
      // |x_j|^2 = -2 (-1/2 |x_j|^2), |i|^2 and 2 p_j are exact; every sum is rounded on its own; sqrtf is correctly
      // rounded, so -sqrtf(max(., 1e-16)) is non-increasing and the largest e_t is the root of the smallest d2_t
      const float isq = -2.0f * __ldg(ihsq + h * 64 + c * 32 + lane);
      float d2_min = __int_as_float(0x7f800000);
      for (int j = 0; j < z.n_ops; ++j) {
        const float sj = u_ok ? __ldg(p.user_scale + j * p.n_users + u) : 0.0f;
        const float xsq = u_ok ? -2.0f * __ldg(ev.user_half_sqnorm + j * p.n_users + u) : 0.0f;
        const float pj = __fmul_rn(col[j * op_stride], m.x * sj);
        const float d2 = __fadd_rn(__fsub_rn(xsq, __fmul_rn(2.0f, pj)), isq);
        if constexpr (kForm == kFormTastesEuclidMax) d2_min = fminf(d2_min, d2);
        else col[j * op_stride] = -sqrtf(fmaxf(d2, 1e-16f));
      }
      if constexpr (kForm == kFormTastesEuclidMax) pred = -sqrtf(fmaxf(d2_min, 1e-16f));
    }
    if constexpr (kForm == kFormTastesMax) {
      pred = -__int_as_float(0x7f800000);
      for (int t = 0; t < n_tastes; ++t) {
        const float su = u_ok ? __ldg(p.user_scale + t * p.n_users + u) : 0.0f;
        pred = fmaxf(pred, operand_value<kForm>(col[t * op_stride], m.x * su));
      }
    } else if constexpr (kForm != kFormTastesEuclidMax) {
      float amax = -__int_as_float(0x7f800000);
      for (int t = 0; t < n_tastes; ++t) {
        const float sa = u_ok ? __ldg(p.user_scale + (n_tastes + t) * p.n_users + u) : 0.0f;
        const float a = operand_value<kForm>(col[(n_tastes + t) * op_stride], m.x * sa);
        col[(n_tastes + t) * op_stride] = a;
        amax = fmaxf(amax, a);
      }
      float sum = 0.0f;
      for (int t = 0; t < n_tastes; ++t) {
        const float ex = expf(__fsub_rn(col[(n_tastes + t) * op_stride], amax));
        col[(n_tastes + t) * op_stride] = ex;
        sum = t == 0 ? ex : __fadd_rn(sum, ex);
      }
      pred = 0.0f;
      for (int t = 0; t < n_tastes; ++t) {
        const float su = u_ok ? __ldg(p.user_scale + t * p.n_users + u) : 0.0f;
        const float pt = operand_value<kForm>(col[t * op_stride], m.x * su);
        const float w = __fdiv_rn(col[(n_tastes + t) * op_stride], sum);
        pred = t == 0 ? __fmul_rn(pt, w) : __fadd_rn(pred, __fmul_rn(pt, w));
      }
    }
    const float ub = (u_ok && p.user_bias != nullptr) ? __ldg(p.user_bias + u) : 0.0f;
    col[0] = __fadd_rn(__fadd_rn(pred, ub), m.y);
  }
}

// Chunk maximum of final scores (tastes forms: collapse_chunk formed them).
__device__ __forceinline__ float chunk_max(const uint32_t (&r)[32]) {
  float cmax = -__int_as_float(0x7f800000);
#pragma unroll
  for (int j = 0; j < 32; ++j) cmax = fmaxf(cmax, __uint_as_float(r[j]));
  return cmax;
}

// Final scores of one 32-column chunk of one user row in form kForm, and their maximum.  Dot / Euclidean: r[] holds
// raw accumulators (ihsq = the chunk's item norms, usq = the row's |u|^2); tastes: r[] already holds final scores.
template <ScoreForm kForm>
__device__ __forceinline__ float score_chunk_as(uint32_t (&r)[32], const float2* meta, const float* ihsq, float su,
                                                float usq, float ubias) {
  if constexpr (is_tastes(kForm)) return chunk_max(r);
  else if constexpr (kForm == kFormEuclid) return score_chunk_euclid(r, meta, ihsq, su, usq, ubias);
  else return score_chunk(r, meta, su, ubias);
}

// Exclusion (kExclude): the final scores of the chunk's columns [base, base + 32) named in list row `xr` become -inf
// (never inserted: the compare is strict and the lists start at -inf).  A select per register, not r[dynamic index],
// which would put r[] into local memory; the FINAL score is masked, not the accumulator (a zero scale would turn -inf into
// NaN).  Returns the new chunk maximum and moves `next` to the row's first listed id >= base + 32.
__device__ __forceinline__ float excl_mask_scores(uint32_t (&r)[32], const TcExcl& x, int32_t xr, int32_t base,
                                                  int32_t& next) {
  const int hi = __ldg(x.indptr + xr + 1);
  int i = excl_lower_bound(x.ids, __ldg(x.indptr + xr), hi, base);
  int32_t e = i < hi ? __ldg(x.ids + i) : 0x7fffffff;
  uint32_t mask = 0;
  while (e < base + 32) {
    mask |= 1u << (e - base);
    ++i;
    e = i < hi ? __ldg(x.ids + i) : 0x7fffffff;
  }
  next = e;
  float cmax = -__int_as_float(0x7f800000);
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    r[j] = ((mask >> j) & 1u) ? 0xff800000u : r[j];
    cmax = fmaxf(cmax, __uint_as_float(r[j]));
  }
  return cmax;
}

// Per-row exclusion state of the exact kernel (empty without exclusion).
template <bool kOn>
struct ExclCursor {
  int32_t row = -1;            // list row of this user row (-1: none)
  int32_t next = 0x7fffffff;   // first listed id >= the current chunk (INT32_MAX: none left)
};
template <>
struct ExclCursor<false> {};

// One 32-column chunk of one user row: final scores, then (top-k mode) the row's listed columns masked (kExclude) and
// the rare inserts, or (dense mode) the store.  `x` is taken by value: a reference bound to the kernel parameter
// changes the generated code of the instantiations without exclusion.  ihsq = the tile's item norms (kFormEuclid).
template <bool kDense, bool kExclude, ScoreForm kForm>
__device__ __forceinline__ void process_chunk(uint32_t (&r)[32], int c, int t, int32_t id0, const float2* meta,
                                              const float* ihsq, float su, float usq, float ubias, float& thr,
                                              float* ls, int32_t* li, const TcParams& p, int64_t u, bool u_ok,
                                              const TcExcl x, ExclCursor<kExclude>& xc) {
  float cmax = score_chunk_as<kForm>(r, meta + c * 32, ihsq + c * 32, su, usq, ubias);
  if constexpr (!kDense) {
    if constexpr (kExclude) {
      const int32_t base = t * kBlockN + c * 32;   // local id of the chunk's first column
      if (xc.next < base + 32) cmax = excl_mask_scores(r, x, xc.row, base, xc.next);
    }
    if (cmax > thr) {   // some column of this chunk enters the row's list (probability ~ 32 k / items seen)
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float s = __uint_as_float(r[j]);
        if (s > thr) thr = list_insert(s, id0 + c * 32 + j, ls, li, p.k);
      }
    }
  } else {
    const int64_t i0 = static_cast<int64_t>(t) * kBlockN + c * 32;
    if (u_ok) {
      float* dst = p.dense_out + u * p.dense_stride + i0;
      if (i0 + 32 <= p.n_items && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
#pragma unroll
        for (int j = 0; j < 32; j += 4)
          *reinterpret_cast<uint4*>(dst + j) = make_uint4(r[j], r[j + 1], r[j + 2], r[j + 3]);
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (i0 + j < p.n_items) dst[j] = __uint_as_float(r[j]);
      }
    }
  }
}

// ---- wide mode (DESIGN.md §3.8) ----
// Each thread's list holds (final score, item id) entries in ascending id order: items arrive in ascending id order and
// a compaction is stable.  An item enters when its score is > thr, the k-th best score the list has kept so far: an
// item whose score equals it has a larger id than the k kept entries that rank ahead of it, so it cannot be in the
// list's top k.  -inf never enters.

// Warp-cooperative compaction of lane src's list (ls / li, cnt > k entries) to exactly its top k by (score desc,
// id asc): the k-th best key by a radix select, every entry above it, and the first entries equal to it -- the lowest
// ids -- up to k.  Returns the k-th best score on every lane.  Called warp-uniformly.
__device__ __forceinline__ float exact_wide_compact(int src, int lane, float* ls_own, int32_t* li_own, int cnt_own,
                                                    int k, uint32_t* hist) {
  const int n = __shfl_sync(0xffffffffu, cnt_own, src);
  float* ls = reinterpret_cast<float*>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(ls_own), src));
  int32_t* li =
      reinterpret_cast<int32_t*>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(li_own), src));
  __syncwarp();   // the owner's appends are visible to every lane
  const uint32_t kth = wide_select(ls, li, n, k, hist, lane);
  int n_gt = 0;
  for (int i = lane; i < n; i += 32) n_gt += wide_key(ls[i]) > kth ? 1 : 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) n_gt += __shfl_xor_sync(0xffffffffu, n_gt, o);
  const int n_eq = k - n_gt;   // entries equal to the k-th best that are kept
  const uint32_t below = (1u << lane) - 1u;
  int n_keep = 0, eq_seen = 0;
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    float s = 0.0f;
    int32_t id = 0;
    uint32_t key = 0;
    if (i < n) {
      s = ls[i];
      id = li[i];
      key = wide_key(s);
    }
    const unsigned eq = __ballot_sync(0xffffffffu, i < n && key == kth);
    const bool kp = i < n && (key > kth || (key == kth && eq_seen + __popc(eq & below) < n_eq));
    const unsigned b = __ballot_sync(0xffffffffu, kp);   // every lane has read its entry of this round
    if (kp) {
      const int dst = n_keep + __popc(b & below);   // <= i: never an entry not yet read
      ls[dst] = s;
      li[dst] = id;
    }
    n_keep += __popc(b);
    eq_seen += __popc(eq);
    __syncwarp();
  }
  return wide_unkey(kth);
}

// Per-row state of the wide mode (empty in the other modes): the list's entry count and its index (u, split, half).
template <bool kOn>
struct WideCursor {
  int cnt = 0;
  int64_t list = 0;
};
template <>
struct WideCursor<false> {};

// The histogram of consumer warp `warp` in the list region of shared memory (wide mode).
__device__ __forceinline__ uint32_t* wide_hist(uint8_t* list_region, int warp) {
  return reinterpret_cast<uint32_t*>(list_region) + (warp - 4) * 256;
}

// The columns of a chunk of final scores that enter a list with threshold thr (bit j: column j).
__device__ __forceinline__ uint32_t exact_wide_admit(const uint32_t (&r)[32], float thr) {
  uint32_t mask = 0;
#pragma unroll
  for (int j = 0; j < 32; ++j) mask |= (__uint_as_float(r[j]) > thr ? 1u : 0u) << j;
  return mask;
}

// Compacts the lists of the lanes in `rows` (each to its top k) and lowers their counts to k.  Warp-uniform.
__device__ __forceinline__ void exact_wide_compact_rows(unsigned rows, int lane, float* ls, int32_t* li, int& cnt,
                                                        float& thr, int k, uint32_t* hist) {
  while (rows != 0u) {
    const int src = __ffs(rows) - 1;
    rows &= rows - 1u;
    const float kth = exact_wide_compact(src, lane, ls, li, cnt, k, hist);
    if (lane == src) {
      thr = kth;
      cnt = k;
    }
  }
  __syncwarp();
}

// One 32-column chunk of the lane's row in wide mode: final scores, the row's listed columns masked (kExclude), then
// the admitted columns appended to the lane's list; lists that could not take them are compacted first.  Lanes without
// a list (owner false) admit nothing.  Warp-uniform.
template <bool kExclude, ScoreForm kForm>
__device__ __forceinline__ void wide_chunk(uint32_t (&r)[32], int c, int t, int32_t id0, const float2* meta,
                                           const float* ihsq, float su, float usq, float ubias, float& thr, float* ls,
                                           int32_t* li, int& cnt, int k, bool owner, const TcExcl x,
                                           ExclCursor<kExclude>& xc, int lane, uint32_t* hist) {
  float cmax = score_chunk_as<kForm>(r, meta + c * 32, ihsq + c * 32, su, usq, ubias);
  if constexpr (kExclude) {
    const int32_t base = t * kBlockN + c * 32;
    if (xc.next < base + 32) cmax = excl_mask_scores(r, x, xc.row, base, xc.next);
  }
  uint32_t mask = (owner && cmax > thr) ? exact_wide_admit(r, thr) : 0u;
  const unsigned full = __ballot_sync(0xffffffffu, cnt + __popc(mask) > exact_wide_cap(k));
  if (full != 0u) {
    exact_wide_compact_rows(full, lane, ls, li, cnt, thr, k, hist);
    if (mask != 0u) mask = exact_wide_admit(r, thr);
  }
  if (mask != 0u) {
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      if ((mask >> j) & 1u) {
        const int e = cnt + __popc(mask & ((1u << j) - 1u));
        ls[e] = __uint_as_float(r[j]);
        li[e] = id0 + c * 32 + j;
      }
    }
    cnt += __popc(mask);
  }
}

// ---- counting mode (DESIGN.md §3.9) ----
// A column (s, id) outranks a pair (t, tid) when s > t or (s == t and id < tid) (r_before): the rank order of
// rank_full.  A pass's targets are a row's pairs 32 p .. 32 p + n - 1 in that order, staged in shared memory as [32][128]
// (column = user row of the block) with (-inf, INT32_MAX) beyond n, which every column outranks.  A column that
// outranks the lowest target outranks the suffix [lb, n) of the targets; it adds 1 to the row's bucket h[lb], and the
// prefix sums of h at the end of the work item are the targets' counts.

// Per-row state of the counting mode (empty in the other modes).  Capture: the row's pairs [lo, hi) and the first
// listed id >= the current chunk.  Count: the pass's first pair lo, its n targets and the lowest of them (+inf: none).
template <bool kOn>
struct CountCursor {
  int32_t lo = 0, hi = 0, n = 0;
  int32_t next = 0x7fffffff;
  float low_s = 0.0f;
  int32_t low_id = 0;
};
template <>
struct CountCursor<false> {};

// Does user block ub hold a row with pairs in this pass (capture: any pair)?  The same test in both roles.
__device__ __forceinline__ bool count_block_live(const TcCount& cn, int ub) {
  return __ldg(cn.block_pairs + ub) > kCountTargets * max(cn.pass, 0);
}

// Capture: the final scores of the row's pairs among the chunk's columns [base, base + 32) go to cn.score.  The pairs'
// columns become a bit mask, and an unrolled walk over the registers in column order stores the marked ones at
// consecutive pair positions (the ids ascend and are distinct): every r[j] has a constant index, so r[] stays in
// registers.  (A select of r[e - base] per pair was lowered to an indexed local-memory copy of r[] that every chunk of
// every pass paid for.)
__device__ __forceinline__ void capture_chunk(const uint32_t (&r)[32], const TcCount& cn, CountCursor<true>& cc,
                                              int32_t base) {
  int i = excl_lower_bound(cn.ids, cc.lo, cc.hi, base);
  int pos = i;
  int32_t e = i < cc.hi ? __ldg(cn.ids + i) : 0x7fffffff;
  uint32_t mask = 0;
  while (e < base + 32) {
    mask |= 1u << (e - base);
    ++i;
    e = i < cc.hi ? __ldg(cn.ids + i) : 0x7fffffff;
  }
  cc.next = e;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    if ((mask >> j) & 1u) {
      cn.score[pos] = __uint_as_float(r[j]);
      ++pos;
    }
  }
}

// Count: every column of the chunk (final scores, ids id0 ..) that outranks the lowest target adds 1 to h[lb], lb found
// by a binary search over the 32 staged targets (ts / ti / h: this row's column, stride kBlockM).  Target 31 is
// outranked whenever the lowest target is, so five steps find lb <= 31 exactly.
__device__ __forceinline__ void count_chunk(const uint32_t (&r)[32], int32_t id0, const float* ts, const int32_t* ti,
                                            int32_t* h, float low_s, int32_t low_id) {
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const float s = __uint_as_float(r[j]);
    const int32_t id = id0 + j;
    if (r_before(s, id, low_s, low_id)) {
      int lb = 0;
#pragma unroll
      for (int step = 16; step > 0; step >>= 1) {
        const int m = lb + step - 1;
        if (!r_before(s, id, ts[m * kBlockM], ti[m * kBlockM])) lb += step;
      }
      h[lb * kBlockM] += 1;
    }
  }
}

// One 32-column chunk of one user row in counting mode: final scores, then the capture of the row's pairs (pass < 0)
// or the row's excluded columns masked (kExclude, excl rows set) and the columns counted, unless the chunk's maximum
// lies below the lowest target.  kCapture (the pairs mode): always the capture, t a virtual tile.
template <bool kExclude, ScoreForm kForm, bool kCapture = false>
__device__ __forceinline__ void count_process_chunk(uint32_t (&r)[32], int c, int t, int32_t id0, const float2* meta,
                                                    const float* ihsq, float su, float usq, float ubias, const TcExcl x,
                                                    ExclCursor<kExclude>& xc, const TcCount cn, CountCursor<true>& cc,
                                                    const float* ts, const int32_t* ti, int32_t* h) {
  float cmax = score_chunk_as<kForm>(r, meta + c * 32, ihsq + c * 32, su, usq, ubias);
  const int32_t base = t * kBlockN + c * 32;
  if (kCapture || cn.pass < 0) {
    if (cc.next < base + 32) capture_chunk(r, cn, cc, base);
    return;
  }
  if constexpr (kExclude) {
    if (xc.next < base + 32) cmax = excl_mask_scores(r, x, xc.row, base, xc.next);
  }
  if (cmax >= cc.low_s) count_chunk(r, id0 + c * 32, ts, ti, h, cc.low_s, cc.low_id);
}

// Dense mode, TMA path: the warp's 32 rows x 32 columns go to a 128B-swizzled staging tile in shared memory and
// leave as ONE cp.async.bulk.tensor store (full 128-byte lines per row, rows / columns beyond the matrix clipped by the
// tensor map).  Direct stores from the row-per-thread layout write 16 bytes per lane to 32 different rows.
__device__ __forceinline__ void store_chunk_tma(const uint32_t (&r)[32], uint32_t stage_addr, int lane,
                                                const CUtensorMap* map_out, int32_t col0, int32_t row0) {
  if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");   // the buffer used two chunks ago
  __syncwarp();
#pragma unroll
  for (int c16 = 0; c16 < 8; ++c16) {
    const uint32_t addr = stage_addr + lane * 128 + ((c16 ^ (lane & 7)) << 4);
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[4 * c16]), "r"(r[4 * c16 + 1]),
                 "r"(r[4 * c16 + 2]), "r"(r[4 * c16 + 3])
                 : "memory");
  }
  fence_proxy_async();
  __syncwarp();
  if (lane == 0) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(map_out)),
                 "r"(stage_addr), "r"(col0), "r"(row0)
                 : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  }
}

// Pairs mode, producer: one B stage (k-block kb2 of a gathered tile, slots = its 128 items) written by the whole
// producer warp.  Lane l copies 16-byte chunk l % 8 of rows l / 8 + 4 j (8 lanes read one 128-byte row segment) to the
// address the 128B swizzle gives it -- the layout a TMA box of the same rows writes -- and an empty slot (-1) is
// zero-filled.  Every lane then
// arrives on the stage's full barrier (initialised to 32 arrivals) once its copies have landed.
template <int kNKB>
__device__ __forceinline__ void gather_b_stage(uint32_t dst, uint64_t* full, const int32_t* slots,
                                               const uint8_t* item_split, int kb2, int lane) {
  constexpr int64_t kRowBytes = 4 * kKBlock * kNKB;   // 2 d_pad fp16 per operand row
  const int c16 = lane % 8;
#pragma unroll 4
  for (int j = 0; j < 32; ++j) {
    const int r = lane / 8 + 4 * j;
    const int32_t item = __ldg(slots + r);
    const uint32_t d = dst + r * 128 + ((c16 ^ (r % 8)) << 4);
    const uint8_t* src = item_split + max(item, 0) * kRowBytes + kb2 * 128 + c16 * 16;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(item >= 0 ? 16 : 0)
                 : "memory");
  }
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(full)) : "memory");
}

// Work item w: (user block, item split, tiles [t0, t1)); the pairs mode reads it from its work list (split 0).
struct WorkItem {
  int ub, sp, t0, t1;
};
template <bool kPairs>
__device__ __forceinline__ WorkItem work_item(int64_t w, const TcParams& p, const TcCount& cn) {
  if constexpr (kPairs) {
    return {__ldg(cn.work + 3 * w), 0, __ldg(cn.work + 3 * w + 1), __ldg(cn.work + 3 * w + 2)};
  } else {
    const int ub = static_cast<int>(w / p.n_splits);
    const int sp = static_cast<int>(w % p.n_splits);
    const int t0 = sp * p.tiles_per_split;
    return {ub, sp, t0, min(t0 + p.tiles_per_split, p.n_tiles)};
  }
}

// kMode: dense, top-k, wide, count or pairs (TcMode).  kNKB = d_pad / 64 k-blocks per operand half.  kExclude (top-k modes): columns named in the row's exclusion list are
// left out of the top-k (excl_mask_scores); the counting mode is always instantiated with it and excludes nothing when
// x.indptr is null.  kForm: the score form, in every mode.  The tastes forms collapse a
// mixture of tastes per (user, item) (collapse_chunk); map_users is then the 3-D map of the stacked operand, a user
// block holds 2 z.per_wg users, and in dense mode map_out's box is 32 columns x z.per_wg rows.
template <TcMode kMode, int kNKB, bool kExclude, ScoreForm kForm>
__global__ void __launch_bounds__(kTcThreads, 1)
score_tc_kernel(const __grid_constant__ CUtensorMap map_users, const __grid_constant__ CUtensorMap map_items,
                const __grid_constant__ CUtensorMap map_out, const TcParams p, const TcExcl x, const TcEuclid e,
                const TcTastes z, const TcWide wl, const TcCount cn) {
  constexpr bool kDense = kMode == kModeDense;
  constexpr bool kWide = kMode == kModeWide;
  constexpr bool kCount = kMode == kModeCount;
  constexpr bool kPairs = kMode == kModePairs;
  uint8_t* smem = smem_base_1024();
  // (the counting mode stages its targets and buckets in the list region of k = kMaxK)
  const SmemLayout L = make_layout(p.n_kblocks, p.n_stages, kMode == kModeTopk ? p.k : (kCount ? kMaxK : 0),
                                   kDense && p.tma_store != 0, kWide);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.bar_off);
  uint64_t* a_full = bars + 0;
  uint64_t* a_empty = bars + 1;
  uint64_t* b_full = bars + 2;
  uint64_t* b_empty = bars + 2 + p.n_stages;

  const int warp = threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  constexpr int n_kb2 = 2 * kNKB;
  // work item w = (user block w / n_splits, item split w % n_splits): the splits of ONE user block go to consecutive
  // CTAs, so a handful of live user blocks (the device-side fallback: ~100 rows of a million) still spreads over the
  // whole machine -- with the block index minor, one live block of 8 x 132 items landed on a quarter of the CTAs
  // (the pairs mode: the work list's items)
  const int64_t n_work = kPairs ? cn.n_work : static_cast<int64_t>(p.n_user_blocks) * p.n_splits;
  // user blocks at or beyond this one hold no rows (every role skips them: the same test in both loops)
  const int live_blocks = p.n_users_live != nullptr
                              ? static_cast<int>(min(static_cast<int64_t>(p.n_user_blocks),
                                                     ceil_div(static_cast<int64_t>(__ldg(p.n_users_live)), kBlockM)))
                              : p.n_user_blocks;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&map_users);
    tma_prefetch_desc(&map_items);
  }
  if (warp == 1 && lane == 0) {
    mbar_init(a_full, 1);
    mbar_init(a_empty, 2 * kConsumerThreads / 32);
    for (int i = 0; i < p.n_stages; ++i) {
      mbar_init(b_full + i, kPairs ? 32 : 1);   // (the pairs mode: every producer lane's gathered copies)
      mbar_init(b_empty + i, 2 * kConsumerThreads / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 0) {
    // ===================================== TMA producer ======================================
    {   // warp-uniform control flow, one elected lane issues
      int stage = 0;       // B ring position
      uint32_t stage_phase = 0;
      uint32_t witer = 0;  // non-empty work items so far
      for (int64_t w = blockIdx.x; w < n_work; w += gridDim.x) {
        const WorkItem wi = work_item<kPairs>(w, p, cn);
        const int ub = wi.ub, t0 = wi.t0, t1 = wi.t1;
        if (t1 <= t0|| ub >= live_blocks || (kCount && !count_block_live(cn, ub))) continue;
        mbar_wait(a_empty, (witer & 1) ^ 1);  // the MMAs of the previous work item no longer read A
        if constexpr (is_tastes(kForm)) {
          // one box of n_ops x per_wg rows per warpgroup half and k-block; a half without users is not loaded
          const int32_t u0 = ub * 2 * z.per_wg;
          const int n_halves = u0 + z.per_wg < p.n_users ? 2 : 1;
          if (elect_one()) {
            mbar_arrive_expect_tx(a_full, n_kb2 * n_halves * z.n_ops * z.per_wg * (kKBlock * 2));
            for (int kb = 0; kb < n_kb2; ++kb)
              for (int h = 0; h < n_halves; ++h)
                tma_load_3d(smem + L.a_off + kb * kATileBytes + h * (kWgRows * 128), &map_users, a_full, kb * kKBlock,
                            u0 + h * z.per_wg, 0, kEvictFirst);
          }
        } else if (elect_one()) {
          mbar_arrive_expect_tx(a_full, n_kb2 * kATileBytes);
          for (int kb = 0; kb < n_kb2; ++kb)
            tma_load_2d(smem + L.a_off + kb * kATileBytes, &map_users, a_full, kb * kKBlock, ub * kBlockM,
                        kEvictFirst);
        }
        __syncwarp();
        ++witer;
        for (int t = t0; t < t1; ++t) {
#pragma unroll
          for (int kb = 0; kb < n_kb2; ++kb) {
            mbar_wait(b_empty + stage, stage_phase ^ 1);
            if constexpr (kPairs) {
              gather_b_stage<kNKB>(smem_u32(smem + L.b_off + stage * kBTileBytes), b_full + stage,
                                   cn.tile_items + static_cast<int64_t>(t) * kBlockN, cn.item_split, kb, lane);
            } else {
              if (elect_one()) {
                mbar_arrive_expect_tx(b_full + stage, kBTileBytes);
                tma_load_2d(smem + L.b_off + stage * kBTileBytes, &map_items, b_full + stage, kb * kKBlock,
                            t * kBlockN, kEvictLast);  // the item operand is re-read by every user block: keep it in L2
              }
              __syncwarp();
            }
            if (++stage == p.n_stages) {   // ring position advances incrementally: no div/mod on the issue path
              stage = 0;
              stage_phase ^= 1;
            }
          }
        }
      }
      if constexpr (kPairs) asm volatile("cp.async.wait_all;" ::: "memory");
    }
  } else if (warp >= 4) {
    // ================================ consumers: wgmma + epilogue ================================
    const int g = warp / 4 - 1;                       // consumer warpgroup: user rows [64 g, 64 g + 64) of the block
    const int wt = threadIdx.x % kConsumerThreads;    // thread of the warpgroup
    const int half = wt / kWgRows;                    // epilogue: column half of the tile this thread scans
    const int row = g * kWgRows + wt % kWgRows;       // epilogue: row inside the user block
    float* ls = reinterpret_cast<float*>(smem + L.list_score_off) + half * (kDense ? 0 : p.k) * kBlockM + row;
    int32_t* li = reinterpret_cast<int32_t*>(smem + L.list_item_off) + half * (kDense ? 0 : p.k) * kBlockM + row;
    float* acc_stage = reinterpret_cast<float*>(smem + L.acc_off + g * kAccStageBytes);
    const float kNegInf = -__int_as_float(0x7f800000);
    uint32_t n_stored = 0;   // dense TMA path: chunks stored by this warp (selects the staging buffer)
    const uint32_t stage_base = smem_u32(smem + L.list_score_off) + static_cast<uint32_t>(warp - 4) * 2u * kStoreTileBytes;
    const uint32_t a_base = smem_u32(smem + L.a_off) + g * (kWgRows * 128);   // this warpgroup's 64 rows
    const uint32_t b_base = smem_u32(smem + L.b_off);
    int stage = 0;
    uint32_t stage_phase = 0, witer = 0;
    float acc[64];

    for (int64_t w = blockIdx.x; w < n_work; w += gridDim.x) {
      const WorkItem wi = work_item<kPairs>(w, p, cn);
      const int ub = wi.ub, sp = wi.sp, t0 = wi.t0, t1 = wi.t1;
      if (ub >= live_blocks || (kCount && !count_block_live(cn, ub)))
        continue;   // (an empty split still emits its sentinel candidates)
      // tastes: this warpgroup's users start at u0; the thread of row q < per_wg owns user u0 + q, later rows own none
      const int64_t u0 = is_tastes(kForm) ? static_cast<int64_t>(ub) * 2 * z.per_wg + g * z.per_wg : 0;
      const int64_t u = is_tastes(kForm) ? u0 + wt % kWgRows : static_cast<int64_t>(ub) * kBlockM + row;
      const bool u_ok = u < p.n_users && (!is_tastes(kForm) || wt % kWgRows < z.per_wg);
      const float su = (!is_tastes(kForm) && u_ok) ? __ldg(p.user_scale + u) : 0.0f;
      const float ubias = (!is_tastes(kForm) && u_ok && p.user_bias != nullptr) ? __ldg(p.user_bias + u) : 0.0f;
      float usq = 0.0f;   // kFormEuclid: |u|^2 (rows at or beyond n_users read nothing)
      if constexpr (kForm == kFormEuclid) usq = u_ok ? -2.0f * __ldg(e.user_half_sqnorm + u) : 0.0f;
      float thr = kNegInf;
      // kExclude: this row's list row and the first listed id >= the current chunk.  Rows of a gathered launch beyond
      // *n_users_live have no map entry and are discarded by the caller: they exclude nothing.
      ExclCursor<kExclude> xc;
      if constexpr (kExclude) {
        if ((!kCount || (x.indptr != nullptr && cn.pass >= 0)) && u_ok && t1 > t0 &&
            (p.n_users_live == nullptr || u < __ldg(p.n_users_live))) {
          xc.row = x.row_map != nullptr ? __ldg(x.row_map + u) : static_cast<int32_t>(u);
          xc.next = excl_next_at(x.indptr, x.ids, xc.row, t0 * kBlockN);
        }
      }
      if constexpr (kMode == kModeTopk) {
        for (int j = 0; j < p.k; ++j) {
          ls[j * kBlockM] = kNegInf;
          li[j * kBlockM] = 0x7fffffff;
        }
      }
      // counting mode: this row's targets and this (row, column half)'s buckets in the list region
      const float* cts = reinterpret_cast<const float*>(smem + L.list_score_off) + row;
      const int32_t* cti = reinterpret_cast<const int32_t*>(smem + L.list_score_off + kCountTargets * kBlockM * 4) + row;
      int32_t* ch = reinterpret_cast<int32_t*>(smem + L.list_item_off) + half * kCountTargets * kBlockM + row;
      CountCursor<kCount || kPairs> cc;
      if constexpr (kCount || kPairs) {
        const int32_t lo = u_ok ? __ldg(cn.indptr + u) : 0;
        const int32_t hi = u_ok ? __ldg(cn.indptr + u + 1) : 0;
        if (kPairs || cn.pass < 0) {
          cc.lo = lo;
          cc.hi = hi;
          if (t1 > t0 && hi > lo) cc.next = excl_next_at(cn.indptr, cn.ids, u, t0 * kBlockN);
        } else {
          cc.lo = lo + kCountTargets * cn.pass;
          cc.n = max(0, min(kCountTargets, hi - cc.lo));
          cc.low_s = __int_as_float(0x7f800000);   // no targets: every chunk is skipped
          if (cc.n > 0) {
            cc.low_s = __ldg(cn.score + cc.lo + cc.n - 1);
            cc.low_id = __ldg(cn.ids + cc.lo + cc.n - 1) + p.item_id_offset;
          }
          if (half == 0) {   // (read by both halves after the epilogue's first barrier)
            float* ts = reinterpret_cast<float*>(smem + L.list_score_off) + row;
            int32_t* ti = reinterpret_cast<int32_t*>(smem + L.list_score_off + kCountTargets * kBlockM * 4) + row;
            for (int j = 0; j < kCountTargets; ++j) {
              ts[j * kBlockM] = j < cc.n ? __ldg(cn.score + cc.lo + j) : kNegInf;
              ti[j * kBlockM] = j < cc.n ? __ldg(cn.ids + cc.lo + j) + p.item_id_offset : 0x7fffffff;
            }
          }
          for (int j = 0; j < kCountTargets; ++j) ch[j * kBlockM] = 0;
        }
      }
      WideCursor<kWide> wc;   // wide mode: this thread's list (u, split, column half) in global memory, empty
      if constexpr (kWide) {
        wc.list = u_ok ? (u * p.n_splits + sp) * 2 + half : 0;
        ls = p.cand_score + wc.list * exact_wide_cap(p.k);
        li = p.cand_item + wc.list * exact_wide_cap(p.k);
      }
      if (t1 > t0) {
        mbar_wait(a_full, witer & 1);
        ++witer;
      }

      for (int t = t0; t < t1; ++t) {
        // ---- 64 rows x 128 items: per B k-block hi: A_hi[kb] B + A_lo[kb] B, per B k-block lo: A_hi[kb] B ----
#pragma unroll
        for (int kb2 = 0; kb2 < n_kb2; ++kb2) {
          mbar_wait(b_full + stage, stage_phase);
          if constexpr (kPairs) fence_proxy_async();   // the gathered stage was written through the generic proxy
          const uint64_t db = wgmma_desc_k_major_sw128(b_base + stage * kBTileBytes);
          const bool b_is_hi = kb2 < kNKB;
          const int kb = b_is_hi ? kb2 : kb2 - kNKB;
          wgmma_fence();
#pragma unroll
          for (int a = 0; a < (b_is_hi ? 2 : 1); ++a) {
            const uint64_t da = wgmma_desc_k_major_sw128(a_base + (a == 0 ? kb : kNKB + kb) * kATileBytes);
#pragma unroll
            for (int ks = 0; ks < kKBlock / kMmaK; ++ks)   // 16 fp16 (32 bytes) inside the swizzle atom = +2
              wgmma_m64n128k16_f16(acc, da + 2u * ks, db + 2u * ks, static_cast<uint32_t>(kb2 > 0 || a > 0 || ks > 0));
          }
          wgmma_commit();
          wgmma_wait<0>();
          __syncwarp();
          if (lane == 0) mbar_arrive(b_empty + stage);   // this warp's part of the MMAs no longer reads the stage
          if (++stage == p.n_stages) {
            stage = 0;
            stage_phase ^= 1;
          }
        }
        // ---- epilogue: two rounds, each stages columns [32 c, 32 c + 32) of both 64-column halves ----
        const int32_t id0 = p.item_id_offset + t * kBlockN;
        const float2* meta = p.item_meta + static_cast<int64_t>(t) * kBlockN;
        const float* ihsq = is_euclid(kForm) ? e.item_half_sqnorm + static_cast<int64_t>(t) * kBlockN : nullptr;
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          named_barrier_sync(1 + g, kConsumerThreads);   // the previous round's rows have been read
#pragma unroll
          for (int i = 0; i < 64; ++i) {
            const int nb = i / 4;                          // 8-column block of the accumulator
            if ((nb % 8) / 4 != c) continue;
            const int col = wgmma_acc_col(wt, i);          // 0..127
            acc_stage[((col / 64) * kWgRows + wgmma_acc_row(wt, i)) * kStageStride + col % 32] = acc[i];
          }
          named_barrier_sync(1 + g, kConsumerThreads);
          if constexpr (is_tastes(kForm)) {   // row q of each half now holds user q's final scores
            collapse_chunk<kForm>(acc_stage, wt, c, meta, ihsq, p, e, z, u0);
            named_barrier_sync(1 + g, kConsumerThreads);
          }
          uint32_t r[32];
          const float* src = acc_stage + (half * kWgRows + wt % kWgRows) * kStageStride;
#pragma unroll
          for (int j = 0; j < 32; ++j) r[j] = __float_as_uint(src[j]);
          const int chunk = half * 2 + c;
          if (kDense && p.tma_store) {
            if constexpr (is_tastes(kForm)) {   // users are rows 0 .. per_wg - 1 (<= 32): the first warp of each half
              if (warp % 2 == 0) {
                store_chunk_tma(r, stage_base + (n_stored & 1) * kStoreTileBytes, lane, &map_out,
                                t * kBlockN + chunk * 32, static_cast<int32_t>(u0));
                ++n_stored;
              }
            } else {
              score_chunk_as<kForm>(r, meta + chunk * 32, ihsq + chunk * 32, su, usq, ubias);
              store_chunk_tma(r, stage_base + (n_stored & 1) * kStoreTileBytes, lane, &map_out,
                              t * kBlockN + chunk * 32, ub * kBlockM + g * kWgRows + (warp % 2) * 32);
              ++n_stored;
            }
          } else if constexpr (kWide) {   // every lane: the compactions are warp-cooperative
            wide_chunk<kExclude, kForm>(r, chunk, t, id0, meta, ihsq, su, usq, ubias, thr, ls, li, wc.cnt, p.k, u_ok, x,
                                        xc, lane, wide_hist(smem + L.list_score_off, warp));
          } else if constexpr (kCount || kPairs) {
            if (!is_tastes(kForm) || wt % kWgRows < z.per_wg)
              count_process_chunk<kExclude, kForm, kPairs>(r, chunk, t, id0, meta, ihsq, su, usq, ubias, x, xc, cn, cc,
                                                           cts, cti, ch);
          } else if (!is_tastes(kForm) || wt % kWgRows < z.per_wg) {
            process_chunk<kDense, kExclude, kForm>(r, chunk, t, id0, meta, ihsq, su, usq, ubias, thr, ls, li, p, u,
                                                   u_ok, x, xc);
          }
        }
      }
      __syncwarp();
      if (t1 > t0 && lane == 0) mbar_arrive(a_empty);   // this warp's MMAs of the work item are complete

      if constexpr (kWide) {
        // the end of the item range: every list to at most k entries, and its count
        exact_wide_compact_rows(__ballot_sync(0xffffffffu, wc.cnt > p.k), lane, ls, li, wc.cnt, thr, p.k,
                                wide_hist(smem + L.list_score_off, warp));
        if (u_ok) wl.list_count[wc.list] = wc.cnt;
      } else if constexpr (kCount) {
        if (cn.pass >= 0) {
          // every column of the work item is counted and the staged targets are read: the buckets' prefix sums are
          // the counts of this (row, column half) over the split (integer adds: the total does not depend on order)
          named_barrier_sync(1 + g, kConsumerThreads);
          int32_t acc_count = 0;
          for (int j = 0; j < cc.n; ++j) {
            acc_count += ch[j * kBlockM];
            if (acc_count != 0) atomicAdd(cn.count + cc.lo + j, acc_count);
          }
        }
      } else if constexpr (!kDense && !kPairs) {
        // both halves have finished the item range: merge the two lists of each row and emit the candidates
        named_barrier_sync(1 + g, kConsumerThreads);
        if (half == 0 && u_ok) {
          const float* l0s = ls;
          const int32_t* l0i = li;
          const float* l1s = ls + p.k * kBlockM;
          const int32_t* l1i = li + p.k * kBlockM;
          float* os = p.cand_score + (u * p.n_splits + sp) * p.k;
          int32_t* oi = p.cand_item + (u * p.n_splits + sp) * p.k;
          int a = 0, b = 0;
          for (int j = 0; j < p.k; ++j) {
            const float sa = l0s[a * kBlockM], sb = l1s[b * kBlockM];
            const int32_t ia = l0i[a * kBlockM], ib = l1i[b * kBlockM];
            const bool take_a = sa > sb || (sa == sb && ia <= ib);
            os[j] = take_a ? sa : sb;
            oi[j] = take_a ? ia : ib;
            a += take_a ? 1 : 0;
            b += take_a ? 0 : 1;
          }
        }
        named_barrier_sync(1 + g, kConsumerThreads);   // lists may be re-initialised for the next work item
      }
    }
  }

  // ---- teardown ----
  if (kDense && p.tma_store && warp >= 4 && lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
namespace {

int pick_stages(int n_kblocks, int k, bool dense_staging, bool wide) {
  for (int s = kMaxStages; s >= 2; --s)
    if (make_layout(n_kblocks, s, k, dense_staging, wide).total + kSmemAlignSlack <= kSmemLimit) return s;
  return 0;
}

}  // namespace

int score_topk_max_k(int32_t d_pad) {
  if (d_pad != 64 && d_pad != 128) return 0;
  return kMaxK;
}

int score_topk_wide_list_capacity(int32_t k) { return k >= 1 && k <= kExactWideMaxK ? exact_wide_cap(k) : 0; }

// Item splits of a dense launch over n_ub user blocks: enough that every SM gets work when there are few user blocks.
static int32_t dense_splits(int64_t n_ub, int64_t n_items) {
  const int64_t n_tiles = ceil_div(n_items, kBlockN);
  int64_t splits = ceil_div(2 * static_cast<int64_t>(sm_count()), n_ub);
  if (splits > n_tiles) splits = n_tiles;
  if (splits < 1) splits = 1;
  return static_cast<int32_t>(splits);
}

// (the kernels of one instantiation, for score_tc: fn[d_pad / 64 - 1])
using TcKernelFn = void (*)(CUtensorMap, CUtensorMap, CUtensorMap, TcParams, TcExcl, TcEuclid, TcTastes, TcWide,
                            TcCount);
template <TcMode kMode, bool kExclude, ScoreForm kForm>
struct TcKernel {
  static constexpr TcKernelFn fn[2] = {score_tc_kernel<kMode, 1, kExclude, kForm>,
                                       score_tc_kernel<kMode, 2, kExclude, kForm>};
};

int score_tc(const ScoreTcArgs& a, cudaStream_t stream) {
  TRK_CHECK_ARG(a.user_split && a.user_scale && a.item_split && a.item_meta, "score_tc: null operand");
  TRK_CHECK_ARG((a.user_half_sqnorm == nullptr) == (a.item_half_sqnorm == nullptr),
                "score_tc: user_half_sqnorm and item_half_sqnorm go together");
  TRK_CHECK_ARG(reinterpret_cast<uintptr_t>(a.item_half_sqnorm) % 16 == 0,
                "score_tc: item_half_sqnorm must be 16-byte aligned");
  const bool euclid = a.user_half_sqnorm != nullptr;
  TRK_CHECK_ARG(a.n_users >= 1 && a.n_items >= 1, "score_tc: empty shape");
  TRK_CHECK_ARG(a.n_users < (1ll << 31) && a.n_items < (1ll << 31) - 512, "score_tc: shape exceeds int32 indexing");
  if (a.d_pad != 64 && a.d_pad != 128) {
    set_error("score_tc: d_pad=%d not supported by the tensor-core kernel (64 or 128)", a.d_pad);
    return TRK_ERR_UNSUPPORTED;
  }
  TRK_CHECK_ARG(reinterpret_cast<uintptr_t>(a.user_split) % 16 == 0 &&
                    reinterpret_cast<uintptr_t>(a.item_split) % 16 == 0 &&
                    reinterpret_cast<uintptr_t>(a.item_meta) % 16 == 0,
                "score_tc: operands must be 16-byte aligned");
  if (a.pairs) {
    TRK_CHECK_ARG(a.pair_indptr && a.pair_ids && a.pair_score && a.tile_items && a.work, "score_pairs: null pair plan");
    TRK_CHECK_ARG(a.n_tiles >= 1 && a.n_work >= 1, "score_pairs: n_tiles=%d and n_work=%d must be positive", a.n_tiles,
                  a.n_work);
    TRK_CHECK_ARG(a.n_tiles <= (1 << 24), "score_pairs: n_tiles=%d exceeds int32 virtual columns", a.n_tiles);
  } else if (a.count) {
    TRK_CHECK_ARG(a.pair_indptr && a.pair_ids && a.pair_score && a.block_pairs, "score_count: null pair list");
    TRK_CHECK_ARG(a.pass >= -1, "score_count: pass=%d < -1", a.pass);
    TRK_CHECK_ARG(a.pass < 0 || a.pair_count, "score_count: null pair_count");
    TRK_CHECK_ARG(a.n_users_live == nullptr, "score_count: no live-row count");
    TRK_CHECK_ARG(a.n_splits >= 1, "score_tc: n_splits < 1");
  } else if (!a.dense) {
    TRK_CHECK_ARG(a.cand_score && a.cand_item && (!a.wide || a.list_count), "score_topk: null output");
    const int max_k = a.wide ? kExactWideMaxK : kMaxK;
    if (a.k < 1 || a.k > max_k) {
      set_error("score_topk: k=%d outside [1, %d]", a.k, max_k);
      return TRK_ERR_UNSUPPORTED;
    }
    TRK_CHECK_ARG(a.n_splits >= 1, "score_tc: n_splits < 1");
  } else {
    TRK_CHECK_ARG(a.dense_out && a.dense_stride >= a.n_items, "score_dense: bad output");
  }
  TRK_CHECK_ARG((a.excl_indptr == nullptr) == (a.excl_ids == nullptr) &&
                    (a.excl_indptr != nullptr || a.excl_row_map == nullptr),
                "score_topk: excl_indptr and excl_ids go together (excl_row_map needs both)");
  // n_tastes != 0: a mixture of tastes on the stacked operand [n_ops, n_users, 2 d_pad] (TcTastes)
  const bool tastes = a.n_tastes != 0;
  TcTastes z = {0, 0, 0};
  if (tastes) {
    // (one operand row per user is the plain kernel: per_wg would exceed the 32 rows of a dense store tile)
    TRK_CHECK_ARG(a.n_tastes >= 2 || (a.n_tastes == 1 && a.attention),
                  "score_tastes: n_tastes=%d needs n_tastes >= 2 or attention", a.n_tastes);
    TRK_CHECK_ARG(a.n_users_live == nullptr, "score_tastes: no live-row count");
    const int n_ops = a.n_tastes <= 64 ? (a.attention ? 2 : 1) * a.n_tastes : 65;
    if (n_ops > kWgRows) {
      set_error("score_tastes: %d operand rows per user (n_tastes=%d%s) exceed %d", n_ops, a.n_tastes,
                a.attention ? ", attention" : "", kWgRows);
      return TRK_ERR_UNSUPPORTED;
    }
    z = {n_ops, a.n_tastes, kWgRows / n_ops};
  }
  const ScoreForm form = tastes ? (euclid ? (a.attention ? kFormTastesEuclidAttention : kFormTastesEuclidMax)
                                          : (a.attention ? kFormTastesAttention : kFormTastesMax))
                                : (euclid ? kFormEuclid : kFormDot);
  // every instantiation:
  //   [dense | top-k | top-k with exclusion | wide | wide with exclusion | count | pairs][form][d_pad / 64 - 1]
  // (the wide mode exists for the forms without a wide filter: Euclidean similarity and attention; a Euclidean mixture
  // of tastes without attention ranks its top k per taste, so its max form has no top-k or wide instantiation; the
  // counting mode takes its exclusion lists at run time; the pairs mode excludes nothing, as dense scores do not)
  static constexpr const TcKernelFn* kKernels[7][6] = {
      {TcKernel<kModeDense, false, kFormDot>::fn, TcKernel<kModeDense, false, kFormEuclid>::fn,
       TcKernel<kModeDense, false, kFormTastesMax>::fn, TcKernel<kModeDense, false, kFormTastesAttention>::fn,
       TcKernel<kModeDense, false, kFormTastesEuclidMax>::fn,
       TcKernel<kModeDense, false, kFormTastesEuclidAttention>::fn},
      {TcKernel<kModeTopk, false, kFormDot>::fn, TcKernel<kModeTopk, false, kFormEuclid>::fn,
       TcKernel<kModeTopk, false, kFormTastesMax>::fn, TcKernel<kModeTopk, false, kFormTastesAttention>::fn, nullptr,
       TcKernel<kModeTopk, false, kFormTastesEuclidAttention>::fn},
      {TcKernel<kModeTopk, true, kFormDot>::fn, TcKernel<kModeTopk, true, kFormEuclid>::fn,
       TcKernel<kModeTopk, true, kFormTastesMax>::fn, TcKernel<kModeTopk, true, kFormTastesAttention>::fn, nullptr,
       TcKernel<kModeTopk, true, kFormTastesEuclidAttention>::fn},
      {nullptr, TcKernel<kModeWide, false, kFormEuclid>::fn, nullptr, TcKernel<kModeWide, false, kFormTastesAttention>::fn,
       nullptr, TcKernel<kModeWide, false, kFormTastesEuclidAttention>::fn},
      {nullptr, TcKernel<kModeWide, true, kFormEuclid>::fn, nullptr, TcKernel<kModeWide, true, kFormTastesAttention>::fn,
       nullptr, TcKernel<kModeWide, true, kFormTastesEuclidAttention>::fn},
      {TcKernel<kModeCount, true, kFormDot>::fn, TcKernel<kModeCount, true, kFormEuclid>::fn,
       TcKernel<kModeCount, true, kFormTastesMax>::fn, TcKernel<kModeCount, true, kFormTastesAttention>::fn,
       TcKernel<kModeCount, true, kFormTastesEuclidMax>::fn,
       TcKernel<kModeCount, true, kFormTastesEuclidAttention>::fn},
      {TcKernel<kModePairs, false, kFormDot>::fn, TcKernel<kModePairs, false, kFormEuclid>::fn,
       TcKernel<kModePairs, false, kFormTastesMax>::fn, TcKernel<kModePairs, false, kFormTastesAttention>::fn,
       TcKernel<kModePairs, false, kFormTastesEuclidMax>::fn,
       TcKernel<kModePairs, false, kFormTastesEuclidAttention>::fn}};
  const int mode_row = a.pairs ? 6 : a.count ? 5 : a.dense ? 0 : (a.wide ? 3 : 1) + (a.excl_indptr != nullptr ? 1 : 0);
  if (kKernels[mode_row][form] == nullptr) {
    if (form == kFormTastesEuclidMax)
      set_error("score_topk: a Euclidean mixture of tastes without attention has no one-sweep top-k: rank each taste "
                "on trk_score_topk%s_euclid_f16x3 and merge the lists", a.wide ? "_wide" : "");
    else
      set_error("score_topk_wide: the wide mode serves the Euclidean and attention forms only");
    return TRK_ERR_UNSUPPORTED;
  }

  TcParams p;
  p.user_scale = a.user_scale;
  p.user_bias = a.user_bias;
  p.item_meta = reinterpret_cast<const float2*>(a.item_meta);
  p.n_users = a.n_users;
  p.n_items = a.n_items;
  p.n_kblocks = a.d_pad / kKBlock;
  p.k = a.dense ? 0 : a.k;
  p.n_tiles = static_cast<int32_t>(ceil_div(a.n_items, kBlockN));
  p.n_user_blocks = static_cast<int32_t>(ceil_div(a.n_users, tastes ? 2 * z.per_wg : kBlockM));
  p.n_splits = a.dense ? dense_splits(p.n_user_blocks, a.n_items) : a.pairs ? 1 : a.n_splits;
  p.tiles_per_split = static_cast<int32_t>(ceil_div(p.n_tiles, p.n_splits));
  p.item_id_offset = a.item_id_offset;
  p.cand_score = a.cand_score;
  p.cand_item = a.cand_item;
  p.dense_out = a.dense_out;
  p.dense_stride = a.dense_stride;
  p.n_users_live = a.n_users_live;
  const TcExcl x = {a.excl_indptr, a.excl_ids, a.excl_row_map};
  const TcEuclid e = {a.user_half_sqnorm, a.item_half_sqnorm};
  p.tma_store = (a.dense && a.dense_stride % 4 == 0 && reinterpret_cast<uintptr_t>(a.dense_out) % 16 == 0) ? 1 : 0;
  // k of the shared-memory lists (the wide mode keeps its lists in global memory; the counting mode stages its targets
  // and buckets in the region of kMaxK)
  const int list_k = a.wide ? 0 : a.count ? kMaxK : p.k;
  p.n_stages = pick_stages(p.n_kblocks, list_k, p.tma_store != 0, a.wide);
  TRK_CHECK_ARG(p.n_stages >= 2, "score_tc: shared memory budget exceeded (d_pad=%d k=%d)", a.d_pad, p.k);

  // operands: [rows, 2 d_pad] fp16 (hi | lo), boxes of one k-block x one tile
  // (tastes: the stacked operand, boxes of one k-block x per_wg users x n_ops operands = one warpgroup's rows)
  CUtensorMap map_users, map_items;
  int rc = tastes ? encode_tiled_3d(&map_users, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, a.user_split, 2 * a.d_pad, a.n_users,
                                    z.n_ops, 4 * a.d_pad, 4 * a.d_pad * a.n_users, kKBlock, z.per_wg, z.n_ops,
                                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B)
                  : encode_tiled_2d(&map_users, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, a.user_split, 2 * a.d_pad, a.n_users,
                                    4 * a.d_pad, kKBlock, kBlockM, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (rc != TRK_OK) return rc;
  rc = encode_tiled_2d(&map_items, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, a.item_split, 2 * a.d_pad, a.n_items, 4 * a.d_pad,
                       kKBlock, kBlockN, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (rc != TRK_OK) return rc;

  CUtensorMap map_out = map_items;   // placeholder when the TMA store path is off
  if (p.tma_store) {
    rc = encode_tiled_2d(&map_out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, a.dense_out, a.n_items, a.n_users,
                         4 * a.dense_stride, 32, tastes ? z.per_wg : 32, CU_TENSOR_MAP_L2_PROMOTION_NONE);
    if (rc != TRK_OK) return rc;
  }
  const uint32_t smem_bytes =
      make_layout(p.n_kblocks, p.n_stages, list_k, p.tma_store != 0, a.wide).total + kSmemAlignSlack;
  const TcKernelFn kernel = kKernels[mode_row][form][p.n_kblocks - 1];
  TRK_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
  const int grid = capped_grid(a.pairs ? a.n_work : static_cast<int64_t>(p.n_user_blocks) * p.n_splits, 1);
  const TcWide wl = {a.list_count};
  const TcCount cn = {a.pair_indptr, a.pair_ids, a.pair_score, a.pair_count, a.block_pairs, a.pairs ? -1 : a.pass,
                      a.n_work, a.tile_items, a.work, static_cast<const uint8_t*>(a.item_split)};
  kernel<<<grid, kTcThreads, smem_bytes, stream>>>(map_users, map_items, map_out, p, x, e, z, wl, cn);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

}  // namespace trk
