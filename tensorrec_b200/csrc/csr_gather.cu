// K1 -- sparse features x dense weights -> dense representation (CSR gather-reduce), HBM-bound.
//
// Reference semantics: tf.sparse_tensor_dense_matmul in LinearRepresentationGraph
// (tensorrec/representation_graphs.py:40), tf.nn.l2_normalize of NormalizedLinearRepresentationGraph (:57) and of
// relative_cosine (tensorrec/recommendation_graphs.py:119-120), project_biases (recommendation_graphs.py:13-17).
//
// Layout / mapping
//   * a block walks tiles of kTileRows consecutive rows (grid-stride, grid = SMs x resident blocks);
//   * the tile's indptr slice and ALL its (col, val) pairs are staged into shared memory with coalesced loads
//     (the nonzeros of consecutive rows are contiguous in CSR), so the index stream is read from HBM exactly once
//     and never through scattered 4-entry requests;
//   * a group of G lanes owns one row and every lane keeps CH float4 accumulators (d = 128: G = 8, CH = 4, so a warp
//     works on four rows at once); kBatch x CH 16-byte gathers are in flight per lane, 32 warps per SM.  The launch
//     bound (4 resident blocks) matters: without it ptxas budgets 32 registers, sinks every gather next to its FMAs and
//     the kernel runs one memory latency per nonzero -- it then reacts to neither byte count nor L2 hints;
//   * outputs are written with streaming stores (single use);
//   * accumulation is fp32 FMA in CSR storage order -> bit-identical from run to run, duplicates are summed;
//   * the epilogue (row still in registers) optionally L2-normalises, writes fp32 and/or the split-fp16 operand
//     (hi | lo, per-row power-of-two scale) that the tensor-core score kernel consumes.

#include "common.cuh"

namespace trk {

constexpr int kGatherThreads = 256;
constexpr int kTileRows = 64;
constexpr int kNnzCap = 3072;  // staged (col,val) pairs per tile: 24 KB

// Weight-row gathers are issued through `asm volatile` and their results pinned by empty volatile asm statements: with
// plain __ldg the compiler sinks every load next to its FMAs to save registers (32 registers, one gather in flight per
// lane: four serialised memory latencies per 4-entry row -- the kernel then ignores both byte count and L2 hints).
// This keeps the loads of a batch together, ahead of the first FMA.
__device__ __forceinline__ float4 ldg_f4_nc(const float* ptr) {
  float4 v;
  asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(ptr));
  return v;
}
__device__ __forceinline__ float ldg_f1_nc(const float* ptr) {
  float v;
  asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(v) : "l"(ptr));
  return v;
}

template <int G>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o, G);
  return v;
}
template <int G>
__device__ __forceinline__ float group_max(float v) {
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o, G));
  return v;
}

// Power-of-two scaling of one row for the split-fp16 operand: returns `up` = 2^s with max|x|*up in [2^14, 2^15)
// (fp16 max is 65504), and *inv = 2^-s.  Zero / non-finite rows use 1.
__device__ __forceinline__ float row_scale_pow2(float max_abs, float* inv) {
  int s = 0;
  if (max_abs > 0.0f && max_abs < __int_as_float(0x7f800000)) {
    const int e = static_cast<int>((__float_as_uint(max_abs) >> 23) & 0xffu) - 127;  // floor(log2) for normals
    s = 14 - e;
    s = s > 126 ? 126 : s;
  }
  *inv = __uint_as_float(static_cast<uint32_t>(127 - s) << 23);
  return __uint_as_float(static_cast<uint32_t>(127 + s) << 23);
}

__device__ __forceinline__ void split_f16(float x, float up, __half* hi, __half* lo) {
  const float xs = x * up;
  const __half h = __float2half_rn(xs);
  *hi = h;
  *lo = __float2half_rn(xs - __half2float(h));
}

// Row epilogue shared by the gather kernel and the dense->split converter.
// VEC: every lane owns CH float4 chunks, chunk index = lane + G*j ; scalar: CH floats, element = lane + G*j.
// Running maxima a thread carries over all the rows it finishes (reduced once per warp at the end of the kernel: one
// atomic per row would serialise a million updates of one address in L2).
struct RowStats {
  float max_norm = 0.0f;    // largest row norm (upper bound, see below)
  float max_scale = 0.0f;   // largest 2^-e among the non-zero rows == the scale of the row with the largest element
};

template <int G, int CH, bool VEC>
__device__ __forceinline__ void row_epilogue(float (&acc)[CH][VEC ? 4 : 1], int lane, int64_t row, bool active,
                                             int d, int n_normalize, float* __restrict__ out_f32,
                                             __half* __restrict__ out_split, int d_pad,
                                             float* __restrict__ out_scale, float* __restrict__ out_norm = nullptr,
                                             RowStats* st = nullptr) {
  constexpr int W = VEC ? 4 : 1;
  for (int n = 0; n < n_normalize; ++n) {
    float ss = 0.0f;
#pragma unroll
    for (int j = 0; j < CH; ++j)
#pragma unroll
      for (int w = 0; w < W; ++w) ss = fmaf(acc[j][w], acc[j][w], ss);
    ss = group_sum<G>(ss);
    const float inv_norm = 1.0f / sqrtf(fmaxf(ss, 1e-12f));  // tf.nn.l2_normalize: x * rsqrt(max(sum x^2, eps))
#pragma unroll
    for (int j = 0; j < CH; ++j)
#pragma unroll
      for (int w = 0; w < W; ++w) acc[j][w] *= inv_norm;
  }
  // (the shuffles above are executed by every lane of the warp; only stores are predicated on `active`)
  float row_ss = 0.0f;
  if (out_norm != nullptr || st != nullptr) {
    // |row|_2 as an UPPER bound (the filter's error bound is proportional to it): inflated by 2^-9, which covers the
    // rounding of this reduction and of the 22-bit split operand
#pragma unroll
    for (int j = 0; j < CH; ++j)
#pragma unroll
      for (int w = 0; w < W; ++w) row_ss = fmaf(acc[j][w], acc[j][w], row_ss);
    row_ss = group_sum<G>(row_ss);
    const float norm = sqrtf(row_ss) * 1.002f;
    if (active && lane == 0) {
      if (out_norm != nullptr) out_norm[row] = norm;
      if (st != nullptr) st->max_norm = fmaxf(st->max_norm, norm);
    }
  }
  if (out_f32 != nullptr && active) {
#pragma unroll
    for (int j = 0; j < CH; ++j) {
      const int e0 = (lane + G * j) * W;
      if (e0 < d) {
        if constexpr (VEC) {
          __stcs(reinterpret_cast<float4*>(out_f32 + row * d + e0), make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]));
        } else {
          __stcs(out_f32 + row * d + e0, acc[j][0]);
        }
      }
    }
  }
  if (out_split != nullptr) {
    float m = 0.0f;
#pragma unroll
    for (int j = 0; j < CH; ++j)
#pragma unroll
      for (int w = 0; w < W; ++w) m = fmaxf(m, fabsf(acc[j][w]));
    m = group_max<G>(m);
    float inv;
    const float up = row_scale_pow2(m, &inv);
    if (!active) return;
    if (lane == 0) {
      out_scale[row] = inv;
      if (st != nullptr && m > 0.0f) st->max_scale = fmaxf(st->max_scale, inv);   // all-zero rows carry the neutral 1
    }
    __half* hi_row = out_split + row * (2 * static_cast<int64_t>(d_pad));
    __half* lo_row = hi_row + d_pad;
#pragma unroll
    for (int j = 0; j < CH; ++j) {
      const int e0 = (lane + G * j) * W;
      if (e0 < d_pad) {  // accumulators beyond d are zero: this writes the zero padding too
        if constexpr (VEC) {
          __half h[4], l[4];
#pragma unroll
          for (int w = 0; w < 4; ++w) split_f16(acc[j][w], up, &h[w], &l[w]);
          __stcs(reinterpret_cast<uint2*>(hi_row + e0), *reinterpret_cast<uint2*>(h));   // streaming: written once
          __stcs(reinterpret_cast<uint2*>(lo_row + e0), *reinterpret_cast<uint2*>(l));
        } else {
          __half h, l;
          split_f16(acc[j][0], up, &h, &l);
          hi_row[e0] = h;
          lo_row[e0] = l;
        }
      }
    }
  }
}

template <int G, int CH, bool VEC>
__global__ void __launch_bounds__(kGatherThreads, 4)
csr_gather_reduce_kernel(const int32_t* __restrict__ indptr, const int32_t* __restrict__ col,
                         const float* __restrict__ val, const float* __restrict__ weights, int64_t rows, int d,
                         int n_normalize, float* __restrict__ out_f32, __half* __restrict__ out_split, int d_pad,
                         float* __restrict__ out_scale, float* __restrict__ out_norm, float* __restrict__ stats) {
  constexpr int W = VEC ? 4 : 1;
  constexpr int kGroups = kGatherThreads / G;
  __shared__ int32_t s_ptr[kTileRows + 1];
  __shared__ int32_t s_col[kNnzCap];
  __shared__ float s_val[kNnzCap];

  const int tid = threadIdx.x;
  const int group = tid / G;
  const int lane = tid % G;
  const int64_t n_tiles = ceil_div(rows, kTileRows);
  RowStats st;

  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t r0 = tile * kTileRows;
    const int nr = static_cast<int>(min(static_cast<int64_t>(kTileRows), rows - r0));
    if (tid <= nr) s_ptr[tid] = indptr[r0 + tid];
    __syncthreads();
    const int p0 = s_ptr[0];
    const int n_tile = s_ptr[nr] - p0;
    const bool staged = n_tile <= kNnzCap;
    if (staged) {
      for (int i = tid; i < n_tile; i += kGatherThreads) {
        s_col[i] = __ldg(col + p0 + i);
        s_val[i] = __ldg(val + p0 + i);
      }
    }
    __syncthreads();

    // warp-uniform trip count: the epilogue uses full-mask shuffles, so every lane must reach it
    for (int rr_base = 0; rr_base < nr; rr_base += kGroups) {
      const int rr = rr_base + group;
      const bool active = rr < nr;
      const int a = active ? s_ptr[rr] : 0, b = active ? s_ptr[rr + 1] : 0;
      float acc[CH][W];
#pragma unroll
      for (int j = 0; j < CH; ++j)
#pragma unroll
        for (int w = 0; w < W; ++w) acc[j][w] = 0.0f;

      // batches of kBatch entries: all gathers of a batch are issued before the first FMA, also for rows with fewer
      // entries left (a scalar tail would serialise one memory latency per entry); FMAs retire in storage order.
      // kBatch x CH loads of 16 bytes are in flight per lane.
      constexpr int kBatch = (CH * W >= 16) ? 2 : 4;
      for (int p = a; p < b; p += kBatch) {
        const int n = min(kBatch, b - p);
        int c[kBatch];
        float v[kBatch];
#pragma unroll
        for (int q = 0; q < kBatch; ++q) {
          const int pq = p + (q < n ? q : 0);
          c[q] = staged ? s_col[pq - p0] : __ldg(col + pq);
          v[q] = staged ? s_val[pq - p0] : __ldg(val + pq);
        }
        float wv[kBatch][CH][W];
#pragma unroll
        for (int q = 0; q < kBatch; ++q) {
          // entries past the end of the row re-read entry 0 (c[q] is clamped above) and are skipped by the FMAs;
          // chunks past d (padding lanes of the split operand) re-read chunk 0 and are zeroed
          const float* wrow = weights + static_cast<int64_t>(c[q]) * d;
#pragma unroll
          for (int j = 0; j < CH; ++j) {
            const int e0 = (lane + G * j) * W;
            const bool in_row = e0 < d;
            if constexpr (VEC) {
              const float4 t = ldg_f4_nc(wrow + (in_row ? e0 : 0));
              wv[q][j][0] = in_row ? t.x : 0.0f;
              wv[q][j][1] = in_row ? t.y : 0.0f;
              wv[q][j][2] = in_row ? t.z : 0.0f;
              wv[q][j][3] = in_row ? t.w : 0.0f;
            } else {
              const float t = ldg_f1_nc(wrow + (in_row ? e0 : 0));
              wv[q][j][0] = in_row ? t : 0.0f;
            }
          }
        }
        // pin: every loaded value passes through an (empty) volatile asm that is ordered after ALL the loads above,
        // so no FMA can be scheduled in between two gathers
#pragma unroll
        for (int q = 0; q < kBatch; ++q)
#pragma unroll
          for (int j = 0; j < CH; ++j)
#pragma unroll
            for (int w = 0; w < W; ++w) asm volatile("" : "+f"(wv[q][j][w]));
#pragma unroll
        for (int q = 0; q < kBatch; ++q)
          if (q < n) {
#pragma unroll
            for (int j = 0; j < CH; ++j)
#pragma unroll
              for (int w = 0; w < W; ++w) acc[j][w] = fmaf(v[q], wv[q][j][w], acc[j][w]);
          }
      }
      row_epilogue<G, CH, VEC>(acc, lane, r0 + rr, active, d, n_normalize, out_f32, out_split, d_pad, out_scale,
                               out_norm, stats != nullptr ? &st : nullptr);
    }
    __syncthreads();  // the next tile overwrites the staging buffers
  }
  if (stats != nullptr) {
    // non-negative floats order like their bit patterns: atomicMax on the bits is order independent -> deterministic
    float mn = st.max_norm, ms = st.max_scale;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn = fmaxf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
      ms = fmaxf(ms, __shfl_xor_sync(0xffffffffu, ms, o));
    }
    if (tid % 32 == 0) {
      atomicMax(reinterpret_cast<int*>(stats + 0), __float_as_int(mn));
      atomicMax(reinterpret_cast<int*>(stats + 1), __float_as_int(ms));
    }
  }
}

// dense fp32 rows -> (optionally normalised) split-fp16 operand; one group per row
template <int G, int CH, bool VEC>
__global__ void __launch_bounds__(kGatherThreads)
split_rows_kernel(const float* __restrict__ repr, int64_t rows, int d, int n_normalize,
                  float* __restrict__ out_f32_inplace, __half* __restrict__ out_split, int d_pad,
                  float* __restrict__ out_scale) {
  constexpr int W = VEC ? 4 : 1;
  constexpr int kGroups = kGatherThreads / G;
  const int group = threadIdx.x / G, lane = threadIdx.x % G;
  for (int64_t row_base = static_cast<int64_t>(blockIdx.x) * kGroups; row_base < rows;
       row_base += static_cast<int64_t>(gridDim.x) * kGroups) {
    const int64_t row = row_base + group;
    const bool active = row < rows;
    float acc[CH][W];
#pragma unroll
    for (int j = 0; j < CH; ++j) {
      const int e0 = (lane + G * j) * W;
      if (active && e0 < d) {
        if constexpr (VEC) {
          const float4 t = *reinterpret_cast<const float4*>(repr + row * d + e0);
          acc[j][0] = t.x; acc[j][1] = t.y; acc[j][2] = t.z; acc[j][3] = t.w;
        } else {
          acc[j][0] = repr[row * d + e0];
        }
      } else {
#pragma unroll
        for (int w = 0; w < W; ++w) acc[j][w] = 0.0f;
      }
    }
    row_epilogue<G, CH, VEC>(acc, lane, row, active, d, n_normalize, out_f32_inplace, out_split, d_pad, out_scale);
  }
}

// project_biases: one thread per row, entries staged per tile of 256 rows; sequential fp32 FMA in CSR order.
constexpr int kBiasTileRows = 256;
__global__ void __launch_bounds__(kBiasTileRows)
csr_project_biases_kernel(const int32_t* __restrict__ indptr, const int32_t* __restrict__ col,
                          const float* __restrict__ val, const float* __restrict__ biases, int64_t rows,
                          float* __restrict__ out) {
  __shared__ int32_t s_ptr[kBiasTileRows + 1];
  __shared__ int32_t s_col[kNnzCap];
  __shared__ float s_val[kNnzCap];
  const int tid = threadIdx.x;
  const int64_t n_tiles = ceil_div(rows, kBiasTileRows);
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t r0 = tile * kBiasTileRows;
    const int nr = static_cast<int>(min(static_cast<int64_t>(kBiasTileRows), rows - r0));
    for (int i = tid; i <= nr; i += kBiasTileRows) s_ptr[i] = indptr[r0 + i];
    __syncthreads();
    const int p0 = s_ptr[0];
    const int n_tile = s_ptr[nr] - p0;
    const bool staged = n_tile <= kNnzCap;
    if (staged) {
      for (int i = tid; i < n_tile; i += kBiasTileRows) {
        s_col[i] = __ldg(col + p0 + i);
        s_val[i] = __ldg(val + p0 + i);
      }
    }
    __syncthreads();
    if (tid < nr) {
      float acc = 0.0f;
      for (int p = s_ptr[tid]; p < s_ptr[tid + 1]; ++p) {
        const int c = staged ? s_col[p - p0] : __ldg(col + p);
        const float v = staged ? s_val[p - p0] : __ldg(val + p);
        acc = fmaf(v, __ldg(biases + c), acc);
      }
      out[r0 + tid] = acc;
    }
    __syncthreads();
  }
}

__global__ void pack_item_meta_kernel(const float* __restrict__ scale, const float* __restrict__ bias, int64_t n,
                                      float2* __restrict__ meta, int64_t n_padded) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n_padded) return;
  float2 m;
  if (i < n) {
    m.x = scale != nullptr ? scale[i] : 1.0f;
    m.y = bias != nullptr ? bias[i] : 0.0f;
  } else {
    m.x = 0.0f;
    m.y = -__int_as_float(0x7f800000);  // -inf: a padded column can never enter a top-k list
  }
  meta[i] = m;
}

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
namespace {

struct RowShape {
  bool vec;
  int g;
  int ch;
};

// units the row group must cover: d (and d_pad when the split operand is written)
bool pick_shape(int d, int d_pad, bool want_split, bool aligned16, RowShape* s) {
  const int cover = want_split ? (d_pad > d ? d_pad : d) : d;
  if (d % 4 == 0 && aligned16) {
    const int units = cover / 4;
    s->vec = true;
    // narrow groups, several 16-byte chunks per lane: a warp then works on 4 (or 2) rows at once, which amortises the
    // per-row control instructions and puts kBatch x CH gathers in flight per lane (scripts/k1_probe.py times the
    // variants)
    if (units <= 8) { s->g = 8; s->ch = 1; }
    else if (units <= 16) { s->g = 8; s->ch = 2; }
    else if (units <= 32) { s->g = 8; s->ch = 4; }
    else if (units <= 64) { s->g = 16; s->ch = 4; }
    else if (units <= 128) { s->g = 32; s->ch = 4; }
    else return false;
    return true;
  }
  s->vec = false;
  s->g = 32;
  if (cover <= 32) s->ch = 1;
  else if (cover <= 64) s->ch = 2;
  else if (cover <= 128) s->ch = 4;
  else if (cover <= 256) s->ch = 8;
  else return false;
  return true;
}

#define TRK_DISPATCH_ROWSHAPE(S, CALL)                          \
  do {                                                          \
    if ((S).vec) {                                              \
      if ((S).g == 8 && (S).ch == 1) { CALL(8, 1, true); }      \
      else if ((S).g == 8 && (S).ch == 2) { CALL(8, 2, true); } \
      else if ((S).g == 8) { CALL(8, 4, true); }                \
      else if ((S).g == 16) { CALL(16, 4, true); }              \
      else { CALL(32, 4, true); }                               \
    } else {                                                    \
      if ((S).ch == 1) { CALL(32, 1, false); }                  \
      else if ((S).ch == 2) { CALL(32, 2, false); }             \
      else if ((S).ch == 4) { CALL(32, 4, false); }             \
      else { CALL(32, 8, false); }                              \
    }                                                           \
  } while (0)

}  // namespace

int csr_gather_reduce(const int32_t* indptr, const int32_t* col, const float* val, const float* weights,
                      int64_t rows, int32_t n_features, int32_t d, int32_t n_normalize, float* out_f32,
                      void* out_split, int32_t d_pad, float* out_scale, float* out_norm, float* stats,
                      cudaStream_t stream) {
  TRK_CHECK_ARG(indptr && weights, "csr_gather_reduce: null indptr/weights");
  TRK_CHECK_ARG(rows >= 0 && d >= 1 && n_features >= 0, "csr_gather_reduce: bad sizes rows=%lld d=%d",
                static_cast<long long>(rows), d);
  TRK_CHECK_ARG(out_f32 || out_split, "csr_gather_reduce: no output buffer");
  TRK_CHECK_ARG(n_normalize >= 0 && n_normalize <= 4, "csr_gather_reduce: n_normalize=%d", n_normalize);
  if (out_split) {
    TRK_CHECK_ARG(out_scale, "csr_gather_reduce: out_split needs out_scale");
    TRK_CHECK_ARG(d_pad >= d && d_pad % 64 == 0, "csr_gather_reduce: d_pad=%d must be a multiple of 64 >= d=%d",
                  d_pad, d);
  }
  if (stats != nullptr) TRK_CHECK_CUDA(cudaMemsetAsync(stats, 0, 3 * sizeof(float), stream));
  if (rows == 0) return TRK_OK;
  const bool aligned = (reinterpret_cast<uintptr_t>(weights) % 16 == 0) &&
                       (out_f32 == nullptr || reinterpret_cast<uintptr_t>(out_f32) % 16 == 0) &&
                       (out_split == nullptr || reinterpret_cast<uintptr_t>(out_split) % 16 == 0);
  RowShape s;
  if (!pick_shape(d, d_pad, out_split != nullptr, aligned, &s)) {
    set_error("csr_gather_reduce: n_components=%d (d_pad=%d) exceeds the fused row width", d, d_pad);
    return TRK_ERR_UNSUPPORTED;
  }
  const int grid = capped_grid(ceil_div(rows, kTileRows), 8);   // 8 x 256 threads resident per SM
#define CALL(G, CH, VEC)                                                                                     \
  csr_gather_reduce_kernel<G, CH, VEC><<<grid, kGatherThreads, 0, stream>>>(                                 \
      indptr, col, val, weights, rows, d, n_normalize, out_f32, static_cast<__half*>(out_split), d_pad, out_scale, \
      out_norm, stats)
  TRK_DISPATCH_ROWSHAPE(s, CALL);
#undef CALL
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

int split_rows(const float* repr, int64_t rows, int32_t d, int32_t n_normalize, float* normalized_inplace,
               void* out_split, int32_t d_pad, float* out_scale, cudaStream_t stream) {
  TRK_CHECK_ARG(repr, "split_rows: null input");
  TRK_CHECK_ARG(rows >= 0 && d >= 1, "split_rows: bad sizes");
  if (out_split) {
    TRK_CHECK_ARG(out_scale, "split_rows: out_split needs out_scale");
    TRK_CHECK_ARG(d_pad >= d && d_pad % 64 == 0, "split_rows: d_pad=%d must be a multiple of 64 >= d=%d", d_pad, d);
  }
  if (rows == 0) return TRK_OK;
  const bool aligned = (reinterpret_cast<uintptr_t>(repr) % 16 == 0) &&
                       (out_split == nullptr || reinterpret_cast<uintptr_t>(out_split) % 16 == 0);
  RowShape s;
  if (!pick_shape(d, d_pad, out_split != nullptr, aligned, &s)) {
    set_error("split_rows: n_components=%d (d_pad=%d) exceeds the fused row width", d, d_pad);
    return TRK_ERR_UNSUPPORTED;
  }
  const int groups = kGatherThreads / s.g;
  const int grid = capped_grid(ceil_div(rows, groups), 8);
#define CALL(G, CH, VEC)                                                 \
  split_rows_kernel<G, CH, VEC><<<grid, kGatherThreads, 0, stream>>>(    \
      repr, rows, d, n_normalize, normalized_inplace, static_cast<__half*>(out_split), d_pad, out_scale)
  TRK_DISPATCH_ROWSHAPE(s, CALL);
#undef CALL
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

int csr_project_biases(const int32_t* indptr, const int32_t* col, const float* val, const float* biases,
                       int64_t rows, float* out, cudaStream_t stream) {
  TRK_CHECK_ARG(indptr && biases && out, "csr_project_biases: null pointer");
  TRK_CHECK_ARG(rows >= 0, "csr_project_biases: rows < 0");
  if (rows == 0) return TRK_OK;
  const int grid = capped_grid(ceil_div(rows, kBiasTileRows), 8);
  csr_project_biases_kernel<<<grid, kBiasTileRows, 0, stream>>>(indptr, col, val, biases, rows, out);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

int pack_item_meta(const float* scale, const float* bias, int64_t n, float* meta, int64_t n_padded,
                   cudaStream_t stream) {
  TRK_CHECK_ARG(meta && n >= 0 && n_padded >= n, "pack_item_meta: bad arguments");
  if (n_padded == 0) return TRK_OK;
  const int threads = 256;
  pack_item_meta_kernel<<<static_cast<unsigned>(ceil_div(n_padded, threads)), threads, 0, stream>>>(
      scale, bias, n, reinterpret_cast<float2*>(meta), n_padded);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

}  // namespace trk
