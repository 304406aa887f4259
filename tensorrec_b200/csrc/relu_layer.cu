// The hidden layer of ReLURepresentationGraph in the fused training step (DESIGN §3.14):
//
//   forward   repr = relu(P + b) . W2                       P = X . W1 [rows, H] from K1, b [H], W2 [H, d]
//   backward  dP   = (d_repr . W2^T) (*) [P + b > 0]        written over P (K1^T turns it into dW1)
//             db   = sum_rows dP
//             dW2  = relu(P + b)^T . d_repr
//
// Both products run on the tensor cores as 3xTF32: every operand x is split into big = tf32(x) and
// small = tf32(x - big), and a product is big.big + big.small + small.big with fp32 accumulation.  tf32 keeps fp32's
// 8-bit exponent, so the split needs no per-row scale and the result is fp32-grade (error bound in DESIGN §3.14).
// The MMAs are the warp-level mma.sync m16n8k8 tf32: its fragments are loaded element by element from shared memory,
// so the transposed operands of the backward (relu(P + b)^T and d_repr as the B operand of dW2) cost nothing extra.
//
// The backward is partitioned by (32-wide H slice, row chunk).  A CTA keeps its slice of W2 in shared memory and its
// slice's dW2 partial in registers over all rows of its chunk, writes its partials to a workspace, and a second launch
// sums the chunks' partials in chunk order.  No atomics: the step stays run-to-run deterministic (sparse_ops.py).
#include <cuda_runtime.h>

#include "common.cuh"

namespace trk {

namespace {

constexpr int kReluMaxHidden = 2048;
constexpr int kReluMaxD = 512;

// forward tile: 64 rows x 128 output columns per CTA, 4 warps of 32 x 64, K (= H) in steps of 32
constexpr int kFwdRows = 64;
constexpr int kFwdCols = 128;
constexpr int kFwdK = 32;
constexpr int kFwdThreads = 128;
constexpr int kFwdAStride = kFwdK + 4;     // conflict-free fragment reads: bank 4 g + t
constexpr int kFwdBStride = kFwdCols + 8;  // bank 8 t + g

// backward: a 32-wide H slice per CTA, 32 rows per iteration, 8 warps
constexpr int kBwdSlice = 32;
constexpr int kBwdRows = 32;
constexpr int kBwdThreads = 256;
constexpr int kBwdPStride = kBwdSlice + 8;   // relu(P + b)^T fragment reads: bank 8 t + g
constexpr int kBwdGStride = kBwdSlice + 1;
constexpr int kBwdTargetCtas = 8 * kSMsH100;  // the row chunking is a function of the shape only, never of the device

__device__ __forceinline__ void split_tf32(float x, uint32_t& big, uint32_t& small) {
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(big) : "f"(x));
  const float rest = x - __uint_as_float(big);
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(small) : "f"(rest));
}

// D += A[16 x 8] . B[8 x 8], tf32 inputs, fp32 accumulate.  Thread (g = lane / 4, t = lane % 4) holds
// a = {A[g][t], A[g + 8][t], A[g][t + 4], A[g + 8][t + 4]}, b = {B[t][g], B[t + 4][g]},
// d = {D[g][2t], D[g][2t + 1], D[g + 8][2t], D[g + 8][2t + 1]}.
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// 3xTF32: the small terms first, so the big product is added last to the smaller partial sums
__device__ __forceinline__ void mma_3xtf32(float (&d)[4], const uint32_t (&a_big)[4], const uint32_t (&a_small)[4],
                                           uint32_t b0_big, uint32_t b1_big, uint32_t b0_small, uint32_t b1_small) {
  mma_tf32(d, a_small, b0_big, b1_big);
  mma_tf32(d, a_big, b0_small, b1_small);
  mma_tf32(d, a_big, b0_big, b1_big);
}

__global__ void __launch_bounds__(kFwdThreads) relu_layer_forward_kernel(const float* __restrict__ pre,
                                                                         const float* __restrict__ bias,
                                                                         const float* __restrict__ w2, int64_t rows,
                                                                         int hidden, int d, float* __restrict__ out) {
  __shared__ __align__(16) float a_s[kFwdRows][kFwdAStride];
  __shared__ __align__(16) float b_s[kFwdK][kFwdBStride];
  const int tid = threadIdx.x, warp = tid / kWarp, lane = tid % kWarp, g = lane / 4, t = lane % 4;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 64;
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * kFwdRows;
  const int c0 = blockIdx.y * kFwdCols;
  float acc[2][8][4];
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 8; ++ni)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[mi][ni][q] = 0.0f;

  for (int k0 = 0; k0 < hidden; k0 += kFwdK) {
    // A = relu(P + b), formed as it is loaded (hidden % 8 == 0: a float4 starting below hidden lies inside the row)
#pragma unroll
    for (int i = tid; i < kFwdRows * kFwdK / 4; i += kFwdThreads) {
      const int r = i / (kFwdK / 4), kq = (i % (kFwdK / 4)) * 4;
      const int64_t row = r0 + r;
      const int k = k0 + kq;
      float4 v = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      if (row < rows && k < hidden) {
        v = __ldg(reinterpret_cast<const float4*>(pre + row * hidden + k));
        const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + k));
        v.x = fmaxf(v.x + bb.x, 0.0f);
        v.y = fmaxf(v.y + bb.y, 0.0f);
        v.z = fmaxf(v.z + bb.z, 0.0f);
        v.w = fmaxf(v.w + bb.w, 0.0f);
      }
      *reinterpret_cast<float4*>(&a_s[r][kq]) = v;
    }
    // B = W2[k0 .. k0 + 32, c0 .. c0 + 128] (d % 4 == 0)
#pragma unroll
    for (int i = tid; i < kFwdK * kFwdCols / 4; i += kFwdThreads) {
      const int k = i / (kFwdCols / 4), cq = (i % (kFwdCols / 4)) * 4;
      const int kk = k0 + k, c = c0 + cq;
      float4 v = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      if (kk < hidden && c < d) v = __ldg(reinterpret_cast<const float4*>(w2 + static_cast<int64_t>(kk) * d + c));
      *reinterpret_cast<float4*>(&b_s[k][cq]) = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kFwdK; kk += 8) {
      uint32_t a_big[2][4], a_small[2][4];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        const int r = wm + 16 * mi + g;
        split_tf32(a_s[r][kk + t], a_big[mi][0], a_small[mi][0]);
        split_tf32(a_s[r + 8][kk + t], a_big[mi][1], a_small[mi][1]);
        split_tf32(a_s[r][kk + t + 4], a_big[mi][2], a_small[mi][2]);
        split_tf32(a_s[r + 8][kk + t + 4], a_big[mi][3], a_small[mi][3]);
      }
#pragma unroll
      for (int ni = 0; ni < 8; ++ni) {
        const int c = wn + 8 * ni + g;
        uint32_t b0, b0s, b1, b1s;
        split_tf32(b_s[kk + t][c], b0, b0s);
        split_tf32(b_s[kk + t + 4][c], b1, b1s);
#pragma unroll
        for (int mi = 0; mi < 2; ++mi) mma_3xtf32(acc[mi][ni], a_big[mi], a_small[mi], b0, b1, b0s, b1s);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int mi = 0; mi < 2; ++mi) {
#pragma unroll
    for (int ni = 0; ni < 8; ++ni) {
      const int c = c0 + wn + 8 * ni + 2 * t;   // even, d even: c < d covers c + 1
      if (c >= d) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t row = r0 + wm + 16 * mi + g + 8 * h;
        if (row < rows)
          *reinterpret_cast<float2*>(out + row * d + c) = make_float2(acc[mi][ni][2 * h], acc[mi][ni][2 * h + 1]);
      }
    }
  }
}

// kNt: n8 tiles of dW2 per warp; the 8 warps cover 2 x 16 H rows and 4 x 8 kNt columns of the slice's dW2, so a
// launch covers d <= 32 kNt.
template <int kNt>
struct BwdSmem {
  static constexpr int kDStride = 32 * kNt + 4;
  static constexpr size_t kBytes =
      sizeof(float) * (2 * kBwdRows * kDStride + kBwdRows * kBwdPStride + kBwdRows * kBwdGStride);
};

template <int kNt>
__global__ void __launch_bounds__(kBwdThreads) relu_layer_backward_kernel(
    float* __restrict__ pre, const float* __restrict__ bias, const float* __restrict__ w2,
    const float* __restrict__ d_out, int64_t rows, int hidden, int d, int64_t rows_per_chunk,
    float* __restrict__ part_w2, float* __restrict__ part_b) {
  constexpr int kDStride = BwdSmem<kNt>::kDStride;
  constexpr int kCover = 32 * kNt;
  extern __shared__ __align__(16) float smem[];
  float* w2_s = smem;                              // [32 H][kDStride]   W2 rows of the slice
  float* do_s = w2_s + kBwdSlice * kDStride;       // [32 rows][kDStride] d_repr rows
  float* z_s = do_s + kBwdRows * kDStride;         // [32 rows][kBwdPStride] P + b
  float* g_s = z_s + kBwdRows * kBwdPStride;       // [32 rows][kBwdGStride] dP

  const int tid = threadIdx.x, warp = tid / kWarp, lane = tid % kWarp, g = lane / 4, t = lane % 4;
  const int h0 = blockIdx.x * kBwdSlice;
  const int chunk = blockIdx.y;
  const int64_t row_begin = static_cast<int64_t>(chunk) * rows_per_chunk;
  const int64_t row_end = row_begin + rows_per_chunk < rows ? row_begin + rows_per_chunk : rows;
  const int k_d = (d + 7) & ~7;

  for (int i = tid; i < kBwdSlice * kCover / 4; i += kBwdThreads) {
    const int h = i / (kCover / 4), jq = (i % (kCover / 4)) * 4;
    float4 v = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if (h0 + h < hidden && jq < d)
      v = __ldg(reinterpret_cast<const float4*>(w2 + static_cast<int64_t>(h0 + h) * d + jq));
    *reinterpret_cast<float4*>(w2_s + h * kDStride + jq) = v;
  }

  // stage A: warp (am, an) owns dP rows 16 am .., H columns 8 an ..; stage B: warp (bm, bn) owns dW2 H rows 16 bm ..,
  // columns 8 kNt bn ..
  const int am = warp & 1, an = warp >> 1;
  const int bm = warp & 1, bn = warp >> 1;
  float acc_w2[kNt][4];
#pragma unroll
  for (int ni = 0; ni < kNt; ++ni)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc_w2[ni][q] = 0.0f;
  float acc_b = 0.0f;

  for (int64_t r0 = row_begin; r0 < row_end; r0 += kBwdRows) {
    for (int i = tid; i < kBwdRows * kCover / 4; i += kBwdThreads) {
      const int r = i / (kCover / 4), jq = (i % (kCover / 4)) * 4;
      float4 v = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      if (r0 + r < row_end && jq < d) v = __ldg(reinterpret_cast<const float4*>(d_out + (r0 + r) * d + jq));
      *reinterpret_cast<float4*>(do_s + r * kDStride + jq) = v;
    }
    for (int i = tid; i < kBwdRows * kBwdSlice; i += kBwdThreads) {
      const int r = i / kBwdSlice, h = i % kBwdSlice;
      float z = 0.0f;    // rows past the chunk and H past hidden: relu 0, no gradient
      if (r0 + r < row_end && h0 + h < hidden) z = pre[(r0 + r) * hidden + h0 + h] + __ldg(bias + h0 + h);
      z_s[r * kBwdPStride + h] = z;
    }
    __syncthreads();

    {  // dP = (d_repr . W2^T) (*) [P + b > 0]
      float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
      const float* arow = do_s + (16 * am + g) * kDStride;
      const float* brow = w2_s + (8 * an + g) * kDStride;
      for (int k = 0; k < k_d; k += 8) {
        uint32_t a_big[4], a_small[4], b0, b0s, b1, b1s;
        split_tf32(arow[k + t], a_big[0], a_small[0]);
        split_tf32(arow[8 * kDStride + k + t], a_big[1], a_small[1]);
        split_tf32(arow[k + t + 4], a_big[2], a_small[2]);
        split_tf32(arow[8 * kDStride + k + t + 4], a_big[3], a_small[3]);
        split_tf32(brow[k + t], b0, b0s);
        split_tf32(brow[k + t + 4], b1, b1s);
        mma_3xtf32(acc, a_big, a_small, b0, b1, b0s, b1s);
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int r = 16 * am + g + 8 * (q / 2), h = 8 * an + 2 * t + (q % 2);
        g_s[r * kBwdGStride + h] = z_s[r * kBwdPStride + h] > 0.0f ? acc[q] : 0.0f;
      }
    }
    __syncthreads();

    // dP over P (coalesced along H), and the slice's db partial in a fixed row order
    for (int i = tid; i < kBwdRows * kBwdSlice; i += kBwdThreads) {
      const int r = i / kBwdSlice, h = i % kBwdSlice;
      if (r0 + r < row_end && h0 + h < hidden) pre[(r0 + r) * hidden + h0 + h] = g_s[r * kBwdGStride + h];
    }
    if (tid < kBwdSlice) {
#pragma unroll 8
      for (int r = 0; r < kBwdRows; ++r) acc_b += g_s[r * kBwdGStride + tid];
    }

    // dW2 slice += relu(P + b)^T . d_repr over these rows (K = the 32 rows)
#pragma unroll
    for (int k = 0; k < kBwdRows; k += 8) {
      uint32_t a_big[4], a_small[4];
      const int h = 16 * bm + g;
      split_tf32(fmaxf(z_s[(k + t) * kBwdPStride + h], 0.0f), a_big[0], a_small[0]);
      split_tf32(fmaxf(z_s[(k + t) * kBwdPStride + h + 8], 0.0f), a_big[1], a_small[1]);
      split_tf32(fmaxf(z_s[(k + t + 4) * kBwdPStride + h], 0.0f), a_big[2], a_small[2]);
      split_tf32(fmaxf(z_s[(k + t + 4) * kBwdPStride + h + 8], 0.0f), a_big[3], a_small[3]);
#pragma unroll
      for (int ni = 0; ni < kNt; ++ni) {
        const int c = 8 * kNt * bn + 8 * ni + g;
        uint32_t b0, b0s, b1, b1s;
        split_tf32(do_s[(k + t) * kDStride + c], b0, b0s);
        split_tf32(do_s[(k + t + 4) * kDStride + c], b1, b1s);
        mma_3xtf32(acc_w2[ni], a_big, a_small, b0, b1, b0s, b1s);
      }
    }
    __syncthreads();   // the next tile overwrites do_s, z_s and g_s
  }

  // this chunk's partials: part_w2 [n_chunks][hidden][d], part_b [n_chunks][hidden]
  float* pw = part_w2 + static_cast<int64_t>(chunk) * hidden * d;
#pragma unroll
  for (int ni = 0; ni < kNt; ++ni) {
    const int c = 8 * kNt * bn + 8 * ni + 2 * t;
    if (c >= d) continue;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int h = h0 + 16 * bm + g + 8 * hh;
      if (h < hidden)
        *reinterpret_cast<float2*>(pw + static_cast<int64_t>(h) * d + c) =
            make_float2(acc_w2[ni][2 * hh], acc_w2[ni][2 * hh + 1]);
    }
  }
  if (tid < kBwdSlice && h0 + tid < hidden) part_b[static_cast<int64_t>(chunk) * hidden + h0 + tid] = acc_b;
}

// d_w2 [hidden * d] then d_bias [hidden]: the chunks' partials summed in chunk order
__global__ void relu_layer_reduce_kernel(const float* __restrict__ part_w2, const float* __restrict__ part_b,
                                         int n_chunks, int hidden, int d, float* __restrict__ d_w2,
                                         float* __restrict__ d_bias) {
  const int64_t n_w = static_cast<int64_t>(hidden) * d;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n_w + hidden;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const bool w = i < n_w;
    const float* src = w ? part_w2 + i : part_b + (i - n_w);
    const int64_t stride = w ? n_w : hidden;
    float s = 0.0f;
    for (int c = 0; c < n_chunks; ++c) s += src[c * stride];
    if (w)
      d_w2[i] = s;
    else
      d_bias[i - n_w] = s;
  }
}

int relu_chunks(int64_t rows, int32_t hidden) {
  const int64_t slices = ceil_div(hidden, kBwdSlice);
  const int64_t tiles = ceil_div(rows, kBwdRows);
  const int64_t want = ceil_div(kBwdTargetCtas, slices);
  const int64_t n = want < tiles ? want : tiles;
  return static_cast<int>(n < 1 ? 1 : n);
}

int check_layer(const char* who, const float* pre, const float* bias, const float* w2, int64_t rows, int32_t hidden,
                int32_t d) {
  TRK_CHECK_ARG(pre && bias && w2, "%s: null input (pre, bias and w2 are required)", who);
  TRK_CHECK_ARG(rows >= 0 && rows < (int64_t(1) << 31), "%s: rows=%lld outside [0, 2^31)", who,
                static_cast<long long>(rows));
  TRK_CHECK_ARG(hidden >= 8 && hidden <= kReluMaxHidden && hidden % 8 == 0,
                "%s: hidden=%d must be a multiple of 8 in [8, %d] (pad with zero units)", who, hidden, kReluMaxHidden);
  TRK_CHECK_ARG(d >= 4 && d <= kReluMaxD && d % 4 == 0,
                "%s: d=%d must be a multiple of 4 in [4, %d] (pad with zero columns)", who, d, kReluMaxD);
  TRK_CHECK_ARG((reinterpret_cast<uintptr_t>(pre) | reinterpret_cast<uintptr_t>(bias) |
                 reinterpret_cast<uintptr_t>(w2)) % 16 == 0,
                "%s: pre, bias and w2 must be 16-byte aligned", who);
  return TRK_OK;
}

template <int kNt>
int launch_backward(float* pre, const float* bias, const float* w2, const float* d_out, int64_t rows, int32_t hidden,
                    int32_t d, int n_chunks, int64_t rows_per_chunk, float* part_w2, float* part_b,
                    cudaStream_t stream) {
  const size_t smem = BwdSmem<kNt>::kBytes;
  TRK_CHECK_CUDA(cudaFuncSetAttribute(relu_layer_backward_kernel<kNt>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      static_cast<int>(smem)));
  const dim3 grid(static_cast<unsigned>(ceil_div(hidden, kBwdSlice)), static_cast<unsigned>(n_chunks));
  relu_layer_backward_kernel<kNt><<<grid, kBwdThreads, smem, stream>>>(pre, bias, w2, d_out, rows, hidden, d,
                                                                       rows_per_chunk, part_w2, part_b);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

}  // namespace

size_t relu_layer_workspace_bytes(int64_t rows, int32_t hidden, int32_t d) {
  if (rows < 0 || hidden < 1 || d < 1) return 0;
  return static_cast<size_t>(relu_chunks(rows, hidden)) * static_cast<size_t>(hidden) * (static_cast<size_t>(d) + 1) *
         sizeof(float);
}

int relu_layer_forward(const float* pre, const float* bias, const float* w2, int64_t rows, int32_t hidden, int32_t d,
                       float* out, cudaStream_t stream) {
  const char* who = "relu_layer_forward";
  int rc = check_layer(who, pre, bias, w2, rows, hidden, d);
  if (rc != TRK_OK) return rc;
  TRK_CHECK_ARG(out, "%s: null output", who);
  TRK_CHECK_ARG(reinterpret_cast<uintptr_t>(out) % 16 == 0, "%s: out must be 16-byte aligned", who);
  if (rows == 0) return TRK_OK;
  const dim3 grid(static_cast<unsigned>(ceil_div(rows, kFwdRows)), static_cast<unsigned>(ceil_div(d, kFwdCols)));
  relu_layer_forward_kernel<<<grid, kFwdThreads, 0, stream>>>(pre, bias, w2, rows, hidden, d, out);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

int relu_layer_backward(float* pre, const float* bias, const float* w2, const float* d_out, int64_t rows,
                        int32_t hidden, int32_t d, float* d_bias, float* d_w2, void* workspace, size_t workspace_bytes,
                        cudaStream_t stream) {
  const char* who = "relu_layer_backward";
  int rc = check_layer(who, pre, bias, w2, rows, hidden, d);
  if (rc != TRK_OK) return rc;
  TRK_CHECK_ARG(d_out, "%s: null d_out", who);
  TRK_CHECK_ARG(d_bias && d_w2, "%s: null output (d_bias and d_w2 are required)", who);
  TRK_CHECK_ARG(workspace, "%s: null workspace", who);
  TRK_CHECK_ARG(reinterpret_cast<uintptr_t>(d_out) % 16 == 0 && reinterpret_cast<uintptr_t>(d_w2) % 8 == 0 &&
                    reinterpret_cast<uintptr_t>(workspace) % 16 == 0,
                "%s: d_out and workspace must be 16-byte aligned, d_w2 8-byte aligned", who);
  const size_t need = relu_layer_workspace_bytes(rows, hidden, d);
  TRK_CHECK_ARG(workspace_bytes >= need, "%s: workspace of %zu bytes, %zu needed (trk_relu_layer_workspace_bytes)", who,
                workspace_bytes, need);
  const int n_chunks = relu_chunks(rows, hidden);
  const int64_t rows_per_chunk = ceil_div(ceil_div(rows, kBwdRows), n_chunks) * kBwdRows;
  float* part_w2 = static_cast<float*>(workspace);
  float* part_b = part_w2 + static_cast<int64_t>(n_chunks) * hidden * d;
  if (d <= 32)
    rc = launch_backward<1>(pre, bias, w2, d_out, rows, hidden, d, n_chunks, rows_per_chunk, part_w2, part_b, stream);
  else if (d <= 64)
    rc = launch_backward<2>(pre, bias, w2, d_out, rows, hidden, d, n_chunks, rows_per_chunk, part_w2, part_b, stream);
  else if (d <= 128)
    rc = launch_backward<4>(pre, bias, w2, d_out, rows, hidden, d, n_chunks, rows_per_chunk, part_w2, part_b, stream);
  else if (d <= 256)
    rc = launch_backward<8>(pre, bias, w2, d_out, rows, hidden, d, n_chunks, rows_per_chunk, part_w2, part_b, stream);
  else
    rc = launch_backward<16>(pre, bias, w2, d_out, rows, hidden, d, n_chunks, rows_per_chunk, part_w2, part_b, stream);
  if (rc != TRK_OK) return rc;
  relu_layer_reduce_kernel<<<capped_grid(ceil_div(static_cast<int64_t>(hidden) * (d + 1), 256), 8), 256, 0, stream>>>(
      part_w2, part_b, n_chunks, hidden, d, d_w2, d_bias);
  TRK_CHECK_LAUNCH();
  return TRK_OK;
}

}  // namespace trk
