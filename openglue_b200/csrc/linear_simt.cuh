// fp32 CUDA-core GEMM with fused epilogue:  Y = epi(alpha * [A|A2] . W^T + bias)
// The exact-arithmetic mode (OG_PREC_FP32) of og_linear_fwd and the on-device ground truth
// for the tensor-core kernels.  128x128x8 tiles, 8x8 outputs per thread, register-prefetched
// double buffering.  Replaces the reference's Conv1d(k=1) calls (attention_gnn.py:24-32,
// models/utils.py:53-57, superglue.py:58) and the score matmul (superglue.py:80-86).
#pragma once
#include "common.cuh"
#include <algorithm>

namespace og {

constexpr int LBM = 128, LBN = 128, LBK = 8;

struct LinearFlags { int vecA, vecW, vecY, vecYt; };

__device__ __forceinline__ void linear_load4(float (&dst)[4], const float* __restrict__ P, int64_t ld,
                                             const float* __restrict__ P2, int64_t ld2,
                                             int k1, int K, int row, int nrows, int k, int vec) {
  dst[0] = dst[1] = dst[2] = dst[3] = 0.f;
  if (row >= nrows || k >= K) return;
  if (vec) {                       // k1, K multiples of 4, rows 16B aligned: never straddles
    const float* src = (k < k1) ? (P + (int64_t)row * ld + k) : (P2 + (int64_t)row * ld2 + (k - k1));
    float4 v = __ldg(reinterpret_cast<const float4*>(src));
    dst[0] = v.x; dst[1] = v.y; dst[2] = v.z; dst[3] = v.w;
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int kk = k + i;
      if (kk < K) dst[i] = (kk < k1) ? __ldg(P + (int64_t)row * ld + kk) : __ldg(P2 + (int64_t)row * ld2 + (kk - k1));
    }
  }
}

__global__ void __launch_bounds__(256, 2) linear_simt_kernel(og_linear_args a, LinearFlags f) {
  __shared__ __align__(16) float As[2][LBK][LBM];
  __shared__ __align__(16) float Bs[2][LBK][LBN];
  const int b = blockIdx.z;
  const float* __restrict__ A = a.A + (int64_t)b * a.strideA;
  const float* __restrict__ A2 = a.A2 ? a.A2 + (int64_t)b * a.strideA2 : nullptr;
  const float* __restrict__ W = a.W + (int64_t)b * a.strideW;
  const int row0 = blockIdx.y * LBM, col0 = blockIdx.x * LBN;
  const int K = a.k1 + a.k2;
  const int tid = threadIdx.x;
  const int lr = tid >> 1, lk = (tid & 1) * 4;
  const int ty = tid >> 4, tx = tid & 15;

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float ra[4], rb[4];
  const int nk = cdiv(K, LBK);
  linear_load4(ra, A, a.lda, A2, a.lda2, a.k1, K, row0 + lr, a.rows, lk, f.vecA);
  linear_load4(rb, W, a.ldw, nullptr, 0, K, K, col0 + lr, a.nout, lk, f.vecW);
#pragma unroll
  for (int i = 0; i < 4; ++i) { As[0][lk + i][lr] = ra[i]; Bs[0][lk + i][lr] = rb[i]; }
  __syncthreads();

  for (int kt = 0; kt < nk; ++kt) {
    const int cur = kt & 1;
    if (kt + 1 < nk) {
      linear_load4(ra, A, a.lda, A2, a.lda2, a.k1, K, row0 + lr, a.rows, (kt + 1) * LBK + lk, f.vecA);
      linear_load4(rb, W, a.ldw, nullptr, 0, K, K, col0 + lr, a.nout, (kt + 1) * LBK + lk, f.vecW);
    }
#pragma unroll
    for (int k = 0; k < LBK; ++k) {
      float4 a0 = *reinterpret_cast<const float4*>(&As[cur][k][ty * 4]);
      float4 a1 = *reinterpret_cast<const float4*>(&As[cur][k][64 + ty * 4]);
      float4 b0 = *reinterpret_cast<const float4*>(&Bs[cur][k][tx * 4]);
      float4 b1 = *reinterpret_cast<const float4*>(&Bs[cur][k][64 + tx * 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
#pragma unroll
      for (int i = 0; i < 4; ++i) { As[cur ^ 1][lk + i][lr] = ra[i]; Bs[cur ^ 1][lk + i][lr] = rb[i]; }
    }
    __syncthreads();
  }

  // epilogue
  // R may alias Y (in-place residual update x <- x + f(x)): each element is read, then written, by the
  // same thread only, so no __restrict__ / non-coherent loads on these two.
  const float* R = a.R ? a.R + (int64_t)b * a.strideR : nullptr;
  float* Y = a.Y ? a.Y + (int64_t)b * a.strideY : nullptr;
  float* __restrict__ Yt = a.Yt ? a.Yt + (int64_t)b * a.strideYt : nullptr;
#pragma unroll
  for (int ih = 0; ih < 2; ++ih) {
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int cb = col0 + jh * 64 + tx * 4;
      float out[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = row0 + ih * 64 + ty * 4 + i;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int c = cb + j;
          float y = acc[ih * 4 + i][jh * 4 + j] * a.alpha;
          if (c < a.nout) {
            if (a.bias) y += __ldg(a.bias + c);
            if (a.relu) y = fmaxf(y, 0.f);
            if (R && r < a.rows) {
              float rv = R[(int64_t)r * a.ldr + c];
              y = a.rscale ? fmaf(__ldg(a.rscale + c), rv, y) : (y + rv);
            }
          }
          out[i][j] = y;
        }
        if (Y && r < a.rows) {
          if (f.vecY && cb + 3 < a.nout) {
            *reinterpret_cast<float4*>(Y + (int64_t)r * a.ldy + cb) = make_float4(out[i][0], out[i][1], out[i][2], out[i][3]);
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) if (cb + j < a.nout) Y[(int64_t)r * a.ldy + cb + j] = out[i][j];
          }
        }
      }
      if (Yt) {
        const int rb0 = row0 + ih * 64 + ty * 4;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int c = cb + j;
          if (c >= a.nout) continue;
          if (f.vecYt && rb0 + 3 < a.rows) {
            *reinterpret_cast<float4*>(Yt + (int64_t)c * a.ldyt + rb0) = make_float4(out[0][j], out[1][j], out[2][j], out[3][j]);
          } else {
#pragma unroll
            for (int i = 0; i < 4; ++i) if (rb0 + i < a.rows) Yt[(int64_t)c * a.ldyt + rb0 + i] = out[i][j];
          }
        }
      }
    }
  }
}

// grid.y counts 128-row tiles and stops at 65535: taller operands run as consecutive launches over row ranges of at most
// LINEAR_MAX_ROWS rows, each with A, A2, R and Y advanced by its first row and Yt by its first column.  The ranges start at
// multiples of 128 rows, so a row's tile, and with it its result, is the same as in one launch.
constexpr int64_t LINEAR_MAX_ROWS = 65535 * (int64_t)LBM;

inline int linear_simt_launch(const og_linear_args& a, cudaStream_t stream) {
  if (a.batch > 65535) return fail(OG_EUNSUPPORTED, "linear: %d batches exceed the grid limit 65535", a.batch);
  LinearFlags f;
  f.vecA = (a.k1 % 4 == 0) && (a.k2 % 4 == 0) && (a.lda % 4 == 0) && (a.strideA % 4 == 0) && aligned16(a.A) &&
           (!a.A2 || ((a.lda2 % 4 == 0) && (a.strideA2 % 4 == 0) && aligned16(a.A2)));
  f.vecW = ((a.k1 + a.k2) % 4 == 0) && (a.ldw % 4 == 0) && (a.strideW % 4 == 0) && aligned16(a.W);
  f.vecY = a.Y && (a.ldy % 4 == 0) && (a.strideY % 4 == 0) && aligned16(a.Y);
  f.vecYt = a.Yt && (a.ldyt % 4 == 0) && (a.strideYt % 4 == 0) && aligned16(a.Yt);
  // the flags hold for every range: r0 is a multiple of 4, so an advanced pointer stays 16-byte aligned where its flag needs it
  for (int64_t r0 = 0; r0 < a.rows; r0 += LINEAR_MAX_ROWS) {
    og_linear_args p = a;
    p.rows = (int)std::min<int64_t>(a.rows - r0, LINEAR_MAX_ROWS);
    p.A += r0 * a.lda;
    if (p.A2) p.A2 += r0 * a.lda2;
    if (p.R) p.R += r0 * a.ldr;
    if (p.Y) p.Y += r0 * a.ldy;
    if (p.Yt) p.Yt += r0;
    dim3 grid(cdiv(p.nout, LBN), cdiv(p.rows, LBM), p.batch);
    if (const int rc = OG_LAUNCH(linear_simt_kernel, grid, 256, 0, stream, p, f)) return rc;
  }
  return OG_OK;
}

}  // namespace og
