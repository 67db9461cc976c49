// fp32 CUDA-core fused multi-head softmax attention (flash-style online softmax; the N x M
// probability tensor the reference materialises at attention.py:12-13,19 never exists).
// Exact-arithmetic mode (OG_PREC_FP32) of og_attention_fwd and on-device ground truth for the
// tensor-core kernel.  One CTA = 64 queries of one (batch, head); key tiles of 64.
#pragma once
#include "common.cuh"
#include <math_constants.h>

namespace og {

struct AttnArgs {
  const float* q; int64_t ldq, strideq;
  const float* k; int64_t ldk, stridek;
  const float* v; int64_t ldv, stridev;
  float* out; int64_t ldo, strideo;
  int batch, nq, nk, num_heads;
  float scale;
  const int* klen;           // padded batch (device, may be null): keys of sequence b = klen[b], clamped into [1, nk]
};

constexpr int ATQ = 64, ATK = 64;

template <int DH>
__global__ void __launch_bounds__(256) attention_simt_kernel(AttnArgs a) {
  constexpr int CPT = (DH >= 64) ? 4 : (DH >= 32 ? 2 : 1);     // output columns per thread
  extern __shared__ __align__(16) float og_attn_smem[];          // 64 KB at DH=64: dynamic
  float (*Qt)[ATQ] = reinterpret_cast<float (*)[ATQ]>(og_attn_smem);
  float (*Kt)[ATK] = reinterpret_cast<float (*)[ATK]>(og_attn_smem + DH * ATQ);
  float (*Vs)[DH] = reinterpret_cast<float (*)[DH]>(og_attn_smem + DH * (ATQ + ATK));
  float (*Pt)[ATQ] = reinterpret_cast<float (*)[ATQ]>(og_attn_smem + DH * (ATQ + ATK) + ATK * DH);

  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * ATQ;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int nk = padded_length(a.klen, b, a.nk);
  const float* __restrict__ Q = a.q + (int64_t)b * a.strideq + h * DH;
  const float* __restrict__ Kp = a.k + (int64_t)b * a.stridek + h * DH;
  const float* __restrict__ Vp = a.v + (int64_t)b * a.stridev + h * DH;

  // Q tile -> Qt (transposed); rows beyond nq are zero
  for (int idx = tid; idx < ATQ * DH; idx += 256) {
    const int r = idx % ATQ, c = idx / ATQ;
    Qt[c][r] = (q0 + r < a.nq) ? __ldg(Q + (int64_t)(q0 + r) * a.ldq + c) : 0.f;
  }

  float m_i[4], l_i[4], o[4][CPT];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m_i[i] = -CUDART_INF_F; l_i[i] = 0.f;
#pragma unroll
    for (int c = 0; c < CPT; ++c) o[i][c] = 0.f;
  }
  const bool pv_active = (tx * CPT < DH);

  for (int k0 = 0; k0 < nk; k0 += ATK) {
    __syncthreads();                                   // previous tile fully consumed (and Qt visible)
    for (int idx = tid; idx < ATK * DH; idx += 256) {
      const int r = idx % ATK, c = idx / ATK;
      const bool ok = (k0 + r < nk);
      Kt[c][r] = ok ? __ldg(Kp + (int64_t)(k0 + r) * a.ldk + c) : 0.f;
    }
    for (int idx = tid; idx < ATK * DH; idx += 256) {
      const int r = idx / DH, c = idx % DH;
      Vs[r][c] = (k0 + r < nk) ? __ldg(Vp + (int64_t)(k0 + r) * a.ldv + c) : 0.f;
    }
    __syncthreads();

    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 8
    for (int kk = 0; kk < DH; ++kk) {
      const float4 q4 = *reinterpret_cast<const float4*>(&Qt[kk][ty * 4]);
      const float4 k4 = *reinterpret_cast<const float4*>(&Kt[kk][tx * 4]);
      const float qv[4] = {q4.x, q4.y, q4.z, q4.w}, kv[4] = {k4.x, k4.y, k4.z, k4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) s[i][j] = fmaf(qv[i], kv[j], s[i][j]);
    }
    // scale (matmul * Dh^-0.5, attention.py:12), mask the key tail, online softmax
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float mx = -CUDART_INF_F;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        s[i][j] = (k0 + tx * 4 + j < nk) ? s[i][j] * a.scale : -CUDART_INF_F;
        mx = fmaxf(mx, s[i][j]);
      }
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
      const float m_new = fmaxf(m_i[i], mx);
      float rs = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) { s[i][j] = expf(s[i][j] - m_new); rs += s[i][j]; }
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) rs += __shfl_xor_sync(0xffffffffu, rs, off);
      const float corr = expf(m_i[i] - m_new);          // exp(-inf) = 0 on the first tile
      l_i[i] = l_i[i] * corr + rs;
      m_i[i] = m_new;
#pragma unroll
      for (int c = 0; c < CPT; ++c) o[i][c] *= corr;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
      *reinterpret_cast<float4*>(&Pt[tx * 4 + j][ty * 4]) = make_float4(s[0][j], s[1][j], s[2][j], s[3][j]);
    __syncthreads();
    if (pv_active) {
#pragma unroll 8
      for (int kk = 0; kk < ATK; ++kk) {
        const float4 p4 = *reinterpret_cast<const float4*>(&Pt[kk][ty * 4]);
        const float pv[4] = {p4.x, p4.y, p4.z, p4.w};
        float vv[CPT];
#pragma unroll
        for (int c = 0; c < CPT; ++c) vv[c] = Vs[kk][tx * CPT + c];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int c = 0; c < CPT; ++c) o[i][c] = fmaf(pv[i], vv[c], o[i][c]);
      }
    }
  }
  if (pv_active) {
    float* __restrict__ O = a.out + (int64_t)b * a.strideo + h * DH;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = q0 + ty * 4 + i;
      if (r >= a.nq) continue;
      const float inv = 1.f / l_i[i];
#pragma unroll
      for (int c = 0; c < CPT; ++c) O[(int64_t)r * a.ldo + tx * CPT + c] = o[i][c] * inv;
    }
  }
}

inline int attention_simt_launch(const AttnArgs& a, int head_dim, cudaStream_t stream) {
  dim3 grid(cdiv(a.nq, ATQ), a.num_heads, a.batch);
#define OG_ATTN_CASE(DH_)                                                                        \
  case DH_: {                                                                                    \
    constexpr int smem = (DH_ * (ATQ + ATK) + ATK * DH_ + ATK * ATQ) * (int)sizeof(float);       \
    if (const int rc = smem_opt_in<attention_simt_kernel<DH_>>(smem)) return rc;                 \
    return OG_LAUNCH(attention_simt_kernel<DH_>, grid, 256, smem, stream, a);                    \
  }
  switch (head_dim) {
    OG_ATTN_CASE(8) OG_ATTN_CASE(16) OG_ATTN_CASE(32) OG_ATTN_CASE(64)
    default: return fail(OG_EUNSUPPORTED, "attention: head_dim %d not in {8,16,32,64}", head_dim);
  }
#undef OG_ATTN_CASE
}

}  // namespace og
