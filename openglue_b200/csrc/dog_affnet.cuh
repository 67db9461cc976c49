// The reference's DoG-AffNet-HardNet front-end (OPENCVDoGAffNetHardNet: models/features/opencv/dog_affnet_harnet.py on
// models/features/opencv/base.py).  Detection and selection are the OpenCV SIFT stages (sift.cuh: og_sift_detect, og_sift_select)
// unchanged; this file describes the selected keypoints, restating kornia_moons and kornia 0.6.3 on the float image.  Stages, for
// the selected rows only and in chunks of rows:
//   affnet    cv2 keypoint -> laf_from_opencv_SIFT_kpts (mrSize 6) -> make_upright -> AffNet's standardised 32x32 patch
//   (AffNet's CNN, im2col + GEMM, outside this file)
//   frames    tanh and the affine frame algebra (kg_affine_frame, orientation preserved) -> OriNet's standardised patch on that LAF
//   (OriNet's six 3x3 convolutions, outside this file)
//   orinet    OriNet's head: the 8x8, padding-1 convolution to 3x3x2, tanh, the mean, atan2 -> the orienter composition
//             (ks_set_orientation) -> HardNet's standardised patch on the final LAF
//   (HardNet's CNN, then og_kgftt_desc_finish)
// The output LAFs [B, out_cap, 2, 3] carry each row's frame from stage to stage: every stage reads its row and writes it back.
#pragma once
#include "kornia_gftt.cuh"

namespace og {

constexpr int KD_ORI_C = 64;                     // OriNet's channels before its head
constexpr int KD_ORI_K = 8;                      // the head's kernel; padding 1 on the 8x8 map gives 3x3 outputs
constexpr int KD_ORI_OUT = 3;

// kornia_moons.feature.laf_from_opencv_SIFT_kpts of one keypoint kp = (x, y, size, angle, response):
// laf_from_center_scale_ori(xy, float32(6 size), float32(-angle)) = [[s cos t, s sin t, x], [-s sin t, s cos t, y]],
// t = deg2rad(-angle) = -angle * pi / 180 in float32.  cos and sin are taken in double and rounded once, so they are the correctly
// rounded float32 values.
__device__ __forceinline__ void kd_laf_from_kp(const float* __restrict__ kp, float a[6]) {
  const float s = __fmul_rn(6.f, kp[2]);
  const float t = __fdiv_rn(__fmul_rn(-kp[3], KS_PI), 180.f);
  const float c = (float)cos((double)t), sn = (float)sin((double)t);
  a[0] = __fmul_rn(s, c); a[1] = __fmul_rn(s, sn); a[2] = kp[0];
  a[3] = __fmul_rn(s, -sn); a[4] = __fmul_rn(s, c); a[5] = kp[1];
}

// Chunk rows [r0, r0 + gridDim.x) of the [B, out_cap] output: row (b, j) is keypoint kp[b, sel[b, j]] for j < n[b].  Writes the
// kornia_moons LAF to lafs[b, j], the cv2 response to scores[b, j] and AffNet's standardised patch on make_upright(LAF) to
// out [rows][32][32]; rows past n[b] get zeros.
template <int THREADS>
__global__ void __launch_bounds__(THREADS) kd_affnet_patch_kernel(KsPyr P, int H, int W, const float* __restrict__ kp, int cap,
                                                                  const int* __restrict__ sel, const int* __restrict__ n, int out_cap,
                                                                  int r0, float* __restrict__ lafs, float* __restrict__ scores,
                                                                  float* __restrict__ out) {
  __shared__ float patch[KG_PS * KG_PS];
  __shared__ float red[THREADS / 32];
  float* o = out + (int64_t)blockIdx.x * KG_PS * KG_PS;
  int b, j;
  const int src = kg_row(r0, out_cap, sel, n, cap, b, j);
  const int64_t row = (int64_t)b * out_cap + j;
  if (src < 0) {
    for (int i = threadIdx.x; i < KG_PS * KG_PS; i += THREADS) o[i] = 0.f;
    if (threadIdx.x < 6) lafs[row * 6 + threadIdx.x] = 0.f;
    if (threadIdx.x == 0) scores[row] = 0.f;
    return;
  }
  const float* k = kp + ((int64_t)b * cap + src) * 5;
  float a[6], u[6];
  kd_laf_from_kp(k, a);
  kg_upright(a, u);
  ks_patch<KG_PS>(P, b, H, W, u, patch);
  __syncthreads();
  kg_standardize<THREADS>(patch, red, o);
  if (threadIdx.x < 6) lafs[row * 6 + threadIdx.x] = a[threadIdx.x];
  if (threadIdx.x == 0) scores[row] = k[4];
}

// After AffNet's CNN: xy [rows][3] (before tanh) and lafs[b, j] -> the affine LAF (orientation preserved) back to lafs[b, j], and
// OriNet's standardised patch on it as it is (not made upright) to out [rows][32][32].  Rows past n[b] get zeros.
template <int THREADS>
__global__ void __launch_bounds__(THREADS) kd_frame_kernel(KsPyr P, int H, int W, const int* __restrict__ n, int out_cap, int r0,
                                                           const float* __restrict__ xy, float* __restrict__ lafs, float* __restrict__ out) {
  __shared__ float patch[KG_PS * KG_PS];
  __shared__ float red[THREADS / 32];
  float* o = out + (int64_t)blockIdx.x * KG_PS * KG_PS;
  int b, j;
  const int src = kg_row(r0, out_cap, nullptr, n, 0, b, j);
  const int64_t row = (int64_t)b * out_cap + j;
  if (src < 0) {
    for (int i = threadIdx.x; i < KG_PS * KG_PS; i += THREADS) o[i] = 0.f;
    if (threadIdx.x < 6) lafs[row * 6 + threadIdx.x] = 0.f;
    return;
  }
  float d[6], a[6];
  for (int e = 0; e < 6; ++e) d[e] = lafs[row * 6 + e];
  kg_affine_frame(xy + (int64_t)blockIdx.x * 3, d, a);
  ks_patch<KG_PS>(P, b, H, W, a, patch);
  __syncthreads();                                          // every thread has read the row before thread < 6 rewrites it
  kg_standardize<THREADS>(patch, red, o);
  if (threadIdx.x < 6) lafs[row * 6 + threadIdx.x] = a[threadIdx.x];
}

// OriNet's head and LAFOrienter(32, angle_detector=OriNet) after OriNet's 3x3 convolutions.  act [rows][8][8][64] (NHWC, after
// the last ReLU); wt [2][8][8][64] and bias [2] the head's Conv2d(64, 2, 8, padding=1).  Per row: the 3x3x2 convolution on CUDA
// cores (each output: lane l sums channels 2l, 2l + 1 over the taps in raster order, then a fixed xor tree), tanh, the mean of
// the 9 values in raster order, angle = atan2(y0 + 1e-8, y1 + 1e-8); lafs[b, j] <- set_laf_orientation(laf, rad2deg(angle) +
// get_laf_orientation(laf)), angle[b, j] <- angle, and HardNet's standardised patch on the new LAF to out [rows][32][32].  Rows
// past n[b] get zeros.  256 threads: warp w computes the outputs w, w + 8 and w + 16 of the 18.
__global__ void __launch_bounds__(256) kd_orinet_head_kernel(KsPyr P, int H, int W, const int* __restrict__ n, int out_cap, int r0,
                                                             const float* __restrict__ act, const float* __restrict__ wt,
                                                             const float* __restrict__ bias, float* __restrict__ lafs,
                                                             float* __restrict__ angle, float* __restrict__ out) {
  constexpr int THREADS = 256, M = KD_ORI_K * KD_ORI_K * KD_ORI_C, NOUT = 2 * KD_ORI_OUT * KD_ORI_OUT;
  __shared__ __align__(16) float x[M];
  __shared__ float y[NOUT];
  __shared__ float la[6];
  __shared__ float red[THREADS / 32];
  float* patch = x;                                         // the activations are dead once y is written
  float* o = out + (int64_t)blockIdx.x * KG_PS * KG_PS;
  int b, j;
  const int src = kg_row(r0, out_cap, nullptr, n, 0, b, j);
  const int64_t row = (int64_t)b * out_cap + j;
  if (src < 0) {
    for (int i = threadIdx.x; i < KG_PS * KG_PS; i += THREADS) o[i] = 0.f;
    if (threadIdx.x < 6) lafs[row * 6 + threadIdx.x] = 0.f;
    if (threadIdx.x == 0) angle[row] = 0.f;
    return;
  }
  const float4* a4 = reinterpret_cast<const float4*>(act + (int64_t)blockIdx.x * M);
  for (int i = threadIdx.x; i < M / 4; i += THREADS) reinterpret_cast<float4*>(x)[i] = __ldg(a4 + i);
  if (threadIdx.x < 6) la[threadIdx.x] = lafs[row * 6 + threadIdx.x];
  __syncthreads();
  const int warp = threadIdx.x / 32, lane = threadIdx.x & 31;
  for (int q = warp; q < NOUT; q += THREADS / 32) {
    const int oc = q / (KD_ORI_OUT * KD_ORI_OUT), oy = (q / KD_ORI_OUT) % KD_ORI_OUT, ox = q % KD_ORI_OUT;
    const float* w = wt + (int64_t)oc * M;
    float s = 0.f;
    for (int ky = 0; ky < KD_ORI_K; ++ky) {
      const int iy = oy + ky - 1;
      if (iy < 0 || iy >= KD_ORI_K) continue;
      for (int kx = 0; kx < KD_ORI_K; ++kx) {
        const int ix = ox + kx - 1;
        if (ix < 0 || ix >= KD_ORI_K) continue;
        const float2 wv = __ldg(reinterpret_cast<const float2*>(w + (ky * KD_ORI_K + kx) * KD_ORI_C) + lane);
        const float2 xv = reinterpret_cast<const float2*>(x + (iy * KD_ORI_K + ix) * KD_ORI_C)[lane];
        s = __fmaf_rn(wv.x, xv.x, s);
        s = __fmaf_rn(wv.y, xv.y, s);
      }
    }
    for (int off = 16; off > 0; off >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, off));
    if (lane == 0) y[q] = tanhf(__fadd_rn(s, bias[oc]));
  }
  __syncthreads();
  if (threadIdx.x == 0) {                                   // the only thread touching la until the next barrier
    float a[6], m[2];
    for (int e = 0; e < 6; ++e) a[e] = la[e];
    for (int c = 0; c < 2; ++c) {                           // AdaptiveAvgPool2d(1)
      float s = 0.f;
      for (int i = 0; i < KD_ORI_OUT * KD_ORI_OUT; ++i) s = __fadd_rn(s, y[c * KD_ORI_OUT * KD_ORI_OUT + i]);
      m[c] = __fdiv_rn(s, (float)(KD_ORI_OUT * KD_ORI_OUT));
    }
    const float an = atan2f(__fadd_rn(m[0], 1e-8f), __fadd_rn(m[1], 1e-8f));
    ks_set_orientation(a, an, la);
    y[0] = an;
  }
  __syncthreads();
  const float ang = y[0];
  float a[6];
  for (int e = 0; e < 6; ++e) a[e] = la[e];
  ks_patch<KG_PS>(P, b, H, W, a, patch);
  __syncthreads();
  kg_standardize<THREADS>(patch, red, o);
  if (threadIdx.x < 6) lafs[row * 6 + threadIdx.x] = a[threadIdx.x];
  if (threadIdx.x == 0) angle[row] = ang;
}

}  // namespace og
