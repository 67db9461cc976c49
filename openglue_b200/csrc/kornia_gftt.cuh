// kornia's GFTT / AffNet / HardNet front-end (the reference's GFTTAffNetHardNet: models/features/hardnet.py on
// models/features/base.py), restated from kornia 0.6.3 on top of the DoG SIFT stages (kornia_sift.cuh).  Stages:
//   pyramid   ScalePyramid(3, 1.6, 32, double_image=False): octave 0 at the input resolution, first blurred by sqrt(1.6^2 - 0.5^2);
//             then CornerGFTT on every Gaussian level (one fused kernel per octave); and kornia's pyrdown patch pyramid.
//   detect    ConvQuadInterp3d(10) on levels 0 .. 4 of the response volume, maxima only; then the SIFT detector's exact top-k,
//             border test and merge (ks_octave_list_kernel<.., 1>, ks_merge_kernel).
//   select    og_ksift_select (run_nms), unchanged.
//   describe  for the selected rows only, in chunks of rows: AffNet's standardised patches on make_upright(laf) -> AffNet's CNN
//             (im2col + GEMM, outside this file) -> tanh and the frame algebra, LAFOrienter(19) unless upright, HardNet's
//             standardised patches on the final LAF -> HardNet's CNN -> zero rows past the counts and F.normalize.
#pragma once
#include "kornia_sift.cuh"

namespace og {

constexpr int KG_PS = 32;                        // AffNet and HardNet patch size
constexpr int KG_TILE = 16;                      // GFTT output tile (threads 16 x 16)
constexpr int KG_HALO = 3;                       // the 7x7 blur's radius

// The 7x7 sigma-1 Gaussian (get_gaussian_kernel2d, float32 outer product) and sigma^4 of the six levels of an octave
struct KgGftt { float k2[49]; float s4[KS_LEVELS]; };

// gftt_response of every Gaussian level of one octave: vol[b][l] (6 levels).  grid (cdiv(w, 16), cdiv(h, 16), B * 6), 256 threads.
// The Sobel products of the 22 x 22 tile (the blur's reflect border applied to their positions; the Sobel's replicate border
// to the level) go to shared memory; each thread blurs one pixel and takes the smaller eigenvalue.
__global__ void __launch_bounds__(256) kg_gftt_kernel(const float* __restrict__ gauss, int h, int w, KgGftt g, float* __restrict__ vol) {
  constexpr int T = KG_TILE + 2 * KG_HALO;
  __shared__ float pxx[T][T], pyy[T][T], pxy[T][T];
  const int z = blockIdx.z, l = z % KS_LEVELS;
  const float* img = gauss + (int64_t)z * h * w;            // [B][6][h][w]: plane z is image z / 6, level z % 6
  const int x0 = blockIdx.x * KG_TILE - KG_HALO, y0 = blockIdx.y * KG_TILE - KG_HALO;
  const int tid = threadIdx.y * KG_TILE + threadIdx.x;
  for (int i = tid; i < T * T; i += 256) {
    const int ty = i / T, tx = i % T;
    const int yy = ks_reflect(y0 + ty, h), xx = ks_reflect(x0 + tx, w);
    auto P = [&](int dy, int dx) { return __ldg(img + (int64_t)min(max(yy + dy, 0), h - 1) * w + min(max(xx + dx, 0), w - 1)); };
    float gx = __fmul_rn(-0.125f, P(-1, -1));
    gx = __fadd_rn(gx, __fmul_rn(0.125f, P(-1, 1)));
    gx = __fadd_rn(gx, __fmul_rn(-0.25f, P(0, -1)));
    gx = __fadd_rn(gx, __fmul_rn(0.25f, P(0, 1)));
    gx = __fadd_rn(gx, __fmul_rn(-0.125f, P(1, -1)));
    gx = __fadd_rn(gx, __fmul_rn(0.125f, P(1, 1)));
    float gy = __fmul_rn(-0.125f, P(-1, -1));
    gy = __fadd_rn(gy, __fmul_rn(-0.25f, P(-1, 0)));
    gy = __fadd_rn(gy, __fmul_rn(-0.125f, P(-1, 1)));
    gy = __fadd_rn(gy, __fmul_rn(0.125f, P(1, -1)));
    gy = __fadd_rn(gy, __fmul_rn(0.25f, P(1, 0)));
    gy = __fadd_rn(gy, __fmul_rn(0.125f, P(1, 1)));
    pxx[ty][tx] = __fmul_rn(gx, gx);
    pyy[ty][tx] = __fmul_rn(gy, gy);
    pxy[ty][tx] = __fmul_rn(gx, gy);
  }
  __syncthreads();
  const int x = blockIdx.x * KG_TILE + threadIdx.x, y = blockIdx.y * KG_TILE + threadIdx.y;
  if (x >= w || y >= h) return;
  float a = 0.f, c = 0.f, bb = 0.f;
  for (int ky = 0; ky < 7; ++ky)
    for (int kx = 0; kx < 7; ++kx) {
      const float k = g.k2[ky * 7 + kx];
      a = __fmaf_rn(k, pxx[threadIdx.y + ky][threadIdx.x + kx], a);
      c = __fmaf_rn(k, pyy[threadIdx.y + ky][threadIdx.x + kx], c);
      bb = __fmaf_rn(k, pxy[threadIdx.y + ky][threadIdx.x + kx], bb);
    }
  const float det = __fsub_rn(__fmul_rn(a, c), __fmul_rn(bb, bb));
  const float tr = __fadd_rn(a, c);
  const float d = sqrtf(fabsf(__fsub_rn(__fmul_rn(tr, tr), __fmul_rn(4.f, det))));
  const float e1 = __fmul_rn(0.5f, __fadd_rn(tr, d)), e2 = __fmul_rn(0.5f, __fsub_rn(tr, d));
  vol[(int64_t)z * h * w + (int64_t)y * w + x] = __fmul_rn(fminf(e1, e2), g.s4[l]);
}

// conv_quad_interp3d responses (maxima only) of levels 0 .. 4 of one octave's 6-level volume: resp [B][5][h][w]
__global__ void kg_response_kernel(const float* __restrict__ vol, int B, int h, int w, float* __restrict__ resp) {
  const int64_t hw = (int64_t)h * w, per = (int64_t)KS_DOG * hw, n = B * per;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / per, r = i % per;
    const int x = (int)(r % w), y = (int)((r / w) % h), l = (int)(r / hw);
    resp[i] = ks_quad_interp(vol + b * KS_LEVELS * hw, 1.f, h, w, l, y, x).resp;
  }
}

// The detector output row of chunk row i: (b, j) of row r0 + i of the [B, out_cap] output, src its detector index (-1: past n[b])
__device__ __forceinline__ int kg_row(int r0, int out_cap, const int* __restrict__ sel, const int* __restrict__ n, int cap_in, int& b,
                                      int& j) {
  const int r = r0 + (int)blockIdx.x;
  b = r / out_cap; j = r % out_cap;
  if (j >= min(n[b], out_cap)) return -1;
  return sel ? sel[(int64_t)b * cap_in + j] : j;
}

// _normalize_input in place on patch[32 * 32] (shared) and the standardised patch to out: (x - mean) / (std + 1e-6), std with
// Bessel's correction
template <int THREADS>
__device__ void kg_standardize(const float* patch, float* red, float* __restrict__ out) {
  constexpr int N = KG_PS * KG_PS;
  float s = 0.f;
  for (int i = threadIdx.x; i < N; i += THREADS) s = __fadd_rn(s, patch[i]);
  s = cta_sum<THREADS>(s, red);
  __syncthreads();
  if (threadIdx.x == 0) red[0] = s;
  __syncthreads();
  const float mean = __fdiv_rn(red[0], (float)N);
  __syncthreads();
  float q = 0.f;
  for (int i = threadIdx.x; i < N; i += THREADS) { const float d = __fsub_rn(patch[i], mean); q = __fmaf_rn(d, d, q); }
  q = cta_sum<THREADS>(q, red);
  __syncthreads();
  if (threadIdx.x == 0) red[0] = q;
  __syncthreads();
  const float den = __fadd_rn(sqrtf(__fdiv_rn(red[0], (float)(N - 1))), 1e-6f);
  for (int i = threadIdx.x; i < N; i += THREADS) out[i] = __fdiv_rn(__fsub_rn(patch[i], mean), den);
  __syncthreads();
}

// make_upright of a LAF's 2x2 part (kornia.feature.laf.make_upright, with its scale_laf by the determinant's root)
__device__ __forceinline__ void kg_upright(const float a[6], float u[6]) {
  const float det = sqrtf(fabsf(__fadd_rn(__fsub_rn(__fmul_rn(a[0], a[4]), __fmul_rn(a[3], a[1])), 1e-10f)));
  const float b2a2 = __fadd_rn(sqrtf(__fadd_rn(__fmul_rn(a[1], a[1]), __fmul_rn(a[0], a[0]))), 1e-9f);
  u[0] = __fmul_rn(det, __fdiv_rn(b2a2, det)); u[1] = 0.f; u[2] = a[2];
  u[3] = __fmul_rn(det, __fdiv_rn(__fadd_rn(__fmul_rn(a[4], a[1]), __fmul_rn(a[3], a[0])), __fmul_rn(b2a2, det)));
  u[4] = __fmul_rn(det, __fdiv_rn(det, b2a2)); u[5] = a[5];
}

// AffNet's input for chunk rows [r0, r0 + gridDim.x): the standardised 32x32 patch of make_upright(lafs_in[sel[b][j]]) (zeros past
// n[b]).  One CTA per row; out [rows][32][32] (NHWC, one channel).
template <int THREADS>
__global__ void __launch_bounds__(THREADS) kg_affnet_patch_kernel(KsPyr P, int H, int W, const float* __restrict__ lafs_in, int cap_in,
                                                                  const int* __restrict__ sel, const int* __restrict__ n, int out_cap,
                                                                  int r0, float* __restrict__ out) {
  __shared__ float patch[KG_PS * KG_PS];
  __shared__ float red[THREADS / 32];
  float* o = out + (int64_t)blockIdx.x * KG_PS * KG_PS;
  int b, j;
  const int src = kg_row(r0, out_cap, sel, n, cap_in, b, j);
  if (src < 0) {
    for (int i = threadIdx.x; i < KG_PS * KG_PS; i += THREADS) o[i] = 0.f;
    return;
  }
  float a[6], u[6];
  for (int e = 0; e < 6; ++e) a[e] = lafs_in[((int64_t)b * cap_in + src) * 6 + e];
  kg_upright(a, u);
  ks_patch<KG_PS>(P, b, H, W, u, patch);
  __syncthreads();
  kg_standardize<THREADS>(patch, red, o);
}

// LAFAffNetShapeEstimator(preserve_orientation=True) after the network: v [3] (AffNet's 8x8-conv output, before tanh) and the
// input LAF d -> the affine LAF a at d's centre, with d's orientation
__device__ __forceinline__ void kg_affine_frame(const float* v, const float d[6], float a[6]) {
  const float t0 = tanhf(v[0]), t1 = tanhf(v[1]), t2 = tanhf(v[2]);   // AdaptiveAvgPool2d(1) of a 1x1 map: the value itself
  // new_laf = [[1 + t0, 0 t0], [t1, 1 + t2]] at the original centre
  const float nl[6] = {__fadd_rn(1.f, t0), __fmul_rn(0.f, t0), d[2], t1, __fadd_rn(1.f, t2), d[5]};
  const float scale_orig = sqrtf(fabsf(__fadd_rn(__fsub_rn(__fmul_rn(d[0], d[4]), __fmul_rn(d[3], d[1])), 1e-10f)));
  const float ori_orig = __fdiv_rn(__fmul_rn(180.f, atan2f(d[1], d[0])), KS_PI);
  const float ellipse = sqrtf(fabsf(__fadd_rn(__fsub_rn(__fmul_rn(nl[0], nl[4]), __fmul_rn(nl[3], nl[1])), 1e-10f)));
  const float coef = __fdiv_rn(scale_orig, ellipse);
  float u[6], s[6];
  kg_upright(nl, u);                                    // scale_laf(make_upright(new_laf), scale_orig / ellipse_scale)
  s[0] = __fmul_rn(u[0], coef); s[1] = __fmul_rn(u[1], coef); s[2] = u[2];
  s[3] = __fmul_rn(u[3], coef); s[4] = __fmul_rn(u[4], coef); s[5] = u[5];
  // set_laf_orientation(s, ori_orig) = rotate_laf(make_upright(s), ori_orig - get_laf_orientation(s))
  const float cur = __fdiv_rn(__fmul_rn(180.f, atan2f(s[1], s[0])), KS_PI);
  const float rad = __fdiv_rn(__fmul_rn(__fsub_rn(ori_orig, cur), KS_PI), 180.f);
  const float cs = cosf(rad), sn = sinf(rad);
  kg_upright(s, u);
  a[0] = __fadd_rn(__fmul_rn(u[0], cs), __fmul_rn(u[1], -sn));
  a[1] = __fadd_rn(__fmul_rn(u[0], sn), __fmul_rn(u[1], cs));
  a[3] = __fadd_rn(__fmul_rn(u[3], cs), __fmul_rn(u[4], -sn));
  a[4] = __fadd_rn(__fmul_rn(u[3], sn), __fmul_rn(u[4], cs));
  a[2] = d[2]; a[5] = d[5];
}

// After AffNet's CNN, chunk rows [r0, r0 + gridDim.x): xy [rows][3] (before tanh) and the detector LAF -> the affine LAF
// (LAFAffNetShapeEstimator with preserve_orientation), then LAFOrienter(19) unless upright; writes the row's LAF, score and angle
// and HardNet's standardised patch on the final LAF (out [rows][32][32]).  Rows past n[b] get zeros.
template <int THREADS>
__global__ void __launch_bounds__(THREADS) kg_frame_kernel(KsPyr P, int H, int W, const float* __restrict__ lafs_in,
                                                           const float* __restrict__ resp_in, int cap_in, const int* __restrict__ sel,
                                                           const int* __restrict__ n, int out_cap, int r0, const float* __restrict__ xy,
                                                           int upright, const KsDescConst* __restrict__ K, float* __restrict__ lafs_out,
                                                           float* __restrict__ scores, float* __restrict__ angle, float* __restrict__ out) {
  __shared__ float patch[KG_PS * KG_PS];                   // the 19-pixel orientation patch, then the 32-pixel HardNet patch
  __shared__ float wa[KS_ORI_PS * KS_ORI_PS], wb[KS_ORI_PS * KS_ORI_PS];
  __shared__ unsigned char bin[KS_ORI_PS * KS_ORI_PS];
  __shared__ float hist[KS_ORI_BINS];
  __shared__ float red[THREADS / 32];
  __shared__ float la[6];
  float* o = out + (int64_t)blockIdx.x * KG_PS * KG_PS;
  int b, j;
  const int src = kg_row(r0, out_cap, sel, n, cap_in, b, j);
  const int64_t row = (int64_t)b * out_cap + j;
  if (src < 0) {
    for (int i = threadIdx.x; i < KG_PS * KG_PS; i += THREADS) o[i] = 0.f;
    if (threadIdx.x < 6) lafs_out[row * 6 + threadIdx.x] = 0.f;
    if (threadIdx.x == 0) { scores[row] = 0.f; if (angle) angle[row] = 0.f; }
    return;
  }
  float d[6], a[6];
  for (int e = 0; e < 6; ++e) d[e] = lafs_in[((int64_t)b * cap_in + src) * 6 + e];
  kg_affine_frame(xy + (int64_t)blockIdx.x * 3, d, a);
  if (threadIdx.x < 6) la[threadIdx.x] = a[threadIdx.x];
  __syncthreads();
  float ang = 0.f;
  if (!upright) ang = ks_orient<THREADS>(P, b, H, W, K, a, patch, wa, wb, bin, hist, la);
  ks_patch<KG_PS>(P, b, H, W, a, patch);
  __syncthreads();
  kg_standardize<THREADS>(patch, red, o);
  if (threadIdx.x < 6) lafs_out[row * 6 + threadIdx.x] = a[threadIdx.x];
  if (threadIdx.x == 0) {
    scores[row] = resp_in[(int64_t)b * cap_in + src];
    if (angle) angle[row] = ang;
  }
}

// 3x3, stride 2, pad 1 im2col on NHWC: out[p, (3 ky + kx) C + c] = x[b, 2 oy + ky - 1, 2 ox + kx - 1, c] (zero padding),
// p over [B, ceil(H / 2), ceil(W / 2)]
__global__ void __launch_bounds__(256) kg_im2col3x3_s2_kernel(const float* __restrict__ x, int B, int H, int W, int C,
                                                              float* __restrict__ out) {
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const int64_t P = (int64_t)B * Ho * Wo;
  const int cv = (C % 4 == 0) ? C / 4 : C;                  // float4 columns when C allows
  const int64_t total = P * 9 * cv;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int c = (int)(i % cv);
    const int tap = (int)((i / cv) % 9);
    const int64_t p = i / (9 * cv);
    const int ox = (int)(p % Wo), oy = (int)((p / Wo) % Ho);
    const int64_t b = p / ((int64_t)Wo * Ho);
    const int sy = 2 * oy + tap / 3 - 1, sx = 2 * ox + tap % 3 - 1;
    const bool in = sy >= 0 && sy < H && sx >= 0 && sx < W;
    if (C % 4 == 0) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (in) v = __ldg(reinterpret_cast<const float4*>(x + ((b * H + sy) * W + sx) * C) + c);
      reinterpret_cast<float4*>(out + p * 9 * C + (int64_t)tap * C)[c] = v;
    } else {
      out[p * 9 * C + (int64_t)tap * C + c] = in ? __ldg(x + ((b * H + sy) * W + sx) * C + c) : 0.f;
    }
  }
}

// HardNet's output rows: F.normalize (x / max(||x||_2, 1e-12)) on rows j < n[b], zeros past them.  One warp per row of [B, out_cap].
__global__ void kg_desc_finish_kernel(float* __restrict__ desc, int B, int out_cap, const int* __restrict__ n) {
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  if (row >= (int64_t)B * out_cap) return;
  const int b = (int)(row / out_cap), j = (int)(row % out_cap), lane = threadIdx.x & 31;
  float4* d = reinterpret_cast<float4*>(desc + row * 128) + lane;
  float4 v = *d;
  if (j >= min(n[b], out_cap)) { *d = make_float4(0.f, 0.f, 0.f, 0.f); return; }
  float s = __fadd_rn(__fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y)), __fadd_rn(__fmul_rn(v.z, v.z), __fmul_rn(v.w, v.w)));
  for (int o = 16; o > 0; o >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
  const float nn = fmaxf(sqrtf(s), 1e-12f);
  *d = make_float4(__fdiv_rn(v.x, nn), __fdiv_rn(v.y, nn), __fdiv_rn(v.z, nn), __fdiv_rn(v.w, nn));
}

}  // namespace og
