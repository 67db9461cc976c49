// SuperPoint front-end (SURVEY.md section 8, row f4): the detector / descriptor network that produces the keypoints the matching
// core consumes when features are not cached (reference models/features/superpoint/model.py:61-129, superpoint/utils.py:4-39).
//
// Layout: activations are NHWC ([B, H, W, C] = [pixels, channels] row-major), so every convolution is a GEMM over pixels:
//   3x3, pad 1:  Y[p, co] = relu(sum_{tap, ci} X[p + off(tap), ci] W[co, tap, ci] + b[co])  = im2col (this file) + the tensor-core GEMM
//                of the library (og_linear_auto_fwd: 3xTF32 wgmma for K = 9 C >= 32, exact fp32 for the 1-channel input layer),
//   1x1:         the GEMM alone.
// The rest of the front-end is HBM-bound index work, one kernel each: 2x2 max-pool, channel L2 norm, cell softmax -> pixel heat
// map -> non-maximum suppression + threshold + border removal, ordered compaction, top-k (bitonic sort in shared memory),
// bilinear descriptor sampling + normalisation.
//
// Non-maximum suppression restates kornia.geometry.subpix.nms2d (kornia >= 0.6.1 per the reference's requirements.txt; kornia is
// not installed in the build container, so THIS piece is pinned to the published algorithm, not to an execution of it):
//   keep x[p] iff x[p] > max(0, x[q] for the k*k - 1 other offsets q of the window, coordinates clamped to the image (replicate padding)).
#pragma once
#include "common.cuh"
#include <algorithm>

namespace og {

// ---------------------------------------------------------------------------------------------------------------------
// im2col for a 3x3 / stride 1 / zero-pad 1 convolution on NHWC: out[p, tap * C + c] = x[b, y + ky - 1, x + kx - 1, c], tap = 3 ky + kx
__global__ void __launch_bounds__(256) im2col3x3_kernel(const float* __restrict__ x, int B, int H, int W, int C, float* __restrict__ out) {
  const int64_t P = (int64_t)B * H * W;
  if (C % 4 == 0) {
    const int c4n = C / 4;
    const int64_t total = P * 9 * c4n;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
      const int c4 = (int)(i % c4n);
      const int tap = (int)((i / c4n) % 9);
      const int64_t p = i / (9 * c4n);
      const int xx = (int)(p % W), yy = (int)((p / W) % H);
      const int64_t b = p / ((int64_t)W * H);
      const int sy = yy + tap / 3 - 1, sx = xx + tap % 3 - 1;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (sy >= 0 && sy < H && sx >= 0 && sx < W) v = __ldg(reinterpret_cast<const float4*>(x + ((b * H + sy) * W + sx) * C) + c4);
      reinterpret_cast<float4*>(out + p * 9 * C + (int64_t)tap * C)[c4] = v;
    }
  } else {
    const int64_t total = P * 9 * C;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
      const int c = (int)(i % C);
      const int tap = (int)((i / C) % 9);
      const int64_t p = i / (9 * C);
      const int xx = (int)(p % W), yy = (int)((p / W) % H);
      const int64_t b = p / ((int64_t)W * H);
      const int sy = yy + tap / 3 - 1, sx = xx + tap % 3 - 1;
      out[i] = (sy >= 0 && sy < H && sx >= 0 && sx < W) ? __ldg(x + ((b * H + sy) * W + sx) * C + c) : 0.f;
    }
  }
}

// 2x2 / stride 2 max-pool on NHWC (H, W even)
__global__ void __launch_bounds__(256) maxpool2x2_kernel(const float* __restrict__ x, int B, int H, int W, int C, float* __restrict__ out) {
  const int Ho = H / 2, Wo = W / 2;
  const int64_t total = (int64_t)B * Ho * Wo * C;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int c = (int)(i % C);
    const int xo = (int)((i / C) % Wo), yo = (int)((i / ((int64_t)C * Wo)) % Ho);
    const int64_t b = i / ((int64_t)C * Wo * Ho);
    const float* s = x + ((b * H + 2 * yo) * W + 2 * xo) * C + c;
    out[i] = fmaxf(fmaxf(s[0], s[C]), fmaxf(s[(int64_t)W * C], s[(int64_t)W * C + C]));
  }
}

// x[r, :] /= ||x[r, :]||_2 (mode 0: torch.norm + div, model.py:70-71)  or  /= max(||.||, eps) (mode 1: F.normalize).  One warp per row.
__global__ void __launch_bounds__(256) row_normalize_kernel(float* __restrict__ x, int64_t rows, int C, int mode, float eps) {
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float* r = x + row * C;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s = fmaf(r[c], r[c], s);
  s = warp_sum(s);
  float nrm = __fsqrt_rn(s);
  if (mode == 1) nrm = fmaxf(nrm, eps);
  for (int c = lane; c < C; c += 32) r[c] = __fdiv_rn(r[c], nrm);
}

// cell probabilities [B, Hc, Wc, 65] (after the channel softmax; channel 64 = "no keypoint") -> per-pixel scores of the H = 8 Hc,
// W = 8 Wc image (model.py:84-86), non-maximum suppression (kornia nms2d, see the header), F.threshold(s, thr, 0) + nonzero
// (model.py:89-92) and remove_borders (utils.py:4-11) in one pass: heat[b, y, x] = the score if the pixel survives, else 0.
__global__ void __launch_bounds__(256) sp_heat_nms_kernel(const float* __restrict__ probs, int B, int Hc, int Wc, int nms, float thr, int border,
                                                          float* __restrict__ heat) {
  const int H = 8 * Hc, W = 8 * Wc, r = nms / 2;
  const int64_t total = (int64_t)B * H * W;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int xx = (int)(i % W), yy = (int)((i / W) % H);
    const int64_t b = i / ((int64_t)W * H);
    const float* pb = probs + b * Hc * Wc * 65;
    auto at = [&](int y, int x) { return __ldg(pb + ((int64_t)(y >> 3) * Wc + (x >> 3)) * 65 + ((y & 7) * 8 + (x & 7))); };
    const float v = at(yy, xx);
    bool keep = v > 0.f && v > thr && yy >= border && yy < H - border && xx >= border && xx < W - border;
    for (int dy = -r; dy <= r && keep; ++dy) {
      const int y2 = min(max(yy + dy, 0), H - 1);
      for (int dx = -r; dx <= r; ++dx) {
        if (dy == 0 && dx == 0) continue;
        const int x2 = min(max(xx + dx, 0), W - 1);
        if (!(v > at(y2, x2))) { keep = false; break; }
      }
    }
    heat[i] = keep ? v : 0.f;
  }
}

// ordered compaction of the surviving pixels of one image (torch.nonzero order = row-major): cand_idx / cand_score [B, cap], count [B]
// (count may exceed cap: the caller checks).  One CTA of 1024 threads per image.
__global__ void __launch_bounds__(1024) sp_compact_kernel(const float* __restrict__ heat, int HW, int cap, int* __restrict__ cand_idx,
                                                          float* __restrict__ cand_score, int* __restrict__ count) {
  __shared__ int warp_tot[32];
  __shared__ int base;
  const int b = blockIdx.x, tid = threadIdx.x;
  const float* h = heat + (int64_t)b * HW;
  if (tid == 0) base = 0;
  __syncthreads();
  for (int p0 = 0; p0 < HW; p0 += 1024) {
    const int p = p0 + tid;
    const float v = p < HW ? h[p] : 0.f;
    const bool on = v != 0.f;
    const int pos = cta_ordered_slot(on, warp_tot, base);
    if (on && pos < cap) { cand_idx[(int64_t)b * cap + pos] = p; cand_score[(int64_t)b * cap + pos] = v; }
  }
  if (tid == 0) count[b] = base;
}

// selection of n_out[b] keypoints of image b from its candidate list: mode[b] = 0 keep the (row-major) order, 1 = the n_out largest
// scores in descending order (torch.topk; equal scores: lower index first).  Outputs keypoints as (x, y) floats (model.py:108),
// scores, both [B, out_cap, ...].  One CTA per image; the sort is cta_topk_sort's, of (score, position) in shared memory.
// Caller contract (not checked on the device): n_out[b] <= min(count[b], cap) and n_out[b] <= out_cap, and max_count >= every count[b]
// (it sizes the shared memory); a larger n_out reads candidate slots that were never written.
__global__ void __launch_bounds__(1024) sp_select_kernel(const int* __restrict__ cand_idx, const float* __restrict__ cand_score,
                                                         const int* __restrict__ count, const int* __restrict__ n_out, const int* __restrict__ mode,
                                                         int cap, int W, int out_cap, float* __restrict__ kpts, float* __restrict__ scores) {
  extern __shared__ __align__(16) unsigned char og_sp_smem[];
  float* key = reinterpret_cast<float*>(og_sp_smem);
  const int b = blockIdx.x, tid = threadIdx.x;
  const int cnt = min(count[b], cap), n = n_out[b];
  const int* ci = cand_idx + (int64_t)b * cap;
  const float* cs = cand_score + (int64_t)b * cap;
  int* val = reinterpret_cast<int*>(key + pow2_ceil(cnt));
  // <0>: the sort strides by blockDim.x.  Here that runs faster than the loop unrolled for the constant 1024 (collate is the
  // other way round), so the choice is deliberate.
  if (mode[b]) cta_topk_sort<0>(cs, cnt, key, val);
  for (int j = tid; j < n; j += 1024) {
    const int src = mode[b] ? val[j] : j;
    const int p = ci[src];
    kpts[((int64_t)b * out_cap + j) * 2 + 0] = (float)(p % W);
    kpts[((int64_t)b * out_cap + j) * 2 + 1] = (float)(p / W);
    scores[(int64_t)b * out_cap + j] = cs[src];
  }
}

// sample_desc_from_points (utils.py:14-31): bilinear grid_sample (align_corners = False, zero padding) of the coarse descriptor map
// at the keypoints + F.normalize.  coarse [B, Hc, Wc, D] NHWC; kpts [B, out_cap, 2] (x, y); desc [B, out_cap, D].  One warp per keypoint.
__global__ void __launch_bounds__(256) sp_sample_desc_kernel(const float* __restrict__ coarse, int Hc, int Wc, int D, const float* __restrict__ kpts,
                                                             const int* __restrict__ n_out, int out_cap, int cell, float* __restrict__ desc) {
  const int b = blockIdx.y;
  const int j = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (j >= n_out[b]) return;
  const float H = (float)(Hc * cell), W = (float)(Wc * cell), half = (float)cell / 2.f;
  float px = kpts[((int64_t)b * out_cap + j) * 2 + 0], py = kpts[((int64_t)b * out_cap + j) * 2 + 1];
  px = (px - half) + 0.5f; py = (py - half) + 0.5f;                      // pts - cell / 2 + 0.5
  px = __fdiv_rn(px, W - half - 0.5f); py = __fdiv_rn(py, H - half - 0.5f);
  px = px * 2.f - 1.f; py = py * 2.f - 1.f;
  const float ix = __fdiv_rn((px + 1.f) * (float)Wc - 1.f, 2.f), iy = __fdiv_rn((py + 1.f) * (float)Hc - 1.f, 2.f);   // grid_sampler_unnormalize
  const float fx = floorf(ix), fy = floorf(iy);
  const int x0 = (int)fx, y0 = (int)fy, x1 = x0 + 1, y1 = y0 + 1;
  const float wx1 = ix - fx, wy1 = iy - fy, wx0 = 1.f - wx1, wy0 = 1.f - wy1;
  const float w00 = wx0 * wy0, w10 = wx1 * wy0, w01 = wx0 * wy1, w11 = wx1 * wy1;       // (nw, ne, sw, se)
  const float* cb = coarse + (int64_t)b * Hc * Wc * D;
  auto ok = [&](int y, int x) { return y >= 0 && y < Hc && x >= 0 && x < Wc; };
  float* o = desc + ((int64_t)b * out_cap + j) * D;
  float ss = 0.f;
  for (int c = lane; c < D; c += 32) {
    float v = 0.f;
    if (ok(y0, x0)) v = fmaf(cb[((int64_t)y0 * Wc + x0) * D + c], w00, v);
    if (ok(y0, x1)) v = fmaf(cb[((int64_t)y0 * Wc + x1) * D + c], w10, v);
    if (ok(y1, x0)) v = fmaf(cb[((int64_t)y1 * Wc + x0) * D + c], w01, v);
    if (ok(y1, x1)) v = fmaf(cb[((int64_t)y1 * Wc + x1) * D + c], w11, v);
    o[c] = v;
    ss = fmaf(v, v, ss);
  }
  ss = warp_sum(ss);
  const float nrm = fmaxf(__fsqrt_rn(ss), 1e-12f);
  __syncwarp();
  for (int c = lane; c < D; c += 32) o[c] = __fdiv_rn(o[c], nrm);
}

inline unsigned sp_grid(int64_t n) { return (unsigned)std::min<int64_t>((n + 255) / 256, 132 * 32); }

}  // namespace og
