// Local features -> matcher inputs, and matches -> the compact match list of stand-alone inference.
//
// prepare_features_kernel: prepare_features_output (reference models/features/utils.py:54-65) with the LAF converters of
// models/laf_converter.py:22-128.  For a local affine frame (LAF) [[a00, a01, x], [a10, a11, y]]:
//   s = sqrt(|(a00 a11 - a10 a01) + 1e-10|)   (kornia get_laf_scale; kornia is not installed in the build container, so this is
//                                               pinned to the published source, not to an execution of it)
//   keypoint = (x, y)                         (lafs[..., -1], kornia get_laf_center)
//   side     = [r or log(r + 0.1), then by method:  scale: log s | rotation: a01/s, a00/s | scale_rotation: log s, a01/s, a00/s |
//               affine: log s, a00/s, a01/s, a10/s, a11/s]
// Every product, difference, sum, quotient and square root is its own IEEE round-to-nearest operation, in ATen's order and without
// FMA contraction, so every column except the logs equals the reference's fp32 result bit for bit wherever ATen's square root is
// correctly rounded (its vectorised CPU sqrt is 1 ulp off on a few frames in a thousand; torch on CUDA rounds correctly, as this
// kernel does); logf is within an ulp of ATen's.
//
// match_compact_kernel: the boolean indexing of OpenGlueMatcher.forward (inference.py:192-209) on og_match_fwd's output.
#pragma once
#include "common.cuh"

namespace og {

__host__ __device__ inline int laf_side_dim(int method) {
  switch (method) {
    case OG_LAF_SCALE: return 1;
    case OG_LAF_ROTATION: return 2;
    case OG_LAF_SCALE_ROTATION: return 3;
    case OG_LAF_AFFINE: return 5;
    default: return 0;
  }
}

// One thread per keypoint.  lafs [R, 2, 3]; responses [R] or NULL (no response column); kpts [R, 2] or NULL; side [R, width].
__global__ void __launch_bounds__(256) prepare_features_kernel(const float* __restrict__ lafs, const float* __restrict__ responses, int64_t R,
                                                               int method, int log_response, float* __restrict__ kpts,
                                                               float* __restrict__ side, int width) {
  const int64_t r = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (r >= R) return;
  const float* l = lafs + r * 6;
  const float a00 = l[0], a01 = l[1], x = l[2], a10 = l[3], a11 = l[4], y = l[5];
  if (kpts) { kpts[r * 2] = x; kpts[r * 2 + 1] = y; }
  float* o = side + r * width;
  if (responses) {
    const float v = responses[r];
    *o++ = log_response ? logf(__fadd_rn(v, 0.1f)) : v;                           // (responses + 0.1).log()
  }
  if (method == OG_LAF_NONE) return;
  const float det = __fadd_rn(__fsub_rn(__fmul_rn(a00, a11), __fmul_rn(a10, a01)), 1e-10f);
  const float s = __fsqrt_rn(fabsf(det));
  if (method != OG_LAF_ROTATION) *o++ = logf(s);
  if (method == OG_LAF_ROTATION || method == OG_LAF_SCALE_ROTATION) {             // flip(lafs[..., 0, :-1]) / s
    *o++ = __fdiv_rn(a01, s);
    *o++ = __fdiv_rn(a00, s);
  } else if (method == OG_LAF_AFFINE) {                                           // flatten(lafs[..., :-1]) / s
    *o++ = __fdiv_rn(a00, s);
    *o++ = __fdiv_rn(a01, s);
    *o++ = __fdiv_rn(a10, s);
    *o++ = __fdiv_rn(a11, s);
  }
}

// Ordered compaction of the matches of B pairs, in boolean-indexing order (pair-major, then i).  A row is a match iff
// matches0[b, i] >= 0 (og_match_fwd leaves -1 elsewhere); its score is not consulted, so a mutual match whose exp underflowed to 0
// still counts when the threshold is negative.  One CTA of 1024 threads walks the B n rows in order (cta_ordered_slot), so the
// output order never depends on scheduling.  total[0] = the number of matches.
__global__ void __launch_bounds__(1024) match_compact_kernel(const int64_t* __restrict__ matches0, const float* __restrict__ mscores0,
                                                             const float* __restrict__ lafs0, const float* __restrict__ lafs1, int rows,
                                                             int n, int m, int64_t* __restrict__ pair, int64_t* __restrict__ ij,
                                                             float* __restrict__ conf, float* __restrict__ out_lafs0,
                                                             float* __restrict__ out_lafs1, float* __restrict__ out_kpts0,
                                                             float* __restrict__ out_kpts1, int64_t* __restrict__ total) {
  __shared__ int warp_tot[32];
  __shared__ int base;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  for (int r0 = 0; r0 < rows; r0 += 1024) {
    const int r = r0 + (int)threadIdx.x;
    const int64_t j = r < rows ? matches0[r] : -1;
    const bool on = j >= 0;
    const int pos = cta_ordered_slot(on, warp_tot, base);
    if (!on) continue;
    const int b = r / n, i = r - b * n;
    pair[pos] = b;
    ij[2 * (int64_t)pos] = i;
    ij[2 * (int64_t)pos + 1] = j;
    conf[pos] = mscores0[r];
    const float* l0 = lafs0 + (int64_t)r * 6;
    const float* l1 = lafs1 + ((int64_t)b * m + j) * 6;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      out_lafs0[(int64_t)pos * 6 + k] = l0[k];
      out_lafs1[(int64_t)pos * 6 + k] = l1[k];
    }
    out_kpts0[2 * (int64_t)pos] = l0[2];
    out_kpts0[2 * (int64_t)pos + 1] = l0[5];
    out_kpts1[2 * (int64_t)pos] = l1[2];
    out_kpts1[2 * (int64_t)pos + 1] = l1[5];
  }
  if (threadIdx.x == 0) total[0] = base;
}

// The kept count of image b of a front-end output padded to K rows, from its device count: of count[b] keypoints the first
// min(count[b], cap) were stored; the top-k keeps max_keypoints of them when max_keypoints >= 0 cuts that number (mode[b] = 1: by
// score) and all of them otherwise (mode[b] = 0: in stored order), as top_k_keypoints (superpoint/utils.py:34-39) decides per
// image.  n_out[b] = that number clamped to K; overflow[b] |= 1 when count[b] > cap or the kept number exceeds K.  mode may be NULL.
__global__ void __launch_bounds__(256) keypoint_counts_kernel(const int* __restrict__ count, int B, int cap, int max_keypoints, int K,
                                                              int* __restrict__ n_out, int* __restrict__ mode, int* __restrict__ overflow) {
  const int b = blockIdx.x * 256 + threadIdx.x;
  if (b >= B) return;
  const int c = count[b], stored = max(0, min(c, cap));
  const bool top = max_keypoints >= 0 && max_keypoints < stored;
  const int keep = top ? max_keypoints : stored;
  n_out[b] = min(keep, K);
  if (mode) mode[b] = top ? 1 : 0;
  if (c > cap || keep > K) overflow[b] = 1;
}

// matches0 / mscores0 [B, n], matches1 / mscores1 [B, m]: -1 and 0 in every slot of a pair with no keypoint in either image
// (len0[b] == 0 or len1[b] == 0).  The padded matcher clamps each length to at least 1, so it matches row 0 of an empty image.
__global__ void __launch_bounds__(256) mask_empty_pairs_kernel(const int* __restrict__ len0, const int* __restrict__ len1, int B, int n, int m,
                                                               int64_t* __restrict__ matches0, float* __restrict__ mscores0,
                                                               int64_t* __restrict__ matches1, float* __restrict__ mscores1) {
  const int64_t rows0 = (int64_t)B * n, total = rows0 + (int64_t)B * m;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const bool first = i < rows0;
    const int64_t r = first ? i : i - rows0;
    const int b = (int)(r / (first ? n : m));
    if (__ldg(len0 + b) > 0 && __ldg(len1 + b) > 0) continue;
    if (first) { matches0[r] = -1; mscores0[r] = 0.f; }
    else { matches1[r] = -1; mscores1[r] = 0.f; }
  }
}

}  // namespace og
