// Ground-truth match generation: the step immediately before the matching core in the reference's training /
// validation step (models/matching_module.py:84-93 -> models/gt_matches_generation.py:17-93, utils/misc.py:21-103).
//   1. reproject keypoints0 with the pair's transformation and keypoints1 with its inverse
//      (homography: utils/misc.py:62-71; relative pose + depth: utils/misc.py:74-103, inverse :37-59)
//   2. nearest neighbour of every reprojected point among the other image's keypoints (torch.cdist + min, :40-44)
//   3. mutual check, UNMATCHED (-1) / IGNORE (-2, unknown depth) marks (:45-51, :72-73)
// The reference's threshold refinements (:56-67, :76-78) write through boolean-mask copies and have no effect;
// they are not reproduced (see oracle/gt_matches_oracle.py).  The two N x M distance matrices (2 x 268 MB at 16 pairs,
// N = M = 2048) are never formed: each thread keeps the running minimum of its query point over shared-memory tiles
// of the targets.  CUDA-core work, ~10 FLOP per point pair.
#pragma once
#include "common.cuh"
#include <math_constants.h>

namespace og {

struct GtPrepared {            // per pair and direction: what the reprojection needs, row-major 3x3
  float m[9];                  // perspective: H (or H^-1).  3d: K_src^-1
  float r[9];                  // 3d: R (or R^T)
  float k[9];                  // 3d: K_dst
  float t[3];                  // 3d: T (or -R^T T)
};

__device__ __forceinline__ void inv3x3(const float* a, float* o) {
  const float c00 = a[4] * a[8] - a[5] * a[7], c01 = a[5] * a[6] - a[3] * a[8], c02 = a[3] * a[7] - a[4] * a[6];
  const float det = a[0] * c00 + a[1] * c01 + a[2] * c02;
  const float id = 1.0f / det;
  o[0] = c00 * id; o[1] = (a[2] * a[7] - a[1] * a[8]) * id; o[2] = (a[1] * a[5] - a[2] * a[4]) * id;
  o[3] = c01 * id; o[4] = (a[0] * a[8] - a[2] * a[6]) * id; o[5] = (a[2] * a[3] - a[0] * a[5]) * id;
  o[6] = c02 * id; o[7] = (a[1] * a[6] - a[0] * a[7]) * id; o[8] = (a[0] * a[4] - a[1] * a[3]) * id;
}

// one thread per (pair, direction): direction 0 maps image 0 -> 1, direction 1 is the inverse transformation
__global__ void gt_prepare_kernel(og_gt_transform tf, int B, GtPrepared* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * B) return;
  const int b = i >> 1, dir = i & 1;
  GtPrepared p;
  if (tf.type == OG_GT_PERSPECTIVE) {
    const float* H = tf.H + 9 * b;
    if (dir == 0) { for (int k = 0; k < 9; ++k) p.m[k] = H[k]; } else inv3x3(H, p.m);          // utils/misc.py:41-44
    for (int k = 0; k < 9; ++k) { p.r[k] = 0.f; p.k[k] = 0.f; }
    p.t[0] = p.t[1] = p.t[2] = 0.f;
  } else {
    const float* Ks = (dir == 0 ? tf.K0 : tf.K1) + 9 * b;                                      // utils/misc.py:50-52
    const float* Kd = (dir == 0 ? tf.K1 : tf.K0) + 9 * b;
    const float* R = tf.R + 9 * b;
    const float* T = tf.T + 3 * b;
    inv3x3(Ks, p.m);                                                                            // utils/misc.py:80
    for (int k = 0; k < 9; ++k) p.k[k] = Kd[k];
    if (dir == 0) {
      for (int k = 0; k < 9; ++k) p.r[k] = R[k];
      p.t[0] = T[0]; p.t[1] = T[1]; p.t[2] = T[2];
    } else {                                                                                    // R^T, -R^T T  (:49-55)
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) p.r[3 * r + c] = R[3 * c + r];
      for (int r = 0; r < 3; ++r) p.t[r] = -(p.r[3 * r] * T[0] + p.r[3 * r + 1] * T[1] + p.r[3 * r + 2] * T[2]);
    }
  }
  out[i] = p;
}

__device__ __forceinline__ void mat3_apply(const float* m, float x, float y, float z, float& ox, float& oy, float& oz) {
  ox = fmaf(m[2], z, fmaf(m[1], y, m[0] * x));
  oy = fmaf(m[5], z, fmaf(m[4], y, m[3] * x));
  oz = fmaf(m[8], z, fmaf(m[7], y, m[6] * x));
}

// one thread per keypoint of image `dir`; out: reprojected xy and validity mask
__global__ void gt_reproject_kernel(const float* __restrict__ kpts, int n, int dir, og_gt_transform tf,
                                    const GtPrepared* __restrict__ prep, float2* __restrict__ out, uint8_t* __restrict__ mask) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const GtPrepared& p = prep[2 * b + dir];
  const float x = kpts[((int64_t)b * n + i) * 2], y = kpts[((int64_t)b * n + i) * 2 + 1];
  const float eps = 1e-8f;
  float ox, oy, oz;
  bool ok = true;
  if (tf.type == OG_GT_PERSPECTIVE) {
    mat3_apply(p.m, x, y, 1.f, ox, oy, oz);                                                     // utils/misc.py:66-69
  } else {
    const float* dsrc = dir == 0 ? tf.depth0 : tf.depth1;
    float depth;
    if (tf.depth_is_image) {                                                                    // utils/misc.py:90-97
      const int dh = dir == 0 ? tf.depth0_h : tf.depth1_h, dw = dir == 0 ? tf.depth0_w : tf.depth1_w;
      int xi = (int)x, yi = (int)y;                                                             // .type(torch.int64): truncation
      xi = min(max(xi, 0), dw - 1); yi = min(max(yi, 0), dh - 1);                               // (the reference would raise out of range)
      depth = dsrc[((int64_t)b * dh + yi) * dw + xi];
    } else {
      depth = dsrc[(int64_t)b * n + i];
    }
    ok = !(fabsf(depth) <= 1e-8f);                                                              // ~isclose(depth, 0): atol 1e-8
    float rx, ry, rz;
    mat3_apply(p.m, x, y, 1.f, rx, ry, rz);                                                     // rays = [x y 1] K0^-T
    rx *= depth; ry *= depth; rz *= depth;
    float cx, cy, cz;
    mat3_apply(p.r, rx, ry, rz, cx, cy, cz);                                                    // R x + T
    cx += p.t[0]; cy += p.t[1]; cz += p.t[2];
    mat3_apply(p.k, cx, cy, cz, ox, oy, oz);                                                    // K1 x
  }
  const float den = oz + eps;
  out[(int64_t)b * n + i] = make_float2(ox / den, oy / den);
  mask[(int64_t)b * n + i] = ok ? 1 : 0;
}

// nearest target of every query point (first index on ties, like torch.min); targets stream through shared memory.
// A padded batch (tlen set) searches each pair's first tlen[b] targets only.
constexpr int GT_TILE = 2048;
__global__ void __launch_bounds__(256) gt_nearest_kernel(const float2* __restrict__ q, int nq, const float* __restrict__ targets, int nt_cap,
                                                         const int* __restrict__ tlen, int* __restrict__ nn) {
  __shared__ float2 tile[GT_TILE];
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  const float2 me = i < nq ? q[(int64_t)b * nq + i] : make_float2(0.f, 0.f);
  const float2* tg = reinterpret_cast<const float2*>(targets) + (int64_t)b * nt_cap;
  const int nt = tlen ? padded_length(tlen, b, nt_cap) : nt_cap;
  float best = CUDART_INF_F;
  int best_j = 0;
  for (int j0 = 0; j0 < nt; j0 += GT_TILE) {
    const int cnt = min(GT_TILE, nt - j0);
    __syncthreads();
    for (int j = threadIdx.x; j < cnt; j += blockDim.x) tile[j] = tg[j0 + j];
    __syncthreads();
#pragma unroll 4
    for (int j = 0; j < cnt; ++j) {
      const float dx = me.x - tile[j].x, dy = me.y - tile[j].y;
      const float d2 = fmaf(dx, dx, dy * dy);
      if (d2 < best) { best = d2; best_j = j0 + j; }
    }
  }
  if (i < nq) nn[(int64_t)b * nq + i] = best_j;
}

// gt[i] = nn[i] if the neighbour points back, else -1; -2 where the reprojection was invalid   (:45-51, :72-73), and in a padded
// batch (alen set) past the pair's length
__global__ void gt_mutual_kernel(const int* __restrict__ nn_a, const int* __restrict__ nn_b, const uint8_t* __restrict__ mask_a,
                                 int na, int nb, const int* __restrict__ alen, int64_t* __restrict__ gt_a) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= na) return;
  if (alen && i >= padded_length(alen, b, na)) { gt_a[(int64_t)b * na + i] = -2; return; }
  const int j = nn_a[(int64_t)b * na + i];
  int64_t g = (nn_b[(int64_t)b * nb + j] == i) ? (int64_t)j : -1;
  if (!mask_a[(int64_t)b * na + i]) g = -2;
  gt_a[(int64_t)b * na + i] = g;
}

inline int64_t gt_matches_workspace_bytes(int B, int n, int m) {
  return align_up((int64_t)2 * B * sizeof(GtPrepared), 256) + align_up((int64_t)B * n * 8, 256) + align_up((int64_t)B * m * 8, 256) +
         align_up((int64_t)B * n, 256) + align_up((int64_t)B * m, 256) + align_up((int64_t)B * n * 4, 256) + align_up((int64_t)B * m * 4, 256);
}

inline int gt_matches_launch(const float* kpts0, const float* kpts1, int B, int n, int m, const og_gt_transform& tf,
                             int64_t* gt0, int64_t* gt1, void* ws, int64_t ws_bytes, cudaStream_t st, const int* lens = nullptr) {
  const int* len0 = lens;                              // padded batch: n_0 .. n_{B-1}, m_0 .. m_{B-1}
  const int* len1 = lens ? lens + B : nullptr;
  if (ws_bytes < gt_matches_workspace_bytes(B, n, m)) return fail(OG_EWORKSPACE, "gt_matches: workspace too small");
  char* w = static_cast<char*>(ws);
  auto take = [&](int64_t bytes) { char* p = w; w += align_up(bytes, 256); return p; };
  GtPrepared* prep = reinterpret_cast<GtPrepared*>(take((int64_t)2 * B * sizeof(GtPrepared)));
  float2* k0t = reinterpret_cast<float2*>(take((int64_t)B * n * 8));
  float2* k1t = reinterpret_cast<float2*>(take((int64_t)B * m * 8));
  uint8_t* mask0 = reinterpret_cast<uint8_t*>(take((int64_t)B * n));
  uint8_t* mask1 = reinterpret_cast<uint8_t*>(take((int64_t)B * m));
  int* nn0 = reinterpret_cast<int*>(take((int64_t)B * n * 4));
  int* nn1 = reinterpret_cast<int*>(take((int64_t)B * m * 4));
  int rc;
  if ((rc = OG_LAUNCH(gt_prepare_kernel, cdiv(2 * B, 64), 64, 0, st, tf, B, prep))) return rc;
  if ((rc = OG_LAUNCH(gt_reproject_kernel, dim3(cdiv(n, 256), B), 256, 0, st, kpts0, n, 0, tf, prep, k0t, mask0))) return rc;
  if ((rc = OG_LAUNCH(gt_reproject_kernel, dim3(cdiv(m, 256), B), 256, 0, st, kpts1, m, 1, tf, prep, k1t, mask1))) return rc;
  if ((rc = OG_LAUNCH(gt_nearest_kernel, dim3(cdiv(n, 256), B), 256, 0, st, k0t, n, kpts1, m, len1, nn0))) return rc;
  if ((rc = OG_LAUNCH(gt_nearest_kernel, dim3(cdiv(m, 256), B), 256, 0, st, k1t, m, kpts0, n, len0, nn1))) return rc;
  if ((rc = OG_LAUNCH(gt_mutual_kernel, dim3(cdiv(n, 256), B), 256, 0, st, nn0, nn1, mask0, n, m, len0, gt0))) return rc;
  return OG_LAUNCH(gt_mutual_kernel, dim3(cdiv(m, 256), B), 256, 0, st, nn1, nn0, mask1, m, n, len1, gt1);
}

}  // namespace og
