// Homography-pretraining pair synthesis: OxfordParis1MDataset.__getitem__ (reference data/oxford_paris_dataset.py:27-66) without
// the decode, the INTER_AREA resize and the colour augmentation, for B images at once.
//
// Per pair, from uint8 RGB [H, W, 3] and 4 corner offsets o (x, y) in [-off, off):
//   H_warp = getPerspectiveTransform(c + o, c),  c = the crop's corners in the full image (off, off) .. (W-off-1, H-off-1)
//   H_true = getPerspectiveTransform(c' + o, c'), c' = the same corners relative to the crop (0, 0) .. (w-1, h-1)
//   image0 = gray(crop(rgb)) / 255,  image1 = gray(crop(warpPerspective(rgb, H_warp, (W, H)))) / 255,  H = fp32(H_true)
// with w = W - 2 off, h = H - 2 off.  Only the crop of the warped image is computed.
//
// The arithmetic is OpenCV's (imgwarp.cpp, matrix_decomp.cpp, color), so every output equals cv2's bit for bit:
//   fit     the 8x8 system of getPerspectiveTransform (src.x * dst.x products formed in float), solved by cv::solve's
//           DECOMP_LU (LUImpl: partial pivoting on the first largest |pivot|, alpha = a[j][i] * (-1 / a[i][i]), back substitution
//           dividing by the pivot), every double operation separately rounded (no FMA contraction); M[8] = 1.  A pivot below
//           100 DBL_EPSILON fails the solve: H = [[0,0,0],[0,0,0],[0,0,1]] (cv::solve zeroes its output).
//   invert  warpPerspective inverts H by invert()'s closed form for 3x3 (cofactors times 1/det3, all zero when det3 == 0).
//   warp    WarpPerspectiveInvoker: in 32x16 (bw0 x bh0) destination blocks, X0 = M0 xb + M1 y + M2 at the block's first
//           column xb, then per column x1 = x - xb:  W = W0 + M6 x1, W = W ? 32 / W : 0, X = rint((X0 + M0 x1) W) (clamped to
//           int), the same for Y; the source pixel is (X >> 5, Y >> 5) (saturated to int16), the fraction (X & 31, Y & 31).
//           remapBilinear: weights (32 - fx)(32 - fy) 32 ... (they sum to 32768), a neighbour outside the image counts as 0
//           (BORDER_CONSTANT 0), each channel (sum + 2^14) >> 15.
//   gray    cvtColor RGB2GRAY on uint8: (9798 R + 19235 G + 3735 B + 2^14) >> 15, then torch.FloatTensor(u8) / 255. (fp32, RN).
#pragma once
#include "common.cuh"

namespace og {

constexpr int HG_THREADS = 256;
static_assert(HG_THREADS == 256, "one thread per entry of the 1/255 table");
constexpr int HG_ROWS = 8;                 // output rows per CTA

// cv::getPerspectiveTransform by one warp, from dst = the rectangle corners (x0, y0), (x0, y1), (x1, y0), (x1, y1) and
// src = dst + o (o: 4 x (x, y) int offsets); a is [8][9] in shared memory (column 8 = the right-hand side).  Element updates of
// one elimination step are independent, so the lanes share them; every element sees OpenCV's operations in OpenCV's order.
// Lane 0 writes M[9].
__device__ __forceinline__ void hg_fit_warp(float x0, float y0, float x1, float y1, const int* __restrict__ o, double (*a)[9], double* M) {
  const int lane = threadIdx.x & 31;
  if (lane < 4) {
    const int i = lane;
    const float dx = i < 2 ? x0 : x1, dy = (i & 1) ? y1 : y0;
    const float sx = __fadd_rn(dx, (float)o[2 * i]), sy = __fadd_rn(dy, (float)o[2 * i + 1]);   // corners_dst + warp_offset (float32)
    double* r0 = a[i];
    double* r1 = a[i + 4];
    r0[0] = r1[3] = sx;
    r0[1] = r1[4] = sy;
    r0[2] = r1[5] = 1.0;
    r0[3] = r0[4] = r0[5] = r1[0] = r1[1] = r1[2] = 0.0;
    r0[6] = __fmul_rn(-sx, dx);
    r0[7] = __fmul_rn(-sy, dx);
    r1[6] = __fmul_rn(-sx, dy);
    r1[7] = __fmul_rn(-sy, dy);
    r0[8] = dx;
    r1[8] = dy;
  }
  __syncwarp();
  bool ok = true;
  for (int i = 0; i < 8 && ok; ++i) {
    int k = i;
    for (int j = i + 1; j < 8; ++j)
      if (fabs(a[j][i]) > fabs(a[k][i])) k = j;
    ok = !(fabs(a[k][i]) < 100.0 * 2.220446049250313e-16);        // DBL_EPSILON * 100
    if (!ok) break;
    if (k != i && lane < 9) { const double t = a[i][lane]; a[i][lane] = a[k][lane]; a[k][lane] = t; }
    __syncwarp();
    const double d = __ddiv_rn(-1.0, a[i][i]);
    // rows i+1 .. 7 x columns i+1 .. 8 (8: the right-hand side): at most 7 x 8 = 56 elements.  An element's update reads only
    // itself, row i and column i, which this step does not write, so the lanes need no ordering among themselves.
    const int cols = 8 - i;
    for (int e = lane; e < (7 - i) * cols; e += 32) {
      const int j = i + 1 + e / cols, c = i + 1 + e % cols;
      const double alpha = __dmul_rn(a[j][i], d);
      a[j][c] = __dadd_rn(a[j][c], __dmul_rn(alpha, a[i][c]));
    }
    __syncwarp();
  }
  if (lane == 0) {
    if (ok) {
      for (int i = 7; i >= 0; --i) {                                // the solution replaces the right-hand side, as in LUImpl
        double s = a[i][8];
        for (int k = i + 1; k < 8; ++k) s = __dsub_rn(s, __dmul_rn(a[i][k], a[k][8]));
        a[i][8] = __ddiv_rn(s, a[i][i]);
      }
      for (int i = 0; i < 8; ++i) M[i] = a[i][8];
    } else {
      for (int i = 0; i < 8; ++i) M[i] = 0.0;
    }
    M[8] = 1.0;
  }
  __syncwarp();
}

// cv::invert(DECOMP_LU) of a 3x3 double matrix: cofactors times 1/det3; all zero when det3 == 0.
__device__ __forceinline__ void hg_invert3(const double* S, double* D) {
#define HG_S(r, c) S[3 * (r) + (c)]
#define HG_C(a, b, c, d) __dsub_rn(__dmul_rn(a, b), __dmul_rn(c, d))
  const double det = __dadd_rn(__dsub_rn(__dmul_rn(HG_S(0, 0), HG_C(HG_S(1, 1), HG_S(2, 2), HG_S(1, 2), HG_S(2, 1))),
                                         __dmul_rn(HG_S(0, 1), HG_C(HG_S(1, 0), HG_S(2, 2), HG_S(1, 2), HG_S(2, 0)))),
                               __dmul_rn(HG_S(0, 2), HG_C(HG_S(1, 0), HG_S(2, 1), HG_S(1, 1), HG_S(2, 0))));
  if (det == 0.0) {
    for (int i = 0; i < 9; ++i) D[i] = 0.0;
    return;
  }
  const double r = __ddiv_rn(1.0, det);
  D[0] = __dmul_rn(HG_C(HG_S(1, 1), HG_S(2, 2), HG_S(1, 2), HG_S(2, 1)), r);
  D[1] = __dmul_rn(HG_C(HG_S(0, 2), HG_S(2, 1), HG_S(0, 1), HG_S(2, 2)), r);
  D[2] = __dmul_rn(HG_C(HG_S(0, 1), HG_S(1, 2), HG_S(0, 2), HG_S(1, 1)), r);
  D[3] = __dmul_rn(HG_C(HG_S(1, 2), HG_S(2, 0), HG_S(1, 0), HG_S(2, 2)), r);
  D[4] = __dmul_rn(HG_C(HG_S(0, 0), HG_S(2, 2), HG_S(0, 2), HG_S(2, 0)), r);
  D[5] = __dmul_rn(HG_C(HG_S(0, 2), HG_S(1, 0), HG_S(0, 0), HG_S(1, 2)), r);
  D[6] = __dmul_rn(HG_C(HG_S(1, 0), HG_S(2, 1), HG_S(1, 1), HG_S(2, 0)), r);
  D[7] = __dmul_rn(HG_C(HG_S(0, 1), HG_S(2, 0), HG_S(0, 0), HG_S(2, 1)), r);
  D[8] = __dmul_rn(HG_C(HG_S(0, 0), HG_S(1, 1), HG_S(0, 1), HG_S(1, 0)), r);
#undef HG_C
#undef HG_S
}

__device__ __forceinline__ int hg_gray(int r, int g, int b) { return (9798 * r + 19235 * g + 3735 * b + (1 << 14)) >> 15; }

// grid (cdiv(h, HG_ROWS), B), HG_THREADS threads.  rgb [B, H, W, 3] uint8 (rows 3 W bytes, no alignment assumed);
// warp_offset [B, 4, 2] int32 (x, y) for the corners (off, off), (off, H-off-1), (W-off-1, off), (W-off-1, H-off-1);
// image0 / image1 [B, h, w] fp32; H_true [B, 3, 3] fp32 (written by the CTAs of row block 0).
__global__ void __launch_bounds__(HG_THREADS) homography_pairs_kernel(const uint8_t* __restrict__ rgb, int H, int W, int off, int bw0,
                                                                       const int* __restrict__ warp_offset, float* __restrict__ image0,
                                                                       float* __restrict__ image1, float* __restrict__ H_true) {
  __shared__ double a_sh[2][8][9];
  __shared__ double M_sh[2][9];
  __shared__ double Mi_sh[9];
  __shared__ float by255[256];                                      // torch.FloatTensor(u8) / 255.: fp32, round to nearest
  by255[threadIdx.x] = __fdiv_rn((float)threadIdx.x, 255.f);
  const int b = blockIdx.y, warp = threadIdx.x >> 5;
  const int h = H - 2 * off, w = W - 2 * off;
  const int* o = warp_offset + 8 * b;
  if (warp < 2 && (warp == 0 || blockIdx.x == 0)) {              // warp 0: H_warp (full image); warp 1: H_true (crop-relative)
    const float c0 = warp == 0 ? (float)off : 0.f;
    const float x1 = warp == 0 ? (float)(W - off - 1) : (float)(w - 1), y1 = warp == 0 ? (float)(H - off - 1) : (float)(h - 1);
    hg_fit_warp(c0, c0, x1, y1, o, a_sh[warp], M_sh[warp]);
    if ((threadIdx.x & 31) == 0) {
      if (warp == 0) hg_invert3(M_sh[0], Mi_sh);
      else
        for (int i = 0; i < 9; ++i) H_true[9 * (int64_t)b + i] = __double2float_rn(M_sh[1][i]);
    }
  }
  __syncthreads();
  double M[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) M[i] = Mi_sh[i];
  const uint8_t* img = rgb + (int64_t)b * H * W * 3;
  const int row0 = blockIdx.x * HG_ROWS, rows = min(HG_ROWS, h - row0);
  for (int e = threadIdx.x; e < rows * w; e += HG_THREADS) {
    const int cy = row0 + e / w, cx = e - (e / w) * w;
    const int y = cy + off, x = cx + off;
    const int64_t out = ((int64_t)b * h + cy) * w + cx;
    const uint8_t* p = img + ((int64_t)y * W + x) * 3;
    image0[out] = by255[hg_gray(p[0], p[1], p[2])];

    const int xb = x / bw0 * bw0;
    const double x1 = (double)(x - xb), yd = (double)y, xbd = (double)xb;
    const double W0 = __dadd_rn(__dadd_rn(__dmul_rn(M[6], xbd), __dmul_rn(M[7], yd)), M[8]);
    double Wd = __dadd_rn(W0, __dmul_rn(M[6], x1));
    Wd = Wd != 0.0 ? __ddiv_rn(32.0, Wd) : 0.0;
    const double X0 = __dadd_rn(__dadd_rn(__dmul_rn(M[0], xbd), __dmul_rn(M[1], yd)), M[2]);
    const double Y0 = __dadd_rn(__dadd_rn(__dmul_rn(M[3], xbd), __dmul_rn(M[4], yd)), M[5]);
    const double fX = fmax((double)INT32_MIN, fmin((double)INT32_MAX, __dmul_rn(__dadd_rn(X0, __dmul_rn(M[0], x1)), Wd)));
    const double fY = fmax((double)INT32_MIN, fmin((double)INT32_MAX, __dmul_rn(__dadd_rn(Y0, __dmul_rn(M[3], x1)), Wd)));
    const int Xi = __double2int_rn(fX), Yi = __double2int_rn(fY);
    const int sx = max(-32768, min(32767, Xi >> 5)), sy = max(-32768, min(32767, Yi >> 5));
    const int fx = Xi & 31, fy = Yi & 31;
    const int wt[4] = {(32 - fx) * (32 - fy) * 32, fx * (32 - fy) * 32, (32 - fx) * fy * 32, fx * fy * 32};
    int acc[3] = {1 << 14, 1 << 14, 1 << 14};
#pragma unroll
    for (int n = 0; n < 4; ++n) {
      const int px = sx + (n & 1), py = sy + (n >> 1);
      if (px >= 0 && px < W && py >= 0 && py < H) {
        const uint8_t* q = img + ((int64_t)py * W + px) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c] += q[c] * wt[n];
      }
    }
    image1[out] = by255[hg_gray(acc[0] >> 15, acc[1] >> 15, acc[2] >> 15)];
  }
}

// WarpPerspectiveInvoker's block width for a W x H destination (BLOCK_SZ 32)
inline int hg_block_width(int H, int W) {
  const int bh0 = H < 16 ? H : 16;
  return 1024 / bh0 < W ? 1024 / bh0 : W;
}

}  // namespace og
