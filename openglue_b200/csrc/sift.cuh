// OpenCV SIFT front-end (DESIGN.md scope f7): the reference's default local features, OPENCV_SIFT (reference
// models/features/opencv/_features.py:10-18, base.py:14-182, torch_wrapper.py:19-49):
//   cv2.SIFT_create(contrastThreshold=-10000, edgeThreshold=-10000).detectAndCompute(gray_u8)  ->  greedy radius NMS  ->  top-k
//   ->  RootSIFT  ->  LAFs (mr_size 6).
// Both thresholds are negative, so every 26-neighbour DoG extremum that survives interpolation is a keypoint and the edge test
// rejects only det <= 0.
//
// The detector restates cv2's published algorithm with its constants: 3 layers per octave, sigma 1.6, first octave -1 (the x2
// INTER_LINEAR upsampled image, blurred by sqrt(1.6^2 - 4 * 0.5^2)), octave count round(log2(min side of the base)) - 2 + 1,
// Gaussian taps computed in double and rounded to float, BORDER_REFLECT_101, nearest-neighbour x2 downsampling from layer 3.
// Where cv2's x86 build (AVX2 dispatch) fixes an arithmetic order, the kernels follow it: the row pass of a blur is a running
// fused multiply-add over the taps except in the last (w mod 4) columns, the column pass folds symmetric taps with fused
// multiply-adds except in the last (w mod 8) columns, the tails unfused (with these rules the blurs equal cv2.GaussianBlur); gradient angles are cv2's fastAtan2 polynomial (fused in the first len - len mod 8 samples
// of a keypoint, as cv::hal::fastAtan2's vector loop, unfused in the tail), never atan2.  cv2's exp32f and powf are not
// restated (the correctly rounded exp and exp2 stand in), so keypoint sizes, orientations and descriptors may differ from cv2's
// in the last bits.
//
// Kernels (one launch per stage, every image of a batch in the same launch):
//   sift_quantize_kernel      (255 * x) truncated to uint8, the torch wrapper's conversion
//   sift_upsample_kernel      uint8 [H, W] -> float [2H, 2W] (cv2 INTER_LINEAR on float: exact for x2)
//   sift_blur_rows_kernel / sift_blur_cols_kernel
//                             separable Gaussian; the column pass also writes the DoG level (this level - the previous one)
//   sift_downsample_kernel    nearest x2
//   sift_extrema_kernel       26-neighbour test + up to 5 interpolation steps + det <= 0 rejection -> located candidates
//   sift_orientation_kernel   one warp per candidate: 36-bin histogram, [1 4 6 4 1] / 16 smoothing, every peak >= 0.8 max
//   sift_sort_unique_kernel   one CTA per image: bitonic sort into cv2's KeyPoint order (x, y, size desc, angle, response desc,
//                             octave desc) + removal of exact duplicates (cv2's removeDuplicatedSorted)
//   sift_select_kernel        one CTA per image: greedy radius NMS (rank = response desc, index asc) in parallel rounds + top-k
//   sift_describe_kernel      one warp per selected keypoint: 4 x 4 x 8 descriptor, clip 0.2, x512, saturate; RootSIFT + LAF
//   sift_rootsift_laf_kernel  RootSIFT + LAF of supplied raw descriptors
#pragma once
#include "common.cuh"
#include <math_constants.h>
#include <float.h>
#include <math.h>

namespace og {

constexpr int SIFT_LAYERS = 3;                 // nOctaveLayers
constexpr int SIFT_GAUSS = SIFT_LAYERS + 3;    // Gaussian levels per octave
constexpr int SIFT_DOGS = SIFT_LAYERS + 2;     // DoG levels per octave
// cv2 keeps sigma as a double: the pyramid's per-level blurs are derived from 1.6 in double, while the initial blur and the
// keypoint size use (float)sigma.
constexpr double SIFT_SIGMA_D = 1.6;
constexpr float SIFT_SIGMA = (float)SIFT_SIGMA_D;
constexpr int SIFT_BORDER = 5;                 // SIFT_IMG_BORDER
constexpr int SIFT_MAX_INTERP = 5;
constexpr int SIFT_ORI_BINS = 36;
constexpr float SIFT_ORI_SIG = 1.5f;
constexpr float SIFT_ORI_RADIUS = 3 * SIFT_ORI_SIG;
constexpr float SIFT_ORI_PEAK = 0.8f;
constexpr int SIFT_D = 4, SIFT_N = 8;          // descriptor: 4 x 4 cells x 8 orientation bins
constexpr int SIFT_DESC = SIFT_D * SIFT_D * SIFT_N;
constexpr int SIFT_HIST = (SIFT_D + 2) * (SIFT_D + 2) * (SIFT_N + 2);
constexpr float SIFT_DESCR_SCL = 3.f, SIFT_DESCR_MAG_THR = 0.2f, SIFT_INT_DESCR = 512.f;
constexpr int SIFT_MAX_TAPS = 32;              // the widest kernel is 27 taps (sigma 3.09)
constexpr int SIFT_MAX_OCTAVES = 16;

struct SiftTaps { float k[SIFT_MAX_TAPS]; int n; };

// A located extremum before orientation assignment: octave o (0 = the upsampled image), layer, pixel, cv2's packed octave word
// and the keypoint in base-image coordinates as adjustLocalExtrema forms it.
struct SiftLoc { int o, layer, r, c, octw; float x, y, size, response; };
static_assert(sizeof(SiftLoc) == 36, "SiftLoc is read back as a 36-byte record (tests/test_sift_stages.py)");

// ---------------------------------------------------------------------------------------------------------------------
// cv2's fastAtan2 (degrees in [0, 360)): the polynomial of cv::hal::fastAtan2.  fused = the vector loop's form (v_fma), else the
// scalar form (cv2.fastAtan2, and the vector loop's tail).
__device__ __forceinline__ float sift_fast_atan2(float y, float x, bool fused) {
  const float r2d = (float)(180.0 / 3.141592653589793);
  const float p1 = 0.9997878412794807f * r2d, p3 = -0.3258083974640975f * r2d;
  const float p5 = 0.1555786518463281f * r2d, p7 = -0.04432655554792128f * r2d;
  const float ax = fabsf(x), ay = fabsf(y);
  const float c = ax >= ay ? __fdiv_rn(ay, __fadd_rn(ax, (float)DBL_EPSILON)) : __fdiv_rn(ax, __fadd_rn(ay, (float)DBL_EPSILON));
  const float c2 = __fmul_rn(c, c);
  float a;
  if (fused) a = __fmul_rn(fmaf(fmaf(fmaf(c2, p7, p5), c2, p3), c2, p1), c);
  else a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
  if (!(ax >= ay)) a = __fsub_rn(90.f, a);
  if (x < 0) a = __fsub_rn(180.f, a);
  if (y < 0) a = __fsub_rn(360.f, a);
  return a;
}

__global__ void __launch_bounds__(256) sift_fast_atan2_kernel(const float* __restrict__ y, const float* __restrict__ x, int64_t n, int fused,
                                                              float* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) out[i] = sift_fast_atan2(y[i], x[i], fused != 0);
}

// cv2's BORDER_REFLECT_101 index (borderInterpolate)
__device__ __forceinline__ int sift_reflect(int p, int len) {
  if (len == 1) return 0;
  while ((unsigned)p >= (unsigned)len) p = p < 0 ? -p : 2 * len - p - 2;
  return p;
}

// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) sift_quantize_kernel(const float* __restrict__ x, int64_t n, uint8_t* __restrict__ u8) {
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256)
    u8[i] = (uint8_t)(int)__fmul_rn(255.f, x[i]);             // numpy astype(uint8) of the float32 product: truncation
}

// uint8 [B, H, W] -> float [B, 2H, 2W]: cv2.resize INTER_LINEAR at exactly x2 (weights 1/4, 3/4, clamped at the borders; exact)
__global__ void __launch_bounds__(256) sift_upsample_kernel(const uint8_t* __restrict__ src, int B, int H, int W, float* __restrict__ dst) {
  const int W2 = 2 * W, H2 = 2 * H;
  const int64_t total = (int64_t)B * H2 * W2;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int x = (int)(i % W2), y = (int)((i / W2) % H2);
    const int64_t b = i / ((int64_t)W2 * H2);
    const uint8_t* s = src + b * H * W;
    const int x0 = (x & 1) ? x >> 1 : (x >> 1) - 1, y0 = (y & 1) ? y >> 1 : (y >> 1) - 1;
    const float fx = (x & 1) ? 0.25f : 0.75f, fy = (y & 1) ? 0.25f : 0.75f;      // weight of x0 + 1 / y0 + 1
    const int xa = max(x0, 0), xb = min(x0 + 1, W - 1), ya = max(y0, 0), yb = min(y0 + 1, H - 1);
    auto row = [&](int yy) { return (float)s[yy * W + xa] * (1.f - fx) + (float)s[yy * W + xb] * fx; };
    dst[i] = row(ya) * (1.f - fy) + row(yb) * fy;
  }
}

// row pass: tmp[y, x] = sum_t k[t] src[y, reflect(x + t - R)] over t in order: a running fused multiply-add in the first
// w - w mod 4 columns (cv2's RowVec_32f, 8 and 4 lanes), product then sum in the rest (its scalar tail)
__global__ void __launch_bounds__(256) sift_blur_rows_kernel(const float* __restrict__ src, int B, int h, int w, SiftTaps taps, float* __restrict__ tmp) {
  const int R = taps.n / 2, vec_end = w & ~3;
  const int64_t total = (int64_t)B * h * w;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int x = (int)(i % w);
    const float* row = src + (i - x);
    const bool inside = x >= R && x + R < w;
    float s = 0.f;
    if (x < vec_end) {
      for (int t = 0; t < taps.n; ++t) s = fmaf(row[inside ? x + t - R : sift_reflect(x + t - R, w)], taps.k[t], s);
    } else {
      for (int t = 0; t < taps.n; ++t) s = __fadd_rn(s, __fmul_rn(row[inside ? x + t - R : sift_reflect(x + t - R, w)], taps.k[t]));
    }
    tmp[i] = s;
  }
}

// column pass: dst[y, x] = k[R] tmp[y, x] + sum_{t=1..R} k[R+t] (tmp[y+t, x] + tmp[y-t, x]) (cv2's SymmColumnVec_32f: fused in the
// first w - w mod 8 columns, unfused in the rest), and, when dog is given, dog = dst - prev (cv2's subtract(next, prev)).
__global__ void __launch_bounds__(256) sift_blur_cols_kernel(const float* __restrict__ tmp, int B, int h, int w, SiftTaps taps,
                                                             float* __restrict__ dst, const float* __restrict__ prev, float* __restrict__ dog) {
  const int R = taps.n / 2, vec_end = w & ~7;
  const int64_t total = (int64_t)B * h * w;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int x = (int)(i % w), y = (int)((i / w) % h);
    const float* col = tmp + (i - x - (int64_t)y * w) + x;
    float s;
    if (x < vec_end) {
      s = fmaf(col[(int64_t)y * w], taps.k[R], 0.f);
      for (int t = 1; t <= R; ++t)
        s = fmaf(__fadd_rn(col[(int64_t)sift_reflect(y + t, h) * w], col[(int64_t)sift_reflect(y - t, h) * w]), taps.k[R + t], s);
    } else {
      s = __fmul_rn(col[(int64_t)y * w], taps.k[R]);
      for (int t = 1; t <= R; ++t)
        s = __fadd_rn(s, __fmul_rn(__fadd_rn(col[(int64_t)sift_reflect(y + t, h) * w], col[(int64_t)sift_reflect(y - t, h) * w]), taps.k[R + t]));
    }
    dst[i] = s;
    if (dog) dog[i] = __fsub_rn(s, prev[i]);
  }
}

// dst [B, h/2, w/2] = src [B, h, w] at (2y, 2x): cv2.resize INTER_NEAREST to (w/2, h/2)
__global__ void __launch_bounds__(256) sift_downsample_kernel(const float* __restrict__ src, int B, int h, int w, float* __restrict__ dst) {
  const int hd = h / 2, wd = w / 2;
  const int64_t total = (int64_t)B * hd * wd;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int x = (int)(i % wd), y = (int)((i / wd) % hd);
    const int64_t b = i / ((int64_t)wd * hd);
    dst[i] = src[(b * h + 2 * y) * w + 2 * x];
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// The pyramid of one octave: Gaussian levels [SIFT_GAUSS][B][h][w], DoG levels [SIFT_DOGS][B][h][w].
struct SiftOctave { float* gauss; float* dog; int h, w; };
struct SiftPyramid { SiftOctave oct[SIFT_MAX_OCTAVES]; int n, B; };

__device__ __forceinline__ float sift_at(const float* img, int w, int r, int c) { return img[(int64_t)r * w + c]; }

// cv2's adjustLocalExtrema with contrastThreshold, edgeThreshold < 0 (the contrast test never rejects; the edge test rejects
// det <= 0 only).  Returns false when the extremum is dropped; else fills loc.
__device__ bool sift_adjust(const SiftOctave& oc, int B, int b, int o, int layer, int r, int c, SiftLoc& loc) {
  const float img_scale = 1.f / 255.f, deriv_scale = img_scale * 0.5f, second_scale = img_scale, cross_scale = img_scale * 0.25f;
  const int h = oc.h, w = oc.w;
  const int64_t plane = (int64_t)h * w;
  float xi = 0.f, xr = 0.f, xc = 0.f;
  int i = 0;
  const float *img = nullptr, *prv = nullptr, *nxt = nullptr;
  for (; i < SIFT_MAX_INTERP; ++i) {
    img = oc.dog + ((int64_t)layer * B + b) * plane;
    prv = img - (int64_t)B * plane;
    nxt = img + (int64_t)B * plane;
    const float dx = __fmul_rn(__fsub_rn(sift_at(img, w, r, c + 1), sift_at(img, w, r, c - 1)), deriv_scale);
    const float dy = __fmul_rn(__fsub_rn(sift_at(img, w, r + 1, c), sift_at(img, w, r - 1, c)), deriv_scale);
    const float ds = __fmul_rn(__fsub_rn(sift_at(nxt, w, r, c), sift_at(prv, w, r, c)), deriv_scale);
    const float v2 = __fmul_rn(sift_at(img, w, r, c), 2.f);
    const float dxx = __fmul_rn(__fsub_rn(__fadd_rn(sift_at(img, w, r, c + 1), sift_at(img, w, r, c - 1)), v2), second_scale);
    const float dyy = __fmul_rn(__fsub_rn(__fadd_rn(sift_at(img, w, r + 1, c), sift_at(img, w, r - 1, c)), v2), second_scale);
    const float dss = __fmul_rn(__fsub_rn(__fadd_rn(sift_at(nxt, w, r, c), sift_at(prv, w, r, c)), v2), second_scale);
    const float dxy = __fmul_rn(__fadd_rn(__fsub_rn(__fsub_rn(sift_at(img, w, r + 1, c + 1), sift_at(img, w, r + 1, c - 1)), sift_at(img, w, r - 1, c + 1)),
                                          sift_at(img, w, r - 1, c - 1)), cross_scale);
    const float dxs = __fmul_rn(__fadd_rn(__fsub_rn(__fsub_rn(sift_at(nxt, w, r, c + 1), sift_at(nxt, w, r, c - 1)), sift_at(prv, w, r, c + 1)),
                                          sift_at(prv, w, r, c - 1)), cross_scale);
    const float dys = __fmul_rn(__fadd_rn(__fsub_rn(__fsub_rn(sift_at(nxt, w, r + 1, c), sift_at(nxt, w, r - 1, c)), sift_at(prv, w, r + 1, c)),
                                          sift_at(prv, w, r - 1, c)), cross_scale);
    // Matx33f(H).solve(dD, DECOMP_LU): Cramer's rule with the float determinant (Matx_FastSolveOp<float, 3, 1>)
    const float a00 = dxx, a01 = dxy, a02 = dxs, a10 = dxy, a11 = dyy, a12 = dys, a20 = dxs, a21 = dys, a22 = dss;
    const float b0 = dx, b1 = dy, b2 = ds;
    auto m = [](float p, float q) { return __fmul_rn(p, q); };
    auto sb = [](float p, float q) { return __fsub_rn(p, q); };
    auto ad = [](float p, float q) { return __fadd_rn(p, q); };
    float det = ad(sb(m(a00, sb(m(a11, a22), m(a21, a12))), m(a01, sb(m(a10, a22), m(a20, a12)))), m(a02, sb(m(a10, a21), m(a20, a11))));
    float X0 = 0.f, X1 = 0.f, X2 = 0.f;
    if (det != 0.f) {
      const float d = __fdiv_rn(1.f, det);
      X0 = m(d, ad(sb(m(b0, sb(m(a11, a22), m(a12, a21))), m(a01, sb(m(b1, a22), m(a12, b2)))), m(a02, sb(m(b1, a21), m(a11, b2)))));
      X1 = m(d, ad(sb(m(a00, sb(m(b1, a22), m(a12, b2))), m(b0, sb(m(a10, a22), m(a12, a20)))), m(a02, sb(m(a10, b2), m(b1, a20)))));
      X2 = m(d, ad(sb(m(a00, sb(m(a11, b2), m(b1, a21))), m(a01, sb(m(a10, b2), m(b1, a20)))), m(b0, sb(m(a10, a21), m(a11, a20)))));
    }
    xi = -X2; xr = -X1; xc = -X0;
    if (fabsf(xi) < 0.5f && fabsf(xr) < 0.5f && fabsf(xc) < 0.5f) break;
    const float big = (float)(INT_MAX / 3);
    if (fabsf(xi) > big || fabsf(xr) > big || fabsf(xc) > big) return false;
    c += __float2int_rn(xc);
    r += __float2int_rn(xr);
    layer += __float2int_rn(xi);
    if (layer < 1 || layer > SIFT_LAYERS || c < SIFT_BORDER || c >= w - SIFT_BORDER || r < SIFT_BORDER || r >= h - SIFT_BORDER) return false;
  }
  if (i >= SIFT_MAX_INTERP) return false;
  img = oc.dog + ((int64_t)layer * B + b) * plane;
  prv = img - (int64_t)B * plane;
  nxt = img + (int64_t)B * plane;
  const float dx = __fmul_rn(__fsub_rn(sift_at(img, w, r, c + 1), sift_at(img, w, r, c - 1)), deriv_scale);
  const float dy = __fmul_rn(__fsub_rn(sift_at(img, w, r + 1, c), sift_at(img, w, r - 1, c)), deriv_scale);
  const float ds = __fmul_rn(__fsub_rn(sift_at(nxt, w, r, c), sift_at(prv, w, r, c)), deriv_scale);
  const float t = __fadd_rn(__fadd_rn(__fmul_rn(dx, xc), __fmul_rn(dy, xr)), __fmul_rn(ds, xi));
  const float contr = __fadd_rn(__fmul_rn(sift_at(img, w, r, c), img_scale), __fmul_rn(t, 0.5f));
  const float v2 = __fmul_rn(sift_at(img, w, r, c), 2.f);
  const float dxx = __fmul_rn(__fsub_rn(__fadd_rn(sift_at(img, w, r, c + 1), sift_at(img, w, r, c - 1)), v2), second_scale);
  const float dyy = __fmul_rn(__fsub_rn(__fadd_rn(sift_at(img, w, r + 1, c), sift_at(img, w, r - 1, c)), v2), second_scale);
  const float dxy = __fmul_rn(__fadd_rn(__fsub_rn(__fsub_rn(sift_at(img, w, r + 1, c + 1), sift_at(img, w, r + 1, c - 1)), sift_at(img, w, r - 1, c + 1)),
                                        sift_at(img, w, r - 1, c - 1)), cross_scale);
  const float det = __fsub_rn(__fmul_rn(dxx, dyy), __fmul_rn(dxy, dxy));
  if (det <= 0.f) return false;
  loc.o = o; loc.layer = layer; loc.r = r; loc.c = c;
  loc.x = __fmul_rn(__fadd_rn((float)c, xc), (float)(1 << o));
  loc.y = __fmul_rn(__fadd_rn((float)r, xr), (float)(1 << o));
  loc.octw = o + (layer << 8) + (__double2int_rn(((double)xi + 0.5) * 255.0) << 16);
  const float e = __fdiv_rn(__fadd_rn((float)layer, xi), (float)SIFT_LAYERS);
  loc.size = __fmul_rn(__fmul_rn(__fmul_rn(SIFT_SIGMA, (float)exp2((double)e)), (float)(1 << o)), 2.f);
  loc.response = fabsf(contr);
  return true;
}

// One thread per pixel of layers 1..3 of octave o, every image: the 26-neighbour test (val > 0 and >= all, or val < 0 and <= all)
// inside the 5-pixel border, then sift_adjust.  Located candidates are appended to loc[b] (order is irrelevant: the sort fixes it).
__global__ void __launch_bounds__(256) sift_extrema_kernel(SiftOctave oc, int B, int o, SiftLoc* __restrict__ loc, int loc_cap,
                                                            int* __restrict__ loc_count) {
  const int h = oc.h, w = oc.w;
  const int ih = h - 2 * SIFT_BORDER, iw = w - 2 * SIFT_BORDER;
  if (ih <= 0 || iw <= 0) return;
  const int64_t plane = (int64_t)h * w;
  const int64_t total = (int64_t)B * SIFT_LAYERS * ih * iw;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int c = (int)(i % iw) + SIFT_BORDER, r = (int)((i / iw) % ih) + SIFT_BORDER;
    const int layer = (int)((i / ((int64_t)iw * ih)) % SIFT_LAYERS) + 1;
    const int b = (int)(i / ((int64_t)iw * ih * SIFT_LAYERS));
    const float* cur = oc.dog + ((int64_t)layer * B + b) * plane + (int64_t)r * w + c;
    const float val = *cur;
    if (!(val > 0.f || val < 0.f)) continue;
    bool ext = true;
    for (int l = -1; l <= 1 && ext; ++l) {
      const float* p = cur + (int64_t)l * B * plane;
      for (int dy = -1; dy <= 1 && ext; ++dy)
        for (int dx = -1; dx <= 1; ++dx) {
          const float v = p[(int64_t)dy * w + dx];
          if (val > 0.f ? !(val >= v) : !(val <= v)) { ext = false; break; }
        }
    }
    if (!ext) continue;
    SiftLoc L;
    if (!sift_adjust(oc, B, b, o, layer, r, c, L)) continue;
    const int slot = atomicAdd(loc_count + b, 1);
    if (slot < loc_cap) loc[(int64_t)b * loc_cap + slot] = L;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Keypoint records: kp [.., 5] = (x, y, size, angle, response) and the packed octave word, as cv2.KeyPoint holds them.
struct SiftKp { float x, y, size, angle, response; int octave; };
__device__ __forceinline__ SiftKp sift_load_kp(const float* kp, const int* oct, int64_t i) {
  SiftKp k;
  k.x = kp[i * 5 + 0]; k.y = kp[i * 5 + 1]; k.size = kp[i * 5 + 2]; k.angle = kp[i * 5 + 3]; k.response = kp[i * 5 + 4]; k.octave = oct[i];
  return k;
}
__device__ __forceinline__ void sift_store_kp(float* kp, int* oct, int64_t i, const SiftKp& k) {
  kp[i * 5 + 0] = k.x; kp[i * 5 + 1] = k.y; kp[i * 5 + 2] = k.size; kp[i * 5 + 3] = k.angle; kp[i * 5 + 4] = k.response; oct[i] = k.octave;
}

// One warp per located candidate: cv2's calcOrientationHist + the peak loop of findScaleSpaceExtrema.  The histogram adds the
// samples in cv2's (row-major) order: each lane owns bins lane and lane + 32 and takes the samples of a 32-sample chunk in turn.
// Every peak becomes a keypoint, with the first-octave scaling applied (pt, size x 1/2; octave byte - 1).
__global__ void __launch_bounds__(256) sift_orientation_kernel(SiftPyramid pyr, const SiftLoc* __restrict__ loc, int loc_cap,
                                                               const int* __restrict__ loc_count, float* __restrict__ kp, int* __restrict__ kp_oct,
                                                               int cap, int* __restrict__ count) {
  __shared__ float hist_s[8][SIFT_ORI_BINS + 4];
  const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int j = blockIdx.x * 8 + warp;
  if (j >= min(loc_count[b], loc_cap)) return;
  const SiftLoc L = loc[(int64_t)b * loc_cap + j];
  const SiftOctave& oc = pyr.oct[L.o];
  const int h = oc.h, w = oc.w;
  const float* img = oc.gauss + ((int64_t)L.layer * pyr.B + b) * h * w;
  const float scl = __fdiv_rn(__fmul_rn(L.size, 0.5f), (float)(1 << L.o));
  const int radius = __float2int_rn(__fmul_rn(SIFT_ORI_RADIUS, scl));
  const float sigma = __fmul_rn(SIFT_ORI_SIG, scl);
  const float expf_scale = __fdiv_rn(-1.f, __fmul_rn(__fmul_rn(2.f, sigma), sigma));
  const int ylo = max(-radius, 1 - L.r), yhi = min(radius, h - 2 - L.r), xlo = max(-radius, 1 - L.c), xhi = min(radius, w - 2 - L.c);
  const int nc = xhi - xlo + 1, len = (yhi >= ylo && xhi >= xlo) ? (yhi - ylo + 1) * nc : 0;
  const int vec_end = len & ~7;
  float h0 = 0.f, h1 = 0.f;
  for (int base = 0; base < len; base += 32) {
    const int k = base + lane;
    int bin = -1;
    float val = 0.f;
    if (k < len) {
      const int ii = ylo + k / nc, jj = xlo + k % nc, y = L.r + ii, x = L.c + jj;
      const float dx = __fsub_rn(sift_at(img, w, y, x + 1), sift_at(img, w, y, x - 1));
      const float dy = __fsub_rn(sift_at(img, w, y - 1, x), sift_at(img, w, y + 1, x));
      const float wt = (float)exp((double)__fmul_rn((float)(ii * ii + jj * jj), expf_scale));
      const bool vec = k < vec_end;
      const float ori = sift_fast_atan2(dy, dx, vec);
      const float mag = vec ? __fsqrt_rn(fmaf(dx, dx, __fmul_rn(dy, dy))) : __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
      bin = __float2int_rn(__fmul_rn((float)SIFT_ORI_BINS / 360.f, ori));
      if (bin >= SIFT_ORI_BINS) bin -= SIFT_ORI_BINS;
      if (bin < 0) bin += SIFT_ORI_BINS;
      val = __fmul_rn(wt, mag);
    }
    const int ns = min(32, len - base);
    for (int s = 0; s < ns; ++s) {
      const int bs = __shfl_sync(0xffffffffu, bin, s);
      const float vs = __shfl_sync(0xffffffffu, val, s);
      if (bs == lane) h0 = __fadd_rn(h0, vs);
      if (bs == lane + 32) h1 = __fadd_rn(h1, vs);
    }
  }
  float* th = hist_s[warp] + 2;                        // temphist[-2 .. n + 1]
  th[lane] = h0;
  if (lane < SIFT_ORI_BINS - 32) th[lane + 32] = h1;
  __syncwarp();
  if (lane < 2) { th[-1 - lane] = th[SIFT_ORI_BINS - 1 - lane]; th[SIFT_ORI_BINS + lane] = th[lane]; }
  __syncwarp();
  // smoothing: cv2's vector loop (fused) covers bins 0..31, its scalar tail 32..35
  auto smooth = [&](int i, bool fused) {
    if (fused) return fmaf(__fadd_rn(th[i - 2], th[i + 2]), 1.f / 16.f, fmaf(__fadd_rn(th[i - 1], th[i + 1]), 4.f / 16.f, __fmul_rn(th[i], 6.f / 16.f)));
    return __fadd_rn(__fadd_rn(__fmul_rn(__fadd_rn(th[i - 2], th[i + 2]), 1.f / 16.f), __fmul_rn(__fadd_rn(th[i - 1], th[i + 1]), 4.f / 16.f)),
                     __fmul_rn(th[i], 6.f / 16.f));
  };
  const float s0 = smooth(lane, true);
  const float s1 = lane < SIFT_ORI_BINS - 32 ? smooth(lane + 32, false) : -CUDART_INF_F;
  __syncwarp();
  float* hist = hist_s[warp];                          // reused: hist[0 .. n - 1]
  hist[lane] = s0;
  if (lane < SIFT_ORI_BINS - 32) hist[lane + 32] = s1;
  const float omax = warp_max(fmaxf(s0, s1));
  __syncwarp();
  const float mag_thr = __fmul_rn(omax, SIFT_ORI_PEAK);
  for (int jb = lane; jb < SIFT_ORI_BINS; jb += 32) {
    const int l = jb > 0 ? jb - 1 : SIFT_ORI_BINS - 1, r2 = jb < SIFT_ORI_BINS - 1 ? jb + 1 : 0;
    const float hj = hist[jb], hl = hist[l], hr = hist[r2];
    if (hj > hl && hj > hr && hj >= mag_thr) {
      float bin = __fadd_rn((float)jb, __fdiv_rn(__fmul_rn(0.5f, __fsub_rn(hl, hr)), __fadd_rn(__fsub_rn(hl, __fmul_rn(2.f, hj)), hr)));
      bin = bin < 0 ? __fadd_rn((float)SIFT_ORI_BINS, bin) : bin >= SIFT_ORI_BINS ? __fsub_rn(bin, (float)SIFT_ORI_BINS) : bin;
      float angle = __fsub_rn(360.f, __fmul_rn(360.f / SIFT_ORI_BINS, bin));
      if (fabsf(__fsub_rn(angle, 360.f)) < FLT_EPSILON) angle = 0.f;
      SiftKp k;                                        // detectAndCompute's firstOctave = -1 rescaling
      k.x = __fmul_rn(L.x, 0.5f); k.y = __fmul_rn(L.y, 0.5f); k.size = __fmul_rn(L.size, 0.5f);
      k.angle = angle; k.response = L.response;
      k.octave = (L.octw & ~255) | ((L.octw - 1) & 255);
      const int slot = atomicAdd(count + b, 1);
      if (slot < cap) sift_store_kp(kp, kp_oct, (int64_t)b * cap + slot, k);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// CTA-wide sort of the indices idx[0 .. pow2_ceil(n)) (entries >= n are padding that sorts last) by before(a, b), in global
// memory; every thread of the CTA calls it.
template <class Before>
__device__ void sift_cta_sort(int* idx, int n, Before before) {
  const int n2 = pow2_ceil(n);
  for (int t = threadIdx.x; t < n2; t += blockDim.x) idx[t] = t;
  __syncthreads();
  cta_bitonic_sort(n2, [&](int lo, int hi) { const int a = idx[lo], c = idx[hi]; return c >= n || (a < n && before(a, c)); },
                   [&](int lo, int hi) { const int a = idx[lo], c = idx[hi]; idx[lo] = c; idx[hi] = a; });
}

// cv2's KeyPoint12_LessThan
__device__ __forceinline__ bool sift_cv_before(const SiftKp& p, const SiftKp& q) {
  if (p.x != q.x) return p.x < q.x;
  if (p.y != q.y) return p.y < q.y;
  if (p.size != q.size) return p.size > q.size;
  if (p.angle != q.angle) return p.angle < q.angle;
  if (p.response != q.response) return p.response > q.response;
  return p.octave > q.octave;
}

// One CTA per image: the orientation kernel's keypoints -> cv2's order without exact duplicates (same x, y, size, angle) into
// out_kp / out_oct [B, cap]; count[b] = the number kept, or a value > cap when a capacity was exceeded (the outputs are then
// incomplete).  With overflow non-null, count[b] is always the number of keypoints written and overflow[b] = 1 marks an image
// whose outputs are incomplete.  work: [B, n2max] ints.
__global__ void __launch_bounds__(1024) sift_sort_unique_kernel(const float* __restrict__ kp, const int* __restrict__ kp_oct, const int* __restrict__ kp_count,
                                                                const int* __restrict__ loc_count, int loc_cap, int cap, int n2max, int* __restrict__ work,
                                                                float* __restrict__ out_kp, int* __restrict__ out_oct, int* __restrict__ count,
                                                                int* __restrict__ overflow) {
  __shared__ int warp_tot[32];
  __shared__ int base;
  const int b = blockIdx.x;
  const int raw = kp_count[b], n = min(raw, cap);
  int* idx = work + (int64_t)b * n2max;
  const float* kb = kp + (int64_t)b * cap * 5;
  const int* ob = kp_oct + (int64_t)b * cap;
  sift_cta_sort(idx, n, [&](int p, int q) { return sift_cv_before(sift_load_kp(kb, ob, p), sift_load_kp(kb, ob, q)); });
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  for (int j0 = 0; j0 < n; j0 += 1024) {
    const int j = j0 + threadIdx.x;
    bool on = false;
    SiftKp k;
    if (j < n) {
      k = sift_load_kp(kb, ob, idx[j]);
      on = j == 0;
      if (!on) {
        const SiftKp p = sift_load_kp(kb, ob, idx[j - 1]);
        on = p.x != k.x || p.y != k.y || p.size != k.size || p.angle != k.angle;
      }
    }
    const int pos = cta_ordered_slot(on, warp_tot, base);
    if (on) sift_store_kp(out_kp, out_oct, (int64_t)b * cap + pos, k);
  }
  if (threadIdx.x == 0) {
    const bool over = raw > cap || loc_count[b] > loc_cap;
    if (overflow) {
      count[b] = base;
      overflow[b] = over ? 1 : 0;
    } else {
      count[b] = over ? max(raw, cap + 1) : base;
    }
  }
}

// One CTA per image: detect_kpts_opencv's selection on keypoints kp [B, cap, 5] (x, y, size, angle, response), count[b] of them:
// greedy radius NMS (nms_keypoints: visit by response desc - equal responses by index asc -, a kept point removes every point
// within radius, inclusive; skipped when radius <= 0), then the max_keypoints largest responses (all when max_keypoints <= 0).
// sel [B, cap]: the kept indices by response desc, index asc; n_sel [B].
// NMS runs in rounds: a point is removed once a higher-ranked neighbour is kept, and kept once every higher-ranked neighbour is
// removed, which is the greedy result.  Neighbours come from the x-sorted order by binary search.  work: [B, 4, n2max] ints.
__global__ void __launch_bounds__(1024) sift_select_kernel(const float* __restrict__ kp, const int* __restrict__ count, int cap, float radius,
                                                           int max_keypoints, int n2max, int* __restrict__ work, int* __restrict__ sel, int* __restrict__ n_sel) {
  __shared__ int warp_tot[32];
  __shared__ int base, changed;
  const int b = blockIdx.x;
  const int n = max(0, min(count[b], cap));
  int* ord = work + (int64_t)b * 4 * n2max;
  int* xo = ord + n2max;
  int* rank = xo + n2max;
  int* state = rank + n2max;                           // 0 undecided, 1 kept, 2 removed
  const float* kb = kp + (int64_t)b * cap * 5;
  auto X = [&](int i) { return kb[(int64_t)i * 5 + 0]; };
  auto Y = [&](int i) { return kb[(int64_t)i * 5 + 1]; };
  auto S = [&](int i) { return kb[(int64_t)i * 5 + 4]; };
  sift_cta_sort(ord, n, [&](int p, int q) { return topk_before(S(p), p, S(q), q); });
  for (int j = threadIdx.x; j < n; j += blockDim.x) { rank[ord[j]] = j; state[j] = radius > 0.f ? 0 : 1; }
  __syncthreads();
  if (radius > 0.f) {
    sift_cta_sort(xo, n, [&](int p, int q) { const float xp = X(p), xq = X(q); return xp < xq || (xp == xq && p < q); });
    const double r = (double)radius, r2 = r * r;
    volatile int* vstate = state;
    for (;;) {
      if (threadIdx.x == 0) changed = 0;
      __syncthreads();
      for (int p = threadIdx.x; p < n; p += blockDim.x) {
        if (vstate[p] != 0) continue;
        const double xp = X(p), yp = Y(p);
        const int rp = rank[p];
        int lo = 0, hi = n;                            // first position with x >= xp - r
        while (lo < hi) { const int m = (lo + hi) >> 1; if ((double)X(xo[m]) < xp - r) lo = m + 1; else hi = m; }
        bool pending = false, removed = false;
        for (int m = lo; m < n; ++m) {
          const int q = xo[m];
          const double xq = X(q);
          if (xq > xp + r) break;
          if (rank[q] >= rp) continue;
          const double dx = xq - xp, dy = (double)Y(q) - yp;
          if (dx * dx + dy * dy > r2) continue;
          const int sq = vstate[q];
          if (sq == 1) { removed = true; break; }
          if (sq == 0) pending = true;
        }
        if (removed) { vstate[p] = 2; changed = 1; }
        else if (!pending) { vstate[p] = 1; changed = 1; }
      }
      __syncthreads();
      const int any = changed;
      __syncthreads();
      if (!any) break;
    }
  }
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  const int kmax = max_keypoints > 0 ? max_keypoints : cap;
  for (int j0 = 0; j0 < n; j0 += 1024) {
    const int j = j0 + threadIdx.x;
    const bool on = j < n && state[ord[j]] == 1;
    const int pos = cta_ordered_slot(on, warp_tot, base);
    if (on && pos < kmax) sel[(int64_t)b * cap + pos] = ord[j];
  }
  if (threadIdx.x == 0) n_sel[b] = min(base, kmax);
}

// ---------------------------------------------------------------------------------------------------------------------
// OpenCVFeatures.normalize_descriptors + lafs_from_opencv_kpts (mr_size 6) for one keypoint, one warp: raw[128] (cv2's integer
// values) -> desc (RootSIFT: L1 normalisation then sqrt; else L2), laf [2, 3], score.  The integer sums are exact, so the division
// and square root are numpy's correctly rounded float32 ones.  scale * cos / sin is rounded once from double: numpy's float32
// cos / sin are not correctly rounded, so a LAF entry may differ from the reference's by an ulp (rarely two).
__device__ void sift_finish(const float* raw_lane4, const SiftKp& k, bool rootsift, float* desc, float* laf, float* score) {
  const int lane = threadIdx.x & 31;
  float s = 0.f;
  for (int q = 0; q < 4; ++q) s += rootsift ? fabsf(raw_lane4[q]) : raw_lane4[q] * raw_lane4[q];
  s = warp_sum(s);                                     // integers below 2^24: exact in any order
  const float nrm = rootsift ? s : __fsqrt_rn(s);
  for (int q = 0; q < 4; ++q) {
    const float v = __fdiv_rn(raw_lane4[q], nrm);
    desc[lane + 32 * q] = rootsift ? __fsqrt_rn(v) : v;
  }
  if (lane == 0) {
    const float sc = (float)(6.0 * (double)k.size);
    const float th = __fmul_rn(-k.angle, (float)(3.141592653589793 / 180.0));
    const float sct = (float)((double)sc * cos((double)th)), sst = (float)((double)sc * sin((double)th));
    laf[0] = sct; laf[1] = sst; laf[2] = k.x;
    laf[3] = -sst; laf[4] = sct; laf[5] = k.y;
    *score = k.response;
  }
}

// One warp per row: sift_finish of supplied raw descriptors raw [N, 128] and keypoints kp [N, 5].
__global__ void __launch_bounds__(256) sift_rootsift_laf_kernel(const float* __restrict__ kp, const float* __restrict__ raw, int64_t N, int rootsift,
                                                                float* __restrict__ lafs, float* __restrict__ scores, float* __restrict__ desc) {
  const int64_t i = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= N) return;
  SiftKp k;
  k.x = kp[i * 5 + 0]; k.y = kp[i * 5 + 1]; k.size = kp[i * 5 + 2]; k.angle = kp[i * 5 + 3]; k.response = kp[i * 5 + 4]; k.octave = 0;
  float v[4];
  for (int q = 0; q < 4; ++q) v[q] = raw[i * SIFT_DESC + lane + 32 * q];
  sift_finish(v, k, rootsift != 0, desc + i * SIFT_DESC, lafs + i * 6, scores + i);
}

// One warp per selected keypoint (b, j < n_sel[b]): cv2's calcDescriptors / calcSIFTDescriptor on the Gaussian level the packed
// octave word names, then sift_finish.  The 4 x 4 x 8 histogram (with its one-cell margin) lives in shared memory; samples are
// generated 32 at a time in cv2's order and added one after another (lanes 0..7 take the 8 trilinear contributions of one
// sample), so every bin sums in cv2's order.  raw_out (optional): cv2's integer-valued descriptor.
__global__ void __launch_bounds__(256) sift_describe_kernel(SiftPyramid pyr, const float* __restrict__ kp, const int* __restrict__ kp_oct, int cap,
                                                            const int* __restrict__ sel, const int* __restrict__ n_sel, int out_cap, int rootsift,
                                                            float* __restrict__ lafs, float* __restrict__ scores, float* __restrict__ desc,
                                                            float* __restrict__ raw_out) {
  __shared__ float hist_s[8][SIFT_HIST];
  __shared__ float stg_v[8][32][8];
  __shared__ int stg_i[8][32];
  __shared__ float acc_s[8][8];
  const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int j = blockIdx.x * 8 + warp;
  if (j >= min(n_sel[b], out_cap)) return;
  const SiftKp k = sift_load_kp(kp, kp_oct, (int64_t)b * cap + sel[(int64_t)b * cap + j]);
  // unpackOctave
  int octave = k.octave & 255;
  const int layer = (k.octave >> 8) & 255;
  octave = octave < 128 ? octave : (-128 | octave);
  const float scale = octave >= 0 ? __fdiv_rn(1.f, (float)(1 << octave)) : (float)(1 << -octave);
  const float size = __fmul_rn(k.size, scale);
  const float ptx = __fmul_rn(k.x, scale), pty = __fmul_rn(k.y, scale);
  const SiftOctave& oc = pyr.oct[octave + 1];
  const int rows = oc.h, cols = oc.w;
  const float* img = oc.gauss + ((int64_t)layer * pyr.B + b) * rows * cols;
  float ori = __fsub_rn(360.f, k.angle);
  if (fabsf(__fsub_rn(ori, 360.f)) < FLT_EPSILON) ori = 0.f;
  const float scl = __fmul_rn(size, 0.5f);
  // calcSIFTDescriptor
  const int px = __float2int_rn(ptx), py = __float2int_rn(pty);
  const float orad = __fmul_rn(ori, (float)(3.141592653589793 / 180.0));
  float cos_t = (float)cos((double)orad), sin_t = (float)sin((double)orad);
  const float bins_per_rad = (float)SIFT_N / 360.f;
  const float exp_scale = __fdiv_rn(-1.f, (float)(SIFT_D * SIFT_D) * 0.5f);
  const float hist_width = __fmul_rn(SIFT_DESCR_SCL, scl);
  int radius = __float2int_rn(__fmul_rn(__fmul_rn(__fmul_rn(hist_width, 1.4142135623730951f), (float)(SIFT_D + 1)), 0.5f));
  radius = min(radius, (int)sqrt((double)cols * cols + (double)rows * rows));
  cos_t = __fdiv_rn(cos_t, hist_width);
  sin_t = __fdiv_rn(sin_t, hist_width);
  float* hist = hist_s[warp];
  for (int t = lane; t < SIFT_HIST; t += 32) hist[t] = 0.f;
  const int side = 2 * radius + 1, nsamp = side * side;
  auto sample = [&](int t, float& c_rot, float& r_rot, float& rbin, float& cbin) {
    const int i = t / side - radius, jj = t % side - radius;
    c_rot = __fsub_rn(__fmul_rn((float)jj, cos_t), __fmul_rn((float)i, sin_t));
    r_rot = __fadd_rn(__fmul_rn((float)jj, sin_t), __fmul_rn((float)i, cos_t));
    rbin = __fsub_rn(__fadd_rn(r_rot, (float)(SIFT_D / 2)), 0.5f);
    cbin = __fsub_rn(__fadd_rn(c_rot, (float)(SIFT_D / 2)), 0.5f);
    const int r = py + i, c = px + jj;
    return rbin > -1.f && rbin < (float)SIFT_D && cbin > -1.f && cbin < (float)SIFT_D && r > 0 && r < rows - 1 && c > 0 && c < cols - 1;
  };
  int len = 0;                                         // pass 1: the number of samples (cv2's len), for the vector / tail split
  for (int t0 = 0; t0 < nsamp; t0 += 32) {
    float a, bb, c, d;
    const bool ok = t0 + lane < nsamp && sample(t0 + lane, a, bb, c, d);
    len += __popc(__ballot_sync(0xffffffffu, ok));
  }
  const int vec_end = len & ~7;
  const int offs[8] = {0, 1, SIFT_N + 2, SIFT_N + 3, (SIFT_D + 2) * (SIFT_N + 2), (SIFT_D + 2) * (SIFT_N + 2) + 1,
                       (SIFT_D + 3) * (SIFT_N + 2), (SIFT_D + 3) * (SIFT_N + 2) + 1};
  __syncwarp();
  int kbase = 0;
  for (int t0 = 0; t0 < nsamp; t0 += 32) {
    const int t = t0 + lane;
    float c_rot, r_rot, rbin, cbin;
    const bool ok = t < nsamp && sample(t, c_rot, r_rot, rbin, cbin);
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    const int pos = __popc(bal & ((1u << lane) - 1u));
    if (ok) {
      const int kk = kbase + pos;
      const int i = t / side - radius, jj = t % side - radius, r = py + i, c = px + jj;
      const float dx = __fsub_rn(sift_at(img, cols, r, c + 1), sift_at(img, cols, r, c - 1));
      const float dy = __fsub_rn(sift_at(img, cols, r - 1, c), sift_at(img, cols, r + 1, c));
      const float wexp = (float)exp((double)__fmul_rn(__fadd_rn(__fmul_rn(c_rot, c_rot), __fmul_rn(r_rot, r_rot)), exp_scale));
      const bool vec = kk < vec_end;
      const float o = sift_fast_atan2(dy, dx, vec);
      const float mag0 = vec ? __fsqrt_rn(fmaf(dx, dx, __fmul_rn(dy, dy))) : __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
      float obin = __fmul_rn(__fsub_rn(o, ori), bins_per_rad);
      const float mag = __fmul_rn(mag0, wexp);
      const int r0 = (int)floorf(rbin), c0 = (int)floorf(cbin);
      int o0 = (int)floorf(obin);
      rbin = __fsub_rn(rbin, (float)r0); cbin = __fsub_rn(cbin, (float)c0); obin = __fsub_rn(obin, (float)o0);
      if (o0 < 0) o0 += SIFT_N;
      if (o0 >= SIFT_N) o0 -= SIFT_N;
      const float v_r1 = __fmul_rn(mag, rbin), v_r0 = __fsub_rn(mag, v_r1);
      const float v_rc11 = __fmul_rn(v_r1, cbin), v_rc10 = __fsub_rn(v_r1, v_rc11);
      const float v_rc01 = __fmul_rn(v_r0, cbin), v_rc00 = __fsub_rn(v_r0, v_rc01);
      const float v_rco111 = __fmul_rn(v_rc11, obin), v_rco110 = __fsub_rn(v_rc11, v_rco111);
      const float v_rco101 = __fmul_rn(v_rc10, obin), v_rco100 = __fsub_rn(v_rc10, v_rco101);
      const float v_rco011 = __fmul_rn(v_rc01, obin), v_rco010 = __fsub_rn(v_rc01, v_rco011);
      const float v_rco001 = __fmul_rn(v_rc00, obin), v_rco000 = __fsub_rn(v_rc00, v_rco001);
      stg_i[warp][pos] = ((r0 + 1) * (SIFT_D + 2) + c0 + 1) * (SIFT_N + 2) + o0;
      float* sv = stg_v[warp][pos];
      sv[0] = v_rco000; sv[1] = v_rco001; sv[2] = v_rco010; sv[3] = v_rco011;
      sv[4] = v_rco100; sv[5] = v_rco101; sv[6] = v_rco110; sv[7] = v_rco111;
    }
    __syncwarp();
    const int nv = __popc(bal);
    for (int s = 0; s < nv; ++s) {
      if (lane < 8) hist[stg_i[warp][s] + offs[lane]] = __fadd_rn(hist[stg_i[warp][s] + offs[lane]], stg_v[warp][s][lane]);
      __syncwarp();
    }
    kbase += nv;
  }
  // circular orientation bins, then the 128 values (cv2's rawDst) into hist[0 .. 127]'s place via registers
  if (lane < SIFT_D * SIFT_D) {
    const int i = lane / SIFT_D, jj = lane % SIFT_D;
    const int idx = ((i + 1) * (SIFT_D + 2) + (jj + 1)) * (SIFT_N + 2);
    hist[idx] = __fadd_rn(hist[idx], hist[idx + SIFT_N]);
    hist[idx + 1] = __fadd_rn(hist[idx + 1], hist[idx + SIFT_N + 1]);
  }
  __syncwarp();
  float v[4];
  for (int q = 0; q < 4; ++q) {
    const int e = lane + 32 * q, cell = e / SIFT_N, kk = e % SIFT_N;
    v[q] = hist[((cell / SIFT_D + 1) * (SIFT_D + 2) + (cell % SIFT_D + 1)) * (SIFT_N + 2) + kk];
  }
  __syncwarp();
  float* dst = hist;                                   // rawDst[0 .. 127]
  for (int q = 0; q < 4; ++q) dst[lane + 32 * q] = v[q];
  __syncwarp();
  // the norms: eight fused accumulators (element e goes to e mod 8, in order), summed as v_reduce_sum does on AVX2
  auto reduce8 = [&]() {
    const float* a = acc_s[warp];
    return __fadd_rn(__fadd_rn(__fadd_rn(a[0], a[1]), __fadd_rn(a[2], a[3])), __fadd_rn(__fadd_rn(a[4], a[5]), __fadd_rn(a[6], a[7])));
  };
  if (lane < 8) {
    float a = 0.f;
    for (int e = lane; e < SIFT_DESC; e += 8) a = fmaf(dst[e], dst[e], a);
    acc_s[warp][lane] = a;
  }
  __syncwarp();
  const float thr = __fmul_rn(__fsqrt_rn(reduce8()), SIFT_DESCR_MAG_THR);
  __syncwarp();
  for (int q = 0; q < 4; ++q) v[q] = fminf(v[q], thr);
  for (int q = 0; q < 4; ++q) dst[lane + 32 * q] = v[q];
  __syncwarp();
  if (lane < 8) {
    float a = 0.f;
    for (int e = lane; e < SIFT_DESC; e += 8) a = fmaf(dst[e], dst[e], a);
    acc_s[warp][lane] = a;
  }
  __syncwarp();
  const float nrm = __fdiv_rn(SIFT_INT_DESCR, fmaxf(__fsqrt_rn(reduce8()), FLT_EPSILON));
  for (int q = 0; q < 4; ++q) v[q] = (float)min(max(__float2int_rn(__fmul_rn(v[q], nrm)), 0), 255);     // saturate_cast<uchar>
  const int64_t row = (int64_t)b * out_cap + j;
  if (raw_out)
    for (int q = 0; q < 4; ++q) raw_out[row * SIFT_DESC + lane + 32 * q] = v[q];
  sift_finish(v, k, rootsift != 0, desc + row * SIFT_DESC, lafs + row * 6, scores + row);
}

// ---------------------------------------------------------------------------------------------------------------------
// Host side: geometry of the pyramid and the Gaussian taps.
// cv2's getGaussianKernel (getGaussianKernelBitExact, in double) rounded to float; n = cvRound(sigma * 8 + 1) | 1 for float images.
inline int sift_gaussian_taps(double sigma, float* k, int cap) {
  const int n = ((int)lrint(sigma * 8 + 1)) | 1;
  if (n > cap) return -1;
  const double scale2X = -0.125 / (sigma * sigma);
  const int n2 = (n - 1) / 2;
  double vals[SIFT_MAX_TAPS], sum = 0.0;
  for (int i = 0, x = 1 - n; i < n2; ++i, x += 2) { vals[i] = exp((double)(x * x) * scale2X); sum += vals[i]; }
  sum = sum * 2.0 + 1.0;
  const double mul1 = 1.0 / sum;
  for (int i = 0; i < n2; ++i) k[i] = k[n - 1 - i] = (float)(vals[i] * mul1);
  k[n2] = (float)mul1;
  return n;
}

inline int sift_num_octaves(int H, int W) {
  const int m = 2 * std::min(H, W);
  return (int)lrint(log((double)m) / log(2.0) - 2) + 1;
}

struct SiftLayout {
  int nO, h[SIFT_MAX_OCTAVES], w[SIFT_MAX_OCTAVES];
  int64_t gauss_off[SIFT_MAX_OCTAVES], dog_off[SIFT_MAX_OCTAVES], tmp_off, u8_off, loc_off, kp_off, oct_off, cnt_off, work_off, total;
  int loc_cap, n2max;
};

// Workspace of og_sift_detect / og_sift_describe for B images of H x W and cap keypoints per image.
inline bool sift_layout(int B, int H, int W, int cap, SiftLayout& L) {
  L.nO = sift_num_octaves(H, W);
  if (L.nO < 1 || L.nO > SIFT_MAX_OCTAVES) return false;
  int64_t off = 0;
  int h = 2 * H, w = 2 * W;
  for (int o = 0; o < L.nO; ++o) {
    L.h[o] = h; L.w[o] = w;
    L.gauss_off[o] = off; off += align_up((int64_t)SIFT_GAUSS * B * h * w * 4, 256);
    L.dog_off[o] = off; off += align_up((int64_t)SIFT_DOGS * B * h * w * 4, 256);
    h /= 2; w /= 2;
  }
  L.tmp_off = off; off += align_up((int64_t)B * 4 * H * W * 4, 256);
  L.u8_off = off; off += align_up((int64_t)B * H * W, 256);
  L.loc_cap = cap;
  L.loc_off = off; off += align_up((int64_t)B * cap * sizeof(SiftLoc), 256);
  L.kp_off = off; off += align_up((int64_t)B * cap * 5 * 4, 256);
  L.oct_off = off; off += align_up((int64_t)B * cap * 4, 256);
  L.cnt_off = off; off += align_up((int64_t)2 * B * 4, 256);
  L.n2max = pow2_ceil(cap);
  L.work_off = off; off += align_up((int64_t)B * 4 * L.n2max * 4, 256);
  L.total = off;
  return true;
}

inline SiftPyramid sift_pyramid(unsigned char* ws, const SiftLayout& L, int B) {
  SiftPyramid p;
  p.n = L.nO; p.B = B;
  for (int o = 0; o < L.nO; ++o) {
    p.oct[o].gauss = reinterpret_cast<float*>(ws + L.gauss_off[o]);
    p.oct[o].dog = reinterpret_cast<float*>(ws + L.dog_off[o]);
    p.oct[o].h = L.h[o]; p.oct[o].w = L.w[o];
  }
  return p;
}

inline unsigned sift_grid(int64_t n) { return (unsigned)std::min<int64_t>((n + 255) / 256, 132 * 32); }

}  // namespace og
