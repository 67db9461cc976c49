// kornia's DoG SIFT (the reference's default online features, SIFT: models/features/sift.py on models/features/base.py), restated
// from kornia 0.6.3.  Stages (each its own entry point in api.cu):
//   pyramid   ScalePyramid(3, 1.6, 32, double_image=True) + BlobDoG for B same-size images: bilinear 2x upsample, Gaussian blurs
//             (separable here; kornia convolves with the 2-D outer-product kernel), [::2, ::2] subsample, DoG.
//   detect    ConvQuadInterp3d(10) on the DoG and on -DoG, the larger response per voxel, the per-octave top-k over every voxel
//             (exact radix select on (response desc, voxel index asc)), LAFs, laf_is_inside_image, the octave -> image mapping
//             and the global top-k (response desc, octave asc, per-octave rank asc).
//   select    base.py's run_nms per image: float32 key sort, unique positions, 9x9 nms2d on the scattered scores, top-k, and
//             optionally the min-stack over the batch.
//   describe  LAFOrienter(19) (skipped when upright) and LAFDescriptor(SIFTDescriptor(41, rootsift)) of the selected LAFs only,
//             on kornia's pyrdown patch pyramid.
#pragma once
#include "common.cuh"

namespace og {

constexpr int KS_LEVELS = 6;                 // n_levels + 3 Gaussian levels per octave
constexpr int KS_DOG = 5;
constexpr int KS_MAX_OCTAVES = 16;
constexpr int KS_MAX_PATCH_LEVELS = 16;
constexpr int KS_MAX_TAPS = 64;
constexpr int KS_MAX_FEATURES = 8192;           // num_features / max_keypoints per image: one CTA sorts them in shared memory
constexpr int KS_ORI_PS = 19, KS_DESC_PS = 41, KS_ORI_BINS = 36;
constexpr float KS_PI = 3.14159265358979323846f;  // kornia.constants.pi (float32)

struct KsTaps { int n; float k[KS_MAX_TAPS]; };
// The Gaussian weightings of the 19- and 41-pixel patches (get_gaussian_kernel2d(PS, PS / sqrt 2)) and SIFT's pooling kernel
struct KsDescConst { float ori_w[KS_ORI_PS * KS_ORI_PS]; float desc_w[KS_DESC_PS * KS_DESC_PS]; float pool[16 * 16]; };


// One octave's slice of the workspace (floats): Gaussian levels [B][6][h][w], DoG [B][5][h][w], responses [B][5][h][w]
struct KsOctave { int h, w; int64_t gauss, dog, resp; };

struct KsLayout {
  int nO, k;                                 // octaves, per-octave candidates (num_features)
  KsOctave oct[KS_MAX_OCTAVES];
  int np;                                    // pyrdown patch-pyramid levels
  int ph[KS_MAX_PATCH_LEVELS], pw[KS_MAX_PATCH_LEVELS];
  int64_t pyr[KS_MAX_PATCH_LEVELS];          // float offsets of the patch-pyramid levels [B][h][w] (level 0 is the input image)
  int64_t tmp;                               // float offset: B * h0 * w0 scratch of the separable blur
  int64_t state, hist, cand, list, scratch, count;   // byte offsets of the detector's selection state
  int64_t consts;                            // byte offset of the descriptor's weight tables (KsDescConst)
  int64_t bytes;
};

// Octave sizes: 2H x 2W (H x W without double_image), then [::2, ::2] while the smaller side stays above 32
// (ScalePyramid.forward).  The per-octave volume the detector reads ("dog") has vol_levels levels: the 5 DoG levels of SIFT, or
// the GFTT responses of all 6 Gaussian levels.
inline bool ks_layout(int B, int H, int W, int k, KsLayout& L, bool double_image = true, int vol_levels = KS_DOG) {
  L = KsLayout{};
  L.k = k;
  int h = double_image ? 2 * H : H, w = double_image ? 2 * W : W;
  int64_t f = 0;
  for (;;) {
    if (L.nO == KS_MAX_OCTAVES) return false;
    KsOctave& o = L.oct[L.nO++];
    o.h = h; o.w = w;
    const int64_t plane = (int64_t)B * h * w;
    o.gauss = f; f += KS_LEVELS * plane;
    o.dog = f; f += vol_levels * plane;
    o.resp = f; f += KS_DOG * plane;
    const int nh = (h + 1) / 2, nw = (w + 1) / 2;
    if (min(nh, nw) <= 32) break;
    h = nh; w = nw;
  }
  L.tmp = f; f += (int64_t)B * L.oct[0].h * L.oct[0].w;
  // patch pyramid for 19-pixel patches (the deeper of the two): level k + 1 exists while level k's smaller side is >= 19
  int ph = H, pw = W;
  L.np = 1; L.ph[0] = H; L.pw[0] = W; L.pyr[0] = -1;
  while (min(ph, pw) >= KS_ORI_PS) {
    if (L.np == KS_MAX_PATCH_LEVELS) return false;
    ph /= 2; pw /= 2;
    L.ph[L.np] = ph; L.pw[L.np] = pw;
    L.pyr[L.np] = f; f += (int64_t)B * max(ph, 1) * max(pw, 1);
    ++L.np;
  }
  int64_t b = align_up(f * 4, 256);
  const int segs = B * L.nO;
  L.state = b; b = align_up(b + (int64_t)segs * 32, 256);
  L.hist = b; b = align_up(b + (int64_t)segs * 256 * 4, 256);
  L.cand = b; b = align_up(b + (int64_t)segs * k * 8, 256);
  L.list = b; b = align_up(b + (int64_t)segs * k * 16, 256);
  L.scratch = b; b = align_up(b + (int64_t)segs * k * 16, 256);
  L.count = b; b = align_up(b + (int64_t)segs * 4, 256);
  L.consts = b; b = align_up(b + (int64_t)sizeof(KsDescConst), 256);
  L.bytes = b;
  return true;
}

// kornia.filters.kernels.gaussian(ksize, sigma) in float32 (the 1-D factor of get_gaussian_kernel2d)
inline void ks_gaussian_taps(int ksize, double sigma, KsTaps& t) {
  t.n = ksize;
  float s = 0.f;
  const float den = (float)(2 * sigma * sigma);
  for (int i = 0; i < ksize; ++i) {
    float x = (float)i - (float)(ksize / 2);
    if (ksize % 2 == 0) x += 0.5f;
    t.k[i] = expf(-(x * x) / den);
  }
  for (int i = 0; i < ksize; ++i) s += t.k[i];
  for (int i = 0; i < ksize; ++i) t.k[i] = t.k[i] / s;
}
// ScalePyramid.get_kernel_size, with forward()'s clamp to the level's smaller side
inline int ks_kernel_size(double sigma, int h, int w) {
  int k = (int)(2.0 * 4.0 * sigma + 1.0);
  if (k % 2 == 0) ++k;
  k = min(k, min(h, w));
  if (k % 2 == 0) ++k;
  return k;
}

__device__ __forceinline__ int ks_reflect(int i, int n) {
  if (n == 1) return 0;
  while (i < 0 || i >= n) i = i < 0 ? -i : 2 * (n - 1) - i;
  return i;
}

// ---- pyramid ----
// F.interpolate(scale_factor=2, bilinear, align_corners=False): source = max(0.5 (dst + 0.5) - 0.5, 0); out: level 0 of the first
// octave ([B][6][2H][2W])
__global__ void ks_upsample_kernel(const float* __restrict__ img, int B, int H, int W, float* __restrict__ out) {
  const int64_t n = (int64_t)B * 4 * H * W;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % (2 * W)), y = (int)((i / (2 * W)) % (2 * H)), b = (int)(i / (4LL * H * W));
    const float sy = fmaxf(0.5f * ((float)y + 0.5f) - 0.5f, 0.f), sx = fmaxf(0.5f * ((float)x + 0.5f) - 0.5f, 0.f);
    const int y0 = (int)sy, x0 = (int)sx;
    const int yp = y0 < H - 1 ? 1 : 0, xp = x0 < W - 1 ? 1 : 0;
    const float ly1 = sy - (float)y0, ly0 = 1.f - ly1, lx1 = sx - (float)x0, lx0 = 1.f - lx1;
    const float* p = img + (int64_t)b * H * W;
    const float v00 = p[y0 * W + x0], v01 = p[y0 * W + x0 + xp], v10 = p[(y0 + yp) * W + x0], v11 = p[(y0 + yp) * W + x0 + xp];
    out[(int64_t)b * KS_LEVELS * 4 * H * W + i % (4LL * H * W)] =
        __fadd_rn(__fmul_rn(ly0, __fadd_rn(__fmul_rn(lx0, v00), __fmul_rn(lx1, v01))),
                  __fmul_rn(ly1, __fadd_rn(__fmul_rn(lx0, v10), __fmul_rn(lx1, v11))));
  }
}

// One pass of the separable Gaussian blur, reflect border: along x (dir 0) or y (dir 1) of B planes of h x w
__global__ void ks_blur_kernel(const float* __restrict__ src, int64_t src_stride, int B, int h, int w, KsTaps t, int dir,
                               float* __restrict__ dst, int64_t dst_stride) {
  const int64_t n = (int64_t)B * h * w;
  const int r = t.n / 2;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % w), y = (int)((i / w) % h), b = (int)(i / ((int64_t)h * w));
    const float* p = src + b * src_stride;
    float acc = 0.f;
    if (dir == 0) {
      for (int j = 0; j < t.n; ++j) acc = __fmaf_rn(t.k[j], p[(int64_t)y * w + ks_reflect(x + j - r, w)], acc);
    } else {
      for (int j = 0; j < t.n; ++j) acc = __fmaf_rn(t.k[j], p[(int64_t)ks_reflect(y + j - r, h) * w + x], acc);
    }
    dst[b * dst_stride + (int64_t)y * w + x] = acc;
  }
}

// DoG levels of one octave: dog[b][l] = gauss[b][l + 1] - gauss[b][l]
__global__ void ks_dog_kernel(const float* __restrict__ gauss, int B, int hw, float* __restrict__ dog) {
  const int64_t n = (int64_t)B * KS_DOG * hw;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / ((int64_t)KS_DOG * hw), r = i % ((int64_t)KS_DOG * hw);
    const float* g = gauss + b * KS_LEVELS * hw + r;
    dog[i] = __fsub_rn(g[hw], g[0]);
  }
}

// The next octave's first level: level 3 of the previous octave at [::2, ::2]
__global__ void ks_subsample_kernel(const float* __restrict__ prev, int B, int h, int w, int nh, int nw, float* __restrict__ out) {
  const int64_t n = (int64_t)B * nh * nw;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % nw), y = (int)((i / nw) % nh), b = (int)(i / ((int64_t)nh * nw));
    out[b * (int64_t)KS_LEVELS * nh * nw + (int64_t)y * nw + x] = prev[b * (int64_t)KS_LEVELS * h * w + 3LL * h * w + (int64_t)(2 * y) * w + 2 * x];
  }
}

// ---- detect ----
struct KsPoint { float resp, s, x, y; };

// conv_quad_interp3d at one voxel of u = sign * DoG (replicate border): the response and the (s, x, y) coordinate
__device__ __forceinline__ KsPoint ks_quad_interp(const float* __restrict__ d, float sign, int h, int w, int l, int y, int x) {
  auto at = [&](int dl, int dy, int dx) {
    const int ll = min(max(l + dl, 0), KS_DOG - 1), yy = min(max(y + dy, 0), h - 1), xx = min(max(x + dx, 0), w - 1);
    return sign * __ldg(d + ((int64_t)ll * h + yy) * w + xx);
  };
  const float c = at(0, 0, 0);
  KsPoint p{c, (float)l, (float)x, (float)y};
  float m = -CUDART_INF_F;
  for (int dl = -1; dl <= 1; ++dl)
    for (int dy = -1; dy <= 1; ++dy)
      for (int dx = -1; dx <= 1; ++dx)
        if (dl | dy | dx) m = fmaxf(m, at(dl, dy, dx));
  if (!(c > m)) return p;
  // spatial_gradient3d 'diff': b = half central differences; the Hessian from the depth-flipped second-order kernel
  const float b0 = __fmul_rn(0.5f, __fsub_rn(at(0, 0, 1), at(0, 0, -1)));
  const float b1 = __fmul_rn(0.5f, __fsub_rn(at(0, 1, 0), at(0, -1, 0)));
  const float b2 = __fmul_rn(0.5f, __fsub_rn(at(1, 0, 0), at(-1, 0, 0)));
  const float c2 = __fmul_rn(-2.f, c);
  const float dxx = __fadd_rn(__fadd_rn(at(0, 0, -1), c2), at(0, 0, 1));
  const float dyy = __fadd_rn(__fadd_rn(at(0, -1, 0), c2), at(0, 1, 0));
  const float dss = __fadd_rn(__fadd_rn(at(-1, 0, 0), c2), at(1, 0, 0));
  const float dxy = __fmul_rn(0.25f, __fadd_rn(__fsub_rn(__fsub_rn(at(0, -1, -1), at(0, -1, 1)), at(0, 1, -1)), at(0, 1, 1)));
  const float dys = __fmul_rn(0.25f, __fsub_rn(__fadd_rn(__fsub_rn(at(-1, 1, 0), at(-1, -1, 0)), at(1, -1, 0)), at(1, 1, 0)));
  const float dxs = __fmul_rn(0.25f, __fsub_rn(__fadd_rn(__fsub_rn(at(-1, 0, 1), at(-1, 0, -1)), at(1, 0, -1)), at(1, 0, 1)));
  // LU with partial pivoting (LAPACK getrf: the first largest |pivot|), "solved" when no pivot is exactly 0
  float A[3][3] = {{dxx, dxy, dxs}, {dxy, dyy, dys}, {dxs, dys, dss}};
  float r[3] = {b0, b1, b2};
  for (int k = 0; k < 3; ++k) {
    int piv = k;
    for (int i = k + 1; i < 3; ++i) if (fabsf(A[i][k]) > fabsf(A[piv][k])) piv = i;
    if (A[piv][k] == 0.f) return p;
    if (piv != k) {
      for (int j = 0; j < 3; ++j) { const float t = A[k][j]; A[k][j] = A[piv][j]; A[piv][j] = t; }
      const float t = r[k]; r[k] = r[piv]; r[piv] = t;
    }
    const float inv = __frcp_rn(A[k][k]);
    for (int i = k + 1; i < 3; ++i) {
      const float f = __fmul_rn(A[i][k], inv);
      for (int j = k + 1; j < 3; ++j) A[i][j] = __fsub_rn(A[i][j], __fmul_rn(f, A[k][j]));
      r[i] = __fsub_rn(r[i], __fmul_rn(f, r[k]));
    }
  }
  float s[3];
  for (int i = 2; i >= 0; --i) {
    float v = r[i];
    for (int j = i + 1; j < 3; ++j) v = __fsub_rn(v, __fmul_rn(A[i][j], s[j]));
    s[i] = __fdiv_rn(v, A[i][i]);
  }
  float dx0 = -s[0], dx1 = -s[1], dx2 = -s[2];
  if (fmaxf(fabsf(dx0), fmaxf(fabsf(dx1), fabsf(dx2))) > 0.7f) dx0 = dx1 = dx2 = 0.f;
  const float dot = __fadd_rn(__fadd_rn(__fmul_rn(b0, dx0), __fmul_rn(b1, dx1)), __fmul_rn(b2, dx2));
  p.resp = __fadd_rn(__fadd_rn(c, __fmul_rn(0.5f, dot)), 10.f);
  // coords = create_meshgrid3d's (s, x, y) + dx.flip(1) = (s + dx2, x + dx1, y + dx0)
  p.s = __fadd_rn((float)l, dx2); p.x = __fadd_rn((float)x, dx1); p.y = __fadd_rn((float)y, dx0);
  return p;
}
__device__ __forceinline__ KsPoint ks_point(const float* d, int h, int w, int l, int y, int x) {
  const KsPoint mx = ks_quad_interp(d, 1.f, h, w, l, y, x), mn = ks_quad_interp(d, -1.f, h, w, l, y, x);
  return mn.resp > mx.resp ? mn : mx;
}

__device__ __forceinline__ uint32_t ks_order(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ks_unorder(uint32_t u) { return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u); }

// Responses of every voxel of one octave
__global__ void ks_response_kernel(const float* __restrict__ dog, int B, int h, int w, float* __restrict__ resp) {
  const int64_t per = (int64_t)KS_DOG * h * w, n = B * per;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / per, r = i % per;
    const int x = (int)(r % w), y = (int)((r / w) % h), l = (int)(r / ((int64_t)h * w));
    resp[i] = ks_point(dog + b * per, h, w, l, y, x).resp;
  }
}

// Radix-select state of one (image, octave) segment: the key prefix found so far, the number of low bits still open, the keys
// still to take among those matching the prefix; done: the keys >= prefix on the resolved bits are exactly the k selected
struct KsSel { unsigned long long prefix; int low, need, done, pad; };

__device__ __forceinline__ unsigned long long ks_key(float r, int64_t idx) {
  return ((unsigned long long)ks_order(r) << 32) | (unsigned long long)(0xffffffffu - (uint32_t)idx);
}
__device__ __forceinline__ bool ks_selected(unsigned long long key, const KsSel& S) {
  return S.low >= 64 || (key >> S.low) >= (S.prefix >> S.low);
}

// One thread per segment (B * nO): the start of the selection, all of an octave's voxels when it has at most k
__global__ void ks_select_init_kernel(KsLayout L, int segs, KsSel* st, unsigned int* hist, int* count) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= segs) return;
  const KsOctave oc = L.oct[s % L.nO];
  const int64_t n = (int64_t)KS_DOG * oc.h * oc.w;
  st[s] = KsSel{0ull, 64, (int)(n < L.k ? n : L.k), n <= L.k ? 1 : 0, 0};
  for (int i = 0; i < 256; ++i) hist[s * 256 + i] = 0;
  count[s] = 0;
}

// Histogram of the next 8-bit digit of the keys that match their segment's prefix; one octave, grid (x, B)
__global__ void ks_hist_kernel(const float* __restrict__ resp, int64_t per, int o, int nO, const KsSel* __restrict__ st,
                               unsigned int* __restrict__ hist) {
  __shared__ unsigned int h[256];
  const int b = blockIdx.y, s = b * nO + o;
  const KsSel S = st[s];
  if (S.done) return;
  for (int i = threadIdx.x; i < 256; i += blockDim.x) h[i] = 0;
  __syncthreads();
  const int sh = S.low - 8;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < per; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long key = ks_key(resp[b * per + i], i);
    if (S.low == 64 || (key >> S.low) == (S.prefix >> S.low)) atomicAdd(&h[(key >> sh) & 255u], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 256; i += blockDim.x) if (h[i]) atomicAdd(&hist[s * 256 + i], h[i]);
}

// One thread per image: picks the digit of segment (b, o) from its histogram and clears the histogram
__global__ void ks_pick_kernel(int B, int o, int nO, KsSel* st, unsigned int* hist) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int s = b * nO + o;
  KsSel S = st[s];
  if (S.done) return;
  unsigned int* h = hist + s * 256;
  int above = 0, d = 255;
  for (; d > 0; --d) {
    if (above + (int)h[d] >= S.need) break;
    above += (int)h[d];
  }
  S.need -= above;
  S.low -= 8;
  S.prefix |= (unsigned long long)d << S.low;
  if ((int)h[d] == S.need || S.low == 0) S.done = 1;
  st[s] = S;
  for (int i = 0; i < 256; ++i) h[i] = 0;
}

// Compacts the selected keys of one octave into cand[s][0 .. k)
__global__ void ks_compact_kernel(const float* __restrict__ resp, int64_t per, int o, int nO, const KsSel* __restrict__ st,
                                  int k, unsigned long long* __restrict__ cand, int* __restrict__ count) {
  const int b = blockIdx.y, s = b * nO + o;
  const KsSel S = st[s];
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < per; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long key = ks_key(resp[b * per + i], i);
    if (ks_selected(key, S)) {
      const int slot = atomicAdd(count + s, 1);
      if (slot < k) cand[(int64_t)s * k + slot] = key;
    }
  }
}

struct KsCand { float resp, scale, x, y; };     // a detector candidate in image pixels (LAF = [[scale, 0, x], [0, scale, y]])

// One segment per CTA: sorts its candidates (response desc, voxel asc), builds their LAFs, zeroes the responses of LAFs that
// touch the octave border, maps them to the image, and sorts again by (zeroed response desc, rank asc): list[s][0 .. n)
// GFTT: the volume holds 6 levels per image, of which the first 5 enter the interpolation, and only maxima count.
template <int THREADS, int GFTT = 0>
__global__ void __launch_bounds__(THREADS) ks_octave_list_kernel(const float* __restrict__ ws_f, KsLayout L, int B, int H, int W,
                                                                 const int* __restrict__ count, KsCand* __restrict__ scratch,
                                                                 KsCand* __restrict__ list, const unsigned long long* __restrict__ cand) {
  extern __shared__ unsigned long long ks_smem[];
  const int s = blockIdx.x, b = s / L.nO, o = s % L.nO, k = L.k;
  const KsOctave oc = L.oct[o];
  const int n = min(count[s], k);
  const int n2 = pow2_ceil(max(n, 1));
  unsigned long long* key = ks_smem;
  for (int j = threadIdx.x; j < n2; j += THREADS) key[j] = j < n ? cand[(int64_t)s * k + j] : 0ull;
  __syncthreads();
  cta_bitonic_sort<THREADS>(n2, [&](int lo, int hi) { return key[lo] > key[hi]; },
                            [&](int lo, int hi) { const auto t = key[lo]; key[lo] = key[hi]; key[hi] = t; });
  const float* dog = ws_f + oc.dog + (int64_t)b * (GFTT ? KS_LEVELS : KS_DOG) * oc.h * oc.w;
  // laf_to_boundary_points(12): the centre, then (sin t, cos t) at torch.linspace(0, 2 pi, 11)
  const float mo = (float)min(oc.h - 1, oc.w - 1), mi = (float)min(H - 1, W - 1);
  for (int j = threadIdx.x; j < n; j += THREADS) {
    const uint32_t idx = 0xffffffffu - (uint32_t)(key[j] & 0xffffffffull);
    const int x = (int)(idx % oc.w), y = (int)((idx / oc.w) % oc.h), l = (int)(idx / ((uint32_t)oc.h * oc.w));
    const KsPoint p = GFTT ? ks_quad_interp(dog, 1.f, oc.h, oc.w, l, y, x) : ks_point(dog, oc.h, oc.w, l, y, x);
    const float sigma = __fmul_rn(1.6f, exp2f(__fdiv_rn(p.s, 3.f)));
    const float sc = __fmul_rn(6.0f, sigma);
    bool good = p.x >= 0.f && p.x <= (float)oc.w && p.y >= 0.f && p.y <= (float)oc.h;
    const float step = __fdiv_rn(2.f * KS_PI, 10.f);
    for (int i = 0; i < 11 && good; ++i) {
      const float t = i < 5 ? __fmul_rn(step, (float)i) : __fsub_rn(2.f * KS_PI, __fmul_rn(step, (float)(10 - i)));
      const float px = __fadd_rn(__fmul_rn(sc, sinf(t)), p.x), py = __fadd_rn(__fmul_rn(sc, cosf(t)), p.y);
      good = px >= 0.f && px <= (float)oc.w && py >= 0.f && py <= (float)oc.h;
    }
    KsCand c;
    c.resp = good ? p.resp : __fmul_rn(p.resp, 0.f);
    c.scale = __fmul_rn(__fdiv_rn(sc, mo), mi);
    c.x = __fmul_rn(__fdiv_rn(p.x, (float)(oc.w - 1)), (float)(W - 1));
    c.y = __fmul_rn(__fdiv_rn(p.y, (float)(oc.h - 1)), (float)(H - 1));
    scratch[(int64_t)s * k + j] = c;
  }
  __syncthreads();
  float* fk = reinterpret_cast<float*>(ks_smem);
  int* fv = reinterpret_cast<int*>(fk + n2);
  for (int j = threadIdx.x; j < n2; j += THREADS) {
    fk[j] = j < n ? scratch[(int64_t)s * k + j].resp : -CUDART_INF_F;
    fv[j] = j < n ? j : INT_MAX;
  }
  __syncthreads();
  cta_bitonic_sort<THREADS>(n2, [&](int lo, int hi) { return topk_before(fk[lo], fv[lo], fk[hi], fv[hi]); },
                            [&](int lo, int hi) {
                              const float a = fk[lo]; fk[lo] = fk[hi]; fk[hi] = a;
                              const int v = fv[lo]; fv[lo] = fv[hi]; fv[hi] = v;
                            });
  for (int j = threadIdx.x; j < n; j += THREADS) list[(int64_t)s * k + j] = scratch[(int64_t)s * k + fv[j]];
}

// Global top-k over the octave lists: element (o, j) goes to rank j + the elements of lower octaves with a response >= its own
// + those of higher octaves with a larger one.  grid (cdiv(k, 256), nO, B)
__global__ void ks_merge_kernel(const KsCand* __restrict__ list, const int* __restrict__ count, int nO, int k, float* __restrict__ lafs,
                                float* __restrict__ resp, int* __restrict__ det_count) {
  const int b = blockIdx.z, o = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = min(count[b * nO + o], k);
  if (o == 0 && j == 0) {
    int tot = 0;
    for (int q = 0; q < nO; ++q) tot += min(count[b * nO + q], k);
    det_count[b] = min(tot, k);
  }
  if (j >= n) return;
  const KsCand c = list[((int64_t)b * nO + o) * k + j];
  int rank = j;
  for (int q = 0; q < nO; ++q) {
    if (q == o) continue;
    const KsCand* lq = list + ((int64_t)b * nO + q) * k;
    int lo = 0, hi = min(count[b * nO + q], k);
    while (lo < hi) {                            // the number of elements that go before c
      const int mid = (lo + hi) >> 1;
      const bool before = q < o ? lq[mid].resp >= c.resp : lq[mid].resp > c.resp;
      if (before) lo = mid + 1; else hi = mid;
    }
    rank += lo;
  }
  if (rank >= k) return;
  float* l = lafs + ((int64_t)b * k + rank) * 6;
  l[0] = c.scale; l[1] = 0.f; l[2] = c.x; l[3] = 0.f; l[4] = c.scale; l[5] = c.y;
  resp[(int64_t)b * k + rank] = c.resp;
}

// Zeroes the detector output rows past det_count[b]
__global__ void ks_det_tail_kernel(const int* __restrict__ det_count, int k, float* __restrict__ lafs, float* __restrict__ resp) {
  const int b = blockIdx.y;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < k; j += gridDim.x * blockDim.x)
    if (j >= det_count[b]) {
      resp[(int64_t)b * k + j] = 0.f;
      for (int e = 0; e < 6; ++e) lafs[((int64_t)b * k + j) * 6 + e] = 0.f;
    }
}

// ---- select: base.py's run_nms ----
// One image per CTA: keys, sort, unique positions, nms2d on the scattered scores; keep[b][j] = 1 for the detector outputs j that
// survive, kept[b] their number.  smem: pow2_ceil(n) x (8 key + 4 x + 4 y) bytes.
template <int THREADS>
__global__ void __launch_bounds__(THREADS) ks_nms_kernel(const float* __restrict__ lafs, const float* __restrict__ resp,
                                                         const int* __restrict__ count, int cap, int H, int W, int radius, int nms,
                                                         unsigned char* __restrict__ keep, int* __restrict__ kept) {
  extern __shared__ unsigned long long ks_smem[];
  __shared__ float red_min[THREADS / 32], red_max[THREADS / 32];
  __shared__ int tot;
  const int b = blockIdx.x;
  const int n = min(max(count[b], 0), cap);
  const int n2 = pow2_ceil(max(n, 1));
  unsigned long long* key = ks_smem;
  int* px = reinterpret_cast<int*>(key + n2);
  int* py = px + n2;
  const float* R = resp + (int64_t)b * cap;
  const float* LA = lafs + (int64_t)b * cap * 6;
  if (threadIdx.x == 0) tot = 0;
  if (!nms) {
    for (int j = threadIdx.x; j < cap; j += THREADS) keep[(int64_t)b * cap + j] = j < n;
    if (threadIdx.x == 0) kept[b] = n;
    return;
  }
  float mn = CUDART_INF_F, mx = -CUDART_INF_F;
  for (int j = threadIdx.x; j < n; j += THREADS) { mn = fminf(mn, R[j]); mx = fmaxf(mx, R[j]); }
  for (int o = 16; o > 0; o >>= 1) { mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o)); mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o)); }
  if ((threadIdx.x & 31) == 0) { red_min[threadIdx.x >> 5] = mn; red_max[threadIdx.x >> 5] = mx; }
  __syncthreads();
  mn = CUDART_INF_F; mx = -CUDART_INF_F;
  for (int w = 0; w < THREADS / 32; ++w) { mn = fminf(mn, red_min[w]); mx = fmaxf(mx, red_max[w]); }
  const float den = __fadd_rn(__fsub_rn(mx, mn), 0.1f);
  for (int j = threadIdx.x; j < n2; j += THREADS) {
    if (j < n) {
      const int x = (int)rintf(LA[j * 6 + 2]), y = (int)rintf(LA[j * 6 + 5]);
      const float ns = __fdiv_rn(__fadd_rn(__fsub_rn(R[j], mn), 0.01f), den);
      const float kv = __fadd_rn((float)((long long)H * x + y), __fsub_rn(1.f, ns));
      key[j] = ((unsigned long long)ks_order(kv) << 32) | (unsigned)j;
    } else {
      key[j] = ~0ull;
    }
  }
  __syncthreads();
  cta_bitonic_sort<THREADS>(n2, [&](int lo, int hi) { return key[lo] < key[hi]; },
                            [&](int lo, int hi) { const auto t = key[lo]; key[lo] = key[hi]; key[hi] = t; });
  for (int p = threadIdx.x; p < n; p += THREADS) {
    const int j = (int)(key[p] & 0xffffffffu);
    px[p] = (int)rintf(LA[j * 6 + 2]); py[p] = (int)rintf(LA[j * 6 + 5]);
  }
  __syncthreads();
  // unique_consecutive on h x + y in sorted order: position p is kept when it starts a run.  The mask holds, per position, the
  // score of the last kept entry written there (index_put_ in sorted order).  Entries of one position are at most 2 apart in key,
  // entries within the window at most H * radius + radius + 2.
  auto uniq = [&](int p) { return p == 0 || px[p] != px[p - 1] || py[p] != py[p - 1]; };
  auto keyval = [&](int p) { return ks_unorder((uint32_t)(key[p] >> 32)); };
  auto mask_at = [&](int p0, int x, int y, bool& occ) {   // the mask value at (x, y), searching sorted entries near p0
    occ = false;
    float v = 0.f;
    const float kc = (float)((long long)H * x + y);
    int lo = 0, hi = n;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (keyval(mid) < kc - 2.f) lo = mid + 1; else hi = mid; }
    for (int q = lo; q < n && keyval(q) <= kc + 2.f; ++q)
      if (uniq(q) && px[q] == x && py[q] == y) { v = R[(int)(key[q] & 0xffffffffu)]; occ = true; }
    return v;
  };
  for (int p = threadIdx.x; p < n; p += THREADS) {
    const int j = (int)(key[p] & 0xffffffffu);
    bool on = false;
    if (uniq(p)) {
      const int x = px[p], y = py[p];
      if (x > 0 && x < W - 1 && y > 0 && y < H - 1) {
        bool occ;
        const float v = mask_at(p, x, y, occ);
        float m = -CUDART_INF_F;
        for (int dx = -radius; dx <= radius; ++dx) {
          const int xx = min(max(x + dx, 0), W - 1);
          for (int dy = -radius; dy <= radius; ++dy) {
            if (!(dx | dy)) continue;
            const int yy = min(max(y + dy, 0), H - 1);
            const float u = mask_at(p, xx, yy, occ);
            m = fmaxf(m, u);
          }
        }
        on = v > m;
      }
    }
    keep[(int64_t)b * cap + j] = on;
  }
  for (int j = n + threadIdx.x; j < cap; j += THREADS) keep[(int64_t)b * cap + j] = 0;
  __syncthreads();
  int c = 0;
  for (int j = threadIdx.x; j < n; j += THREADS) c += keep[(int64_t)b * cap + j];
  c = warp_sum(c);
  if ((threadIdx.x & 31) == 0) atomicAdd(&tot, c);
  __syncthreads();
  if (threadIdx.x == 0) kept[b] = tot;
}

// The first min(kept, max_keypoints) survivors in detector order (= torch.topk of their scores, equal scores by detector index),
// kept = the batch minimum with min_stack: sel[b][0 .. n_sel[b]).  One image per CTA.
__global__ void ks_select_kernel(const unsigned char* __restrict__ keep, const int* __restrict__ kept, int B, int cap, int max_keypoints,
                                 int min_stack, int* __restrict__ sel, int* __restrict__ n_sel) {
  __shared__ int warp_tot[32];
  __shared__ int base;
  const int b = blockIdx.x;
  int want = kept[b];
  if (min_stack) for (int q = 0; q < B; ++q) want = min(want, kept[q]);
  if (max_keypoints > 0) want = min(want, max_keypoints);
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  for (int j0 = 0; j0 < cap; j0 += blockDim.x) {
    const int j = j0 + threadIdx.x;
    const bool on = j < cap && keep[(int64_t)b * cap + j];
    const int slot = cta_ordered_slot(on, warp_tot, base);
    if (on && slot < want) sel[(int64_t)b * cap + slot] = j;
  }
  if (threadIdx.x == 0) n_sel[b] = want;
}

// ---- describe ----
// kornia pyrdown: the 5x5 binomial (reflect) then bilinear to (h / 2, w / 2), align_corners=False, scale = h / (h / 2)
__global__ void ks_pyrdown_blur_kernel(const float* __restrict__ src, int B, int h, int w, float* __restrict__ dst) {
  const float k1[5] = {1.f, 4.f, 6.f, 4.f, 1.f};
  const int64_t n = (int64_t)B * h * w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % w), y = (int)((i / w) % h), b = (int)(i / ((int64_t)h * w));
    const float* p = src + (int64_t)b * h * w;
    float acc = 0.f;
    for (int dy = 0; dy < 5; ++dy) {
      const int yy = ks_reflect(y + dy - 2, h);
      for (int dx = 0; dx < 5; ++dx)
        acc = __fmaf_rn(__fdiv_rn(k1[dy] * k1[dx], 256.f), p[(int64_t)yy * w + ks_reflect(x + dx - 2, w)], acc);
    }
    dst[i] = acc;
  }
}
__global__ void ks_pyrdown_resize_kernel(const float* __restrict__ src, int B, int h, int w, int nh, int nw, float* __restrict__ dst) {
  const int64_t n = (int64_t)B * nh * nw;
  const float scy = __fdiv_rn((float)h, (float)nh), scx = __fdiv_rn((float)w, (float)nw);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % nw), y = (int)((i / nw) % nh), b = (int)(i / ((int64_t)nh * nw));
    const float sy = fmaxf(__fsub_rn(__fmul_rn(scy, (float)y + 0.5f), 0.5f), 0.f), sx = fmaxf(__fsub_rn(__fmul_rn(scx, (float)x + 0.5f), 0.5f), 0.f);
    const int y0 = (int)sy, x0 = (int)sx;
    const int yp = y0 < h - 1 ? 1 : 0, xp = x0 < w - 1 ? 1 : 0;
    const float ly1 = sy - (float)y0, ly0 = 1.f - ly1, lx1 = sx - (float)x0, lx0 = 1.f - lx1;
    const float* p = src + (int64_t)b * h * w;
    const float v00 = p[y0 * w + x0], v01 = p[y0 * w + x0 + xp], v10 = p[(y0 + yp) * w + x0], v11 = p[(y0 + yp) * w + x0 + xp];
    dst[i] = __fadd_rn(__fmul_rn(ly0, __fadd_rn(__fmul_rn(lx0, v00), __fmul_rn(lx1, v01))),
                       __fmul_rn(ly1, __fadd_rn(__fmul_rn(lx0, v10), __fmul_rn(lx1, v11))));
  }
}

// Fills the descriptor's weight tables: kornia's float32 Gaussian weightings and the SIFT pooling kernel.  One thread.
__global__ void ks_desc_const_kernel(KsDescConst* K) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  auto fill = [](float* out, int ps) {
    float g[KS_DESC_PS];
    const double sigma = (double)ps / sqrt(2.0);
    const float den = (float)(2 * sigma * sigma);
    float s = 0.f;
    for (int i = 0; i < ps; ++i) { const float x = (float)(i - ps / 2); g[i] = expf(-(x * x) / den); }
    for (int i = 0; i < ps; ++i) s += g[i];
    for (int i = 0; i < ps; ++i) g[i] = g[i] / s;
    for (int i = 0; i < ps; ++i) for (int j = 0; j < ps; ++j) out[i * ps + j] = __fmul_rn(g[i], g[j]);
  };
  fill(K->ori_w, KS_ORI_PS);
  fill(K->desc_w, KS_DESC_PS);
  for (int i = 0; i < 16; ++i)
    for (int j = 0; j < 16; ++j) {
      const float a = 8.f - fabsf((float)i + 0.5f - 8.f), b = 8.f - fabsf((float)j + 0.5f - 8.f);
      K->pool[i * 16 + j] = __fmul_rn(a, b) / 64.f;
    }
}

struct KsPyr { int n; int h[KS_MAX_PATCH_LEVELS], w[KS_MAX_PATCH_LEVELS]; const float* p[KS_MAX_PATCH_LEVELS]; };

// extract_patches_from_pyramid for one LAF into patch[PS * PS] (shared), every thread of the CTA
template <int PS>
__device__ void ks_patch(const KsPyr& P, int b, int H, int W, const float a[6], float* patch) {
  const float m = (float)min(H - 1, W - 1);
  const float n00 = __fdiv_rn(a[0], m), n01 = __fdiv_rn(a[1], m), n02 = __fdiv_rn(a[2], (float)(W - 1));
  const float n10 = __fdiv_rn(a[3], m), n11 = __fdiv_rn(a[4], m), n12 = __fdiv_rn(a[5], (float)(H - 1));
  // scale = 2 get_laf_scale(denormalize_laf(nlaf, img)) / PS
  const float d00 = __fmul_rn(n00, m), d01 = __fmul_rn(n01, m), d10 = __fmul_rn(n10, m), d11 = __fmul_rn(n11, m);
  const float det = __fadd_rn(__fsub_rn(__fmul_rn(d00, d11), __fmul_rn(d10, d01)), 1e-10f);
  const float scale = __fdiv_rn(__fmul_rn(2.f, sqrtf(fabsf(det))), (float)PS);
  int lvl = (int)fminf(fmaxf(log2f(scale), 0.f), (float)max(0, min(H, W) / PS - 1));
  int levels = 1;                                 // levels the extraction visits for PS
  while (levels < P.n && min(P.h[levels - 1], P.w[levels - 1]) >= PS) ++levels;
  if (lvl >= levels) {
    for (int i = threadIdx.x; i < PS * PS; i += blockDim.x) patch[i] = 0.f;
    return;
  }
  const int h = P.h[lvl], w = P.w[lvl];
  const float mk = (float)min(h - 1, w - 1);
  const float A00 = __fmul_rn(n00, mk), A01 = __fmul_rn(n01, mk), A02 = __fmul_rn(n02, (float)(w - 1));
  const float A10 = __fmul_rn(n10, mk), A11 = __fmul_rn(n11, mk), A12 = __fmul_rn(n12, (float)(h - 1));
  const float* img = P.p[lvl] + (int64_t)b * h * w;
  const float step = __fdiv_rn(2.f, (float)(PS - 1));
  for (int i = threadIdx.x; i < PS * PS; i += blockDim.x) {
    const int r = i / PS, c = i % PS;
    auto base = [&](int j) {                        // linspace(-1, 1, PS) * (PS - 1) / PS
      const float v = j < PS / 2 ? __fadd_rn(-1.f, __fmul_rn(step, (float)j)) : __fsub_rn(1.f, __fmul_rn(step, (float)(PS - 1 - j)));
      return __fdiv_rn(__fmul_rn(v, (float)(PS - 1)), (float)PS);
    };
    const float bx = base(c), by = base(r);
    const float gx = __fadd_rn(__fadd_rn(__fmul_rn(bx, A00), __fmul_rn(by, A01)), A02);
    const float gy = __fadd_rn(__fadd_rn(__fmul_rn(bx, A10), __fmul_rn(by, A11)), A12);
    const float ux = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, gx), (float)w), 1.f), uy = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, gy), (float)h), 1.f);
    float ix = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(ux, 1.f), (float)w), 1.f), 2.f);
    float iy = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(uy, 1.f), (float)h), 1.f), 2.f);
    ix = fminf(fmaxf(ix, 0.f), (float)(w - 1)); iy = fminf(fmaxf(iy, 0.f), (float)(h - 1));
    const float fx = floorf(ix), fy = floorf(iy);
    const int x0 = (int)fx, y0 = (int)fy;
    const float nw_ = __fmul_rn(__fsub_rn(fx + 1.f, ix), __fsub_rn(fy + 1.f, iy)), ne = __fmul_rn(__fsub_rn(ix, fx), __fsub_rn(fy + 1.f, iy));
    const float sw = __fmul_rn(__fsub_rn(fx + 1.f, ix), __fsub_rn(iy, fy)), se = __fmul_rn(__fsub_rn(ix, fx), __fsub_rn(iy, fy));
    float v = __fmul_rn(nw_, img[(int64_t)y0 * w + x0]);
    if (x0 + 1 < w) v = __fadd_rn(v, __fmul_rn(ne, img[(int64_t)y0 * w + x0 + 1]));
    if (y0 + 1 < h) v = __fadd_rn(v, __fmul_rn(sw, img[(int64_t)(y0 + 1) * w + x0]));
    if (x0 + 1 < w && y0 + 1 < h) v = __fadd_rn(v, __fmul_rn(se, img[(int64_t)(y0 + 1) * w + x0 + 1]));
    patch[i] = v;
  }
}

// LAFOrienter(19) on the LAF a (every thread of the CTA, a in registers, la its shared copy): the dominant orientation of its
// 19-pixel patch; a <- set_laf_orientation(a, rad2deg(angle) + get_laf_orientation(a)).  Returns the angle (radians).
template <int THREADS>
__device__ float ks_orient(const KsPyr& P, int b, int H, int W, const KsDescConst* __restrict__ K, float a[6], float* patch, float* wa,
                           float* wb, unsigned char* bin, float* hist, float* la) {
  ks_patch<KS_ORI_PS>(P, b, H, W, a, patch);
  __syncthreads();
  constexpr int N = KS_ORI_PS * KS_ORI_PS;
  const float two_pi = __fmul_rn(2.f, KS_PI);
  for (int i = threadIdx.x; i < N; i += THREADS) {
    const int r = i / KS_ORI_PS, c = i % KS_ORI_PS;
    auto P_ = [&](int rr, int cc) { return patch[min(max(rr, 0), KS_ORI_PS - 1) * KS_ORI_PS + min(max(cc, 0), KS_ORI_PS - 1)]; };
    // normalised Sobel (taps / 8), replicate border
    float gx = __fmul_rn(-0.125f, P_(r - 1, c - 1));
    gx = __fadd_rn(gx, __fmul_rn(0.125f, P_(r - 1, c + 1)));
    gx = __fadd_rn(gx, __fmul_rn(-0.25f, P_(r, c - 1)));
    gx = __fadd_rn(gx, __fmul_rn(0.25f, P_(r, c + 1)));
    gx = __fadd_rn(gx, __fmul_rn(-0.125f, P_(r + 1, c - 1)));
    gx = __fadd_rn(gx, __fmul_rn(0.125f, P_(r + 1, c + 1)));
    float gy = __fmul_rn(-0.125f, P_(r - 1, c - 1));
    gy = __fadd_rn(gy, __fmul_rn(-0.25f, P_(r - 1, c)));
    gy = __fadd_rn(gy, __fmul_rn(-0.125f, P_(r - 1, c + 1)));
    gy = __fadd_rn(gy, __fmul_rn(0.125f, P_(r + 1, c - 1)));
    gy = __fadd_rn(gy, __fmul_rn(0.25f, P_(r + 1, c)));
    gy = __fadd_rn(gy, __fmul_rn(0.125f, P_(r + 1, c + 1)));
    const float mag = __fmul_rn(sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), 1e-8f)), K->ori_w[i]);
    const float ori = __fadd_rn(atan2f(gy, __fadd_rn(gx, 1e-8f)), two_pi);
    const float ob = __fdiv_rn(__fmul_rn((float)KS_ORI_BINS, __fadd_rn(ori, KS_PI)), two_pi);
    const float f = floorf(ob);
    const float w1 = __fsub_rn(ob, f);
    int b0 = (int)f % KS_ORI_BINS;
    bin[i] = (unsigned char)b0;
    wa[i] = __fmul_rn(__fsub_rn(1.f, w1), mag);
    wb[i] = __fmul_rn(w1, mag);
  }
  __syncthreads();
  if (threadIdx.x < KS_ORI_BINS) {              // adaptive_avg_pool2d: the bin's sum over the patch in raster order / N
    const int q = threadIdx.x;
    float s = 0.f;
    for (int i = 0; i < N; ++i) {
      const int b0 = bin[i], b1 = (b0 + 1) % KS_ORI_BINS;
      s = __fadd_rn(s, __fadd_rn(b0 == q ? wa[i] : 0.f, b1 == q ? wb[i] : 0.f));
    }
    hist[q] = __fdiv_rn(s, (float)N);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float best = -CUDART_INF_F;
    int bi = 0;
    for (int q = 0; q < KS_ORI_BINS; ++q) {       // circular conv1d [0.33, 0.34, 0.33], then the first maximum
      const float v = __fadd_rn(__fadd_rn(__fmul_rn(0.33f, hist[(q + KS_ORI_BINS - 1) % KS_ORI_BINS]), __fmul_rn(0.34f, hist[q])),
                                __fmul_rn(0.33f, hist[(q + 1) % KS_ORI_BINS]));
      if (v > best) { best = v; bi = q; }
    }
    const float an = -__fsub_rn(__fdiv_rn(__fmul_rn(two_pi, (float)bi), (float)KS_ORI_BINS), KS_PI);
    // set_laf_orientation(laf, rad2deg(an) + prev): rotate_laf(make_upright(laf), new - prev)
    const float prev = __fdiv_rn(__fmul_rn(180.f, atan2f(a[1], a[0])), KS_PI);
    const float nd = __fadd_rn(__fdiv_rn(__fmul_rn(180.f, an), KS_PI), prev);
    const float rad = __fdiv_rn(__fmul_rn(__fsub_rn(nd, prev), KS_PI), 180.f);
    const float cs = cosf(rad), sn = sinf(rad);
    const float det = sqrtf(fabsf(__fadd_rn(__fsub_rn(__fmul_rn(a[0], a[4]), __fmul_rn(a[3], a[1])), 1e-10f)));
    const float b2a2 = __fadd_rn(sqrtf(__fadd_rn(__fmul_rn(a[1], a[1]), __fmul_rn(a[0], a[0]))), 1e-9f);
    const float u00 = __fmul_rn(det, __fdiv_rn(b2a2, det)), u01 = 0.f;
    const float u10 = __fmul_rn(det, __fdiv_rn(__fadd_rn(__fmul_rn(a[4], a[1]), __fmul_rn(a[3], a[0])), __fmul_rn(b2a2, det)));
    const float u11 = __fmul_rn(det, __fdiv_rn(det, b2a2));
    la[0] = __fadd_rn(__fmul_rn(u00, cs), __fmul_rn(u01, -sn));
    la[1] = __fadd_rn(__fmul_rn(u00, sn), __fmul_rn(u01, cs));
    la[3] = __fadd_rn(__fmul_rn(u10, cs), __fmul_rn(u11, -sn));
    la[4] = __fadd_rn(__fmul_rn(u10, sn), __fmul_rn(u11, cs));
    hist[0] = an;
  }
  __syncthreads();
  const float ang = hist[0];
  for (int e = 0; e < 6; ++e) a[e] = la[e];
  __syncthreads();
  return ang;
}

// One CTA per output row (j, b): orientation (unless upright) and the SIFT descriptor of LAF sel[b][j] of lafs_in; rows past
// n[b] are written as zeros.

template <int THREADS>
__global__ void __launch_bounds__(THREADS) ks_describe_kernel(KsPyr P, int H, int W, const float* __restrict__ lafs_in,
                                                              const float* __restrict__ resp_in, int cap_in, const int* __restrict__ sel,
                                                              const int* __restrict__ n, int out_cap, int upright, int rootsift,
                                                              const KsDescConst* __restrict__ K, float* __restrict__ lafs_out,
                                                              float* __restrict__ scores, float* __restrict__ desc, float* __restrict__ angle) {
  __shared__ float patch[KS_DESC_PS * KS_DESC_PS];
  __shared__ float wa[KS_DESC_PS * KS_DESC_PS], wb[KS_DESC_PS * KS_DESC_PS];
  __shared__ unsigned char bin[KS_DESC_PS * KS_DESC_PS];
  __shared__ float hist[KS_ORI_BINS];
  __shared__ float d[128];
  __shared__ float red[THREADS / 32];
  __shared__ float la[6];
  const int j = blockIdx.x, b = blockIdx.y;
  const int64_t row = (int64_t)b * out_cap + j;
  if (j >= min(n[b], out_cap)) {
    if (threadIdx.x < 6) lafs_out[row * 6 + threadIdx.x] = 0.f;
    if (threadIdx.x == 0) { scores[row] = 0.f; if (angle) angle[row] = 0.f; }
    if (threadIdx.x < 128) desc[row * 128 + threadIdx.x] = 0.f;
    return;
  }
  const int src = sel ? sel[(int64_t)b * cap_in + j] : j;
  if (threadIdx.x < 6) la[threadIdx.x] = lafs_in[((int64_t)b * cap_in + src) * 6 + threadIdx.x];
  __syncthreads();
  float a[6];
  for (int e = 0; e < 6; ++e) a[e] = la[e];
  float ang = 0.f;
  if (!upright) ang = ks_orient<THREADS>(P, b, H, W, K, a, patch, wa, wb, bin, hist, la);
  ks_patch<KS_DESC_PS>(P, b, H, W, a, patch);
  __syncthreads();
  constexpr int N = KS_DESC_PS * KS_DESC_PS;
  const float two_pi = __fmul_rn(2.f, KS_PI);
  for (int i = threadIdx.x; i < N; i += THREADS) {
    const int r = i / KS_DESC_PS, c = i % KS_DESC_PS;
    auto P_ = [&](int rr, int cc) { return patch[min(max(rr, 0), KS_DESC_PS - 1) * KS_DESC_PS + min(max(cc, 0), KS_DESC_PS - 1)]; };
    const float gx = __fsub_rn(__fmul_rn(0.5f, P_(r, c + 1)), __fmul_rn(0.5f, P_(r, c - 1)));
    const float gy = __fsub_rn(__fmul_rn(0.5f, P_(r + 1, c)), __fmul_rn(0.5f, P_(r - 1, c)));
    const float mag = __fmul_rn(sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), 1e-10f)), K->desc_w[i]);
    const float ori = __fadd_rn(atan2f(gy, __fadd_rn(gx, 1e-10f)), two_pi);
    const float ob = __fdiv_rn(__fmul_rn(8.f, ori), two_pi);
    const float f = floorf(ob);
    const float w1 = __fsub_rn(ob, f);
    bin[i] = (unsigned char)((int)f % 8);
    wa[i] = __fmul_rn(__fsub_rn(1.f, w1), mag);
    wb[i] = __fmul_rn(w1, mag);
  }
  __syncthreads();
  if (threadIdx.x < 128) {                          // 16x16 stride-10 pad-4 pooling of angle bin q, cell (cy, cx)
    const int q = threadIdx.x / 16, cy = (threadIdx.x / 4) % 4, cx = threadIdx.x % 4;
    float s = 0.f;
    for (int ky = 0; ky < 16; ++ky) {
      const int y = cy * 10 - 4 + ky;
      if (y < 0 || y >= KS_DESC_PS) continue;
      for (int kx = 0; kx < 16; ++kx) {
        const int x = cx * 10 - 4 + kx;
        if (x < 0 || x >= KS_DESC_PS) continue;
        const int i = y * KS_DESC_PS + x;
        const int b0 = bin[i], b1 = (b0 + 1) % 8;
        const float v = __fadd_rn(b0 == q ? wa[i] : 0.f, b1 == q ? wb[i] : 0.f);
        s = __fmaf_rn(K->pool[ky * 16 + kx], v, s);
      }
    }
    d[threadIdx.x] = s;
  }
  __syncthreads();
  auto norm_sum = [&](int p) {                      // sum of d^2 (p = 2) or |d| (p = 1) in a fixed order
    float v = 0.f;
    if (threadIdx.x < 128) v = p == 2 ? __fmul_rn(d[threadIdx.x], d[threadIdx.x]) : fabsf(d[threadIdx.x]);
    const float t = cta_sum<THREADS>(v, red);
    __syncthreads();
    if (threadIdx.x == 0) red[0] = t;
    __syncthreads();
    const float r = red[0];
    __syncthreads();
    return r;
  };
  float nn = fmaxf(sqrtf(norm_sum(2)), 1e-12f);
  if (threadIdx.x < 128) d[threadIdx.x] = fminf(fmaxf(__fdiv_rn(d[threadIdx.x], nn), 0.f), 0.2f);
  __syncthreads();
  nn = fmaxf(sqrtf(norm_sum(2)), 1e-12f);
  if (threadIdx.x < 128) d[threadIdx.x] = __fdiv_rn(d[threadIdx.x], nn);
  __syncthreads();
  if (rootsift) {
    nn = fmaxf(norm_sum(1), 1e-12f);
    if (threadIdx.x < 128) d[threadIdx.x] = sqrtf(__fadd_rn(__fdiv_rn(d[threadIdx.x], nn), 1e-10f));
    __syncthreads();
  }
  if (threadIdx.x < 128) desc[row * 128 + threadIdx.x] = d[threadIdx.x];
  if (threadIdx.x < 6) lafs_out[row * 6 + threadIdx.x] = a[threadIdx.x];
  if (threadIdx.x == 0) {
    scores[row] = resp_in[(int64_t)b * cap_in + src];
    if (angle) angle[row] = ang;
  }
}

}  // namespace og
