// Metric (triplet / margin) terms of the reference's matching loss and their gradient with respect to the context descriptors:
// criterion(..., margin=mu)['metric_loss'] (reference utils/losses.py:56-99 on utils/misc.py:106-113).
//
//   x_i = normalize(c0[b, :, i]),  y_j = normalize(c1[b, :, j])          (F.normalize, eps 1e-12)
//   dist_ij = 0.25 |x_i - y_j|^2 = 0.25 max(|x_i|^2 + |y_j|^2 - 2 x_i.y_j, 0)     (cdist's matrix-product form)
//   dist' = dist with +inf at every (i, gt0[i]) of a matched row
//   n0(i) = argmin_j dist'[i, :],  n1(j) = argmin_i dist'[:, j],  u0(i) = argmin_j dist[i, :],  u1(j) = argmin_i dist[:, j]
//   per pair:  w_M  sum_{i: gt0[i] = j >= 0} ( [dist_ij - dist_{i,n0(i)} + mu]_+ + [dist_ij - dist_{n1(j),j} + mu]_+ )
//            + w_U0 sum_{i: gt0[i] = -1} [mu - dist_{i,u0(i)}]_+  +  w_U1 sum_{j: gt1[j] = -1} [mu - dist_{u1(j),j}]_+
//   metric_loss = sum over pairs / B          (w = 1 / |set| per pair; an empty set adds nothing; IGNORE (-2) is in no set but
//                                              stays a candidate of every argmin)
//
// Schedule (og_metric_loss_fwd, one stream, no host synchronisation, no float atomics):
//   1. X = c0^T, Y = c1^T (og_transpose), rows normalised (og_row_normalize mode 1), squared norms (metric_sqnorm_kernel)
//   2. Gram G = X Y^T on the training step's GEMM (og_linear_auto_fwd: 3xTF32 wgmma or the exact fp32 kernel)
//   3. hard negatives: one warp per row (n0, u0), column strips per row block (n1, u1 partial) merged in row-block order;
//      every comparison is on (value, index), so ties go to the lowest index as torch.argmin's do; the distances of the
//      selections are kept and the hinges below use exactly those values
//   4. loss: one CTA per pair, fixed-order block sums, the last CTA sums the pairs in pair order (criterion_kernel's pattern);
//      with a gradient it also records each term's hinge derivative (1, 1/2 at 0 as torch.maximum, or 0) x weight x grad_scale
//   5. gradient (optional): a dense D = d loss / d dist [B, n, m] and its transpose, every element summing its own terms in one
//      fixed order (the n1 term of a column is the sum over its anchors in row order), with the row / column sums of D;
//      dX^T = -0.5 (D Y)^T and dY^T = -0.5 (D^T X)^T on the same GEMM (transposed outputs), then the normalisation backward
//      adds 0.5 rowsum(D) x (resp. colsum) and writes dc0 [B, d, n], dc1 [B, d, m].
//   For r = |x - y|^2 <= 0 the gradient is taken as 0.5 (x - y) like everywhere else (the reference's sqrt gives NaN there).
#pragma once
#include "common.cuh"
#include "train_ops.cuh"
#include <math_constants.h>
#include <climits>

namespace og {

constexpr int METRIC_THREADS = 256;
constexpr int METRIC_COLS = 128;            // columns per CTA of the column pass

// the one formula every selection and every hinge reads (explicit roundings: no contraction differences between kernels)
__device__ __forceinline__ float metric_dist(float sx, float sy, float g) {
  return __fmul_rn(0.25f, fmaxf(__fmaf_rn(-2.f, g, __fadd_rn(sx, sy)), 0.f));
}
// (v, i) before (bv, bi): smaller value, on a tie the lower index
__device__ __forceinline__ bool metric_before(float v, int i, float bv, int bi) { return v < bv || (v == bv && i < bi); }
__device__ __forceinline__ void metric_warp_argmin(float& v, int& i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (metric_before(ov, oi, v, i)) { v = ov; i = oi; }
  }
}
__device__ __forceinline__ float hinge(float x) { return fmaxf(x, 0.f); }
__device__ __forceinline__ float hinge_grad(float x) { return x > 0.f ? 1.f : (x == 0.f ? 0.5f : 0.f); }   // torch.maximum(x, 0)
__device__ __forceinline__ bool is_match(int64_t g, int m) { return g >= 0 && g < m; }

// squared norms of the rows of the normalised operands (X and Y back to back: rows = B (n + m)); one warp per row
__global__ void __launch_bounds__(256) metric_sqnorm_kernel(const float* __restrict__ x, int64_t rows, int d, float* __restrict__ sq) {
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* r = x + row * d;
  float s = 0.f;
  for (int c = lane; c < d; c += 32) s = fmaf(r[c], r[c], s);
  s = warp_sum(s);
  if (lane == 0) sq[row] = s;
}

struct MetricArgs {
  const int64_t* gt0; const int64_t* gt1;    // [B, n], [B, m]
  int B, n, m, ldg;                          // G / D: [B, n, ldg]
  float margin;
  const float* G;                            // Gram [B, n, ldg]
  const float* sqx; const float* sqy;        // [B n], [B m]
  int64_t *n0, *u0, *n1, *u1;                // outputs: [B, n], [B, n], [B, m], [B, m]
  float *dn0, *du0, *dpos;                   // [B n]: dist of n0, u0 and of the positive (matched rows)
  float *dn1, *du1;                          // [B m]
  float* part;                               // column pass: [B][chunks][4][m] (masked value, index, unmasked value, index)
  int chunks, rows_per_chunk;
  float* per_pair; unsigned int* counter; float* loss;
  float grad_scale; int want_grad;
  float *posc, *n0c, *u0c, *a1c;             // [B n] gradient coefficients of the row-side terms
  float *n1c, *u1c;                          // [B m] column-side coefficients
  int *cnt, *first;                          // [B m] anchors naming each column: count, lowest row
};

// rows: one warp per (b, i) -> n0, u0 (+ the distances of the selections and of the positive)
__global__ void __launch_bounds__(256) metric_rows_kernel(MetricArgs a) {
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= (int64_t)a.B * a.n) return;
  const int b = (int)(row / a.n);
  const int64_t g = a.gt0[row];
  const float sx = a.sqx[row];
  const float* G = a.G + row * a.ldg;
  const float* sy = a.sqy + (int64_t)b * a.m;
  float bm = CUDART_INF_F, bu = CUDART_INF_F;
  int jm = 0, ju = 0;
  for (int j = lane; j < a.m; j += 32) {                  // ascending j per lane: a strict '<' keeps the lowest index
    const float v = metric_dist(sx, sy[j], G[j]);
    if (v < bu) { bu = v; ju = j; }
    if (j == g) a.dpos[row] = v;
    else if (v < bm) { bm = v; jm = j; }
  }
  metric_warp_argmin(bm, jm);
  metric_warp_argmin(bu, ju);
  if (bm == CUDART_INF_F) bm = metric_dist(sx, sy[jm], G[jm]);    // every column masked (m == 1): index 0, its real distance
  if (lane == 0) { a.n0[row] = jm; a.u0[row] = ju; a.dn0[row] = bm; a.du0[row] = bu; }
}

// columns, stage 1: a CTA owns METRIC_COLS columns x one block of rows and scans it in row order
__global__ void __launch_bounds__(METRIC_COLS) metric_cols_kernel(MetricArgs a) {
  __shared__ int64_t s_g[256];
  __shared__ float s_sx[256];
  const int b = blockIdx.z, ch = blockIdx.y;
  const int j = blockIdx.x * METRIC_COLS + threadIdx.x;
  const int r0 = ch * a.rows_per_chunk, r1 = min(r0 + a.rows_per_chunk, a.n);
  const float sy = j < a.m ? a.sqy[(int64_t)b * a.m + j] : 0.f;
  float bm = CUDART_INF_F, bu = CUDART_INF_F;
  int im = 0, iu = 0;
  for (int t0 = r0; t0 < r1; t0 += 256) {
    const int tn = min(256, r1 - t0);
    __syncthreads();
    for (int t = threadIdx.x; t < tn; t += METRIC_COLS) {
      s_g[t] = a.gt0[(int64_t)b * a.n + t0 + t];
      s_sx[t] = a.sqx[(int64_t)b * a.n + t0 + t];
    }
    __syncthreads();
    if (j < a.m) {
      const float* G = a.G + ((int64_t)b * a.n + t0) * a.ldg + j;
      for (int t = 0; t < tn; ++t) {
        const float v = metric_dist(s_sx[t], sy, G[(int64_t)t * a.ldg]);
        if (v < bu) { bu = v; iu = t0 + t; }
        if (s_g[t] != j && v < bm) { bm = v; im = t0 + t; }
      }
    }
  }
  if (j < a.m) {
    float* p = a.part + ((int64_t)b * a.chunks + ch) * 4 * a.m;
    p[j] = bm; p[a.m + j] = __int_as_float(im); p[2 * a.m + j] = bu; p[3 * a.m + j] = __int_as_float(iu);
  }
}

// columns, stage 2: merge the row blocks in order -> n1, u1 (+ their distances)
__global__ void __launch_bounds__(256) metric_cols_merge_kernel(MetricArgs a) {
  const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (t >= (int64_t)a.B * a.m) return;
  const int b = (int)(t / a.m), j = (int)(t % a.m);
  float bm = CUDART_INF_F, bu = CUDART_INF_F;
  int im = 0, iu = 0;
  for (int ch = 0; ch < a.chunks; ++ch) {
    const float* p = a.part + ((int64_t)b * a.chunks + ch) * 4 * a.m;
    const float vm = p[j], vu = p[2 * a.m + j];
    const int jm = __float_as_int(p[a.m + j]), ju = __float_as_int(p[3 * a.m + j]);
    if (metric_before(vm, jm, bm, im)) { bm = vm; im = jm; }
    if (metric_before(vu, ju, bu, iu)) { bu = vu; iu = ju; }
  }
  if (bm == CUDART_INF_F)                                   // every row masked (n == 1, or all rows name j): index 0, its distance
    bm = metric_dist(a.sqx[(int64_t)b * a.n + im], a.sqy[t], a.G[((int64_t)b * a.n + im) * a.ldg + j]);
  a.n1[t] = im; a.u1[t] = iu; a.dn1[t] = bm; a.du1[t] = bu;
}

// the hinge arguments, one expression each (the loss and its gradient read the same values)
__device__ __forceinline__ float pos_arg(float dpos, float dneg, float mu) { return __fadd_rn(__fsub_rn(dpos, dneg), mu); }
__device__ __forceinline__ float neg_arg(float dneg, float mu) { return __fsub_rn(mu, dneg); }

// loss: one CTA per pair; the last CTA to finish sums the pairs in pair order
__global__ void __launch_bounds__(METRIC_THREADS) metric_loss_kernel(MetricArgs a) {
  __shared__ float red[METRIC_THREADS / 32];
  __shared__ float s_w[3];
  __shared__ bool last;
  const int b = blockIdx.x, n = a.n, m = a.m;
  const float mu = a.margin;
  const int64_t* g0 = a.gt0 + (int64_t)b * n;
  const int64_t* g1 = a.gt1 + (int64_t)b * m;
  const int64_t ro = (int64_t)b * n, co = (int64_t)b * m;
  if (a.want_grad)
    for (int j = threadIdx.x; j < m; j += METRIC_THREADS) { a.cnt[co + j] = 0; a.first[co + j] = INT_MAX; }
  __syncthreads();
  float s0 = 0.f, s1 = 0.f, su0 = 0.f, su1 = 0.f, cm = 0.f, cu0 = 0.f, cu1 = 0.f;
  for (int i = threadIdx.x; i < n; i += METRIC_THREADS) {
    const int64_t g = g0[i];
    if (is_match(g, m)) {
      s0 += hinge(pos_arg(a.dpos[ro + i], a.dn0[ro + i], mu));
      s1 += hinge(pos_arg(a.dpos[ro + i], a.dn1[co + g], mu));
      cm += 1.f;
      if (a.want_grad) { atomicAdd(a.cnt + co + g, 1); atomicMin(a.first + co + g, i); }     // integer: order-free
    } else if (g == -1) {
      su0 += hinge(neg_arg(a.du0[ro + i], mu));
      cu0 += 1.f;
    }
  }
  for (int j = threadIdx.x; j < m; j += METRIC_THREADS)
    if (g1[j] == -1) { su1 += hinge(neg_arg(a.du1[co + j], mu)); cu1 += 1.f; }
  const float t0 = cta_sum<METRIC_THREADS>(s0, red), t1 = cta_sum<METRIC_THREADS>(s1, red);
  const float tu0 = cta_sum<METRIC_THREADS>(su0, red), tu1 = cta_sum<METRIC_THREADS>(su1, red);
  const float nm = cta_sum<METRIC_THREADS>(cm, red), nu0 = cta_sum<METRIC_THREADS>(cu0, red), nu1 = cta_sum<METRIC_THREADS>(cu1, red);
  if (threadIdx.x == 0) {
    float l = 0.f;
    if (nm > 0.f) l += (t0 + t1) / nm;
    if (nu0 > 0.f) l += tu0 / nu0;
    if (nu1 > 0.f) l += tu1 / nu1;
    a.per_pair[b] = l;
    const float gB = a.grad_scale / (float)a.B;
    s_w[0] = nm > 0.f ? gB / nm : 0.f;
    s_w[1] = nu0 > 0.f ? gB / nu0 : 0.f;
    s_w[2] = nu1 > 0.f ? gB / nu1 : 0.f;
    last = last_cta_arrive(a.counter);
  }
  __syncthreads();
  if (a.want_grad) {
    const float wm = s_w[0], w0 = s_w[1], w1 = s_w[2];
    for (int i = threadIdx.x; i < n; i += METRIC_THREADS) {
      const int64_t g = g0[i];
      float pc = 0.f, c0 = 0.f, cu = 0.f, c1 = 0.f;
      if (is_match(g, m)) {
        const float h0 = hinge_grad(pos_arg(a.dpos[ro + i], a.dn0[ro + i], mu));
        const float h1 = hinge_grad(pos_arg(a.dpos[ro + i], a.dn1[co + g], mu));
        pc = wm * (h0 + h1); c0 = -wm * h0; c1 = -wm * h1;
      } else if (g == -1) {
        cu = -w0 * hinge_grad(neg_arg(a.du0[ro + i], mu));
      }
      a.posc[ro + i] = pc; a.n0c[ro + i] = c0; a.u0c[ro + i] = cu; a.a1c[ro + i] = c1;
    }
    __syncthreads();                                        // a1c, cnt, first of this pair are visible to the whole CTA
    for (int j = threadIdx.x; j < m; j += METRIC_THREADS) {
      const int c = a.cnt[co + j];
      float s = 0.f;
      if (c == 1) s = a.a1c[ro + a.first[co + j]];
      else if (c > 1)                                       // several anchors name this column: their sum in row order
        for (int i = a.first[co + j]; i < n; ++i) if (g0[i] == j) s += a.a1c[ro + i];
      a.n1c[co + j] = s;
      a.u1c[co + j] = g1[j] == -1 ? -w1 * hinge_grad(neg_arg(a.du1[co + j], mu)) : 0.f;
    }
  }
  if (last && threadIdx.x == 0) a.loss[0] = last_cta_sum(a.per_pair, a.B) / (float)a.B;     // pair order: deterministic
}

// D = d loss / d dist (TRANS = 0: [B, n, ldo] rows i) or D^T (TRANS = 1: [B, m, ldo] rows j), one warp per output row, pad
// columns written as 0; half the row sum goes to rsum.  Every element adds its terms in the same order in both forms.
template <int TRANS>
__global__ void __launch_bounds__(256) metric_dgrad_kernel(MetricArgs a, float* __restrict__ out, int ldo, float* __restrict__ rsum) {
  const int R = TRANS ? a.m : a.n, C = TRANS ? a.n : a.m;
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= (int64_t)a.B * R) return;
  const int b = (int)(row / R), r = (int)(row % R);
  const int64_t ro = (int64_t)b * a.n, co = (int64_t)b * a.m;
  float* o = out + row * ldo;
  float s = 0.f;
  for (int c = lane; c < ldo; c += 32) {
    float v = 0.f;
    if (c < C) {
      const int i = TRANS ? c : r, j = TRANS ? r : c;
      if (a.gt0[ro + i] == j) v += a.posc[ro + i];
      if (a.n0[ro + i] == j) v += a.n0c[ro + i];
      if (a.u0[ro + i] == j) v += a.u0c[ro + i];
      if (a.n1[co + j] == i) v += a.n1c[co + j];
      if (a.u1[co + j] == i) v += a.u1c[co + j];
    }
    o[c] = v;
    s += v;
  }
  s = warp_sum(s);
  if (lane == 0) rsum[row] = 0.5f * s;
}

// normalisation backward for both sides: one thread per (side, b, k) with k the keypoint, so every access to the [B, d, N]
// tensors is coalesced.  g = P + rs x_hat (P = -0.5 (D Y)^T, rs = 0.5 rowsum D), then F.normalize's backward:
// |x| >= eps: (g - (g . x_hat) x_hat) / |x|;   else g / eps.
__global__ void __launch_bounds__(256) metric_norm_bwd_kernel(const float* __restrict__ c0, const float* __restrict__ c1,
                                                              const float* __restrict__ P0, int ldp0, const float* __restrict__ P1, int ldp1,
                                                              const float* __restrict__ rs0, const float* __restrict__ rs1,
                                                              float* __restrict__ dc0, float* __restrict__ dc1, int B, int d, int n, int m) {
  const float eps = 1e-12f;
  int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
  const float *c, *P, *rs; float* dc; int N, ldp;
  if (t < (int64_t)B * n) { c = c0; P = P0; rs = rs0; dc = dc0; N = n; ldp = ldp0; }
  else { t -= (int64_t)B * n; if (t >= (int64_t)B * m) return; c = c1; P = P1; rs = rs1; dc = dc1; N = m; ldp = ldp1; }
  const int b = (int)(t / N), k = (int)(t % N);
  const float* x = c + (int64_t)b * d * N + k;
  const float* p = P + (int64_t)b * d * ldp + k;
  float* o = dc + (int64_t)b * d * N + k;
  float s = 0.f;
  for (int q = 0; q < d; ++q) { const float v = x[(int64_t)q * N]; s = fmaf(v, v, s); }
  const float nrm = sqrtf(s), den = fmaxf(nrm, eps), r = rs[t];
  float dot = 0.f;
  for (int q = 0; q < d; ++q) {
    const float xh = x[(int64_t)q * N] / den;
    dot = fmaf(fmaf(r, xh, p[(int64_t)q * ldp]), xh, dot);
  }
  for (int q = 0; q < d; ++q) {
    const float xh = x[(int64_t)q * N] / den;
    const float g = fmaf(r, xh, p[(int64_t)q * ldp]);
    o[(int64_t)q * N] = nrm >= eps ? (g - dot * xh) / nrm : g / eps;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// workspace: every region 256-byte aligned; the gradient regions and the operand-split scratch only when asked for
struct MetricLayout {
  int64_t counter, per_pair, X, sq, G, rsel, csel, part, coef, icol, Dt, XT, YT, P0, P1, rs, split, total;
  int ldn, ldm, chunks, rows_per_chunk;
};

inline MetricLayout metric_layout(int B, int n, int m, int d, bool grad, bool split) {
  MetricLayout L;
  L.ldn = (int)align_up(n, 4); L.ldm = (int)align_up(m, 4);
  L.rows_per_chunk = std::max(64, cdiv(n, 32));
  L.chunks = cdiv(n, L.rows_per_chunk);
  const int64_t Bn = (int64_t)B * n, Bm = (int64_t)B * m;
  int64_t o = 0;
  auto take = [&](int64_t bytes) { const int64_t at = o; o += align_up(std::max<int64_t>(bytes, 4), 256); return at; };
  L.counter = take(4);
  L.per_pair = take(4 * (int64_t)B);
  L.X = take(4 * (Bn + Bm) * d);                     // X [B n, d] then Y [B m, d]: one normalisation launch for both
  L.sq = take(4 * (Bn + Bm));
  L.G = take(4 * Bn * L.ldm);                        // Gram, then D
  L.rsel = take(4 * 3 * Bn);                         // dn0, du0, dpos
  L.csel = take(4 * 2 * Bm);                         // dn1, du1
  L.part = take(4 * 4 * (int64_t)B * L.chunks * m);
  L.coef = take(4 * (4 * Bn + 2 * Bm));              // posc, n0c, u0c, a1c | n1c, u1c
  L.icol = take(4 * 2 * Bm);                         // cnt, first
  L.Dt = L.XT = L.YT = L.P0 = L.P1 = L.rs = L.split = -1;
  if (grad) {
    L.Dt = take(4 * Bm * L.ldn);
    L.XT = take(4 * (int64_t)B * d * L.ldn);
    L.YT = take(4 * (int64_t)B * d * L.ldm);
    L.P0 = take(4 * (int64_t)B * d * L.ldn);
    L.P1 = take(4 * (int64_t)B * d * L.ldm);
    L.rs = take(4 * (Bn + Bm));
  }
  if (split)                                         // og_linear_auto_fwd's split W: the largest W operand is d x max(ld) per pair
    L.split = take(4 * 2 * (align_up((int64_t)B * d * std::max(L.ldn, L.ldm), 64) + 64));
  L.total = o;
  return L;
}

inline int64_t metric_workspace_bytes(int B, int n, int m, int d, int want_grad, int precision) {
  return metric_layout(B, n, m, d, want_grad != 0, precision == OG_PREC_TF32X3).total;
}

// one batched GEMM of the schedule: Y (or Yt) = alpha A W^T, all operands [B][rows, ld] with K contiguous
inline int metric_gemm(const float* A, int64_t lda, const float* W, int64_t ldw, int K, int rows, int nout, int B, float alpha,
                       float* Y, int64_t ldy, float* Yt, int64_t ldyt, int precision, float* split, cudaStream_t st) {
  og_linear_args g = {};
  g.A = A; g.lda = lda; g.strideA = (int64_t)rows * lda;
  g.k1 = K; g.k2 = 0;
  g.W = W; g.ldw = ldw; g.strideW = (int64_t)nout * ldw;
  g.rows = rows; g.nout = nout; g.batch = B; g.alpha = alpha;
  g.Y = Y; g.ldy = ldy; g.strideY = (int64_t)rows * ldy;
  g.Yt = Yt; g.ldyt = ldyt; g.strideYt = (int64_t)nout * ldyt;
  return og_linear_auto_fwd(&g, precision, split, st);
}

inline int metric_loss_launch(const float* c0, const float* c1, const int64_t* gt0, const int64_t* gt1, int B, int d, int n, int m,
                              float margin, int precision, float* loss, int64_t* n0, int64_t* u0, int64_t* n1, int64_t* u1,
                              float* dc0, float* dc1, float grad_scale, void* ws, int64_t ws_bytes, cudaStream_t st) {
  const bool grad = dc0 != nullptr;
  const MetricLayout L = metric_layout(B, n, m, d, grad, precision == OG_PREC_TF32X3);
  if (ws_bytes < L.total) return fail(OG_EWORKSPACE, "metric_loss: workspace too small (%lld < %lld bytes)", (long long)ws_bytes,
                                      (long long)L.total);
  char* base = static_cast<char*>(ws);
  auto F = [&](int64_t off) { return off < 0 ? nullptr : reinterpret_cast<float*>(base + off); };
  const int64_t Bn = (int64_t)B * n, Bm = (int64_t)B * m;
  float* X = F(L.X);
  float* Y = X + Bn * d;
  float* split = F(L.split);
  int rc;
  // 1. normalised operands and their squared norms
  if ((rc = transpose_launch(c0, n, (int64_t)d * n, X, d, (int64_t)n * d, B, d, n, 1, st))) return rc;
  if ((rc = transpose_launch(c1, m, (int64_t)d * m, Y, d, (int64_t)m * d, B, d, m, 1, st))) return rc;
  if ((rc = og_row_normalize(X, Bn + Bm, d, 1, 1e-12f, st))) return rc;
  if ((rc = OG_LAUNCH(metric_sqnorm_kernel, (unsigned)((Bn + Bm + 7) / 8), 256, 0, st, X, Bn + Bm, d, F(L.sq)))) return rc;
  // 2. Gram
  if ((rc = metric_gemm(X, d, Y, d, d, n, m, B, 1.f, F(L.G), L.ldm, nullptr, 0, precision, split, st))) return rc;
  // 3. selections
  MetricArgs a = {};
  a.gt0 = gt0; a.gt1 = gt1; a.B = B; a.n = n; a.m = m; a.ldg = L.ldm; a.margin = margin;
  a.G = F(L.G); a.sqx = F(L.sq); a.sqy = F(L.sq) + Bn;
  a.n0 = n0; a.u0 = u0; a.n1 = n1; a.u1 = u1;
  a.dn0 = F(L.rsel); a.du0 = a.dn0 + Bn; a.dpos = a.du0 + Bn;
  a.dn1 = F(L.csel); a.du1 = a.dn1 + Bm;
  a.part = F(L.part); a.chunks = L.chunks; a.rows_per_chunk = L.rows_per_chunk;
  a.counter = reinterpret_cast<unsigned int*>(base + L.counter); a.per_pair = F(L.per_pair); a.loss = loss;
  a.grad_scale = grad_scale; a.want_grad = grad ? 1 : 0;
  a.posc = F(L.coef); a.n0c = a.posc + Bn; a.u0c = a.n0c + Bn; a.a1c = a.u0c + Bn; a.n1c = a.a1c + Bn; a.u1c = a.n1c + Bm;
  a.cnt = reinterpret_cast<int*>(base + L.icol); a.first = a.cnt + Bm;
  if ((rc = OG_LAUNCH(metric_rows_kernel, (unsigned)((Bn + 7) / 8), 256, 0, st, a))) return rc;
  if ((rc = OG_LAUNCH(metric_cols_kernel, dim3(cdiv(m, METRIC_COLS), L.chunks, B), METRIC_COLS, 0, st, a))) return rc;
  if ((rc = OG_LAUNCH(metric_cols_merge_kernel, (unsigned)((Bm + 255) / 256), 256, 0, st, a))) return rc;
  // 4. loss (+ gradient coefficients)
  OG_CUDA(cudaMemsetAsync(a.counter, 0, 4, st));
  if ((rc = OG_LAUNCH(metric_loss_kernel, B, METRIC_THREADS, 0, st, a))) return rc;
  if (!grad) return OG_OK;
  // 5. gradient: D (over the Gram, which is no longer read) and D^T, then the two GEMMs and the normalisation backward
  float* D = F(L.G);
  float* Dt = F(L.Dt);
  float* rs = F(L.rs);
  if ((rc = OG_LAUNCH(metric_dgrad_kernel<0>, (unsigned)((Bn + 7) / 8), 256, 0, st, a, D, L.ldm, rs))) return rc;
  if ((rc = OG_LAUNCH(metric_dgrad_kernel<1>, (unsigned)((Bm + 7) / 8), 256, 0, st, a, Dt, L.ldn, rs + Bn))) return rc;
  float* XT = F(L.XT);
  float* YT = F(L.YT);
  OG_CUDA(cudaMemsetAsync(XT, 0, 4 * (size_t)B * d * L.ldn, st));       // zero K padding of the GEMM operands
  OG_CUDA(cudaMemsetAsync(YT, 0, 4 * (size_t)B * d * L.ldm, st));
  if ((rc = transpose_launch(X, d, (int64_t)n * d, XT, L.ldn, (int64_t)d * L.ldn, B, n, d, 1, st))) return rc;
  if ((rc = transpose_launch(Y, d, (int64_t)m * d, YT, L.ldm, (int64_t)d * L.ldm, B, m, d, 1, st))) return rc;
  if ((rc = metric_gemm(D, L.ldm, YT, L.ldm, L.ldm, n, d, B, -0.5f, nullptr, 0, F(L.P0), L.ldn, precision, split, st))) return rc;
  if ((rc = metric_gemm(Dt, L.ldn, XT, L.ldn, L.ldn, m, d, B, -0.5f, nullptr, 0, F(L.P1), L.ldm, precision, split, st))) return rc;
  return OG_LAUNCH(metric_norm_bwd_kernel, (unsigned)((Bn + Bm + 255) / 256), 256, 0, st, c0, c1, F(L.P0), L.ldn, F(L.P1), L.ldm,
                   rs, rs + Bn, dc0, dc1, B, d, n, m);
}

}  // namespace og
