// Kernels that only the TRAINING step needs (SURVEY.md section 8, row f1): what torch autograd and nn.BatchNorm1d do for the
// reference in MatchingTrainingModule.training_step (models/matching_module.py:71-105) around the contractions - batch-norm
// with batch statistics (models/utils.py:48-58: Conv1d -> ReLU -> BatchNorm1d) and its backward, the column reductions behind
// bias / affine gradients, the row softmax of the materialised attention matrix and its backward (models/superglue/
// attention.py:8-19), transposes for the "dW = dY^T X" contractions, and the residual mix (superglue.py:59-62).
// All activations are row-major [rows, channels] (rows = batch x keypoints), the layout of the inference path.
// Every reduction runs in a fixed order (no atomics): the training step is bit-reproducible.
#pragma once
#include "common.cuh"
#include <math_constants.h>
#include <algorithm>

namespace og {

// ---------------------------------------------------------------------------------------------------------------------
// batched transpose / pitch-changing copy
//   transpose: out[b][c * ld_out + r] = in[b][r * ld_in + c];   copy: out[b][r * ld_out + c] = in[b][r * ld_in + c]
__global__ void __launch_bounds__(256) transpose_kernel(const float* __restrict__ in, int64_t ld_in, int64_t stride_in,
                                                        float* __restrict__ out, int64_t ld_out, int64_t stride_out, int rows, int cols) {
  __shared__ float tile[32][33];
  const float* ib = in + (int64_t)blockIdx.z * stride_in;
  float* ob = out + (int64_t)blockIdx.z * stride_out;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int r = r0 + ty + 8 * j, c = c0 + tx;
    if (r < rows && c < cols) tile[ty + 8 * j][tx] = ib[(int64_t)r * ld_in + c];
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int c = c0 + ty + 8 * j, r = r0 + tx;
    if (r < rows && c < cols) ob[(int64_t)c * ld_out + r] = tile[tx][ty + 8 * j];
  }
}
__global__ void __launch_bounds__(256) copy2d_kernel(const float* __restrict__ in, int64_t ld_in, int64_t stride_in,
                                                     float* __restrict__ out, int64_t ld_out, int64_t stride_out, int rows, int cols) {
  const float* ib = in + (int64_t)blockIdx.z * stride_in;
  float* ob = out + (int64_t)blockIdx.z * stride_out;
  for (int r = blockIdx.y; r < rows; r += gridDim.y)
    for (int c = blockIdx.x * 256 + threadIdx.x; c < cols; c += gridDim.x * 256) ob[(int64_t)r * ld_out + c] = ib[(int64_t)r * ld_in + c];
}

inline int transpose_launch(const float* in, int64_t ld_in, int64_t stride_in, float* out, int64_t ld_out, int64_t stride_out,
                            int batch, int rows, int cols, int transpose, cudaStream_t st) {
  if (batch <= 0 || rows <= 0 || cols <= 0) return OG_OK;
  if (transpose) {
    dim3 grid(cdiv(cols, 32), cdiv(rows, 32), batch);
    if (grid.y > 65535 || grid.z > 65535) return fail(OG_EUNSUPPORTED, "transpose: %d rows x %d batches exceed the grid limits", rows, batch);
    return OG_LAUNCH(transpose_kernel, grid, 256, 0, st, in, ld_in, stride_in, out, ld_out, stride_out, rows, cols);
  }
  dim3 grid(std::min(cdiv(cols, 256), 64), std::min(rows, 4096), batch);
  if (grid.z > 65535) return fail(OG_EUNSUPPORTED, "copy2d: %d batches exceed the grid limits", batch);
  return OG_LAUNCH(copy2d_kernel, grid, 256, 0, st, in, ld_in, stride_in, out, ld_out, stride_out, rows, cols);
}

// ---------------------------------------------------------------------------------------------------------------------
// column reductions over the rows of a [rows, cols] matrix, up to two results per column.  Stage 1: block (64 columns, 4
// row lanes) x row chunk -> partial[chunk][2][cols]; stage 2: fixed-order sum over the chunks + a per-mode finish.
//   MODE 0  sum      o0 = sum x (y - z)            (y, z optional: 1 and 0)           db, d mix
//   MODE 1  mean     o0 = mean relu?(x)                                                 BN statistics, pass 1
//   MODE 2  var      o0 = mean (relu?(x) - mu[c])^2                                     BN statistics, pass 2
//   MODE 3  bn-bwd   o0 = sum dy,  o1 = sum dy xhat,  xhat = (relu?(a) - mu) invstd     d beta, d gamma
// A padded batch (len set) reduces over the real rows only: row r is slot r % cap of pair r / cap, real below len[r / cap], and the
// means divide by their count, sum_b len[b].
struct ColReduceArgs {
  const float* x; int64_t ldx;         // MODE 3: dy
  const float* y; int64_t ldy;         // MODE 0: optional factor; MODE 3: a (pre-activation)
  const float* z; int64_t ldz;         // MODE 0: optional subtrahend
  const float* mu; const float* invstd;
  int rows, cols, relu;
  float* partial;                      // [chunks][2][cols]
  float* out0; float* out1;
  int chunks, rows_per_chunk;
  const int* len; int cap;             // padded batch (null otherwise): per-pair lengths [rows / cap], clamped into [1, cap]
};
constexpr int COLRED_MAX_CHUNKS = 256;

// rows a padded reduction counts: sum_b len[b] (rows when len is null)
__device__ __forceinline__ int padded_count(const int* len, int rows, int cap) {
  if (!len) return rows;
  int t = 0;
  for (int b = 0; b < rows / cap; ++b) t += padded_length(len, b, cap);
  return t;
}
__device__ __forceinline__ bool padded_real(const int* len, int r, int cap) {
  return !len || r % cap < padded_length(len, r / cap, cap);
}

template <int MODE>
__global__ void __launch_bounds__(256) colreduce_stage1(ColReduceArgs a) {
  __shared__ float s0[4][64], s1[4][64];
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  const int c = blockIdx.x * 64 + tx;
  const int rb = blockIdx.y * a.rows_per_chunk, re = min(rb + a.rows_per_chunk, a.rows);
  float acc0 = 0.f, acc1 = 0.f;
  if (c < a.cols) {
    float mu = 0.f, is = 0.f;
    if (MODE == 2 || MODE == 3) mu = __ldg(a.mu + c);
    if (MODE == 3) is = __ldg(a.invstd + c);
    for (int r = rb + ty; r < re; r += 4) {
      if (a.len && !padded_real(a.len, r, a.cap)) continue;
      float v = a.x[(int64_t)r * a.ldx + c];
      if (MODE == 0) {
        if (a.y) { float f = a.y[(int64_t)r * a.ldy + c]; if (a.z) f -= a.z[(int64_t)r * a.ldz + c]; v *= f; }
        acc0 += v;
      } else if (MODE == 1) {
        if (a.relu) v = fmaxf(v, 0.f);
        acc0 += v;
      } else if (MODE == 2) {
        if (a.relu) v = fmaxf(v, 0.f);
        const float d = v - mu;
        acc0 = fmaf(d, d, acc0);
      } else {
        float act = a.y[(int64_t)r * a.ldy + c];
        if (a.relu) act = fmaxf(act, 0.f);
        acc0 += v;
        acc1 = fmaf(v, (act - mu) * is, acc1);
      }
    }
  }
  s0[ty][tx] = acc0; s1[ty][tx] = acc1;
  __syncthreads();
  if (ty == 0 && c < a.cols) {
    float* p = a.partial + (int64_t)blockIdx.y * 2 * a.cols;
    p[c] = (s0[0][tx] + s0[1][tx]) + (s0[2][tx] + s0[3][tx]);
    if (MODE == 3) p[a.cols + c] = (s1[0][tx] + s1[1][tx]) + (s1[2][tx] + s1[3][tx]);
  }
}
template <int MODE>
__global__ void __launch_bounds__(256) colreduce_stage2(ColReduceArgs a) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= a.cols) return;
  float t0 = 0.f, t1 = 0.f;
  for (int k = 0; k < a.chunks; ++k) {
    t0 += a.partial[(int64_t)k * 2 * a.cols + c];
    if (MODE == 3) t1 += a.partial[(int64_t)k * 2 * a.cols + a.cols + c];
  }
  if (MODE == 1 || MODE == 2) t0 = __fdiv_rn(t0, (float)padded_count(a.len, a.rows, a.cap));
  a.out0[c] = t0;
  if (MODE == 3) a.out1[c] = t1;
}
inline int64_t colreduce_workspace_floats(int cols) { return (int64_t)COLRED_MAX_CHUNKS * 2 * cols; }

template <int MODE>
inline int colreduce_launch(ColReduceArgs a, cudaStream_t st) {
  if (a.cols <= 0) return OG_OK;
  a.chunks = std::max(1, std::min(COLRED_MAX_CHUNKS, cdiv(a.rows, 64)));
  a.rows_per_chunk = cdiv(std::max(a.rows, 1), a.chunks);
  a.chunks = std::max(1, cdiv(a.rows, a.rows_per_chunk));
  if (const int rc = OG_LAUNCH(colreduce_stage1<MODE>, dim3(cdiv(a.cols, 64), a.chunks), 256, 0, st, a)) return rc;
  return OG_LAUNCH(colreduce_stage2<MODE>, cdiv(a.cols, 256), 256, 0, st, a);
}

// ---------------------------------------------------------------------------------------------------------------------
// BatchNorm1d with batch statistics (torch.nn.functional.batch_norm, training=True): y = gamma (r - mu) / sqrt(var + eps) + beta,
// r = relu(a) when the ReLU in front of the norm is fused in; var is the biased variance; the running statistics move by
// `momentum` towards (mu, unbiased var).  A padded batch (len set) counts its real rows, sum_b len[b] (ColReduceArgs).
// Guarded form (og_bn_train_fwd_guarded): a nullable device flag `skip` leaves the running statistics untouched when it reads
// non-zero, and a nullable `num_batches_tracked` is incremented by 1 - *skip (by 1 without a flag) - BatchNorm1d's counter kept
// on the device.  Null pointers give the unguarded arithmetic.
__global__ void __launch_bounds__(256) bn_finish_stats_kernel(const float* __restrict__ mean, const float* __restrict__ var, int cols, int rows_all,
                                                              const int* __restrict__ len, int cap, float eps, float momentum,
                                                              float* __restrict__ invstd, float* __restrict__ running_mean,
                                                              float* __restrict__ running_var, const int* __restrict__ skip,
                                                              long long* __restrict__ num_batches_tracked) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= cols) return;
  const bool skipped = skip && *skip;
  if (num_batches_tracked && c == 0 && !skipped) *num_batches_tracked += 1;
  const int rows = padded_count(len, rows_all, cap);
  const float v = var[c];
  invstd[c] = __fdiv_rn(1.f, __fsqrt_rn(v + eps));
  if (skipped) return;
  if (running_mean) running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean[c];
  if (running_var) {
    const float unbiased = rows > 1 ? v * __fdiv_rn((float)rows, (float)(rows - 1)) : v;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
  }
}
__global__ void __launch_bounds__(256) bn_apply_kernel(const float* __restrict__ a, int64_t lda, int rows, int cols, int relu,
                                                       const float* __restrict__ mean, const float* __restrict__ invstd,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                                       float* __restrict__ y, int64_t ldy) {
  const int64_t n = (int64_t)rows * cols;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
    const int r = (int)(i / cols), c = (int)(i % cols);
    float v = a[(int64_t)r * lda + c];
    if (relu) v = fmaxf(v, 0.f);
    y[(int64_t)r * ldy + c] = fmaf((v - mean[c]) * invstd[c], gamma[c], beta[c]);
  }
}
// da = [a > 0] gamma invstd (dy - dbeta / n - xhat dgamma / n);  a padded batch (len set): n = sum_b len[b], da = 0 on its padding rows
__global__ void __launch_bounds__(256) bn_bwd_apply_kernel(const float* __restrict__ dy, int64_t lddy, const float* __restrict__ a, int64_t lda,
                                                           int rows, int cols, int relu, const float* __restrict__ mean,
                                                           const float* __restrict__ invstd, const float* __restrict__ gamma,
                                                           const float* __restrict__ dgamma, const float* __restrict__ dbeta,
                                                           float* __restrict__ da, int64_t ldda, const int* __restrict__ len, int cap) {
  const int64_t n = (int64_t)rows * cols;
  const float inv_n = __fdiv_rn(1.f, (float)padded_count(len, rows, cap));
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
    const int r = (int)(i / cols), c = (int)(i % cols);
    if (len && !padded_real(len, r, cap)) { da[(int64_t)r * ldda + c] = 0.f; continue; }
    const float pre = a[(int64_t)r * lda + c];
    const float act = relu ? fmaxf(pre, 0.f) : pre;
    const float xhat = (act - mean[c]) * invstd[c];
    float g = gamma[c] * invstd[c] * (dy[(int64_t)r * lddy + c] - dbeta[c] * inv_n - xhat * dgamma[c] * inv_n);
    if (relu && !(pre > 0.f)) g = 0.f;
    da[(int64_t)r * ldda + c] = g;
  }
}
inline unsigned eltwise_grid(int64_t n) { return (unsigned)std::min<int64_t>((n + 255) / 256, 132 * 16); }

// ---------------------------------------------------------------------------------------------------------------------
// row softmax of a materialised [rows, cols] matrix (in place) and its backward  dS = scale P (dP - sum_j P dP)  (in place of dP).
// One warp per row.  Padded keys (len set): row r belongs to sequence r / seq_rows, whose first len[r / seq_rows] columns are its
// keys; P = 0 and dS = 0 over the other columns of the capacity `cols`.
__device__ __forceinline__ int softmax_row_cols(const int* len, int64_t row, int64_t seq_rows, int cols) {
  return len ? padded_length(len, (int)(row / seq_rows), cols) : cols;
}
__global__ void __launch_bounds__(256) softmax_rows_kernel(float* __restrict__ S, int64_t ld, int64_t rows, int cols_all,
                                                           const int* __restrict__ len, int64_t seq_rows) {
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float* s = S + row * ld;
  const int cols = softmax_row_cols(len, row, seq_rows, cols_all);
  for (int j = cols + lane; j < cols_all; j += 32) s[j] = 0.f;
  float mx = -CUDART_INF_F;
  for (int j = lane; j < cols; j += 32) mx = fmaxf(mx, s[j]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int j = lane; j < cols; j += 32) { const float e = expf(s[j] - mx); s[j] = e; sum += e; }
  sum = warp_sum(sum);
  const float inv = __fdiv_rn(1.f, sum);
  for (int j = lane; j < cols; j += 32) s[j] *= inv;
}
__global__ void __launch_bounds__(256) softmax_bwd_rows_kernel(const float* __restrict__ P, float* __restrict__ dP, int64_t ld, int64_t rows,
                                                               int cols_all, float scale, const int* __restrict__ len, int64_t seq_rows) {
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* p = P + row * ld;
  float* g = dP + row * ld;
  const int cols = softmax_row_cols(len, row, seq_rows, cols_all);
  for (int j = cols + lane; j < cols_all; j += 32) g[j] = 0.f;
  float dot = 0.f;
  for (int j = lane; j < cols; j += 32) dot = fmaf(p[j], g[j], dot);
  dot = warp_sum(dot);
  for (int j = lane; j < cols; j += 32) g[j] = scale * p[j] * (g[j] - dot);
}

// out[r * ld + c] (+)= sum_s part[s][r * cols + c], s ascending: the reduction behind the split-K weight gradients
// (dW = sum over row chunks of dY_s^T X_s: one batched GEMM fills the GPU where a single [nout, K] output would occupy four CTAs)
__global__ void __launch_bounds__(256) sum_batches_kernel(const float* __restrict__ part, int S, int rows, int cols, float* __restrict__ out,
                                                          int64_t ld, int accumulate) {
  const int64_t n = (int64_t)rows * cols;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
    float t = 0.f;
    for (int k = 0; k < S; ++k) t += part[(int64_t)k * n + i];
    float* o = out + (i / cols) * ld + (i % cols);
    *o = accumulate ? *o + t : t;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// element-wise
__global__ void __launch_bounds__(256) axpby_kernel(const float* __restrict__ x, const float* __restrict__ y, float a, float b,
                                                    float* __restrict__ out, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256)
    out[i] = y ? fmaf(a, x[i], b * y[i]) : a * x[i];
}
// residual mix (superglue.py:59-62): alpha = sigmoid(mix[c]);  fwd: out = alpha g + (1 - alpha) l;
// bwd: dg = alpha dm, dl = (1 - alpha) dm (either may be NULL)
__global__ void __launch_bounds__(256) mix_fwd_kernel(const float* __restrict__ g, const float* __restrict__ l, const float* __restrict__ mix,
                                                      float* __restrict__ out, int64_t rows, int d) {
  const int64_t n = rows * d;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
    const float al = __fdiv_rn(1.f, 1.f + expf(-mix[i % d]));
    out[i] = al * g[i] + (1.f - al) * l[i];
  }
}
__global__ void __launch_bounds__(256) mix_bwd_kernel(const float* __restrict__ dm, const float* __restrict__ mix, float* __restrict__ dg,
                                                      float* __restrict__ dl, int64_t rows, int d) {
  const int64_t n = rows * d;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
    const float al = __fdiv_rn(1.f, 1.f + expf(-mix[i % d]));
    if (dg) dg[i] = al * dm[i];
    if (dl) dl[i] = (1.f - al) * dm[i];
  }
}
// d mix[c] = colsum[c] alpha (1 - alpha),  colsum[c] = sum_r dm (g - l)
__global__ void __launch_bounds__(256) mix_param_grad_kernel(const float* __restrict__ colsum, const float* __restrict__ mix, float* __restrict__ dmix, int d) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= d) return;
  const float al = __fdiv_rn(1.f, 1.f + expf(-mix[c]));
  dmix[c] = colsum[c] * al * (1.f - al);
}

// ---------------------------------------------------------------------------------------------------------------------
// the skip of the reference's training_step (models/matching_module.py:96-97), decided on the device.  lengths [2B]: n_0 .. n_{B-1},
// m_0 .. m_{B-1} as the front-ends wrote them.  skip = 1 when an image has no keypoint (the reference's `data is None`) or when one
// side's real rows total fewer than 2 (what BatchNorm1d raises on: one value per channel), else 0.  One warp.
__global__ void __launch_bounds__(32) train_guard_kernel(const int* __restrict__ lengths, int B, int* __restrict__ skip) {
  const int lane = threadIdx.x;
  bool empty = false;
  unsigned tot[2] = {0u, 0u};                                 // saturated at 2: only "fewer than 2" matters
  for (int i = lane; i < 2 * B; i += 32) {
    const int l = lengths[i];
    empty |= l <= 0;
    unsigned& t = tot[i >= B];
    t = min(t + (unsigned)max(l, 0), 2u);
  }
  empty = __any_sync(0xffffffffu, empty);
  const unsigned s0 = __reduce_add_sync(0xffffffffu, tot[0]), s1 = __reduce_add_sync(0xffffffffu, tot[1]);
  if (lane == 0) *skip = (empty || s0 < 2u || s1 < 2u) ? 1 : 0;
}
// a skipped step's outputs: loss[0 .. nloss) = NaN and x[0 .. n) = 0 when *skip != 0; nothing is written otherwise
__global__ void __launch_bounds__(256) train_skip_outputs_kernel(const int* __restrict__ skip, float* __restrict__ loss, int nloss,
                                                                 float* __restrict__ x, int64_t n) {
  if (!*skip) return;
  const int64_t i0 = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (i0 < nloss) loss[i0] = CUDART_NAN_F;
  for (int64_t i = i0; i < n; i += (int64_t)gridDim.x * 256) x[i] = 0.f;
}

}  // namespace og
