// Mutual-argmax match extraction on the inner n x m block of the log-assignment.
// Replaces models/matching_module.py:174-187 and the reverse direction of inference.py:176-190.
// torch.max(dim) semantics: on ties the LOWEST index wins.
#pragma once
#include "common.cuh"
#include <math_constants.h>

namespace og {

constexpr int MATCH_ROW_CHUNK = 64;     // rows per column-pass chunk

// Pair b's rows and columns: n, m, or in a padded batch of B pairs (lens non-null) lens[b] and lens[B + b] clamped into [1, n] / [1, m]
__device__ __forceinline__ int2 match_lengths(const int* lens, int b, int B, int n, int m) {
  if (!lens) return make_int2(n, m);
  return make_int2(padded_length(lens, b, n), padded_length(lens + B, b, m));
}

// one warp per row: (max, first argmax) over columns 0..m-1 (the pair's; a padded batch's rows past its length are skipped)
__global__ void __launch_bounds__(256) match_rowmax_kernel(const float* __restrict__ scores, int n, int m, const int* lens,
                                                            float* __restrict__ rowval, int* __restrict__ rowidx) {
  const int b = blockIdx.y;
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int2 len = match_lengths(lens, b, gridDim.y, n, m);
  if (row >= len.x) return;
  const float* src = scores + ((int64_t)b * (n + 1) + row) * (m + 1);
  float best = -CUDART_INF_F; int bi = 0x7fffffff;
  for (int c = lane; c < len.y; c += 32) {
    const float x = __ldg(src + c);
    if (x > best || bi == 0x7fffffff) { best = x; bi = c; }      // strict > keeps the first index
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, off);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  if (lane == 0) { rowval[(int64_t)b * n + row] = best; rowidx[(int64_t)b * n + row] = bi; }
}

// one thread per column per row-chunk: partial (max, first argmax) over the chunk's rows (a chunk past a padded pair's rows: -inf,
// which never wins the strict comparison of match_colreduce_kernel)
__global__ void __launch_bounds__(256) match_colmax_kernel(const float* __restrict__ scores, int n, int m, const int* lens, int chunks,
                                                            float* __restrict__ pval, int* __restrict__ pidx) {
  const int b = blockIdx.z, chunk = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int2 len = match_lengths(lens, b, gridDim.z, n, m);
  if (c >= len.y) return;
  const int r0 = chunk * MATCH_ROW_CHUNK, r1 = min(r0 + MATCH_ROW_CHUNK, len.x);
  if (r0 >= r1) {
    pval[((int64_t)b * chunks + chunk) * m + c] = -CUDART_INF_F;
    pidx[((int64_t)b * chunks + chunk) * m + c] = r0;
    return;
  }
  const float* src = scores + (int64_t)b * (n + 1) * (m + 1) + c;
  float best = __ldg(src + (int64_t)r0 * (m + 1)); int bi = r0;
  for (int r = r0 + 1; r < r1; ++r) {
    const float x = __ldg(src + (int64_t)r * (m + 1));
    if (x > best) { best = x; bi = r; }
  }
  pval[((int64_t)b * chunks + chunk) * m + c] = best;
  pidx[((int64_t)b * chunks + chunk) * m + c] = bi;
}

__global__ void __launch_bounds__(256) match_colreduce_kernel(int n, int m, int chunks, const float* __restrict__ pval,
                                                               const int* __restrict__ pidx, int* __restrict__ colidx) {
  const int b = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= m) return;
  float best = pval[((int64_t)b * chunks) * m + c]; int bi = pidx[((int64_t)b * chunks) * m + c];
  for (int k = 1; k < chunks; ++k) {
    const float x = pval[((int64_t)b * chunks + k) * m + c];
    if (x > best) { best = x; bi = pidx[((int64_t)b * chunks + k) * m + c]; }
  }
  colidx[(int64_t)b * m + c] = bi;
}

// padded batch: -1 / 0 past the pair's lengths
__global__ void __launch_bounds__(256) match_finalize_kernel(int n, int m, const int* lens, float thr, const float* __restrict__ rowval,
                                                              const int* __restrict__ rowidx, const int* __restrict__ colidx,
                                                              int64_t* __restrict__ matches0, float* __restrict__ mscores0,
                                                              int64_t* __restrict__ matches1, float* __restrict__ mscores1) {
  const int b = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int* ri = rowidx + (int64_t)b * n;
  const int* ci = colidx + (int64_t)b * m;
  const float* rv = rowval + (int64_t)b * n;
  const int2 len = match_lengths(lens, b, gridDim.y, n, m);    // rows / columns past them: -1 / 0
  if (t >= len.x && t < n) {
    if (matches0) matches0[(int64_t)b * n + t] = -1;
    if (mscores0) mscores0[(int64_t)b * n + t] = 0.f;
  }
  if (t >= len.y && t < m) {
    if (matches1) matches1[(int64_t)b * m + t] = -1;
    if (mscores1) mscores1[(int64_t)b * m + t] = 0.f;
  }
  if (t < len.x) {
    const int j = ri[t];
    const bool mutual = (ci[j] == t);
    const float ms = mutual ? expf(rv[t]) : 0.f;
    const bool valid = mutual && (ms > thr);
    if (matches0) matches0[(int64_t)b * n + t] = valid ? (int64_t)j : -1;
    if (mscores0) mscores0[(int64_t)b * n + t] = ms;
  }
  if (t < len.y && (matches1 || mscores1)) {
    const int i = ci[t];
    const bool mutual1 = (ri[i] == t);
    const bool mutual0_i = (ci[ri[i]] == i);
    const float ms0_i = mutual0_i ? expf(rv[i]) : 0.f;
    const float ms1 = mutual1 ? ms0_i : 0.f;
    const bool valid1 = mutual1 && (mutual0_i && ms0_i > thr);
    if (matches1) matches1[(int64_t)b * m + t] = valid1 ? (int64_t)i : -1;
    if (mscores1) mscores1[(int64_t)b * m + t] = ms1;
  }
}

inline int64_t match_workspace_bytes(int B, int n, int m) {
  const int chunks = cdiv(n, MATCH_ROW_CHUNK);
  return align_up((int64_t)B * n * 4, 256) * 2 + align_up((int64_t)B * m * 4, 256) +
         align_up((int64_t)B * chunks * m * 4, 256) * 2;
}

// lens (padded batch, device): n_0 .. n_{B-1}, then m_0 .. m_{B-1}; n, m are the capacity
inline int match_launch(const float* scores, int B, int n, int m, float thr, int64_t* matches0, float* mscores0, int64_t* matches1,
                        float* mscores1, void* ws, int64_t ws_bytes, cudaStream_t stream, const int* lens = nullptr) {
  if (ws_bytes < match_workspace_bytes(B, n, m)) return fail(OG_EWORKSPACE, "match: workspace too small");
  const int chunks = cdiv(n, MATCH_ROW_CHUNK);
  char* w = static_cast<char*>(ws);
  float* rowval = reinterpret_cast<float*>(w); w += align_up((int64_t)B * n * 4, 256);
  int* rowidx = reinterpret_cast<int*>(w); w += align_up((int64_t)B * n * 4, 256);
  int* colidx = reinterpret_cast<int*>(w); w += align_up((int64_t)B * m * 4, 256);
  float* pval = reinterpret_cast<float*>(w); w += align_up((int64_t)B * chunks * m * 4, 256);
  int* pidx = reinterpret_cast<int*>(w);
  int rc;
  if ((rc = OG_LAUNCH(match_rowmax_kernel, dim3(cdiv(n, 8), B), 256, 0, stream, scores, n, m, lens, rowval, rowidx))) return rc;
  if ((rc = OG_LAUNCH(match_colmax_kernel, dim3(cdiv(m, 256), chunks, B), 256, 0, stream, scores, n, m, lens, chunks, pval, pidx)))
    return rc;
  if ((rc = OG_LAUNCH(match_colreduce_kernel, dim3(cdiv(m, 256), B), 256, 0, stream, n, m, chunks, pval, pidx, colidx))) return rc;
  return OG_LAUNCH(match_finalize_kernel, dim3(cdiv(std::max(n, m), 256), B), 256, 0, stream, n, m, lens, thr, rowval, rowidx,
                   colidx, matches0, mscores0, matches1, mscores1);
}

}  // namespace og
