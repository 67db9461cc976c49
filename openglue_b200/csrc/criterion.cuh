// Matching loss of the reference's training step and its gradient with respect to the log-scores.
// Replaces criterion (reference utils/losses.py:7-53) for margin = None - the value of every shipped config
// (config/*.yaml: `margin: null`, `metric_weight: 0.0`), where 'metric_loss' is identically 0:
//
//   per pair b:   L_b = - mean_{i: gt0[i] >= 0} scores[b, i, gt0[i]]
//                       - 0.5 * ( mean_{i: gt0[i] == -1} scores[b, i, M]  +  mean_{j: gt1[j] == -1} scores[b, N, j] )
//   loss = sum_b L_b / B            (a pair with an empty set contributes nothing for that set, as unique_consecutive
//                                    in the reference never sees it; IGNORE (-2) entries are in no set)
//
// HBM-bound gather: 3 * (N + M) scalars per pair.  One CTA per pair, fixed-order block reduction, the per-pair terms are
// summed by the last CTA to finish in pair order: deterministic, no float atomics.
// The gradient is the scatter of the same weights (everything else is zero): dscores[b, i, gt0[i]] = -1 / (B c_m), ...
#pragma once
#include "common.cuh"

namespace og {

constexpr int CRIT_THREADS = 256;

struct CritArgs {
  const float* scores;          // [B, n+1, m+1]
  const int64_t* gt0;           // [B, n]
  const int64_t* gt1;           // [B, m]
  int B, n, m;
  float* per_pair;              // [B] workspace
  unsigned int* counter;        // workspace, zeroed before launch
  float* loss;                  // [2]: {loss, metric_loss}
  float* dscores;               // optional [B, n+1, m+1], zero-filled by the caller: receives d loss / d scores
  float grad_scale;             // upstream gradient of 'loss' (nll_weight)
  const int* lens;              // padded batch (null otherwise): n_0 .. n_{B-1}, m_0 .. m_{B-1}; pair b is the [n_b + 1, m_b + 1] block of
                                // its capacity-strided scores (dustbins at n_b, m_b), its labels past the lengths are ignored
};

__global__ void __launch_bounds__(CRIT_THREADS) criterion_kernel(CritArgs a) {
  __shared__ float red[CRIT_THREADS / 32];
  __shared__ float s_cnt[3];
  __shared__ bool last;
  const int b = blockIdx.x;
  const int n = a.lens ? padded_length(a.lens, b, a.n) : a.n, m = a.lens ? padded_length(a.lens + a.B, b, a.m) : a.m;
  const int64_t ld = a.m + 1;
  const float* S = a.scores + (int64_t)b * (a.n + 1) * ld;
  const int64_t* g0 = a.gt0 + (int64_t)b * a.n;
  const int64_t* g1 = a.gt1 + (int64_t)b * a.m;
  float sm = 0.f, su0 = 0.f, su1 = 0.f, cm = 0.f, cu0 = 0.f, cu1 = 0.f;
  for (int i = threadIdx.x; i < n; i += CRIT_THREADS) {
    const int64_t g = g0[i];
    if (g >= 0 && g < m) { sm += S[(int64_t)i * ld + g]; cm += 1.f; }
    else if (g == -1)    { su0 += S[(int64_t)i * ld + m]; cu0 += 1.f; }
  }
  for (int j = threadIdx.x; j < m; j += CRIT_THREADS)
    if (g1[j] == -1) { su1 += S[(int64_t)n * ld + j]; cu1 += 1.f; }
  const float tm = cta_sum<CRIT_THREADS>(sm, red), tu0 = cta_sum<CRIT_THREADS>(su0, red), tu1 = cta_sum<CRIT_THREADS>(su1, red);
  const float nm = cta_sum<CRIT_THREADS>(cm, red), nu0 = cta_sum<CRIT_THREADS>(cu0, red), nu1 = cta_sum<CRIT_THREADS>(cu1, red);
  if (threadIdx.x == 0) {
    float l = 0.f;
    if (nm > 0.f) l -= tm / nm;
    if (nu0 > 0.f) l -= 0.5f * tu0 / nu0;
    if (nu1 > 0.f) l -= 0.5f * tu1 / nu1;
    a.per_pair[b] = l;
    s_cnt[0] = nm; s_cnt[1] = nu0; s_cnt[2] = nu1;
    last = last_cta_arrive(a.counter);
  }
  __syncthreads();
  if (a.dscores) {                                          // d loss / d scores: the same gather, scattered
    float* D = a.dscores + (int64_t)b * (a.n + 1) * ld;
    const float wm = s_cnt[0] > 0.f ? -a.grad_scale / (s_cnt[0] * a.B) : 0.f;
    const float w0 = s_cnt[1] > 0.f ? -0.5f * a.grad_scale / (s_cnt[1] * a.B) : 0.f;
    const float w1 = s_cnt[2] > 0.f ? -0.5f * a.grad_scale / (s_cnt[2] * a.B) : 0.f;
    for (int i = threadIdx.x; i < n; i += CRIT_THREADS) {
      const int64_t g = g0[i];
      if (g >= 0 && g < m) D[(int64_t)i * ld + g] = wm;       // a row holds at most one of the two
      else if (g == -1)    D[(int64_t)i * ld + m] = w0;
    }
    for (int j = threadIdx.x; j < m; j += CRIT_THREADS)
      if (g1[j] == -1) D[(int64_t)n * ld + j] = w1;
  }
  if (last && threadIdx.x == 0) {
    a.loss[0] = last_cta_sum(a.per_pair, a.B) / (float)a.B;       // pair order: deterministic
    a.loss[1] = 0.f;                                               // metric_loss with margin = None (utils/losses.py:56-58, 83-85)
  }
}

inline int64_t criterion_workspace_bytes(int B) { return 256 + align_up((int64_t)B * 4, 256); }

inline int criterion_launch(const float* scores, const int64_t* gt0, const int64_t* gt1, int B, int n, int m, float* loss,
                            float* dscores, float grad_scale, void* ws, int64_t ws_bytes, cudaStream_t stream,
                            const int* lens = nullptr) {
  if (ws_bytes < criterion_workspace_bytes(B)) return fail(OG_EWORKSPACE, "criterion: workspace too small");
  CritArgs a;
  a.scores = scores; a.gt0 = gt0; a.gt1 = gt1; a.B = B; a.n = n; a.m = m;
  a.counter = static_cast<unsigned int*>(ws);
  a.per_pair = reinterpret_cast<float*>(static_cast<char*>(ws) + 256);
  a.loss = loss; a.dscores = dscores; a.grad_scale = grad_scale; a.lens = lens;
  OG_CUDA(cudaMemsetAsync(a.counter, 0, 4, stream));
  return OG_LAUNCH(criterion_kernel, B, CRIT_THREADS, 0, stream, a);
}

}  // namespace og
