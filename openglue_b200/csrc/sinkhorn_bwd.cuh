// Backward pass of the dustbin-augmented log-domain Sinkhorn (SURVEY.md section 8, row f1): the gradient of
//     scores = Z + u_T + v_T - norm,   Z = S_aug / reg,   u_t = log_a - LSE_j(Z + v_{t-1}),   v_t = log_b - LSE_i(Z + u_t)
// with respect to S_aug, through all T unrolled iterations - what torch autograd computes for the reference's
// SuperGlue.get_matching_probs / log_otp_solver (superglue.py:88-111, optimal_transport.py:4-28) in training_step
// (matching_module.py:99-105), without keeping T copies of the (N+1) x (M+1) matrix.
//
// With G = d loss / d scores:   ubar_T = G 1,  vbar_T = G^T 1,  Zbar = G, and for t = T .. 1
//     P2_ij = exp(Z_ij + u_t,i + v_t,j - log_b_j)   (column-normalised)     Zbar -= vbar_t,j P2_ij ;  ubar_t,i -= sum_j vbar_t,j P2_ij
//     P1_ij = exp(Z_ij + u_t,i + v_{t-1},j - log_a_i) (row-normalised)      Zbar -= ubar_t,i P1_ij ;  vbar_{t-1},j = - sum_i ubar_t,i P1_ij
// P1 = P2 * wq_j / a_i with wq_j = exp(v_{t-1},j - v_t,j + log_b_j), so one sweep over Z with ONE exponential per element
// serves both reductions of an iteration - the forward kernel's structure, built from the same pieces (csrc/sinkhorn.cuh:
// strips of rows, W warps per row, bulk-copy row ring, per-pair barrier, deterministic column reduction, one plan and one
// launcher), with u_t / v_t read from the history the forward pass recorded.  The matrix gradient is then one more pass with
// Z in registers:
//     Zbar_ij = G_ij - sum_t exp(Z_ij + u_t,i + cvec_t,j) (vbar_t,j + coef_t,i wq_t,j),   coef_t,i = ubar_t,i / a_i
// (T exponentials per element from the MUFU pipe, no HBM traffic beyond Z, G and the result).
// HBM-bound like the forward pass: T sweeps over Z.  d loss / d S = Zbar[:N, :M] / reg; d loss / d dustbin = the sum of
// Zbar's last row and column / reg.
#pragma once
#include "sinkhorn.cuh"

namespace og {

struct SinkBwdArgs {
  static constexpr bool kBackward = true;
  const float* S; int64_t lds, strideS;
  const float* dustbin;
  int B, n, m, iters;
  float reg, norm, log_a_last, log_b_last;
  const float* hist_u;                   // [B][T][n+1]
  const float* hist_v;                   // [B][T+1][m+1]
  const float* ubar_init;                // [B][n+1]  row sums of G
  const float* vbar_init;                // [B][m+1]  column sums of G
  float* hist_coef;                      // [B][T][n+1]   ubar_t,i / a_i
  float* hist_cvec;                      // [B][T][m+1]   v_t,j - log_b_j
  float* hist_vbar;                      // [B][T][m+1]   vbar_t,j
  float* hist_wq;                        // [B][T][m+1]   exp(v_{t-1},j - v_t,j + log_b_j)
  float* partial;                        // [2][B][SP][mpad]
  unsigned int* barrier;
  int SP, rows_per_strip, mpad;
  const int* len_n;                      // padded batch (null otherwise), as SinkArgs: pair b is the [len_n[b], len_m[b]] block of the
  const int* len_m;                      // capacity; every history row and G keep the capacity's strides (n + 1, m + 1)
};

template <int V, int W, int SLOTS>
__global__ void __launch_bounds__(SINK_WARPS * 32, (V <= 8) ? 2 : 1) sinkhorn_bwd_kernel(SinkBwdArgs a) {
  extern __shared__ __align__(128) float og_sinkb_smem[];
  using Strip = SinkStrip<V, W>;
  constexpr int C = Strip::C, MC = Strip::MC, G = Strip::G;
  float* cvec_s = og_sinkb_smem;                       // [MC + 4]  v_t,j - log_b_j  (-inf for the padding columns; [MC] = dustbin column)
  float* vbar_s = cvec_s + MC + 4;                     // [MC + 4]  vbar_t,j
  float* wq_s = vbar_s + MC + 4;                       // [MC + 4]
  float* red = wq_s + MC + 4;                          // [G][mpad]
  float* ring = red + G * a.mpad;                      // [SINK_WARPS][SLOTS][C]
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + SINK_WARPS * SLOTS * C);
  float* xr = reinterpret_cast<float*>(bars + SINK_WARPS * SLOTS);               // [2][G][W] partial row sums
  const SinkPair P(a, blockIdx.x / a.SP);
  const Strip s(a, P.n, P.m);
  const int n = P.n, m = P.m, T = a.iters, b = s.b, tid = s.tid;
  const int64_t n1 = a.n + 1, m1 = a.m + 1;           // the capacity's row lengths of the histories
  const float ia_reg = expf(-P.norm), ia_last = expf(-P.log_a_last);      // 1 / a_i
  SinkRowRing<V, W, SLOTS, false, SinkBwdArgs> rows(a, s, ring, bars);
  const float dz = rows.dz;

  for (int j = tid; j <= MC; j += blockDim.x) {        // vbar_T = column sums of G
    float vb = 0.f;
    if (j < m) vb = __ldg(a.vbar_init + b * m1 + j);
    else if (j == MC) vb = __ldg(a.vbar_init + b * m1 + m);
    vbar_s[j] = vb;
  }
  __syncthreads();

  rows.prime();
  uint32_t rowpar = 0;
  for (int it = T - 1; it >= 0; --it) {
    // column constants of iteration t = it + 1 (every CTA of the pair builds the same values)
    const float* vt = a.hist_v + ((int64_t)b * (T + 1) + it + 1) * m1;
    const float* vtm1 = vt - m1;
    for (int j = tid; j <= MC; j += blockDim.x) {
      float cv = -CUDART_INF_F, wq = 0.f;
      const int jj = (j < m) ? j : (j == MC ? m : -1);
      if (jj >= 0) {
        const float lb = (jj < m) ? P.norm : P.log_b_last;
        cv = __ldcg(vt + jj) - lb;
        wq = expf(__ldcg(vtm1 + jj) - cv);
      }
      cvec_s[j] = cv; wq_s[j] = wq;
    }
    __syncthreads();
    if (s.strip == 0) {                                // history for the matrix-gradient pass
      const int64_t o = ((int64_t)b * T + it) * m1;
      for (int j = tid; j <= m; j += blockDim.x) {
        const int js = (j < m) ? j : MC;
        a.hist_cvec[o + j] = cvec_s[js]; a.hist_vbar[o + j] = vbar_s[js]; a.hist_wq[o + j] = wq_s[js];
      }
    }
    float4 cacc[V];
#pragma unroll
    for (int k = 0; k < V; ++k) cacc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    float cacc_m = 0.f;
    const float cv_m = cvec_s[MC], vb_m = vbar_s[MC];
    const float* ut = a.hist_u + ((int64_t)b * T + it) * n1;

    for (int row = s.r0 + s.grp; row < s.r1; row += G) {
      float4 z[V];
      rows.take(row, z);
      const float u_i = __ldcg(ut + row);
      float rs = 0.f;
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const int c = s.c0 + 4 * (s.lane + 32 * k);
        const float4 cv = *reinterpret_cast<const float4*>(cvec_s + c);
        const float4 vb = *reinterpret_cast<const float4*>(vbar_s + c);
        z[k].x = ex2_approx(((z[k].x + cv.x) + u_i) * LOG2E_F);     // P2_ij <= 1: no shift needed; padding: 2^-inf = 0
        z[k].y = ex2_approx(((z[k].y + cv.y) + u_i) * LOG2E_F);
        z[k].z = ex2_approx(((z[k].z + cv.z) + u_i) * LOG2E_F);
        z[k].w = ex2_approx(((z[k].w + cv.w) + u_i) * LOG2E_F);
        rs = fmaf(z[k].x, vb.x, rs); rs = fmaf(z[k].y, vb.y, rs); rs = fmaf(z[k].z, vb.z, rs); rs = fmaf(z[k].w, vb.w, rs);
      }
      const float e_m = (s.sub == 0) ? ex2_approx(((dz + cv_m) + u_i) * LOG2E_F) : 0.f;
      float r_i = warp_sum(rs) + e_m * vb_m;
      if (W > 1) {
        const float* x = sink_row_exchange(xr, r_i, s, rowpar);
        r_i = 0.f;
#pragma unroll
        for (int w2 = 0; w2 < W; ++w2) r_i += x[w2];
      }
      const float ub0 = (it == T - 1) ? __ldg(a.ubar_init + b * n1 + row) : 0.f;
      const float coef = (ub0 - r_i) * ((row < n) ? ia_reg : ia_last);      // ubar_t,i / a_i
      if (s.sub == 0 && s.lane == 0) a.hist_coef[((int64_t)b * T + it) * n1 + row] = coef;
#pragma unroll
      for (int k = 0; k < V; ++k) {
        cacc[k].x = fmaf(z[k].x, coef, cacc[k].x); cacc[k].y = fmaf(z[k].y, coef, cacc[k].y);
        cacc[k].z = fmaf(z[k].z, coef, cacc[k].z); cacc[k].w = fmaf(z[k].w, coef, cacc[k].w);
      }
      cacc_m = fmaf(e_m, coef, cacc_m);
    }
    if (it > 0) rows.prime();                          // the next iteration's first rows fly during the reduction
    // vbar_{t-1},j = - wq_j sum_i coef_i e_ij
    sink_column_reduce(a, s, red, cacc, cacc_m, T - 1 - it, [&](int j, float c) { vbar_s[j] = -wq_s[j] * c; });
  }
}

// ---- small kernels around the sweeps ------------------------------------------------------------------------------
// row sums of G [B, n+1, m+1]: one warp per row (a padded batch: over the pair's m_b + 1 columns, len_m set)
__global__ void __launch_bounds__(256) sinkb_rowsum_kernel(const float* __restrict__ G, int rows_total, int m1_cap, int n1,
                                                           const int* __restrict__ len_m, float* __restrict__ out) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows_total) return;
  const float* g = G + (int64_t)row * m1_cap;
  const int m1 = len_m ? padded_length(len_m, row / n1, m1_cap - 1) + 1 : m1_cap;
  float s = 0.f;
  for (int j = lane; j < m1; j += 32) s += __ldg(g + j);
  s = warp_sum(s);
  if (lane == 0) out[row] = s;
}
// column sums of G, two deterministic stages: strips of 64 rows -> partial [B][RS][m+1] -> out [B][m+1]
constexpr int SINKB_RS_ROWS = 64;
__global__ void __launch_bounds__(256) sinkb_colsum_kernel(const float* __restrict__ G, int n1, int m1, const int* __restrict__ len_n,
                                                           float* __restrict__ partial) {
  const int b = blockIdx.z, rs = blockIdx.y, j = blockIdx.x * 256 + threadIdx.x;
  if (j >= m1) return;
  const int i0 = rs * SINKB_RS_ROWS;
  const int i1 = min(i0 + SINKB_RS_ROWS, len_n ? padded_length(len_n, b, n1 - 1) + 1 : n1);
  const float* g = G + ((int64_t)b * n1 + i0) * m1 + j;
  float s = 0.f;
  for (int i = i0; i < i1; ++i, g += m1) s += __ldg(g);
  partial[((int64_t)b * gridDim.y + rs) * m1 + j] = s;
}
__global__ void __launch_bounds__(256) sinkb_colsum_finish_kernel(const float* __restrict__ partial, int nrs, int m1, float* __restrict__ out) {
  const int b = blockIdx.y, j = blockIdx.x * 256 + threadIdx.x;
  if (j >= m1) return;
  float s = 0.f;
  for (int r = 0; r < nrs; ++r) s += partial[((int64_t)b * nrs + r) * m1 + j];
  out[(int64_t)b * m1 + j] = s;
}

// matrix gradient: tile of 64 rows x 128 columns per CTA (8 rows x 4 columns per thread), loop over the T iterations
constexpr int SINKB_TR = 64, SINKB_TC = 128;
__global__ void __launch_bounds__(256) sinkb_dz_kernel(SinkBwdArgs a, const float* __restrict__ G, float* __restrict__ dZ, float inv_reg) {
  const int b = blockIdx.z;
  const int n = padded_length(a.len_n, b, a.n), m = padded_length(a.len_m, b, a.m), T = a.iters;
  const int64_t n1 = a.n + 1, m1 = a.m + 1;                  // capacity strides (a padded pair's block is [n + 1, m + 1] of it)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i0 = blockIdx.y * SINKB_TR + warp * 8;            // my 8 rows
  const int j0 = blockIdx.x * SINKB_TC + lane * 4;            // my 4 columns
  const bool unit_reg = (a.reg == 1.0f);
  const float dzv = unit_reg ? __ldg(a.dustbin) : __fdiv_rn(__ldg(a.dustbin), a.reg);
  float z[8][4], acc[8][4];
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const int i = i0 + r;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int j = j0 + c;
      float v = 0.f;
      if (i <= n && j <= m) {
        if (i < n && j < m) { v = __ldg(a.S + (int64_t)b * a.strideS + (int64_t)i * a.lds + j); if (!unit_reg) v = __fdiv_rn(v, a.reg); }
        else v = dzv;
      }
      z[r][c] = v * LOG2E_F;                                  // exponent arguments are kept in the log2 domain
      acc[r][c] = 0.f;
    }
  }
  for (int it = 0; it < T; ++it) {
    const float* ut = a.hist_u + ((int64_t)b * T + it) * n1;
    const float* cf = a.hist_coef + ((int64_t)b * T + it) * n1;
    const int64_t co = ((int64_t)b * T + it) * m1;
    float cv[4], vb[4], wq[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int j = j0 + c;
      const bool ok = j <= m;
      cv[c] = ok ? __ldg(a.hist_cvec + co + j) * LOG2E_F : -CUDART_INF_F;
      vb[c] = ok ? __ldg(a.hist_vbar + co + j) : 0.f;
      wq[c] = ok ? __ldg(a.hist_wq + co + j) : 0.f;
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int i = min(i0 + r, n);
      const float u2 = __ldg(ut + i) * LOG2E_F, coef = __ldg(cf + i);
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const float e = ex2_approx((z[r][c] + cv[c]) + u2);
        acc[r][c] = fmaf(e, fmaf(coef, wq[c], vb[c]), acc[r][c]);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const int i = i0 + r;
    if (i > a.n) continue;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int j = j0 + c;
      if (j > a.m) continue;
      const int64_t o = ((int64_t)b * n1 + i) * m1 + j;
      dZ[o] = (i <= n && j <= m) ? (__ldg(G + o) - acc[r][c]) * inv_reg : 0.f;     // 0 outside a padded pair's block
    }
  }
}
// d loss / d dustbin = sum of dZ's last row and last column (the corner once): one CTA per pair, fixed order, then pairs in order.
// A padded pair (lens set) sums its own dustbin row n_b and column m_b.
__global__ void __launch_bounds__(256) sinkb_dustbin_kernel(const float* __restrict__ dZ, int B, int n_cap, int m_cap, const int* __restrict__ lens,
                                                            float* __restrict__ per_pair, unsigned int* counter, float* __restrict__ out) {
  __shared__ float red[8];
  const int b = blockIdx.x;
  const int64_t ld = m_cap + 1;
  const int n = lens ? padded_length(lens, b, n_cap) : n_cap, m = lens ? padded_length(lens + B, b, m_cap) : m_cap;
  const float* d = dZ + (int64_t)b * (n_cap + 1) * ld;
  float s = 0.f;
  for (int j = threadIdx.x; j <= m; j += 256) s += d[(int64_t)n * ld + j];
  for (int i = threadIdx.x; i < n; i += 256) s += d[(int64_t)i * ld + m];
  const float t = cta_sum<256>(s, red);
  if (threadIdx.x == 0) {
    per_pair[b] = t;
    if (last_cta_arrive(counter)) *out = last_cta_sum(per_pair, B);
  }
}

// history the forward pass records for the backward pass: u [B][T][n+1] then v [B][T+1][m+1]
inline int64_t sinkhorn_hist_floats(int B, int n, int m, int T) { return (int64_t)B * T * (n + 1) + (int64_t)B * (T + 1) * (m + 1); }

inline int64_t sinkhorn_bwd_workspace_bytes(int B, int n, int m, int T) {
  SinkPlan p;
  if (sinkhorn_plan(true, B, n, m, &p) != OG_OK) return -1;
  const int64_t nrs = cdiv(n + 1, SINKB_RS_ROWS);
  int64_t f = 0;
  f += align_up((int64_t)B * (n + 1), 64) + align_up((int64_t)B * (m + 1), 64);                 // ubar_init, vbar_init
  f += align_up((int64_t)B * nrs * (m + 1), 64);                                                // column-sum partials
  f += align_up((int64_t)B * T * (n + 1), 64) + 3 * align_up((int64_t)B * T * (m + 1), 64);     // coef, cvec, vbar, wq histories
  f += align_up(2LL * B * SINK_MAX_STRIPS * p.mpad, 64) + align_up((int64_t)B, 64);             // strip partials, per-pair dustbin sums
  return SINK_BARRIER_BYTES + 256 + f * 4;
}

// G = d loss / d scores [B, n+1, m+1] (dense) -> dZ = d loss / d S_aug [B, n+1, m+1], ddustbin [1]
inline int sinkhorn_bwd_launch(const float* S, int64_t lds, int64_t strideS, const float* dustbin, int B, int n, int m, int iters, float reg,
                               const float* hist, const float* G, float* dZ, float* ddustbin, void* ws, int64_t ws_bytes,
                               cudaStream_t stream, const int* lens = nullptr) {
  SinkPlan p;
  if (const int rc = sinkhorn_plan(true, B, n, m, &p)) return rc;
  if (ws_bytes < sinkhorn_bwd_workspace_bytes(B, n, m, iters)) return fail(OG_EWORKSPACE, "sinkhorn_bwd: workspace too small");
  if (const int rc = sinkhorn_check_rows("sinkhorn_bwd", S, lds, strideS, m)) return rc;
  if (lens && n > SINK_MAX_ROWS) return fail(OG_EUNSUPPORTED, "sinkhorn_bwd: a padded batch has at most %d rows, not %d", SINK_MAX_ROWS, n);
  if (lens)
    if (const int rc = sinkhorn_log_tables(stream)) return rc;
  const int T = iters;
  const int64_t nrs = cdiv(n + 1, SINKB_RS_ROWS);
  char* w = static_cast<char*>(ws);
  unsigned int* barrier = reinterpret_cast<unsigned int*>(w); w += SINK_BARRIER_BYTES;
  unsigned int* counter = reinterpret_cast<unsigned int*>(w); w += 256;
  float* f = reinterpret_cast<float*>(w);
  auto take = [&](int64_t nfl) { float* r = f; f += align_up(nfl, 64); return r; };
  float* ubar_init = take((int64_t)B * (n + 1));
  float* vbar_init = take((int64_t)B * (m + 1));
  float* colpart = take((int64_t)B * nrs * (m + 1));
  float* hist_coef = take((int64_t)B * T * (n + 1));
  float* hist_cvec = take((int64_t)B * T * (m + 1));
  float* hist_vbar = take((int64_t)B * T * (m + 1));
  float* hist_wq = take((int64_t)B * T * (m + 1));
  float* partial = take(2LL * B * SINK_MAX_STRIPS * p.mpad);
  float* per_pair = take(B);
  const SinkConsts k = sinkhorn_consts(n, m);
  const int m1 = m + 1, n1 = n + 1;
  int rc;
  const int* len_n = lens;
  const int* len_m = lens ? lens + B : nullptr;
  if ((rc = OG_LAUNCH(sinkb_rowsum_kernel, cdiv(B * n1, 8), 256, 0, stream, G, B * n1, m1, n1, len_m, ubar_init))) return rc;
  if ((rc = OG_LAUNCH(sinkb_colsum_kernel, dim3(cdiv(m1, 256), (unsigned)nrs, B), 256, 0, stream, G, n1, m1, len_n, colpart))) return rc;
  if ((rc = OG_LAUNCH(sinkb_colsum_finish_kernel, dim3(cdiv(m1, 256), B), 256, 0, stream, colpart, (int)nrs, m1, vbar_init))) return rc;
  SinkBwdArgs a;
  a.S = S; a.lds = lds; a.strideS = strideS; a.dustbin = dustbin; a.B = B; a.n = n; a.m = m; a.iters = T; a.reg = reg;
  a.norm = k.norm; a.log_a_last = k.log_a_last; a.log_b_last = k.log_b_last;
  a.hist_u = hist; a.hist_v = hist + (int64_t)B * T * (n + 1);
  a.ubar_init = ubar_init; a.vbar_init = vbar_init;
  a.hist_coef = hist_coef; a.hist_cvec = hist_cvec; a.hist_vbar = hist_vbar; a.hist_wq = hist_wq;
  a.partial = partial; a.barrier = barrier; a.SP = p.SP; a.rows_per_strip = p.rows_per_strip; a.mpad = p.mpad;
  a.len_n = len_n; a.len_m = len_m;
  if (T > 0) {
    rc = sinkhorn_for_each_launch(p, B, barrier, stream, [&](int b0, int nb) {
      SinkBwdArgs g = a;
      g.B = nb;
      g.S = S + (int64_t)b0 * strideS;
      g.hist_u = a.hist_u + (int64_t)b0 * T * n1; g.hist_v = a.hist_v + (int64_t)b0 * (T + 1) * m1;
      g.ubar_init = ubar_init + (int64_t)b0 * n1; g.vbar_init = vbar_init + (int64_t)b0 * m1;
      g.hist_coef = hist_coef + (int64_t)b0 * T * n1; g.hist_cvec = hist_cvec + (int64_t)b0 * T * m1;
      g.hist_vbar = hist_vbar + (int64_t)b0 * T * m1; g.hist_wq = hist_wq + (int64_t)b0 * T * m1;
      g.len_n = lens ? len_n + b0 : nullptr; g.len_m = lens ? len_m + b0 : nullptr;
      if (p.V == 4 && p.W == 1) return sinkhorn_coop_launch<sinkhorn_bwd_kernel<4, 1, 2>, 4, 1, 2>(g, p, stream);
      if (p.V == 4)             return sinkhorn_coop_launch<sinkhorn_bwd_kernel<4, 2, 2>, 4, 2, 2>(g, p, stream);
      if (p.V == 8)             return sinkhorn_coop_launch<sinkhorn_bwd_kernel<8, 2, 2>, 8, 2, 2>(g, p, stream);
      if (p.W == 2)             return sinkhorn_coop_launch<sinkhorn_bwd_kernel<16, 2, 1>, 16, 2, 1>(g, p, stream);
      return sinkhorn_coop_launch<sinkhorn_bwd_kernel<16, 4, 1>, 16, 4, 1>(g, p, stream);
    });
    if (rc != OG_OK) return rc;
  }
  if ((rc = OG_LAUNCH(sinkb_dz_kernel, dim3(cdiv(m1, SINKB_TC), cdiv(n1, SINKB_TR), B), 256, 0, stream, a, G, dZ, 1.f / reg))) return rc;
  OG_CUDA(cudaMemsetAsync(counter, 0, 4, stream));
  return OG_LAUNCH(sinkb_dustbin_kernel, B, 256, 0, stream, dZ, B, n, m, lens, per_pair, counter, ddustbin);
}

}  // namespace og
