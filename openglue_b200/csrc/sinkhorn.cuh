// Dustbin-augmented log-domain Sinkhorn, all iterations in ONE persistent cooperative launch.
// Replaces SuperGlue.get_matching_probs (superglue.py:88-111) + log_otp_solver
// (optimal_transport.py:4-28).
//
// Formulation (algebraically the reference's iteration, one sweep + one exp per element):
//   row i:      t_ij = z_ij + v_j,  mx_i = max_j t_ij,  e_ij = exp(t_ij - mx_i),  S_i = sum_j e_ij
//               u_i  = log_a_i - (mx_i + log S_i)                     [= log_a - LSE_j(Z + v)]
//   column j:   exp(z_ij + u_i) = e_ij * (a_i / S_i) * exp(-v_j)  =>
//               c_j = sum_i e_ij * a_i / S_i ,   v_j <- log_b_j + v_j - log c_j
//                                                                     [= log_b - LSE_i(Z + u)]
// so a row is read once per iteration, kept in registers between its row reduction and its
// column contribution, and the augmented (n+1) x (m+1) matrix is never materialised: the
// dustbin row and column are the constant dustbin score and are generated in registers.
//
// Decomposition: pair b is cut into SP strips of whole rows, one CTA per strip; a row is shared by W warps
// (a warp owns 128 V consecutive columns: V float4s per lane => m <= 128 V W <= 8192; the warps of a row
// combine their (max, sum) through shared memory and one named barrier per row).  Column sums are reduced
// warp -> CTA (shared memory) -> grid (per-strip partials in global memory, double buffered),
// with one grid-wide barrier per iteration; every CTA of a pair then rebuilds v redundantly
// in a fixed order (deterministic, no atomics on data).
#pragma once
#include "common.cuh"
#include <math_constants.h>
#include <algorithm>
#include <stdlib.h>

namespace og {

struct SinkArgs {
  const float* S; int64_t lds, strideS;
  const float* dustbin;
  int B, n, m, iters;
  float reg;
  float norm, log_a_last, log_b_last;   // -log(n+m), norm + log(m), norm + log(n)   (superglue.py:98-101)
  float* scores;                         // [B, n+1, m+1]
  float* u;                              // [B, n+1]   workspace
  float* partial;                        // [2, B, SP, mpad] workspace
  unsigned int* barrier;                 // [B] counters, one per pair, 128 bytes apart; zeroed before launch
  int SP, rows_per_strip, mpad;
  float* hist_u;                         // optional [B][iters][n+1]: u_t of every iteration  (kept for the backward pass,
  float* hist_v;                         // optional [B][iters+1][m+1]: v_t, row 0 = v_0 = 0   csrc/sinkhorn_bwd.cuh)
  int res_q16;                           // fraction (Q16) of the rows that are loaded with the L2 evict_last policy (see sink_policy)
  int pf_rows;                           // L2 prefetch distance beyond the ring, in rows of a group (0 = off)
};

constexpr int SINK_WARPS = 8;
constexpr int64_t SINK_BARRIER_BYTES = 256 * 128;     // one 128-byte line per pair of a launch (<= SM count pairs)
constexpr float LOG2E_F = 1.4426950408889634f;

__device__ __forceinline__ void grid_barrier(unsigned int* counter, unsigned int target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter, 1u);
    unsigned int seen;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(counter) : "memory");
    } while (seen < target);
    __threadfence();
  }
  __syncthreads();
}

// --- shared-memory row ring fed by bulk async copies (TMA 1-D): decouples HBM latency from the math ---

__device__ __forceinline__ uint32_t sink_smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void sink_mbar_init(uint64_t* bar) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(sink_smem_u32(bar)) : "memory");
}
// L2 residency: the score matrix is read `iters` + 1 times and never written, but at the headline shape (16 pairs x 2048^2 x 4 B
// = 268 MB) it is five times the 50 MB L2, and with plain LRU-like replacement a cyclic sweep over it hits nothing.  So a FIXED subset - the first res_rows rows of every strip, ~RES_MB in total - is loaded with
// the evict_last policy and everything else with evict_first: the subset stays in L2 across the iterations and only the rest
// streams from HBM.  The subset is INTERLEAVED with the streamed rows (round k of a strip is kept iff floor((k+1) f) != floor(k f)):
// with a contiguous block of resident rows every CTA would sit in its L2 phase at the same time and leave HBM idle, then all
// stream together.  The final pass reads every row with evict_first, which hands
// the lines back to the kernels that follow.
__device__ __forceinline__ uint64_t sink_policy(bool keep) {
  uint64_t p;
  if (keep) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  else      asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void sink_row_copy(float* dst, const float* src, uint32_t bytes, uint64_t* bar, uint64_t policy) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sink_smem_u32(bar)), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
               ::"r"(sink_smem_u32(dst)), "l"(src), "r"(bytes), "r"(sink_smem_u32(bar)), "l"(policy) : "memory");
}
__device__ __forceinline__ void sink_row_copy(float* dst, const float* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sink_smem_u32(bar)), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(sink_smem_u32(dst)), "l"(src), "r"(bytes), "r"(sink_smem_u32(bar)) : "memory");
}
// L2 prefetch of a row segment that the ring will ask for a few rows later: the 2-deep ring covers ~2 row times, about the loaded
// HBM latency; a segment that is already in L2 when its bulk copy is issued arrives in a fraction of that
__device__ __forceinline__ void sink_row_prefetch(const float* src, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void sink_mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(sink_smem_u32(bar)), "r"(parity) : "memory");
  } while (!ok);
}

// fp32 pairs: Hopper has no packed fp32 arithmetic, so each pair operation is two scalar round-to-nearest operations (the
// intrinsics keep the compiler from contracting them, so the results match a packed-pair implementation bit for bit)
typedef unsigned long long f32x2;
__device__ __forceinline__ f32x2 pk2(float x, float y) { f32x2 r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(x), "f"(y)); return r; }
__device__ __forceinline__ void upk2(f32x2 v, float& x, float& y) { asm("mov.b64 {%0, %1}, %2;" : "=f"(x), "=f"(y) : "l"(v)); }
#define OG_F32X2_OP(name, expr)                                        \
  __device__ __forceinline__ f32x2 name(f32x2 a, f32x2 b) {            \
    float ax, ay, bx, by; upk2(a, ax, ay); upk2(b, bx, by);            \
    auto op = [](float u, float v) { return expr; };                   \
    return pk2(op(ax, bx), op(ay, by));                                \
  }
OG_F32X2_OP(add2, __fadd_rn(u, v))
OG_F32X2_OP(sub2, __fsub_rn(u, v))
OG_F32X2_OP(mul2, __fmul_rn(u, v))
#undef OG_F32X2_OP
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) {
  float ax, ay, bx, by, cx, cy; upk2(a, ax, ay); upk2(b, bx, by); upk2(c, cx, cy);
  return pk2(__fmaf_rn(ax, bx, cx), __fmaf_rn(ay, by, cy));
}

// V: float4s per lane of a warp's column segment (C = 128 V columns);  W: warps that share one row (a row group covers
// W C columns; the warps exchange (max, sum) of their segments through shared memory and one named barrier per row);
// SLOTS: ring depth per warp.  Configurations with V <= 8 need <= 128 registers and <= 106 KB of shared memory: two CTAs
// per SM, so one CTA streams while the other sits in its per-iteration reduction / barrier phase.
template <int V, int W, int SLOTS>
__global__ void __launch_bounds__(SINK_WARPS * 32, (V <= 8) ? 2 : 1) sinkhorn_kernel(SinkArgs a) {
  extern __shared__ __align__(128) float og_sink_smem[];
  constexpr int C = 128 * V;                           // columns of one warp's segment = floats per ring slot
  constexpr int MC = W * C;                            // columns a row group covers (m <= MC)
  constexpr int G = SINK_WARPS / W;                    // row groups = rows in progress per CTA
  float* v_s = og_sink_smem;                           // [MC + 4]  v_j for j < m, -inf for m <= j < MC (masks the padding
                                                       //           columns in the sweep without per-element selects), v_s[MC] = v_dustbin
  float* red = og_sink_smem + MC + 4;                  // [G][mpad]
  float* ring = red + G * a.mpad;                      // [SINK_WARPS][SLOTS][C]
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + SINK_WARPS * SLOTS * C);   // [SINK_WARPS][SLOTS]
  float2* xr = reinterpret_cast<float2*>(bars + SINK_WARPS * SLOTS);             // [2][G][W] (max, sum) of a segment
  const int b = blockIdx.x / a.SP, strip = blockIdx.x % a.SP;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int grp = warp / W, sub = warp % W;
  const int c0 = sub * C;                              // first column of this warp's segment
  const int n = a.n, m = a.m;
  const int r0 = strip * a.rows_per_strip;
  const int r1 = min(r0 + a.rows_per_strip, n + 1);
  const int r1_real = min(r1, n);                      // rows that exist in memory (the dustbin row does not)
  const float* __restrict__ Sb = a.S + (int64_t)b * a.strideS;
  const bool unit_reg = (a.reg == 1.0f);
  const float dz = unit_reg ? __ldg(a.dustbin) : __fdiv_rn(__ldg(a.dustbin), a.reg);   // Z = M / reg
  const float a_reg = expf(a.norm), a_last = expf(a.log_a_last);
  const int seg_cols = min(m, c0 + C) - c0;            // <= 0: this warp's segment lies beyond the last column
  const bool has_seg = seg_cols > 0;
  const bool seg_full = seg_cols == C;                 // warp-uniform
  const uint32_t seg_bytes = has_seg ? (uint32_t)(((seg_cols + 3) / 4) * 16) : 0u;     // <= 4 * (lds - c0): inside the padded row
  float* my_ring = ring + warp * SLOTS * C;
  uint64_t* my_bars = bars + warp * SLOTS;

  if (lane == 0) {
    for (int sl = 0; sl < SLOTS; ++sl) sink_mbar_init(&my_bars[sl]);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int j = tid; j < MC; j += blockDim.x) v_s[j] = (j < m) ? 0.f : -CUDART_INF_F;
  if (tid == 0) v_s[MC] = 0.f;
  __syncthreads();

  uint32_t issued = 0, consumed = 0;                   // per-warp ring counters (real rows only)
  const uint64_t pol_keep = sink_policy(true), pol_stream = sink_policy(false);
  auto keep_row = [&](int row) {                       // does this row belong to the L2-resident subset?
    const uint32_t k = (uint32_t)(row - r0) / (uint32_t)G;
    return ((k + 1) * (uint32_t)a.res_q16 >> 16) != (k * (uint32_t)a.res_q16 >> 16);
  };
  bool last_sweep = (a.iters == 0);                    // the sweep being FETCHED is the final pass (set below)
  auto prefetch_first = [&]() {                        // first SLOTS rows of this warp's group
    if (lane == 0 && has_seg) {
      for (int sl = 0; sl < SLOTS; ++sl) {
        const int row = r0 + grp + sl * G;
        if (row < r1_real) {
          sink_row_copy(my_ring + (issued % SLOTS) * C, Sb + (int64_t)row * a.lds + c0, seg_bytes, &my_bars[issued % SLOTS],
                        (!last_sweep && keep_row(row)) ? pol_keep : pol_stream);
          ++issued;
        }
      }
      for (int sl = SLOTS; sl < SLOTS + a.pf_rows; ++sl) {
        const int row = r0 + grp + sl * G;
        if (row < r1_real) sink_row_prefetch(Sb + (int64_t)row * a.lds + c0, seg_bytes);
      }
    }
  };
  // fetch this warp's segment of row `row` into registers (float4 k = pairs 2k, 2k+1); refill the slot with the row SLOTS ahead
  auto take_row = [&](int row, f32x2 (&z)[2 * V]) {
    if (row < n) {
      if (has_seg) {
        const uint32_t sl = consumed % SLOTS, ph = (consumed / SLOTS) & 1;
        sink_mbar_wait(&my_bars[sl], ph);
        const ulonglong2* src = reinterpret_cast<const ulonglong2*>(my_ring + sl * C);
        if (seg_full) {                                // the whole segment lies inside the row: no masks (the common case)
#pragma unroll
          for (int k = 0; k < V; ++k) { const ulonglong2 q = src[lane + 32 * k]; z[2 * k] = q.x; z[2 * k + 1] = q.y; }
        } else {
#pragma unroll
          for (int k = 0; k < V; ++k) {
            const int idx = lane + 32 * k;
            const int c = c0 + 4 * idx;
            float4 q = (c < m) ? reinterpret_cast<const float4*>(src)[idx] : make_float4(0.f, 0.f, 0.f, 0.f);
            if (c < m && c + 3 >= m) {                 // the float4 that straddles column m: its tail is row padding (any bits)
              if (c + 1 >= m) q.y = 0.f;
              if (c + 2 >= m) q.z = 0.f;
              q.w = 0.f;
            }
            z[2 * k] = pk2(q.x, q.y); z[2 * k + 1] = pk2(q.z, q.w);
          }
        }
        ++consumed;
        __syncwarp();                                  // every lane has its part of the row in registers
        const int nxt = row + SLOTS * G;
        if (lane == 0 && nxt < r1_real) {
          sink_row_copy(my_ring + sl * C, Sb + (int64_t)nxt * a.lds + c0, seg_bytes, &my_bars[sl],
                        (!last_sweep && keep_row(nxt)) ? pol_keep : pol_stream);
          ++issued;
        }
        const int pfr = nxt + a.pf_rows * G;
        if (lane == 0 && a.pf_rows > 0 && pfr < r1_real) sink_row_prefetch(Sb + (int64_t)pfr * a.lds + c0, seg_bytes);
        if (!unit_reg) {
#pragma unroll
          for (int k = 0; k < 2 * V; ++k) {
            float x, y; upk2(z[k], x, y);
            z[k] = pk2(__fdiv_rn(x, a.reg), __fdiv_rn(y, a.reg));
          }
        }
      } else {
#pragma unroll
        for (int k = 0; k < 2 * V; ++k) z[k] = 0ull;   // masked through v = -inf
      }
    } else {                                           // the dustbin row is the constant dustbin score
#pragma unroll
      for (int k = 0; k < 2 * V; ++k) z[k] = pk2(dz, dz);
    }
  };

  prefetch_first();
  uint32_t rowpar = 0;                                 // parity of the exchange buffer (alternates per row of the group)
  const f32x2 log2e2 = pk2(LOG2E_F, LOG2E_F);
  for (int it = 0; it < a.iters; ++it) {
    if (tid == 0) OG_TRACE_EVT(0, it);
    f32x2 cacc[2 * V];
#pragma unroll
    for (int k = 0; k < 2 * V; ++k) cacc[k] = 0ull;
    float cacc_m = 0.f;
    const float v_m = v_s[MC];

    for (int row = r0 + grp; row < r1; row += G) {
      f32x2 z[2 * V];
#ifdef OG_TRACE
      const int tr = (it == 20 && tid == 0) ? (row - r0) / G : 1 << 20;     // row timeline of warp 0 in iteration 20
#define OG_SINK_ROW_EVT(e) OG_TRACE_EVT(e, tr)
#else
#define OG_SINK_ROW_EVT(e) do { } while (0)
#endif
      OG_SINK_ROW_EVT(5);
      take_row(row, z);
      OG_SINK_ROW_EVT(6);
      // t = z + v, masked; maximum over this warp's segment (the dustbin column entry belongs to segment 0)
      const float t_m = dz + v_m;
      float mx = (sub == 0) ? t_m : -CUDART_INF_F;
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const ulonglong2 vv = *reinterpret_cast<const ulonglong2*>(v_s + c0 + 4 * (lane + 32 * k));   // columns >= m: finite z + (-inf) = -inf, e = 0
        z[2 * k] = add2(z[2 * k], vv.x); z[2 * k + 1] = add2(z[2 * k + 1], vv.y);
        float x0, x1, x2, x3; upk2(z[2 * k], x0, x1); upk2(z[2 * k + 1], x2, x3);
        mx = fmaxf(mx, fmaxf(fmaxf(x0, x1), fmaxf(x2, x3)));
      }
      mx = warp_max(mx);
      OG_SINK_ROW_EVT(7);
      const float mxs = (mx == -CUDART_INF_F) ? 0.f : mx;               // an all-padding segment: e = 2^-inf = 0, not NaN
      const f32x2 mxs2 = pk2(mxs, mxs);
      f32x2 sum2a = 0ull, sum2b = 0ull;
#pragma unroll
      for (int k = 0; k < 2 * V; ++k) {
        float x, y; upk2(mul2(sub2(z[k], mxs2), log2e2), x, y);
        z[k] = pk2(ex2_approx(x), ex2_approx(y));
        if (k & 1) sum2b = add2(sum2b, z[k]); else sum2a = add2(sum2a, z[k]);
      }
      float sa, sb; upk2(add2(sum2a, sum2b), sa, sb);
      const float e_m = (sub == 0) ? ex2_approx((t_m - mxs) * LOG2E_F) : 0.f;
      float s_i = warp_sum(sa + sb) + e_m;
      OG_SINK_ROW_EVT(8);
      float mxg = mx, f_w = 1.f;
      if (W > 1) {                                     // combine the segments of the row: S = sum_w S_w 2^(mx_w - mx)
        float2* x = xr + (rowpar * G + grp) * W;
        if (lane == 0) x[sub] = make_float2(mx, s_i);
        asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "n"(W * 32) : "memory");
        float2 p[W];
#pragma unroll
        for (int w2 = 0; w2 < W; ++w2) { p[w2] = x[w2]; mxg = fmaxf(mxg, p[w2].x); }
        s_i = 0.f;
#pragma unroll
        for (int w2 = 0; w2 < W; ++w2) s_i = fmaf(p[w2].y, ex2_approx((p[w2].x - mxg) * LOG2E_F), s_i);   // fixed order: identical in every warp
        f_w = ex2_approx((mx - mxg) * LOG2E_F);
        rowpar ^= 1u;
      }
      OG_SINK_ROW_EVT(9);
      const float w_i = __fdiv_rn((row < n) ? a_reg : a_last, s_i) * f_w;
      if ((it == a.iters - 1 || a.hist_u) && sub == 0 && lane == 0) {
        const float u_i = ((row < n) ? a.norm : a.log_a_last) - (mxg + logf(s_i));
        if (it == a.iters - 1) a.u[(int64_t)b * (n + 1) + row] = u_i;
        if (a.hist_u) a.hist_u[((int64_t)b * a.iters + it) * (n + 1) + row] = u_i;
      }
      const f32x2 w2 = pk2(w_i, w_i);
#pragma unroll
      for (int k = 0; k < 2 * V; ++k) cacc[k] = fma2(z[k], w2, cacc[k]);
      cacc_m = fmaf(e_m, w_i, cacc_m);
      OG_SINK_ROW_EVT(10);
    }
    if (tid == 0) OG_TRACE_EVT(1, it);
    last_sweep = (it == a.iters - 1);
    prefetch_first();                                 // next sweep's (or the final pass's) first rows fly during the reduction
    // warp -> CTA: a row group's warps own disjoint column segments of red[grp]
    float* myred = red + grp * a.mpad;
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const int c = c0 + 4 * (lane + 32 * k);
      if (c < m) *reinterpret_cast<ulonglong2*>(myred + c) = make_ulonglong2(cacc[2 * k], cacc[2 * k + 1]);   // entries >= m are zero
    }
    __syncthreads();                                  // (a) all float4 column sums are in `red`
    if (sub == 0 && lane == 0) myred[m] = cacc_m;     // column m = dustbin column (may overlap a float4 tail)
    __syncthreads();
    float* part = a.partial + ((int64_t)(it & 1) * a.B * a.SP + (int64_t)b * a.SP + strip) * a.mpad;
    for (int j = tid; j <= m; j += blockDim.x) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < G; ++w) s += red[w * a.mpad + j];
      part[j] = s;
    }
    // only the SP CTAs of this pair exchange data: a per-pair barrier (own 128-byte line) lets the pairs drift apart,
    // so HBM keeps streaming for the other pairs while one pair sits in its reduction / barrier phase
    if (tid == 0) OG_TRACE_EVT(2, it);
    grid_barrier(a.barrier + 32 * b, (unsigned int)(it + 1) * (unsigned int)a.SP);
    if (tid == 0) OG_TRACE_EVT(3, it);
    // every CTA of the pair rebuilds v (fixed summation order => bitwise identical across CTAs)
    const float* pb = a.partial + ((int64_t)(it & 1) * a.B * a.SP + (int64_t)b * a.SP) * a.mpad;
    // float4 columns, all SP loads of a thread in flight together (this phase is pure L2 latency: every CTA of the pair waits on it)
    for (int j4 = tid; 4 * j4 <= m; j4 += blockDim.x) {
      float4 c = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 8
      for (int s = 0; s < a.SP; ++s) {
        const float4 q = __ldcg(reinterpret_cast<const float4*>(pb + (int64_t)s * a.mpad) + j4);
        c.x += q.x; c.y += q.y; c.z += q.z; c.w += q.w;
      }
      const float cc[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int j = 4 * j4 + e;
        if (j < m) v_s[j] = a.norm + v_s[j] - logf(cc[e]);
        else if (j == m) v_s[MC] = a.log_b_last + v_s[MC] - logf(cc[e]);
      }
    }
    __syncthreads();
    if (tid == 0) OG_TRACE_EVT(4, it);
    if (a.hist_v && strip == 0) {                     // every CTA of the pair holds the same v: one of them records it
      float* hv = a.hist_v + ((int64_t)b * (a.iters + 1) + it + 1) * (m + 1);
      for (int j = tid; j <= m; j += blockDim.x) hv[j] = (j < m) ? v_s[j] : v_s[MC];
    }
  }

  // final pass: scores = Z + u + v - norm   (optimal_transport.py:28, superglue.py:111)
  {
    const float v_m = v_s[MC];
    for (int row = r0 + grp; row < r1; row += G) {
      f32x2 zp[2 * V];
      take_row(row, zp);
      float u_i = 0.f;
      if (a.iters > 0) {
        if (lane == 0) u_i = __ldcg(a.u + (int64_t)b * (n + 1) + row);
        u_i = __shfl_sync(0xffffffffu, u_i, 0);
      }
      float* out = a.scores + ((int64_t)b * (n + 1) + row) * (m + 1);
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const int c = c0 + 4 * (lane + 32 * k);
        if (c < m) {
          const float4 vv = *reinterpret_cast<const float4*>(v_s + c);
          float z0, z1, z2, z3; upk2(zp[2 * k], z0, z1); upk2(zp[2 * k + 1], z2, z3);
          if (c + 0 < m) out[c + 0] = (z0 + u_i) + vv.x - a.norm;
          if (c + 1 < m) out[c + 1] = (z1 + u_i) + vv.y - a.norm;
          if (c + 2 < m) out[c + 2] = (z2 + u_i) + vv.z - a.norm;
          if (c + 3 < m) out[c + 3] = (z3 + u_i) + vv.w - a.norm;
        }
      }
      if (sub == 0 && lane == 0) out[m] = (dz + u_i) + v_m - a.norm;
    }
  }
}

struct SinkPlan { int V, W, slots, occ, SP, rows_per_strip, mpad, pairs_per_launch; size_t smem; };
constexpr int SINK_MAX_COLS = 8192;
constexpr int SINK_L2_RESIDENT_MB = 0;   // of the 50 MB L2
constexpr int SINK_L2_PREFETCH_ROWS = 0;

template <int V, int W, int SLOTS>
constexpr size_t sinkhorn_smem(int mpad) {
  constexpr int C = 128 * V, G = SINK_WARPS / W;
  return ((size_t)(W * C + 4) + (size_t)G * mpad + (size_t)SINK_WARPS * SLOTS * C) * sizeof(float) +
         (size_t)SINK_WARPS * SLOTS * sizeof(uint64_t) + (size_t)2 * G * W * sizeof(float2) + 128;
}

// strips per pair / pairs per cooperative launch for p->occ co-resident CTAs per SM
inline void sinkhorn_decompose(SinkPlan* p, int B, int n) {
  const int sms = device_info().ok ? device_info().sm_count : 132;
  const int slots_total = sms * p->occ;                 // co-resident CTAs of the cooperative launch
  p->pairs_per_launch = std::min(B < slots_total ? B : slots_total, (int)(SINK_BARRIER_BYTES / 128));
  // experiment knobs: OG_SINK_PAIRS = pairs per launch (L2 blocking), OG_SINK_SP = max strips per pair
  static const int env_pairs = [] { const char* e = getenv("OG_SINK_PAIRS"); return e ? atoi(e) : 0; }();
  static const int env_sp = [] { const char* e = getenv("OG_SINK_SP"); return e ? atoi(e) : 32; }();
  if (env_pairs > 0 && env_pairs < p->pairs_per_launch) p->pairs_per_launch = env_pairs;
  int sp = slots_total / p->pairs_per_launch;
  if (sp > env_sp) sp = env_sp;
  const int max_sp = cdiv(n + 1, SINK_WARPS / p->W);
  if (sp > max_sp) sp = max_sp;
  if (sp < 1) sp = 1;
  p->SP = sp;
  p->rows_per_strip = cdiv(n + 1, sp);
}

inline int sinkhorn_plan(int B, int n, int m, SinkPlan* p) {
  p->mpad = (int)align_up(m + 1, 4);
  if (m <= 512)       { p->V = 4;  p->W = 1; p->slots = 2; p->occ = 2; p->smem = sinkhorn_smem<4, 1, 2>(p->mpad); }
  else if (m <= 1024) { p->V = 4;  p->W = 2; p->slots = 2; p->occ = 2; p->smem = sinkhorn_smem<4, 2, 2>(p->mpad); }
  else if (m <= 2048) { p->V = 8;  p->W = 2; p->slots = 2; p->occ = 2; p->smem = sinkhorn_smem<8, 2, 2>(p->mpad); }
  else if (m <= 4096) { p->V = 16; p->W = 2; p->slots = 2; p->occ = 1; p->smem = sinkhorn_smem<16, 2, 2>(p->mpad); }
  else if (m <= SINK_MAX_COLS) { p->V = 16; p->W = 4; p->slots = 1; p->occ = 1; p->smem = sinkhorn_smem<16, 4, 1>(p->mpad); }
  else return fail(OG_EUNSUPPORTED, "sinkhorn: m = %d > %d columns not supported (swap the images)", m, SINK_MAX_COLS);
  static const int env_occ = [] { const char* e = getenv("OG_SINK_OCC"); return e ? atoi(e) : 0; }();      // experiment: force 1 CTA / SM
  // experiment: OG_SINK_CFG=VWS picks another instantiation for 1024 < m <= 2048 (824 = V 8, W 2, 4 slots; 1612; 444)
  static const int env_cfg = [] { const char* e = getenv("OG_SINK_CFG"); return e ? atoi(e) : 0; }();
  if (m > 1024 && m <= 2048) {
    if (env_cfg == 824)  { p->V = 8;  p->W = 2; p->slots = 4; p->occ = 1; p->smem = sinkhorn_smem<8, 2, 4>(p->mpad); }
    if (env_cfg == 1612) { p->V = 16; p->W = 1; p->slots = 2; p->occ = 1; p->smem = sinkhorn_smem<16, 1, 2>(p->mpad); }
    if (env_cfg == 444)  { p->V = 4;  p->W = 4; p->slots = 4; p->occ = 2; p->smem = sinkhorn_smem<4, 4, 4>(p->mpad); }
  }
  if (env_occ == 1) p->occ = 1;
  sinkhorn_decompose(p, B, n);
  return OG_OK;
}

inline int64_t sinkhorn_workspace_bytes(int B, int n, int m) {
  SinkPlan p;
  if (sinkhorn_plan(B, n, m, &p) != OG_OK) return -1;
  // sized for the largest strip count any occupancy setting may choose (the plan depends on the device only through the SM count)
  const int64_t sp_max = std::max(p.SP, 32);
  return SINK_BARRIER_BYTES + align_up((int64_t)B * (n + 1) * 4, 256) + align_up(2LL * B * sp_max * p.mpad * 4, 256);
}

template <int V, int W, int SLOTS>
inline int sinkhorn_launch_v(SinkArgs a, const SinkPlan& p, cudaStream_t stream) {
  constexpr size_t smem_max = sinkhorn_smem<V, W, SLOTS>(128 * V * W + 4);     // largest request of this instantiation: m = 128 V W
  static_assert(smem_max <= OG_SMEM_OPTIN_MAX, "sinkhorn_kernel: shared memory beyond what one block may opt in to");
  if (const int rc = smem_opt_in<sinkhorn_kernel<V, W, SLOTS>>((int)smem_max)) return rc;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(a.B * a.SP);
  cfg.blockDim = dim3(SINK_WARPS * 32);
  cfg.dynamicSmemBytes = p.smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  OG_CUDA(cudaLaunchKernelEx(&cfg, sinkhorn_kernel<V, W, SLOTS>, a));
  launch_counter()++;
  return OG_OK;
}

inline int sinkhorn_launch(const float* S, int64_t lds, int64_t strideS, const float* dustbin, int B, int n, int m,
                           int iters, float reg, float* scores, void* ws, int64_t ws_bytes, cudaStream_t stream,
                           float* hist_u = nullptr, float* hist_v = nullptr) {
  SinkPlan p;
  int rc = sinkhorn_plan(B, n, m, &p);
  if (rc != OG_OK) return rc;
  if (ws_bytes < sinkhorn_workspace_bytes(B, n, m)) return fail(OG_EWORKSPACE, "sinkhorn: workspace too small");
  if (lds % 4 != 0 || lds < m || (reinterpret_cast<uintptr_t>(S) & 15) || strideS % 4 != 0)
    return fail(OG_EINVAL, "sinkhorn: S rows must be 16-byte aligned (lds %% 4 == 0, lds >= m)");
  char* w = static_cast<char*>(ws);
  unsigned int* barrier = reinterpret_cast<unsigned int*>(w); w += SINK_BARRIER_BYTES;
  float* u = reinterpret_cast<float*>(w); w += align_up((int64_t)B * (n + 1) * 4, 256);
  float* partial = reinterpret_cast<float*>(w);
  // host-side constants exactly as the reference builds them (float32 throughout)
  const float norm = -logf((float)(n + m));
  const float log_a_last = norm + (float)log((double)m);     // log_a[-1] += math.log(n_cols)
  const float log_b_last = norm + (float)log((double)n);     // log_b[-1] += math.log(n_rows)
  if (hist_v) OG_CUDA(cudaMemsetAsync(hist_v, 0, (size_t)B * (iters + 1) * (m + 1) * sizeof(float), stream));   // row 0 of every pair = v_0 = 0
  for (int b0 = 0; b0 < B; b0 += p.pairs_per_launch) {
    const int nb = std::min(p.pairs_per_launch, B - b0);
    SinkArgs a;
    a.S = S + (int64_t)b0 * strideS; a.lds = lds; a.strideS = strideS; a.dustbin = dustbin;
    a.B = nb; a.n = n; a.m = m; a.iters = iters; a.reg = reg;
    a.norm = norm; a.log_a_last = log_a_last; a.log_b_last = log_b_last;
    a.scores = scores + (int64_t)b0 * (n + 1) * (m + 1);
    a.u = u; a.partial = partial; a.barrier = barrier;
    a.SP = p.SP; a.rows_per_strip = p.rows_per_strip; a.mpad = p.mpad;
    a.hist_u = hist_u ? hist_u + (int64_t)b0 * iters * (n + 1) : nullptr;
    a.hist_v = hist_v ? hist_v + (int64_t)b0 * (iters + 1) * (m + 1) : nullptr;
    {                                                  // L2-resident subset: ~res_mb MB of this launch's matrices (OG_SINK_L2_MB, 0 = off)
      static const int res_mb = [] { const char* e = getenv("OG_SINK_L2_MB"); return e ? atoi(e) : SINK_L2_RESIDENT_MB; }();
      const double total = (double)nb * n * (double)m * 4.0;
      const double frac = total > 0 ? std::min(1.0, res_mb * 1048576.0 / total) : 0.0;
      a.res_q16 = (int)(frac * 65536.0);
      static const int pf = [] { const char* e = getenv("OG_SINK_PF"); return e ? atoi(e) : SINK_L2_PREFETCH_ROWS; }();
      a.pf_rows = pf;
    }
    OG_CUDA(cudaMemsetAsync(barrier, 0, (size_t)nb * 128, stream));
    if (p.V == 8 && p.slots == 4)   rc = sinkhorn_launch_v<8, 2, 4>(a, p, stream);
    else if (p.V == 16 && p.W == 1) rc = sinkhorn_launch_v<16, 1, 2>(a, p, stream);
    else if (p.V == 4 && p.W == 4)  rc = sinkhorn_launch_v<4, 4, 4>(a, p, stream);
    else if (p.V == 4 && p.W == 1)  rc = sinkhorn_launch_v<4, 1, 2>(a, p, stream);
    else if (p.V == 4)              rc = sinkhorn_launch_v<4, 2, 2>(a, p, stream);
    else if (p.V == 8)              rc = sinkhorn_launch_v<8, 2, 2>(a, p, stream);
    else if (p.W == 2)              rc = sinkhorn_launch_v<16, 2, 2>(a, p, stream);
    else                            rc = sinkhorn_launch_v<16, 4, 1>(a, p, stream);
    if (rc != OG_OK) return rc;
  }
  return OG_OK;
}

}  // namespace og
