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
//
// The backward pass (sinkhorn_bwd.cuh) sweeps the same strips in the same way, so the pieces both kernels are made of live
// here: the strip geometry (SinkStrip), the bulk-copy row ring (SinkRowRing), the exchange among the warps of a row
// (sink_row_exchange), the column reduction (sink_column_reduce), the plan (band table, occupancy, strips) and the launcher.
#pragma once
#include "common.cuh"
#include "tc_common.cuh"
#include <math_constants.h>
#include <algorithm>
#include <mutex>
#include <type_traits>
#include <vector>

namespace og {

struct SinkArgs {
  static constexpr bool kBackward = false;
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
  int rows_smem;                         // resident kernel: rows per warp held in shared memory
  float* vglob;                          // resident kernel: [B, mpad] 64-bit words, v as each strip publishes its columns
  float* hist_u;                         // optional [B][iters][n+1]: u_t of every iteration  (kept for the backward pass,
  float* hist_v;                         // optional [B][iters+1][m+1]: v_t, row 0 = v_0 = 0   csrc/sinkhorn_bwd.cuh)
  const int* len_n;                      // padded batch (null otherwise): pair b has len_n[b] rows and len_m[b] columns of the
  const int* len_m;                      // capacity n x m (clamped into [1, n] / [1, m]); S outside that block is never read
};

constexpr int SINK_WARPS = 8;
constexpr int64_t SINK_BARRIER_BYTES = 256 * 128;     // one 128-byte line per pair of a launch (<= SM count pairs)
constexpr int SINK_MAX_COLS = 8192;
constexpr int SINK_MAX_STRIPS = 32;                    // strips per pair at most (the strip-partial workspace is sized for it)
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
// W C columns; the warps exchange what they know of their segments through shared memory and one named barrier per row);
// G = SINK_WARPS / W row groups = rows in progress per CTA.  A warp works on rows r0 + grp, r0 + grp + G, ... of its strip
// [r0, r1) (row n is the dustbin row), columns [c0, c0 + C) of each.
// n, m: the pair's rows and columns, a.n and a.m or, in a padded batch, its own lengths (r1 <= r0 for a strip past them).
template <int V, int W>
struct SinkStrip {
  static constexpr int C = 128 * V, MC = W * C, G = SINK_WARPS / W;
  int b, strip, tid, lane, grp, sub, c0, r0, r1, n, m;
  template <class Args>
  __device__ __forceinline__ SinkStrip(const Args& a, int rows, int cols) : n(rows), m(cols) {
    b = blockIdx.x / a.SP; strip = blockIdx.x % a.SP;
    tid = threadIdx.x; lane = tid & 31;
    grp = (tid >> 5) / W; sub = (tid >> 5) % W;
    c0 = sub * C;
    r0 = strip * a.rows_per_strip;
    r1 = min(r0 + a.rows_per_strip, n + 1);
  }
};

// The lengths of pair b and the constants of its marginals (SinkConsts): the arguments' own, or in a padded batch (a.len_n set) the
// pair's, from the tables of the host's logarithms (sinkhorn_log_tables), so that a pair at the capacity gets the very bits a
// uniform batch gets.  A uniform batch never reads the tables.
constexpr int SINK_MAX_ROWS = 65536;                   // rows of a padded batch's capacity at most (the size of the tables)
__device__ float og_sink_logf_tab[SINK_MAX_ROWS + SINK_MAX_COLS + 1];   // [k] = logf((float)k), the host's libm
__device__ float og_sink_log_tab[SINK_MAX_ROWS + 1];                    // [k] = (float)log((double)k)
struct SinkPair {
  int n, m;
  float norm, log_a_last, log_b_last;
  template <class Args>
  __device__ __forceinline__ SinkPair(const Args& a, int b) {
    n = padded_length(a.len_n, b, a.n);
    m = padded_length(a.len_m, b, a.m);
    if (a.len_n) {
      norm = -og_sink_logf_tab[n + m];
      log_a_last = norm + og_sink_log_tab[m];
      log_b_last = norm + og_sink_log_tab[n];
    } else {
      norm = a.norm; log_a_last = a.log_a_last; log_b_last = a.log_b_last;
    }
  }
};

// One warp's slice of the shared-memory row ring, fed by bulk async copies (TMA 1-D) so that HBM latency overlaps the math of
// the rows before: SLOTS segments of C floats, one mbarrier each.  Every sweep visits the warp's rows in the same order;
// `consumed` counts the real rows taken so far and gives each its slot and phase.  EVICT_FIRST loads with the L2 evict_first
// policy (the forward pass): at the headline shape the score matrix is five times the 50 MB L2 and is swept cyclically, so
// its lines would hit nothing and only push out those of the kernels that follow.
template <int V, int W, int SLOTS, bool EVICT_FIRST, class Args>
struct SinkRowRing {
  static constexpr int C = 128 * V, G = SINK_WARPS / W;
  float* slot;                                         // [SLOTS][C]
  uint64_t* bar;                                       // [SLOTS]
  const Args& a;
  const float* seg;                                    // this warp's column segment of row 0 of the pair
  int first, end_real, n, c0, lane;                    // first row of the warp; rows >= end_real do not exist in memory; row n: dustbin
  uint32_t bytes, consumed;                            // bytes of a segment: 0 when it lies beyond the pair's last column
  bool full;                                           // the whole segment lies inside the pair's row (warp-uniform)
  float dz;                                            // the dustbin score divided by reg, Z = M / reg
  uint64_t policy;

  __device__ __forceinline__ SinkRowRing(const Args& args, const SinkStrip<V, W>& s, float* ring, uint64_t* bars) : a(args) {
    const int warp = s.grp * W + s.sub;
    slot = ring + warp * SLOTS * C;
    bar = bars + warp * SLOTS;
    seg = a.S + (int64_t)s.b * a.strideS + s.c0;
    first = s.r0 + s.grp;
    end_real = min(s.r1, s.n);
    n = s.n;
    c0 = s.c0; lane = s.lane;
    const int seg_cols = min(s.m, c0 + C) - c0;        // <= 0: this warp's segment lies beyond the pair's last column
    bytes = seg_cols > 0 ? (uint32_t)(((seg_cols + 3) / 4) * 16) : 0u;     // <= 4 * (lds - c0): inside the padded row
    full = seg_cols == C;
    consumed = 0;
    dz = (a.reg == 1.0f) ? __ldg(a.dustbin) : __fdiv_rn(__ldg(a.dustbin), a.reg);
    if (lane == 0) {
      for (int sl = 0; sl < SLOTS; ++sl) tc::mbar_init(&bar[sl], 1);
      tc::fence_barrier_init();
    }
    if (EVICT_FIRST) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(policy));
  }

  __device__ __forceinline__ void copy(uint32_t sl, int row) {
    tc::mbar_arrive_expect_tx(&bar[sl], bytes);
    const float* src = seg + (int64_t)row * a.lds;
    if (EVICT_FIRST)
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                   ::"r"(tc::smem_u32(slot + sl * C)), "l"(src), "r"(bytes), "r"(tc::smem_u32(&bar[sl])), "l"(policy) : "memory");
    else
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                   ::"r"(tc::smem_u32(slot + sl * C)), "l"(src), "r"(bytes), "r"(tc::smem_u32(&bar[sl])) : "memory");
  }

  // Starts the copies of the first SLOTS rows of the next sweep.  Called only when a sweep follows: copies nobody waits for
  // could still be writing into shared memory when the CTA exits.
  __device__ __forceinline__ void prime() {
    if (lane == 0 && bytes) {
      for (int sl = 0; sl < SLOTS; ++sl) {
        const int row = first + sl * G;
        if (row < end_real) copy((consumed + sl) % SLOTS, row);
      }
    }
  }

  // This warp's segment of row `row` in registers (columns >= m zero, divided by reg), and the slot refilled with the row SLOTS
  // ahead.  The dustbin row is the constant dustbin score.  In a padded batch the columns m .. a.m - 1 of a row are padding of any
  // bits (NaN + -inf would be NaN), so they are neither copied nor read.
  __device__ __forceinline__ void take(int row, float4 (&z)[V]) {
    if (row >= n) {
#pragma unroll
      for (int k = 0; k < V; ++k) z[k] = make_float4(dz, dz, dz, dz);
      return;
    }
    if (!bytes) {
#pragma unroll
      for (int k = 0; k < V; ++k) z[k] = make_float4(0.f, 0.f, 0.f, 0.f);     // the kernels mask these columns
      return;
    }
    const uint32_t sl = consumed % SLOTS, ph = (consumed / SLOTS) & 1;
    while (!tc::mbar_try_wait(&bar[sl], ph)) {}
    const float4* src = reinterpret_cast<const float4*>(slot + sl * C);
    if (full) {                                        // no masks (the common case)
#pragma unroll
      for (int k = 0; k < V; ++k) z[k] = src[lane + 32 * k];
    } else {                                           // the pair's columns, reloaded: this path is rare and keeps no register
      const int m = padded_length(a.len_m, blockIdx.x / a.SP, a.m);
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const int idx = lane + 32 * k;
        const int c = c0 + 4 * idx;
        float4 q = (c < m) ? src[idx] : make_float4(0.f, 0.f, 0.f, 0.f);
        if (c < m && c + 3 >= m) {                     // the float4 that straddles column m: its tail is padding (any bits)
          if (c + 1 >= m) q.y = 0.f;
          if (c + 2 >= m) q.z = 0.f;
          q.w = 0.f;
        }
        z[k] = q;
      }
    }
    ++consumed;
    // The refill is an async-proxy write to the slot the lanes have just read through the generic proxy.  The memory model orders
    // the two only through a proxy fence; without it, whether the bulk copy can overtake the reads depends on the schedule nvcc
    // emits (16 pairs of 2048 x 2048 gave run-to-run differences on an H100 for a schedule that did not hide it).
    const int nxt = row + SLOTS * G;
    if (nxt < end_real) tc::fence_proxy_async();
    __syncwarp();                                      // every lane has its part of the row in registers
    if (lane == 0 && nxt < end_real) copy(sl, nxt);
    if (a.reg != 1.0f) {
      const float reg = a.reg;
#pragma unroll
      for (int k = 0; k < V; ++k) {
        z[k].x = __fdiv_rn(z[k].x, reg); z[k].y = __fdiv_rn(z[k].y, reg);
        z[k].z = __fdiv_rn(z[k].z, reg); z[k].w = __fdiv_rn(z[k].w, reg);
      }
    }
  }
};

// The W warps of a row group publish one value each (`mine`) and meet at the group's named barrier; the returned W values are
// in warp order, the same in every warp.  The buffer xr [2][G][W] alternates halves row by row (rowpar), so a warp that runs
// ahead into the next row cannot overwrite values another warp has yet to read.
template <int V, int W, class X>
__device__ __forceinline__ const X* sink_row_exchange(X* xr, X mine, const SinkStrip<V, W>& s, uint32_t& rowpar) {
  X* x = xr + (rowpar * SinkStrip<V, W>::G + s.grp) * W;
  if (s.lane == 0) x[s.sub] = mine;
  asm volatile("bar.sync %0, %1;" ::"r"(1 + s.grp), "n"(W * 32) : "memory");
  rowpar ^= 1u;
  return x;
}

// Column sums of sweep `k` (0, 1, ... in launch order): warp (cacc: this warp's segment; cacc_m: the dustbin column, counted by
// segment 0) -> CTA (red [G][mpad]: the row groups' warps own disjoint columns of their row) -> this strip's partial in global
// memory (buffer k & 1 of two) -> barrier among the SP CTAs of the pair -> every CTA of the pair rebuilds the sums in the same
// fixed order (bitwise identical across CTAs) and calls update(j, sum) for j < m and update(MC, sum) for the dustbin column.
// sink_strip_sums is its first part: the strip's column sums, passed to store(j, sum) for j <= m.
template <int V, int W, class Args, class Store>
__device__ __forceinline__ void sink_strip_sums(const Args& a, const SinkStrip<V, W>& s, float* red, const float4 (&cacc)[V],
                                                float cacc_m, Store store) {
  const int m = s.m;
  float* myred = red + s.grp * a.mpad;
#pragma unroll
  for (int q = 0; q < V; ++q) {
    const int c = s.c0 + 4 * (s.lane + 32 * q);
    if (c < m) *reinterpret_cast<float4*>(myred + c) = cacc[q];     // entries >= m are zero
  }
  __syncthreads();                                    // (a) all float4 column sums are in `red`
  if (s.sub == 0 && s.lane == 0) myred[m] = cacc_m;   // column m = dustbin column (may overlap a float4 tail)
  __syncthreads();
  for (int j = s.tid; j <= m; j += blockDim.x) {
    float sum = 0.f;
#pragma unroll
    for (int w = 0; w < SinkStrip<V, W>::G; ++w) sum += red[w * a.mpad + j];
    store(j, sum);
  }
}

template <int V, int W, class Args, class Update>
__device__ __forceinline__ void sink_column_reduce(const Args& a, const SinkStrip<V, W>& s, float* red, const float4 (&cacc)[V],
                                                   float cacc_m, int k, Update update) {
  const int m = s.m;
  const int64_t buf = (int64_t)(k & 1) * a.B * a.SP + (int64_t)s.b * a.SP;
  float* part = a.partial + (buf + s.strip) * a.mpad;
  sink_strip_sums(a, s, red, cacc, cacc_m, [&](int j, float sum) { part[j] = sum; });
  // only the SP CTAs of this pair exchange data: a per-pair barrier (own 128-byte line) lets the pairs drift apart,
  // so HBM keeps streaming for the other pairs while one pair sits in its reduction / barrier phase
  grid_barrier(a.barrier + 32 * s.b, (unsigned int)(k + 1) * (unsigned int)a.SP);
  const float* pb = a.partial + buf * a.mpad;
  // float4 columns, all SP loads of a thread in flight together (this phase is pure L2 latency: every CTA of the pair waits on it)
  for (int j4 = s.tid; 4 * j4 <= m; j4 += blockDim.x) {
    float4 c = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 8
    for (int sp = 0; sp < a.SP; ++sp) {
      const float4 q = __ldcg(reinterpret_cast<const float4*>(pb + (int64_t)sp * a.mpad) + j4);
      c.x += q.x; c.y += q.y; c.z += q.z; c.w += q.w;
    }
    const float cc[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int j = 4 * j4 + e;
      if (j < m) update(j, cc[e]);
      else if (j == m) update(SinkStrip<V, W>::MC, cc[e]);
    }
  }
  __syncthreads();
}

// What a warp publishes in the row exchange of NR rows: (max, sum) of its segment of each row.
template <int NR> using SinkRowStat = std::conditional_t<NR == 1, float2, float4>;

// NR (1 or 2) rows of a forward sweep (iteration `it`), rows row0 and row0 + G, from this warp's segments q[r] of them: t = z + v,
// each row's (max, sum) over the W warps of its group, u_i (stored in the last iteration and in hist_u when recorded) and the row's
// share e_ij a_i / S_i of the column sums, added to cacc (cacc_m: the dustbin column, counted by segment 0) row by row in order.
// v_s: v of the pair in shared memory, v_m = v_s[MC].  Two rows share one read of v and one exchange, and their reduction chains
// are independent, so one row's shuffles run under the other's exponentials; each row's arithmetic is the same for NR = 1 and 2.
template <int V, int W, int NR>
__device__ __forceinline__ void sink_fwd_rows(const SinkArgs& a, const SinkPair& P, const SinkStrip<V, W>& s, const float4 (*q)[V],
                                              const float* v_s, float v_m, float dz, float a_reg, float a_last, SinkRowStat<NR>* xr,
                                              uint32_t& rowpar, int row0, int it, f32x2 (&cacc)[2 * V], float& cacc_m) {
  static_assert(NR == 1 || NR == 2, "one or two rows at a time");
  const int n = P.n, c0 = s.c0, lane = s.lane, sub = s.sub;
  const f32x2 log2e2 = pk2(LOG2E_F, LOG2E_F);
  f32x2 z[NR][2 * V];
#pragma unroll
  for (int r = 0; r < NR; ++r)
#pragma unroll
    for (int k = 0; k < V; ++k) { z[r][2 * k] = pk2(q[r][k].x, q[r][k].y); z[r][2 * k + 1] = pk2(q[r][k].z, q[r][k].w); }
  // t = z + v, masked; maximum over this warp's segment (the dustbin column entry belongs to segment 0)
  const float t_m = dz + v_m;
  float mx[NR];
#pragma unroll
  for (int r = 0; r < NR; ++r) mx[r] = (sub == 0) ? t_m : -CUDART_INF_F;
#pragma unroll
  for (int k = 0; k < V; ++k) {
    const ulonglong2 vv = *reinterpret_cast<const ulonglong2*>(v_s + c0 + 4 * (lane + 32 * k));   // columns >= m: z = 0 (SinkRowRing), 0 + (-inf) = -inf, e = 0
#pragma unroll
    for (int r = 0; r < NR; ++r) {
      z[r][2 * k] = add2(z[r][2 * k], vv.x); z[r][2 * k + 1] = add2(z[r][2 * k + 1], vv.y);
      float x0, x1, x2, x3; upk2(z[r][2 * k], x0, x1); upk2(z[r][2 * k + 1], x2, x3);
      mx[r] = fmaxf(mx[r], fmaxf(fmaxf(x0, x1), fmaxf(x2, x3)));
    }
  }
#pragma unroll
  for (int r = 0; r < NR; ++r) mx[r] = warp_max(mx[r]);
  float s_i[NR], e_m[NR];
#pragma unroll
  for (int r = 0; r < NR; ++r) {
    const float mxs = (mx[r] == -CUDART_INF_F) ? 0.f : mx[r];      // an all-padding segment: e = 2^-inf = 0, not NaN
    const f32x2 mxs2 = pk2(mxs, mxs);
    f32x2 sum2a = 0ull, sum2b = 0ull;
#pragma unroll
    for (int k = 0; k < 2 * V; ++k) {
      float x, y; upk2(mul2(sub2(z[r][k], mxs2), log2e2), x, y);
      z[r][k] = pk2(ex2_approx(x), ex2_approx(y));
      if (k & 1) sum2b = add2(sum2b, z[r][k]); else sum2a = add2(sum2a, z[r][k]);
    }
    float sa, sb; upk2(add2(sum2a, sum2b), sa, sb);
    s_i[r] = sa + sb;
    e_m[r] = (sub == 0) ? ex2_approx((t_m - mxs) * LOG2E_F) : 0.f;
  }
#pragma unroll
  for (int r = 0; r < NR; ++r) s_i[r] = warp_sum(s_i[r]) + e_m[r];
  float mxg[NR], f_w[NR];
#pragma unroll
  for (int r = 0; r < NR; ++r) { mxg[r] = mx[r]; f_w[r] = 1.f; }
  if (W > 1) {                                     // combine the segments of each row: S = sum_w S_w 2^(mx_w - mx)
    SinkRowStat<NR> mine;
    if constexpr (NR == 1) mine = make_float2(mx[0], s_i[0]);
    else mine = make_float4(mx[0], s_i[0], mx[1], s_i[1]);
    const SinkRowStat<NR>* x = sink_row_exchange(xr, mine, s, rowpar);
    float pm[NR][W], ps[NR][W];
#pragma unroll
    for (int w2 = 0; w2 < W; ++w2) {
      const SinkRowStat<NR> p = x[w2];
      pm[0][w2] = p.x; ps[0][w2] = p.y;
      if constexpr (NR == 2) { pm[1][w2] = p.z; ps[1][w2] = p.w; }
    }
#pragma unroll
    for (int r = 0; r < NR; ++r) {
#pragma unroll
      for (int w2 = 0; w2 < W; ++w2) mxg[r] = fmaxf(mxg[r], pm[r][w2]);
      s_i[r] = 0.f;
#pragma unroll
      for (int w2 = 0; w2 < W; ++w2) s_i[r] = fmaf(ps[r][w2], ex2_approx((pm[r][w2] - mxg[r]) * LOG2E_F), s_i[r]);   // fixed order: identical in every warp
      f_w[r] = ex2_approx((mx[r] - mxg[r]) * LOG2E_F);
    }
  }
  float w_i[NR];
#pragma unroll
  for (int r = 0; r < NR; ++r) w_i[r] = __fdiv_rn((row0 + r * SinkStrip<V, W>::G < n) ? a_reg : a_last, s_i[r]) * f_w[r];
  if ((it == a.iters - 1 || a.hist_u) && sub == 0 && lane == 0) {
#pragma unroll
    for (int r = 0; r < NR; ++r) {
      const int row = row0 + r * SinkStrip<V, W>::G;
      const float u_i = ((row < n) ? P.norm : P.log_a_last) - (mxg[r] + logf(s_i[r]));
      if (it == a.iters - 1) a.u[(int64_t)s.b * (a.n + 1) + row] = u_i;
      if (a.hist_u) a.hist_u[((int64_t)s.b * a.iters + it) * (a.n + 1) + row] = u_i;
    }
  }
#pragma unroll
  for (int r = 0; r < NR; ++r) {
    const f32x2 w2 = pk2(w_i[r], w_i[r]);
#pragma unroll
    for (int k = 0; k < 2 * V; ++k) cacc[k] = fma2(z[r][k], w2, cacc[k]);
    cacc_m = fmaf(e_m[r], w_i[r], cacc_m);
  }
}

// The final pass over one row: scores = Z + u + v - norm   (optimal_transport.py:28, superglue.py:111).  Rows are a.m + 1 apart.
template <int V, int W>
__device__ __forceinline__ void sink_fwd_score_row(const SinkArgs& a, const SinkPair& P, const SinkStrip<V, W>& s, const float4 (&z)[V],
                                                   const float* v_s, float v_m, float dz, int row) {
  const int m = P.m, c0 = s.c0, lane = s.lane;
  float u_i = 0.f;
  if (a.iters > 0) {
    if (lane == 0) u_i = __ldcg(a.u + (int64_t)s.b * (a.n + 1) + row);
    u_i = __shfl_sync(0xffffffffu, u_i, 0);
  }
  float* out = a.scores + ((int64_t)s.b * (a.n + 1) + row) * (a.m + 1);
#pragma unroll
  for (int k = 0; k < V; ++k) {
    const int c = c0 + 4 * (lane + 32 * k);
    if (c < m) {
      const float4 vv = *reinterpret_cast<const float4*>(v_s + c);
      if (c + 0 < m) out[c + 0] = (z[k].x + u_i) + vv.x - P.norm;
      if (c + 1 < m) out[c + 1] = (z[k].y + u_i) + vv.y - P.norm;
      if (c + 2 < m) out[c + 2] = (z[k].z + u_i) + vv.z - P.norm;
      if (c + 3 < m) out[c + 3] = (z[k].w + u_i) + vv.w - P.norm;
    }
  }
  if (s.sub == 0 && lane == 0) out[m] = (dz + u_i) + v_m - P.norm;
}

// Padded batch, after the final pass: -inf over the strip's share of the padding of the pair's [a.n + 1, a.m + 1] block, the
// columns past its dustbin column in its rows and every column of the capacity's rows past its dustbin row.
template <int V, int W>
__device__ __forceinline__ void sink_fill_padding(const SinkArgs& a, const SinkStrip<V, W>& s) {
  const int rend = min(s.r0 + a.rows_per_strip, a.n + 1);
  for (int row = s.r0; row < rend; ++row) {
    float* out = a.scores + ((int64_t)s.b * (a.n + 1) + row) * (a.m + 1);
    for (int c = (row <= s.n ? s.m + 1 : 0) + s.tid; c <= a.m; c += blockDim.x) out[c] = -CUDART_INF_F;
  }
}

// SLOTS: ring depth per warp.  Configurations with V <= 8 need <= 128 registers and <= 106 KB of shared memory: two CTAs per
// SM, so one CTA streams while the other sits in its per-iteration reduction / barrier phase.
template <int V, int W, int SLOTS>
__global__ void __launch_bounds__(SINK_WARPS * 32, (V <= 8) ? 2 : 1) sinkhorn_kernel(SinkArgs a) {
  extern __shared__ __align__(128) float og_sink_smem[];
  using Strip = SinkStrip<V, W>;
  constexpr int C = Strip::C, MC = Strip::MC, G = Strip::G;
  float* v_s = og_sink_smem;                           // [MC + 4]  v_j for j < m, -inf for m <= j < MC (masks the padding
                                                       //           columns in the sweep without per-element selects), v_s[MC] = v_dustbin
  float* red = og_sink_smem + MC + 4;                  // [G][mpad]
  float* ring = red + G * a.mpad;                      // [SINK_WARPS][SLOTS][C]
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + SINK_WARPS * SLOTS * C);   // [SINK_WARPS][SLOTS]
  float2* xr = reinterpret_cast<float2*>(bars + SINK_WARPS * SLOTS);             // [2][G][W] (max, sum) of a segment
  const SinkPair P(a, blockIdx.x / a.SP);
  const Strip s(a, P.n, P.m);
  const int m = P.m;
  const float a_reg = expf(P.norm), a_last = expf(P.log_a_last);
  SinkRowRing<V, W, SLOTS, true, SinkArgs> rows(a, s, ring, bars);
  const float dz = rows.dz;

  for (int j = s.tid; j < MC; j += blockDim.x) v_s[j] = (j < m) ? 0.f : -CUDART_INF_F;
  if (s.tid == 0) v_s[MC] = 0.f;
  __syncthreads();

  rows.prime();
  uint32_t rowpar = 0;                                 // parity of the exchange buffer (alternates per row of the group)
  for (int it = 0; it < a.iters; ++it) {
    f32x2 cacc[2 * V];
#pragma unroll
    for (int k = 0; k < 2 * V; ++k) cacc[k] = 0ull;
    float cacc_m = 0.f;
    const float v_m = v_s[MC];

    for (int row = s.r0 + s.grp; row < s.r1; row += G) {
      float4 q[V];
      rows.take(row, q);
      sink_fwd_rows<V, W, 1>(a, P, s, &q, v_s, v_m, dz, a_reg, a_last, xr, rowpar, row, it, cacc, cacc_m);
    }
    rows.prime();                                      // next sweep's (or the final pass's) first rows fly during the reduction
    float4 c4[V];
#pragma unroll
    for (int k = 0; k < V; ++k) { upk2(cacc[2 * k], c4[k].x, c4[k].y); upk2(cacc[2 * k + 1], c4[k].z, c4[k].w); }
    sink_column_reduce(a, s, red, c4, cacc_m, it, [&](int j, float c) {
      v_s[j] = ((j < MC) ? P.norm : P.log_b_last) + v_s[j] - logf(c);
    });
    if (a.hist_v && s.strip == 0) {                   // every CTA of the pair holds the same v: one of them records it
      float* hv = a.hist_v + (int64_t)(a.m + 1) * (s.b * (a.iters + 1) + it + 1);     // capacity rows; the pair's dustbin at m
      for (int j = s.tid; j <= m; j += blockDim.x) hv[j] = (j < m) ? v_s[j] : v_s[MC];
    }
  }

  const float v_m = v_s[MC];
  for (int row = s.r0 + s.grp; row < s.r1; row += G) {
    float4 z[V];
    rows.take(row, z);
    sink_fwd_score_row(a, P, s, z, v_s, v_m, dz, row);
  }
  if (a.len_n) sink_fill_padding(a, s);
}

// A value and the iteration (from 1) it belongs to, as one 64-bit word: a single-copy-atomic store and load carry both, so a reader
// that sees the tag it waits for also sees the value, with no fence.
__device__ __forceinline__ void sink_put(uint64_t* p, float x, uint32_t tag) {
  asm volatile("st.relaxed.gpu.global.b64 [%0], %1;" ::"l"(p), "l"(((uint64_t)tag << 32) | __float_as_uint(x)) : "memory");
}
__device__ __forceinline__ uint64_t sink_get(const uint64_t* p) {
  uint64_t w;
  asm volatile("ld.relaxed.gpu.global.b64 %0, [%1];" : "=l"(w) : "l"(p) : "memory");
  return w;
}
// x[u] = the value at at(u) once its tag is `tag` (0 where at(u) is null).  The N loads are in flight together, and so are the
// reloads of the words that were not ready: a wait costs one memory round trip, not one per word.  SINK_POLL covers the
// (m + 1) / 256 <= 9 words of v a thread reads for m <= 2048, and the strips a thread sums at the plan's strip counts.
constexpr int SINK_POLL = 16;
template <int N, class At>
__device__ __forceinline__ void sink_take(float (&x)[N], At at, uint32_t tag) {
  uint64_t w[N];
#pragma unroll
  for (int u = 0; u < N; ++u) { const uint64_t* p = at(u); w[u] = p ? sink_get(p) : (uint64_t)tag << 32; }
  for (;;) {
    bool ready = true;
#pragma unroll
    for (int u = 0; u < N; ++u) ready &= (uint32_t)(w[u] >> 32) == tag;
    if (ready) break;
#pragma unroll
    for (int u = 0; u < N; ++u)
      if ((uint32_t)(w[u] >> 32) != tag) w[u] = sink_get(at(u));
  }
#pragma unroll
  for (int u = 0; u < N; ++u) x[u] = __uint_as_float((uint32_t)w[u]);
}

// The resident kernel's form of sink_strip_sums, in half the shared memory: the upper half of the row groups parks its column sums
// in red [G/2][mpad] (the dustbin column in redm [G]), the lower half adds its own to them, and store(j, sum) gets the G/2 folded
// sums added in order (a fixed order: the same bits in every run).
template <int V, int W, class Args, class Store>
__device__ __forceinline__ void sink_strip_sums_folded(const Args& a, const SinkStrip<V, W>& s, float* red, float* redm,
                                                       const float4 (&cacc)[V], float cacc_m, Store store) {
  constexpr int H = SinkStrip<V, W>::G / 2;
  const int m = s.m;
  float4* fold = reinterpret_cast<float4*>(red + (s.grp % H) * a.mpad);
  if (s.grp >= H) {
#pragma unroll
    for (int q = 0; q < V; ++q) {
      const int c = s.c0 + 4 * (s.lane + 32 * q);
      if (c < m) fold[c / 4] = cacc[q];                // entries >= m are zero
    }
  }
  if (s.sub == 0 && s.lane == 0) redm[s.grp] = cacc_m;
  __syncthreads();
  if (s.grp < H) {
#pragma unroll
    for (int q = 0; q < V; ++q) {
      const int c = s.c0 + 4 * (s.lane + 32 * q);
      if (c < m) {
        const float4 o = fold[c / 4];
        fold[c / 4] = make_float4(cacc[q].x + o.x, cacc[q].y + o.y, cacc[q].z + o.z, cacc[q].w + o.w);
      }
    }
  }
  __syncthreads();
  for (int j = s.tid; j <= m; j += blockDim.x) {
    float sum = 0.f;
#pragma unroll
    for (int h = 0; h < H; ++h) sum += (j < m) ? red[h * a.mpad + j] : redm[h] + redm[h + H];
    store(j, sum);
  }
}

// The resident kernel: the streaming kernel's sweep over score rows held on chip.  Its CTAs (one per SM) load their strip's rows
// once, in the first sweep, through a one-slot ring: a warp keeps its first RR rows in registers (RR V float4s per lane, fully
// unrolled, so only compile-time indices) and the rest in shared memory (`held`, [slots][SINK_WARPS][C]), so each score matrix is
// read from HBM once per launch instead of once per sweep.  The ring is the warp's last held slot, which its last row fills (a
// dedicated slot where no row is held in shared memory).  After the first sweep a warp works on its rows two at a time
// (sink_fwd_rows<2>: rows k and k + 1 of the warp, one read of v, one exchange, the two rows' reduction chains interleaved), an odd
// last row alone; the first sweep and the final score pass go one row at a time.  The rows are added into the column sums in the
// same order either way.  RR is even, so a pair never straddles registers and shared memory.  The strips number up to the SM
// count, so instead of every CTA summing every strip's partial (SP partials of the pair per CTA and iteration from L2) each strip
// sums the partials of its own 1/SP of the columns in a fixed order and publishes v there (vglob), and every CTA of the pair reads
// v back.  Partials and v travel as (value, iteration + 1) words (sink_put / sink_take), so a reader waits for exactly the words it
// needs and the pair needs no barrier: a strip writes its next partials only after it has read all of v, which every owner
// publishes only after it has read all partials of its columns, so one buffer of each suffices.  Both are zeroed before each launch.
template <int V, int W, int RR>
__global__ void __launch_bounds__(SINK_WARPS * 32, 1) sinkhorn_resident_kernel(SinkArgs a) {
  static_assert(RR % 2 == 0, "the register rows go two at a time");
  extern __shared__ __align__(128) float og_sink_smem[];
  using Strip = SinkStrip<V, W>;
  constexpr int C = Strip::C, MC = Strip::MC, G = Strip::G, NT = SINK_WARPS * 32, HS = SINK_WARPS * (C / 4);
  const int slots = max(a.rows_smem, 1);
  float* v_s = og_sink_smem;                                              // [MC + 4]  as in sinkhorn_kernel
  float* red = v_s + MC + 4;                                              // [G / 2][mpad]
  float* gsum = red + G / 2 * a.mpad;                                     // [NT]  per-group sums of a strip's columns
  float4* held = reinterpret_cast<float4*>(gsum + NT);                    // [slots][SINK_WARPS][C / 4]
  uint64_t* bars = reinterpret_cast<uint64_t*>(held + (size_t)slots * HS);   // [SINK_WARPS]
  float2* xr = reinterpret_cast<float2*>(bars + SINK_WARPS);             // [2][G][W]  one row's (max, sum)
  float4* xr2 = reinterpret_cast<float4*>(xr + 2 * G * W);               // [2][G][W]  two rows'
  float* redm = reinterpret_cast<float*>(xr2 + 2 * G * W);               // [G]
  const SinkPair P(a, blockIdx.x / a.SP);
  const Strip s(a, P.n, P.m);
  const int m = P.m, lane = s.lane, row0 = s.r0 + s.grp;
  const float a_reg = expf(P.norm), a_last = expf(P.log_a_last);
  float4* mine = held + (s.grp * W + s.sub) * (C / 4);
  SinkRowRing<V, W, 1, true, SinkArgs> rows(a, s, reinterpret_cast<float*>(held + (size_t)(slots - 1) * HS), bars);
  const float dz = rows.dz;
  uint64_t* vg = reinterpret_cast<uint64_t*>(a.vglob) + (int64_t)s.b * a.mpad;

  for (int j = s.tid; j < MC; j += blockDim.x) v_s[j] = (j < m) ? 0.f : -CUDART_INF_F;
  if (s.tid == 0) v_s[MC] = 0.f;
  __syncthreads();

  rows.prime();
  uint32_t rowpar = 0;
  float4 zr[RR / 2][2][V];                             // the warp's rows row0 + k G, k < RR
  for (int it = 0; it <= a.iters; ++it) {             // it == iters: the final pass
    const bool last = it == a.iters;
    f32x2 cacc[2 * V];
#pragma unroll
    for (int k = 0; k < 2 * V; ++k) cacc[k] = 0ull;
    float cacc_m = 0.f;
    const float v_m = v_s[MC];
    auto one = [&](int row, const float4 (*q)[V]) {
      sink_fwd_rows<V, W, 1>(a, P, s, q, v_s, v_m, dz, a_reg, a_last, xr, rowpar, row, it, cacc, cacc_m);
    };
    if (it == 0 || last) {
      auto visit = [&](int row, const float4 (&q)[V]) {
        if (last) sink_fwd_score_row(a, P, s, q, v_s, v_m, dz, row);
        else one(row, &q);
      };
#pragma unroll
      for (int k = 0; k < RR; ++k) {
        const int row = row0 + k * G;
        if (row < s.r1) {
          if (it == 0) rows.take(row, zr[k / 2][k % 2]);
          visit(row, zr[k / 2][k % 2]);
        }
      }
      float4* h = mine;
      for (int row = row0 + RR * G; row < s.r1; row += G, h += HS) {
        float4 q[V];
        if (it == 0) {
          rows.take(row, q);
#pragma unroll
          for (int k = 0; k < V; ++k) h[lane + 32 * k] = q[k];
        } else {
#pragma unroll
          for (int k = 0; k < V; ++k) q[k] = h[lane + 32 * k];
        }
        visit(row, q);
      }
      if (last) {
        if (a.len_n) sink_fill_padding(a, s);
        break;
      }
    } else {
      auto two = [&](int row, const float4 (*q)[V]) {
        sink_fwd_rows<V, W, 2>(a, P, s, q, v_s, v_m, dz, a_reg, a_last, xr2, rowpar, row, it, cacc, cacc_m);
      };
#pragma unroll
      for (int k = 0; k < RR; k += 2) {
        const int row = row0 + k * G;
        if (row + G < s.r1) two(row, zr[k / 2]);
        else if (row < s.r1) one(row, zr[k / 2]);
      }
      const float4* h = mine;
      int row = row0 + RR * G;
      for (; row + G < s.r1; row += 2 * G, h += 2 * HS) {
        float4 q[2][V];
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
          for (int k = 0; k < V; ++k) q[r][k] = h[r * HS + lane + 32 * k];
        two(row, q);
      }
      if (row < s.r1) {
        float4 q[1][V];
#pragma unroll
        for (int k = 0; k < V; ++k) q[0][k] = h[lane + 32 * k];
        one(row, q);
      }
    }

    float4 c4[V];
#pragma unroll
    for (int k = 0; k < V; ++k) { upk2(cacc[2 * k], c4[k].x, c4[k].y); upk2(cacc[2 * k + 1], c4[k].z, c4[k].w); }
    const uint32_t tag = it + 1;
    uint64_t* pt = reinterpret_cast<uint64_t*>(a.partial) + (int64_t)s.b * a.SP * a.mpad;
    sink_strip_sums_folded(a, s, red, redm, c4, cacc_m, [&](int j, float sum) { sink_put(pt + (int64_t)s.strip * a.mpad + j, sum, tag); });
    // this strip's columns [lo, lo + S): NG thread groups sum strips g, g + NG, ... of a column, then the groups are added in
    // order (a fixed order: the same bits in every run)
    const int S = cdiv(m + 1, a.SP), lo = s.strip * S, NG = S >= NT ? 1 : NT / S;
    auto publish = [&](int j, float c) {
      sink_put(vg + j, ((j < m) ? P.norm + v_s[j] : P.log_b_last + v_s[MC]) - logf(c), tag);
    };
    for (int i = s.tid; i < S * NG; i += NT) {
      const int j = lo + i % S;
      float sum = 0.f;
      if (j <= m) {
        for (int sp0 = i / S; sp0 < a.SP; sp0 += SINK_POLL * NG) {
          float x[SINK_POLL];
          sink_take<SINK_POLL>(x, [&](int u) { const int sp = sp0 + u * NG; return sp < a.SP ? pt + (int64_t)sp * a.mpad + j : nullptr; }, tag);
#pragma unroll
          for (int u = 0; u < SINK_POLL; ++u) sum += x[u];
        }
      }
      if (NG > 1) gsum[i] = sum;
      else if (j <= m) publish(j, sum);
    }
    if (NG > 1) {
      __syncthreads();
      for (int i = s.tid; i < S && lo + i <= m; i += NT) {
        float sum = gsum[i];
        for (int g = 1; g < NG; ++g) sum += gsum[g * S + i];
        publish(lo + i, sum);
      }
    }
    for (int j0 = s.tid; j0 <= m; j0 += SINK_POLL * NT) {
      float x[SINK_POLL];
      sink_take<SINK_POLL>(x, [&](int u) { const int j = j0 + u * NT; return j <= m ? vg + j : nullptr; }, tag);
#pragma unroll
      for (int u = 0; u < SINK_POLL; ++u) {
        const int j = j0 + u * NT;
        if (j <= m) v_s[(j < m) ? j : MC] = x[u];
      }
    }
    __syncthreads();
  }
}

// resident: the plan is for sinkhorn_resident_kernel (slots = 1, occ = 1); rows_reg / rows_smem: rows per warp in registers /
// in shared memory
struct SinkPlan { int V, W, slots, occ, SP, rows_per_strip, mpad, pairs_per_launch; size_t smem; bool resident; int rows_reg, rows_smem; };

// Dynamic shared memory of one CTA: the column vectors of MC + 4 floats (forward: v; backward: cvec, vbar, wq), the row groups'
// column sums [G][mpad], the row ring [SINK_WARPS][slots][C] and its mbarriers, the row exchange [2][G][W] (forward: (max, sum);
// backward: a sum) and 128 bytes of slack.
constexpr size_t sinkhorn_smem(bool backward, int V, int W, int slots, int mpad) {
  const int C = 128 * V, G = SINK_WARPS / W, vecs = backward ? 3 : 1;
  const size_t xbytes = backward ? sizeof(float) : sizeof(float2);
  return ((size_t)vecs * (W * C + 4) + (size_t)G * mpad + (size_t)SINK_WARPS * slots * C) * sizeof(float) +
         (size_t)SINK_WARPS * slots * sizeof(uint64_t) + (size_t)2 * G * W * xbytes + 128;
}

// The instantiation, its shared memory, the occupancy and the strip decomposition of either pass.  Both passes use the same V and
// W per column band; the backward keeps three column vectors in shared memory where the forward keeps one, so for
// 2048 < m <= 4096 it has ONE ring slot per warp (two would need 246 KB, more than a block may opt in to).  Two CTAs per SM
// (__launch_bounds__ allows it for V <= 8) while two blocks, each with the 1 KB the runtime reserves, fit in 227 KB.
inline int sinkhorn_plan(bool backward, int B, int n, int m, SinkPlan* p) {
  const char* who = backward ? "sinkhorn_bwd" : "sinkhorn";
  if (m <= 512)                { p->V = 4;  p->W = 1; p->slots = 2; }
  else if (m <= 1024)          { p->V = 4;  p->W = 2; p->slots = 2; }
  else if (m <= 2048)          { p->V = 8;  p->W = 2; p->slots = 2; }
  else if (m <= 4096)          { p->V = 16; p->W = 2; p->slots = backward ? 1 : 2; }
  else if (m <= SINK_MAX_COLS) { p->V = 16; p->W = 4; p->slots = 1; }
  else return fail(OG_EUNSUPPORTED, "%s: m = %d > %d columns not supported (swap the images)", who, m, SINK_MAX_COLS);
  p->mpad = (int)align_up(m + 1, 4);
  p->smem = sinkhorn_smem(backward, p->V, p->W, p->slots, p->mpad);
  p->occ = (p->V <= 8 && 2 * (p->smem + 1024) <= OG_SMEM_OPTIN_MAX) ? 2 : 1;
  // strips per pair / pairs per cooperative launch for p->occ co-resident CTAs per SM
  const int sms = device_info().ok ? device_info().sm_count : 132;
  const int ctas = sms * p->occ;                       // co-resident CTAs of the cooperative launch
  p->pairs_per_launch = std::min(B < ctas ? B : ctas, (int)(SINK_BARRIER_BYTES / 128));
  int sp = std::min(ctas / p->pairs_per_launch, SINK_MAX_STRIPS);
  const int max_sp = cdiv(n + 1, SINK_WARPS / p->W);
  if (sp > max_sp) sp = max_sp;
  if (sp < 1) sp = 1;
  p->SP = sp;
  p->rows_per_strip = cdiv(n + 1, sp);
  return OG_OK;
}

// Dynamic shared memory of a resident CTA: v [MC + 4], the folded column sums [G/2][mpad], the column groups' sums [256] float4,
// the held rows [max(rows_smem, 1)][SINK_WARPS][C] (the last slot is the first sweep's row ring), the mbarriers, the row exchanges
// of one and of two rows, the dustbin column's sums [G] and 128 bytes.
constexpr size_t sinkhorn_resident_smem(int V, int W, int mpad, int rows_smem) {
  const int C = 128 * V, G = SINK_WARPS / W;
  return ((size_t)(W * C + 4) + (size_t)G / 2 * mpad + 4 * SINK_WARPS * 32 + (size_t)SINK_WARPS * std::max(rows_smem, 1) * C) *
             sizeof(float) +
         SINK_WARPS * sizeof(uint64_t) + (size_t)2 * G * W * (sizeof(float2) + sizeof(float4)) + G * sizeof(float) + 128;
}

// The resident plan, where it fits and pays: the bands up to 2048 columns (V <= 8; RR = 16 / V rows per warp in registers, 64
// registers per thread, which leaves room for the second row a warp works on; even, so that rows pair up within registers), as
// many rows per warp in shared memory as the opt-in limit leaves, at most one CTA per SM, a pair on at most half the SMs.  The
// pairs are spread evenly over the launches and each pair of a launch over as many SMs as the launch leaves it.  One launch
// always pays: the streaming kernel leaves most SMs idle there.  Over several launches the resident kernel is taken only where
// its modelled sweep time, over all launches, beats the streaming kernel's 2.7 TB/s.  Both rates were measured on an H100 80GB
// HBM3 (700 W) with og_sinkhorn_fwd, the sweep model with the kernel sweeping one row at a time: about 3.8 us (exchanges) +
// R (0.4 + 0.0625 V) us for R rows per warp (8 rows of 2048 columns: 11.0 us; 17 rows of 1024: 14.0 us).  Two rows at a time
// the sweep takes less (8 rows of 2048 columns: 9.6 us), so the model errs towards streaming: 16 pairs of 2048 x 2048 (eight
// launches) run resident, 7.8 ms against 9.9 ms streaming, while 32 pairs of 1024 x 1024 (four launches) stream.  Returns false
// where the streaming kernel runs instead.
inline bool sinkhorn_resident_plan(int B, int n, int m, SinkPlan* p) {
  if (m > 2048 || sinkhorn_plan(false, B, n, m, p) != OG_OK) return false;
  const int G = SINK_WARPS / p->W, rr = 16 / p->V, C = 128 * p->V;
  const int sms = device_info().ok ? device_info().sm_count : 132;
  const int rs_max = 1 + (int)((OG_SMEM_OPTIN_MAX - sinkhorn_resident_smem(p->V, p->W, p->mpad, 1)) / (SINK_WARPS * C * sizeof(float)));
  const int sp_min = cdiv(n + 1, G * (rr + rs_max));  // strips a pair needs
  if (2 * sp_min > sms) return false;
  const int rounds = cdiv(B, std::min(B, sms / sp_min));
  p->pairs_per_launch = cdiv(B, rounds);
  const int sp = std::min(sms / p->pairs_per_launch, cdiv(n + 1, G));
  p->rows_per_strip = cdiv(n + 1, sp);
  p->SP = cdiv(n + 1, p->rows_per_strip);
  const int rows_per_warp = cdiv(p->rows_per_strip, G);
  const double resident_us = rounds * (3.8 + rows_per_warp * (0.4 + 0.0625 * p->V));
  const double streaming_us = 4.0 * B * (n + 1) * (m + 1) / 2.7e6;
  if (rounds > 1 && resident_us >= streaming_us) return false;
  p->rows_reg = rr;
  p->rows_smem = std::max(0, rows_per_warp - rr);
  p->smem = sinkhorn_resident_smem(p->V, p->W, p->mpad, p->rows_smem);
  p->slots = 1; p->occ = 1; p->resident = true;
  return true;
}

// OG_SINK_RESIDENT=0 runs every forward Sinkhorn on the streaming kernel; 1 (default): the resident kernel where its plan fits.
inline int& sink_resident_mode() {
  static int v = [] { const char* e = getenv("OG_SINK_RESIDENT"); return e ? (atoi(e) != 0) : 1; }();
  return v;
}

inline int sinkhorn_check_rows(const char* who, const float* S, int64_t lds, int64_t strideS, int m) {
  if (lds % 4 != 0 || lds < m || !aligned16(S) || strideS % 4 != 0)
    return fail(OG_EINVAL, "%s: S rows must be 16-byte aligned (lds %% 4 == 0, lds >= m)", who);
  return OG_OK;
}

// host-side constants exactly as the reference builds them (float32 throughout)
struct SinkConsts { float norm, log_a_last, log_b_last; };
inline SinkConsts sinkhorn_consts(int n, int m) {
  const float norm = -logf((float)(n + m));
  return {norm, norm + (float)log((double)m),        // log_a[-1] += math.log(n_cols)
          norm + (float)log((double)n)};             // log_b[-1] += math.log(n_rows)
}

// One cooperative launch of Kernel = <pass kernel><V, W, SLOTS> over a.B pairs.
template <auto Kernel, int V, int W, int SLOTS, class Args>
inline int sinkhorn_coop_launch(const Args& a, const SinkPlan& p, cudaStream_t stream) {
  constexpr size_t smem_max = sinkhorn_smem(Args::kBackward, V, W, SLOTS, 128 * V * W + 4);   // largest request: m = 128 V W
  static_assert(smem_max <= OG_SMEM_OPTIN_MAX, "Sinkhorn kernel: shared memory beyond what one block may opt in to");
  if (const int rc = smem_opt_in<Kernel>((int)smem_max)) return rc;
  return launch(Args::kBackward ? "sinkhorn_bwd_kernel" : "sinkhorn_kernel", Kernel, LaunchAttr::cooperative, dim3(a.B * a.SP),
                dim3(SINK_WARPS * 32), p.smem, stream, a);
}

// Calls launch(b0, nb) for pairs [b0, b0 + nb): as many pairs per cooperative launch as the plan allows, each launch with the
// barrier counters of its pairs zeroed.
template <class Launch>
inline int sinkhorn_for_each_launch(const SinkPlan& p, int B, unsigned int* barrier, cudaStream_t stream, Launch&& launch) {
  for (int b0 = 0; b0 < B; b0 += p.pairs_per_launch) {
    const int nb = std::min(p.pairs_per_launch, B - b0);
    OG_CUDA(cudaMemsetAsync(barrier, 0, (size_t)nb * 128, stream));
    if (const int rc = launch(b0, nb)) return rc;
  }
  return OG_OK;
}

// The larger of the two kernels' needs, whichever the switch selects: rows of mpad floats after the barriers and u are the strip
// partials [2][B][SINK_MAX_STRIPS] (streaming) or, as 64-bit words, [pairs_per_launch][SP] and then vglob [pairs_per_launch]
// (resident).
inline int64_t sinkhorn_workspace_bytes(int B, int n, int m) {
  SinkPlan p, r;
  if (sinkhorn_plan(false, B, n, m, &p) != OG_OK) return -1;
  int64_t rows = 2LL * B * SINK_MAX_STRIPS;
  if (sinkhorn_resident_plan(B, n, m, &r)) rows = std::max<int64_t>(rows, 2LL * (r.SP + 1) * r.pairs_per_launch);
  return SINK_BARRIER_BYTES + align_up((int64_t)B * (n + 1) * 4, 256) + align_up(rows * p.mpad * 4, 256);
}

// The tables SinkPair reads in a padded batch, from the host's own logf / log (bit for bit what sinkhorn_consts computes), copied to the
// current device at its first padded Sinkhorn.  That copy is synchronous, so it cannot be part of a stream capture: a capture
// needs one padded call on the device before it.
inline int sinkhorn_log_tables(cudaStream_t stream) {
  static bool done[OG_MAX_DEVICES] = {};
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  bool& d = done[current_device()];
  if (d) return OG_OK;
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  OG_CUDA(cudaStreamIsCapturing(stream, &cap));
  if (cap != cudaStreamCaptureStatusNone)
    return fail(OG_EUNSUPPORTED, "sinkhorn (padded): the first padded call on a device uploads its tables and cannot be captured; "
                                 "run one padded call before the capture");
  static std::vector<float> lf, l;
  if (lf.empty()) {
    lf.resize(SINK_MAX_ROWS + SINK_MAX_COLS + 1); l.resize(SINK_MAX_ROWS + 1);
    for (size_t k = 0; k < lf.size(); ++k) lf[k] = logf((float)k);
    for (size_t k = 0; k < l.size(); ++k) l[k] = (float)log((double)k);
  }
  OG_CUDA(cudaMemcpyToSymbol(og_sink_logf_tab, lf.data(), lf.size() * sizeof(float)));
  OG_CUDA(cudaMemcpyToSymbol(og_sink_log_tab, l.data(), l.size() * sizeof(float)));
  d = true;
  return OG_OK;
}

template <int V, int W>
inline int sinkhorn_resident_launch(const SinkArgs& a, const SinkPlan& p, cudaStream_t stream) {
  constexpr auto kernel = sinkhorn_resident_kernel<V, W, 16 / V>;
  if (const int rc = smem_opt_in<kernel>((int)OG_SMEM_OPTIN_MAX)) return rc;
  return launch("sinkhorn_resident_kernel", kernel, LaunchAttr::cooperative, dim3(a.B * a.SP), dim3(SINK_WARPS * 32), p.smem,
                stream, a);
}

inline int sinkhorn_kernel_launch(const SinkArgs& a, const SinkPlan& p, cudaStream_t stream) {
  if (p.resident) {
    if (p.W == 1) return sinkhorn_resident_launch<4, 1>(a, p, stream);
    return p.V == 4 ? sinkhorn_resident_launch<4, 2>(a, p, stream) : sinkhorn_resident_launch<8, 2>(a, p, stream);
  }
  if (p.V == 4 && p.W == 1) return sinkhorn_coop_launch<sinkhorn_kernel<4, 1, 2>, 4, 1, 2>(a, p, stream);
  if (p.V == 4)             return sinkhorn_coop_launch<sinkhorn_kernel<4, 2, 2>, 4, 2, 2>(a, p, stream);
  if (p.V == 8)             return sinkhorn_coop_launch<sinkhorn_kernel<8, 2, 2>, 8, 2, 2>(a, p, stream);
  if (p.W == 2)             return sinkhorn_coop_launch<sinkhorn_kernel<16, 2, 2>, 16, 2, 2>(a, p, stream);
  return sinkhorn_coop_launch<sinkhorn_kernel<16, 4, 1>, 16, 4, 1>(a, p, stream);
}

// lens (padded batch, device): n_0 .. n_{B-1}, then m_0 .. m_{B-1}; n, m are the capacity and the plan is the capacity's.
inline int sinkhorn_launch(const float* S, int64_t lds, int64_t strideS, const float* dustbin, int B, int n, int m,
                           int iters, float reg, float* scores, void* ws, int64_t ws_bytes, cudaStream_t stream,
                           float* hist_u = nullptr, float* hist_v = nullptr, const int* lens = nullptr) {
  if (lens && n > SINK_MAX_ROWS) return fail(OG_EUNSUPPORTED, "sinkhorn: a padded batch has at most %d rows, not %d", SINK_MAX_ROWS, n);
  if (lens)
    if (const int rc = sinkhorn_log_tables(stream)) return rc;
  SinkPlan p;
  const bool resident = !hist_u && !hist_v && sink_resident_mode() && sinkhorn_resident_plan(B, n, m, &p);
  if (!resident) {
    if (const int rc = sinkhorn_plan(false, B, n, m, &p)) return rc;
    p.resident = false;
  }
  if (ws_bytes < sinkhorn_workspace_bytes(B, n, m)) return fail(OG_EWORKSPACE, "sinkhorn: workspace too small");
  if (const int rc = sinkhorn_check_rows("sinkhorn", S, lds, strideS, m)) return rc;
  char* w = static_cast<char*>(ws);
  unsigned int* barrier = reinterpret_cast<unsigned int*>(w); w += SINK_BARRIER_BYTES;
  float* u = reinterpret_cast<float*>(w); w += align_up((int64_t)B * (n + 1) * 4, 256);
  float* partial = reinterpret_cast<float*>(w);
  const SinkConsts k = sinkhorn_consts(n, m);
  if (hist_v) OG_CUDA(cudaMemsetAsync(hist_v, 0, (size_t)B * (iters + 1) * (m + 1) * sizeof(float), stream));   // row 0 of every pair = v_0 = 0
  return sinkhorn_for_each_launch(p, B, barrier, stream, [&](int b0, int nb) {
    SinkArgs a;
    a.S = S + (int64_t)b0 * strideS; a.lds = lds; a.strideS = strideS; a.dustbin = dustbin;
    a.B = nb; a.n = n; a.m = m; a.iters = iters; a.reg = reg;
    a.norm = k.norm; a.log_a_last = k.log_a_last; a.log_b_last = k.log_b_last;
    a.scores = scores + (int64_t)b0 * (n + 1) * (m + 1);
    a.u = u; a.partial = partial; a.barrier = barrier;
    a.SP = p.SP; a.rows_per_strip = p.rows_per_strip; a.mpad = p.mpad;
    a.rows_smem = p.resident ? p.rows_smem : 0;
    a.vglob = partial + 2LL * p.pairs_per_launch * p.SP * p.mpad;
    if (p.resident) OG_CUDA(cudaMemsetAsync(partial, 0, 8LL * (p.SP + 1) * p.pairs_per_launch * p.mpad, stream));
    a.hist_u = hist_u ? hist_u + (int64_t)b0 * iters * (n + 1) : nullptr;
    a.hist_v = hist_v ? hist_v + (int64_t)b0 * (iters + 1) * (m + 1) : nullptr;
    a.len_n = lens ? lens + b0 : nullptr;
    a.len_m = lens ? lens + B + b0 : nullptr;
    return sinkhorn_kernel_launch(a, p, stream);
  });
}

}  // namespace og
