// Hopper (sm_90a) fused multi-head softmax attention with fp32-grade accuracy from hi/lo operand pairs.
// Replaces softmax_attention (reference models/superglue/attention.py:8-19); the N x M probability tensor never leaves registers.
//
// One CTA = 128 queries of one (batch, head), two warpgroups of 64 query rows; key blocks of 128 (fp16) / 64 (tf32).  One thread
// stages the K_i hi/lo and V_i^T hi/lo tiles by TMA into a ring of mbarrier-guarded stages (128-byte swizzled rows) that both
// warpgroups read; in the fp16 form it is a separate producer warpgroup and the two consumer warpgroups ping-pong (below).
//   S_i  = Q . K_i^T      wgmma, A = Q hi/lo in registers (split once per CTA), B = K_i hi/lo tiles [keys x Dh] (K-major)
//   P_i  = exp(S_i scale - m_i)   in the accumulator registers (row max / sum over the four lanes that share a row)
//   O_i  = P_i . V_i      wgmma, A = P_i hi/lo in registers, B = V_i^T hi/lo tiles [Dh x keys] (K-major); fresh accumulator
//   acc  = acc * exp(m_{i-1} - m_i) + O_i      in registers, round-to-nearest
// Every contraction is three MMAs (lo.hi + hi.lo + hi.hi).  Two operand forms:
//   3xTF32: Q fp32, K / V^T tf32-exact hi/lo fp32 tensors (csrc/linear_sm90.cuh, TcLinearArgs split outputs); head_dim 32 or 64.
//   3xFP16: Q fp32 scaled by sQ = f16_scale_for(q_amax), K / V^T fp16 hi/lo written with the scales k_scale / v_scale; P is formed
//           as 2^14 exp(...) (its row maximum 2^14 keeps the hi/lo pair resolving 2^-39 of it); head_dim 64.
//
// Operand layouts in HBM:
//   Q        fp32  [rows, ldq]            keypoint-major, head h = columns [h*Dh, (h+1)*Dh)
//   K hi/lo        [batch*nk, ldk]        keypoint-major
//   Vt hi/lo       [batch*d, ldvt]        channel-major (the reference's own [B, d, M] layout)
#pragma once
#include "tc_common.cuh"
#include <math_constants.h>

namespace og {

struct TcAttnArgs {
  const float* q; int64_t ldq, strideq;        // strideq: floats between batch items
  float* out; int64_t ldo, strideo;
  int batch, nq, nk, num_heads, d;
  float scale;
  const int* klen;           // padded batch (device, may be null): keys of sequence b = klen[b] clamped into [1, nk]; the operands
                             // keep the capacity's layout (sequence b's keys from row b nk)
};

struct F16AttnScales {
  const float* q_amax;           // device: max |Q| (tracked by the projection GEMM)
  const float* k_scale;          // device: scale K hi/lo were written with
  const float* v_scale;          // device: scale V^T hi/lo were written with
  float* out_amax;               // optional: max |out| (atomicMax; zeroed by the caller)
  int swap_halves;               // debug probe of the packed register operand layout (must be 0)
};

namespace tca {
constexpr int BM = 128;
constexpr float LOG2E = 1.4426950408889634f;
constexpr float P_SHIFT = 14.f;                 // fp16 form: P is written as 2^14 p
template <int DH, bool F16> struct Cfg {
  static constexpr int ESZ = F16 ? 2 : 4;
  static constexpr int BOX = 128 / ESZ;                  // elements per 128-byte row of a TMA box
  static constexpr int BNK = F16 ? 128 : 64;             // keys per block
  static constexpr int THREADS = F16 ? 384 : 256;        // fp16: TMA producer warpgroup + two consumer warpgroups
  static constexpr int K_TILE = BNK * DH * ESZ;          // K_i hi (or lo): DH / BOX boxes of [BNK keys x 128 B]
  static constexpr int V_TILE = DH * BNK * ESZ;          // V_i^T hi (or lo): BNK / BOX boxes of [DH channels x 128 B]
  static constexpr int STAGE = 2 * K_TILE + 2 * V_TILE;
  static constexpr int STAGES = 3;
  static constexpr int SMEM_BYTES = 1024 + STAGES * STAGE + 128;
  // Runs in the 228 KB shared-memory configuration, as the GEMM kernels do (preferred carveout set at launch): a kernel in
  // another configuration makes the SMs switch between neighbours, which measured 5 % on the GEMMs of a step.
  static_assert(SMEM_BYTES <= OG_SMEM_OPTIN_MAX, "dynamic shared memory of one block");
};
}  // namespace tca

// B descriptor of K step kk of a [rows x (elements per K step * steps)] operand tile staged as boxes of 128-byte rows
template <int ROWS, int STEP_BYTES>
__device__ __forceinline__ uint64_t tile_desc(uint32_t tile, int kk) {
  const int byte = kk * STEP_BYTES;
  return tc::make_wgdesc_sw128(tile + (byte >> 7) * ROWS * 128 + (byte & 127));
}

// Issues the TMA loads of key block i into stage st (one thread): K_i hi/lo, then V_i^T hi/lo.  Key rows of the next batch
// item are masked by the consumers; rows and columns past the tensor are zero-filled.
template <int DH, bool F16>
__device__ __forceinline__ void attention_issue(uint8_t* st, uint64_t* full, const CUtensorMap* mkh, const CUtensorMap* mkl,
                                                const CUtensorMap* mvh, const CUtensorMap* mvl, const TcAttnArgs& a, int h, int b,
                                                int i) {
  using C = tca::Cfg<DH, F16>;
  tc::mbar_arrive_expect_tx(full, C::STAGE);
#pragma unroll
  for (int j = 0; j < DH / C::BOX; ++j) {
    tc::tma_load_2d(st + j * C::BNK * 128, mkh, full, h * DH + j * C::BOX, b * a.nk + i * C::BNK);
    tc::tma_load_2d(st + C::K_TILE + j * C::BNK * 128, mkl, full, h * DH + j * C::BOX, b * a.nk + i * C::BNK);
  }
#pragma unroll
  for (int j = 0; j < C::BNK / C::BOX; ++j) {
    tc::tma_load_2d(st + 2 * C::K_TILE + j * DH * 128, mvh, full, i * C::BNK + j * C::BOX, b * a.d + h * DH);
    tc::tma_load_2d(st + 2 * C::K_TILE + C::V_TILE + j * DH * 128, mvl, full, i * C::BNK + j * C::BOX, b * a.d + h * DH);
  }
}

// Online-softmax step over the two rows of this thread for one key block held in p (accumulator layout, NJ blocks of 8 keys:
// p[4j + 2hh + e] = row g + 8hh, key 8j + 2t + e): masks keys >= nk (the sequence's keys), returns the correction factors of the
// running sums.
template <int NJ, bool F16>
__device__ __forceinline__ void attention_softmax(float (&p)[4 * NJ], int k0, int t, int nk, float c1, float (&m_run)[2],
                                                  float (&mc_run)[2], float (&l_run)[2], float (&corr)[2]) {
  using namespace tca;
  if (k0 + 8 * NJ > nk) {                                    // k0: first key of the block
    const int kbase = k0 + 2 * t;
#pragma unroll
    for (int j = 0; j < NJ; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) if (kbase + 8 * j + (e & 1) >= nk) p[4 * j + e] = -CUDART_INF_F;
  }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float mx = -CUDART_INF_F;
#pragma unroll
    for (int j = 0; j < NJ; ++j) mx = fmaxf(mx, fmaxf(p[4 * j + 2 * hh], p[4 * j + 2 * hh + 1]));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    const float m_new = fmaxf(m_run[hh], mx);
    const float mc = F16 ? fmaf(m_new, c1, -P_SHIFT) : m_new * c1;
    corr[hh] = ex2_approx(mc_run[hh] - mc);
    float r = 0.f;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float& x = p[4 * j + 2 * hh + e];
        x = ex2_approx(fmaf(x, c1, -mc));
        r += x;
      }
    }
    l_run[hh] = fmaf(l_run[hh], corr[hh], r);
    m_run[hh] = m_new; mc_run[hh] = mc;
  }
}

// Normalises the running output of this thread's two rows (acc: accumulator layout over DH columns), stores it and returns
// max |out| of what it stored.
template <int DH>
__device__ __forceinline__ float attention_store(const float (&acc)[DH / 2], const float (&l_run)[2], float inv_sv, int qr, int t,
                                                 const TcAttnArgs& a, int h, int b) {
  float omax = 0.f;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float l = l_run[hh];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = inv_sv / l;
    const int row = qr + 8 * hh;
    if (row >= a.nq) continue;
    float* orow = a.out + (int64_t)b * a.strideo + (int64_t)row * a.ldo + h * DH;
#pragma unroll
    for (int j = 0; j < DH / 8; ++j) {
      const float2 v = make_float2(acc[4 * j + 2 * hh] * inv, acc[4 * j + 2 * hh + 1] * inv);
      *reinterpret_cast<float2*>(orow + 8 * j + 2 * t) = v;
      omax = fmaxf(omax, fmaxf(fabsf(v.x), fabsf(v.y)));
    }
  }
  return omax;
}

// ---- 3xFP16 form, warp-specialized.  Warpgroup 0 is the TMA producer: it gives registers back (setmaxnreg) and one thread
// fills a 3-deep ring of [128 keys] K / V^T hi/lo stages (64 KB each).  Warpgroups 1 and 2 own 64 query rows each and take
// 240 registers: the Q hi/lo fragments (split once), the 64 x 128 logits, the P hi/lo fragments and the two output
// accumulators.  (Q staged in shared memory instead needs the 228 KB shared-memory configuration; see Cfg.)  Per key block a
// consumer issues, in one turn of a ping-pong over two named barriers, S_i = Q.K_i^T (12 wgmma m64n128) and
// O_{i-1} = P_{i-1}.V_{i-1} (24 wgmma m64n64), then hands the turn to the other consumer, whose wgmmas keep the tensor pipe busy
// while this one waits for its own, folds O_{i-1} and runs the softmax of S_i and the split of P_i.  (Starting that softmax as soon as S_i is done, while
// O_{i-1} is still in the pipe, measured no faster on an H100.)  A stage is released by one thread per consumer once its P.V
// has completed; three stages, because two leave the consumers waiting for TMA.
template <int DH>
__device__ __forceinline__ void attention_f16_ws(const CUtensorMap* mkh, const CUtensorMap* mkl, const CUtensorMap* mvh,
                                                 const CUtensorMap* mvl, const TcAttnArgs& a, const F16AttnScales& sc,
                                                 uint8_t* smem) {
  using namespace tca;
  using namespace tc;
  using C = Cfg<DH, true>;
  constexpr int S = C::STAGES, BNK = C::BNK;
  constexpr int QK = DH / 16, PK = BNK / 16, NJ = BNK / 8;   // wgmmas (x3) per Q.K^T and per P.V; 8-key blocks of S
  constexpr int TURN = 1;                                     // named barriers TURN + consumer
  static_assert(DH * 2 == 128, "one 128-byte row per K row");
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + S * C::STAGE);
  uint64_t* empty = full + S;
  volatile uint32_t* timeout_flag = reinterpret_cast<uint32_t*>(empty + S);   // a consumer's wait on `full` timed out

  const int q0 = blockIdx.x * BM, h = blockIdx.y, b = blockIdx.z;
  const int nk = padded_length(a.klen, b, a.nk);      // the producer and both consumers run the same key blocks
  const int nblk = cdiv(nk, BNK);
  const int wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    for (int i = 0; i < S; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }
    *timeout_flag = 0;
    fence_barrier_init();
    prefetch_tensormap(mkh); prefetch_tensormap(mkl);
    prefetch_tensormap(mvh); prefetch_tensormap(mvl);
  }
  __syncthreads();
  grid_dependency_wait();

  if (wg == 0) {                                             // ---- producer
    setmaxnreg_dec<24>();
    if (threadIdx.x == 0) {
      for (int i = 0; i < nblk; ++i) {
        const int s = i % S;
        if (i >= S) mbar_wait(&empty[s], (i / S - 1) & 1);
        attention_issue<DH, true>(smem + s * C::STAGE, &full[s], mkh, mkl, mvh, mvl, a, h, b, i);
      }
      mbar_wait(&empty[(nblk - 1) % S], ((nblk - 1) / S) & 1);   // both consumers are done with the last stage
      if (*timeout_flag) asm volatile("trap;");
    }
    return;
  }
  setmaxnreg_inc<240>();                                     // ---- consumers
  const int c = wg - 1, tid = threadIdx.x & 127, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const float s_q = f16_scale_for(__ldcg(sc.q_amax));
  const float c1 = a.scale * LOG2E / (s_q * __ldcg(sc.k_scale));   // logits arrive multiplied by sQ sK
  const float inv_sv = 1.f / __ldcg(sc.v_scale);

  // Q fragments of this warp's rows r, r + 8 (the m64nNk16 A layout: e = (row r | r + 8) x (columns 2t | 2t + 8) of K step kk)
  const float* qb = a.q + (int64_t)b * a.strideq + h * DH;
  uint32_t qh[QK][4], ql[QK][4];
#pragma unroll
  for (int kk = 0; kk < QK; ++kk)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int grow = q0 + c * 64 + warp * 16 + g + (e & 1) * 8, col = kk * 16 + 2 * t + (e >> 1) * 8;
      const float2 v = grow < a.nq ? *reinterpret_cast<const float2*>(qb + (int64_t)grow * a.ldq + col) : make_float2(0.f, 0.f);
      split_f16x2(v.x * s_q, v.y * s_q, qh[kk][e], ql[kk][e]);
    }

  float acc[DH / 2], o[DH / 2], p[4 * NJ];
#pragma unroll
  for (int k = 0; k < DH / 2; ++k) acc[k] = 0.f;
  float m_run[2] = {-CUDART_INF_F, -CUDART_INF_F}, mc_run[2] = {-CUDART_INF_F, -CUDART_INF_F}, l_run[2] = {0.f, 0.f};
  float corr[2];
  uint32_t phi[PK][4], plo[PK][4];
  uint32_t timed_out = 0;

  auto issue_qk = [&](int s) {
    const uint32_t khi = smem_u32(smem + s * C::STAGE), klo = khi + C::K_TILE;
#pragma unroll
    for (int kk = 0; kk < QK; ++kk) {
      const uint64_t bh = tile_desc<BNK, 32>(khi, kk), bl = tile_desc<BNK, 32>(klo, kk);
      wgmma_f16_m64n128(p, ql[kk], bh, kk ? 1 : 0);
      wgmma_f16_m64n128(p, qh[kk], bl, 1);
      wgmma_f16_m64n128(p, qh[kk], bh, 1);
    }
  };
  auto issue_pv = [&](int s) {
    const uint32_t vhi = smem_u32(smem + s * C::STAGE) + 2 * C::K_TILE, vlo = vhi + C::V_TILE;
#pragma unroll
    for (int kk = 0; kk < PK; ++kk) {
      const uint64_t dhi = tile_desc<DH, 32>(vhi, kk), dlo = tile_desc<DH, 32>(vlo, kk);
      wgmma_f16_m64n64(o, plo[kk], dhi, kk ? 1 : 0);
      wgmma_f16_m64n64(o, phi[kk], dlo, 1);
      wgmma_f16_m64n64(o, phi[kk], dhi, 1);
    }
  };
  auto split_p = [&]() {
#pragma unroll
    for (int kk = 0; kk < PK; ++kk)
#pragma unroll
      for (int e = 0; e < 4; ++e) {                          // keys 16kk + {0..7 | 8..15}: accumulator blocks 2kk, 2kk + 1
        const int base = 4 * (2 * kk + (e >> 1)) + 2 * (e & 1);
        split_f16x2(p[base], p[base + 1], phi[kk][e], plo[kk][e]);
        if (sc.swap_halves) { phi[kk][e] = __byte_perm(phi[kk][e], 0, 0x1032); plo[kk][e] = __byte_perm(plo[kk][e], 0, 0x1032); }
      }
  };
  auto release_and_fold = [&](int s) {                       // after the P.V group of stage s has completed
    if (tid == 0) mbar_arrive(&empty[s]);
#pragma unroll
    for (int k = 0; k < DH / 2; ++k) acc[k] = fmaf(acc[k], corr[(k >> 1) & 1], o[k]);
  };

  // consumer 0 takes the first turn; consumer 1 skips its last hand-over, so both barriers end balanced
  if (c == 1) named_bar_arrive(TURN + 0, 256);
  // key block 0: S_0 only
  mbar_wait_flag(&full[0], 0, timed_out);
  named_bar_sync(TURN + c, 256);
  fence_operands(p);
  wgmma_fence();
  issue_qk(0);
  wgmma_commit();
  named_bar_arrive(TURN + (c ^ 1), 256);
  wgmma_wait<0>();
  fence_operands(p);
  attention_softmax<NJ, true>(p, 0, t, nk, c1, m_run, mc_run, l_run, corr);
  split_p();

#pragma unroll 1
  for (int i = 1; i < nblk; ++i) {                           // S_i, then O_{i-1}
    const int s = i % S, sp = (i - 1) % S;
    mbar_wait_flag(&full[s], (i / S) & 1, timed_out);
    named_bar_sync(TURN + c, 256);
    fence_operands(p);
    fence_operands(o);
    wgmma_fence();
    issue_qk(s);
    issue_pv(sp);
    wgmma_commit();
    named_bar_arrive(TURN + (c ^ 1), 256);
    wgmma_wait<0>();
    fence_operands(p);
    fence_operands(o);
    release_and_fold(sp);
    attention_softmax<NJ, true>(p, i * BNK, t, nk, c1, m_run, mc_run, l_run, corr);
    split_p();
  }

  // last key block: O_{nblk-1} only.  A timeout is published before the turn barrier, which orders it before the last release.
  if (timed_out) *timeout_flag = 1;
  named_bar_sync(TURN + c, 256);
  fence_operands(o);
  wgmma_fence();
  issue_pv((nblk - 1) % S);
  wgmma_commit();
  if (c == 0) named_bar_arrive(TURN + 1, 256);
  wgmma_wait<0>();
  fence_operands(o);
  release_and_fold((nblk - 1) % S);

  float omax = attention_store<DH>(acc, l_run, inv_sv, q0 + c * 64 + warp * 16 + g, t, a, h, b);
  if (sc.out_amax) {
    omax = warp_max(omax);
    if (lane == 0 && omax > 0.f) atomic_amax(sc.out_amax, omax);
  }
}

// ---- 3xTF32 form: two warpgroups of 64 query rows, key blocks of 64.  Thread 0 stages the K / V^T hi/lo tiles; Q hi/lo stays in
// registers for the whole CTA; each warpgroup waits for its Q.K^T chain, runs the softmax, then issues and waits for P.V.
template <int DH>
__device__ __forceinline__ void attention_tf32(const CUtensorMap* mkh, const CUtensorMap* mkl, const CUtensorMap* mvh,
                                               const CUtensorMap* mvl, const TcAttnArgs& a, uint8_t* smem) {
  using namespace tca;
  using namespace tc;
  using C = Cfg<DH, false>;
  constexpr int S = C::STAGES, BNK = C::BNK;
  constexpr int QK = DH / 8;                                 // wgmmas (x3) per QK^T
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + S * C::STAGE);
  uint64_t* empty = full + S;

  const int q0 = blockIdx.x * BM, h = blockIdx.y, b = blockIdx.z;
  const int nk = padded_length(a.klen, b, a.nk);
  const int nblk = cdiv(nk, BNK);
  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  if (threadIdx.x == 0) {
    for (int i = 0; i < S; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
    fence_barrier_init();
    prefetch_tensormap(mkh); prefetch_tensormap(mkl);
    prefetch_tensormap(mvh); prefetch_tensormap(mvl);
  }
  __syncthreads();
  grid_dependency_wait();

  if (threadIdx.x == 0)
    for (int i = 0; i < S && i < nblk; ++i) attention_issue<DH, false>(smem + i * C::STAGE, &full[i], mkh, mkl, mvh, mvl, a, h, b, i);

  // ---- Q fragments (rows r, r + 8 of this warp's 16-row slice), split once
  const int qr = q0 + wg * 64 + warp * 16 + g;
  const float c1 = a.scale * LOG2E;
  const float* qb = a.q + (int64_t)b * a.strideq + h * DH;
  uint32_t qhi[QK][4], qlo[QK][4];
#pragma unroll
  for (int kk = 0; kk < QK; ++kk) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {                            // e: (row qr | qr + 8) x (column group 0 | 1)
      const int row = qr + (e & 1) * 8;
      const int col = kk * 8 + t + (e >> 1) * 4;
      split_tf32(row < a.nq ? qb[(int64_t)row * a.ldq + col] : 0.f, qhi[kk][e], qlo[kk][e]);
    }
  }

  float acc[DH / 2];
#pragma unroll
  for (int k = 0; k < DH / 2; ++k) acc[k] = 0.f;
  float m_run[2] = {-CUDART_INF_F, -CUDART_INF_F}, mc_run[2] = {-CUDART_INF_F, -CUDART_INF_F}, l_run[2] = {0.f, 0.f};

#pragma unroll 1
  for (int i = 0; i < nblk; ++i) {
    if (threadIdx.x == 0 && i >= 1 && i - 1 + S < nblk) {
      const int sr = (i - 1) % S;
      mbar_wait(&empty[sr], ((i - 1) / S) & 1);
      attention_issue<DH, false>(smem + sr * C::STAGE, &full[sr], mkh, mkl, mvh, mvl, a, h, b, i - 1 + S);
    }
    const int s = i % S;
    mbar_wait(&full[s], (i / S) & 1);
    const uint32_t st = smem_u32(smem + s * C::STAGE);
    const uint32_t khi = st, klo = st + C::K_TILE, vhi = st + 2 * C::K_TILE, vlo = vhi + C::V_TILE;

    // ---- S = Q K^T  (64 x 64 per warpgroup; p[4j + 2h + e] = row g + 8h, key 8j + 2t + e)
    float p[32];
    fence_operands(p);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < QK; ++kk) {
      const uint64_t dhi = tile_desc<BNK, 32>(khi, kk), dlo = tile_desc<BNK, 32>(klo, kk);
      wgmma_tf32_m64n64(p, qlo[kk], dhi, kk ? 1 : 0);
      wgmma_tf32_m64n64(p, qhi[kk], dlo, 1);
      wgmma_tf32_m64n64(p, qhi[kk], dhi, 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_operands(p);

    float corr[2];
    attention_softmax<8, false>(p, i * BNK, t, nk, c1, m_run, mc_run, l_run, corr);

    // ---- O_i = P V_i  (64 x DH per warpgroup)
    // the tf32 A fragment of keys 8j .. 8j+7 wants (row, key t) and (row, key t + 4); the accumulator holds keys 2t, 2t + 1:
    // fetch them from the lanes 4g + t/2 and 4g + 2 + t/2 of the same row quad
    float o[DH / 2];
    const int src0 = (lane & ~3) | (t >> 1), src1 = src0 + 2;
    const bool odd = t & 1;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      uint32_t phi[4][4], plo[4][4];
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int j = half * 4 + jj;
#pragma unroll
        for (int e = 0; e < 4; ++e) {                        // e: (row g | g + 8) x (key t | t + 4)
          const int reg = 4 * j + 2 * (e & 1), src = (e >> 1) ? src1 : src0;
          const float x0 = __shfl_sync(0xffffffffu, p[reg], src), x1 = __shfl_sync(0xffffffffu, p[reg + 1], src);
          split_tf32(odd ? x1 : x0, phi[jj][e], plo[jj][e]);
        }
      }
      fence_operands(o);
      wgmma_fence();
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int kk = half * 4 + jj;
        const uint64_t dhi = tile_desc<DH, 32>(vhi, kk), dlo = tile_desc<DH, 32>(vlo, kk);
        if constexpr (DH == 64) {
          wgmma_tf32_m64n64(o, plo[jj], dhi, kk ? 1 : 0);
          wgmma_tf32_m64n64(o, phi[jj], dlo, 1);
          wgmma_tf32_m64n64(o, phi[jj], dhi, 1);
        } else {
          wgmma_tf32_m64n32(o, plo[jj], dhi, kk ? 1 : 0);
          wgmma_tf32_m64n32(o, phi[jj], dlo, 1);
          wgmma_tf32_m64n32(o, phi[jj], dhi, 1);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_operands(o);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);                   // this warp's wgmmas have read the stage
#pragma unroll
    for (int k = 0; k < DH / 2; ++k) acc[k] = fmaf(acc[k], corr[(k >> 1) & 1], o[k]);
  }
  attention_store<DH>(acc, l_run, 1.f, qr, t, a, h, b);
}

template <int DH, bool F16>
__global__ void __launch_bounds__(tca::Cfg<DH, F16>::THREADS, 1) attention_sm90_kernel(const __grid_constant__ CUtensorMap map_khi,
                                                                                       const __grid_constant__ CUtensorMap map_klo,
                                                                                       const __grid_constant__ CUtensorMap map_vhi,
                                                                                       const __grid_constant__ CUtensorMap map_vlo,
                                                                                       TcAttnArgs a, F16AttnScales sc) {
  static_assert(DH == 64 || (DH == 32 && !F16), "head_dim 64 (both forms) or 32 (tf32)");
  tc::launch_dependents();
  extern __shared__ uint8_t og_att_smem_raw[];
  uint8_t* smem = tc::align_smem_1024(og_att_smem_raw);
  if constexpr (F16) attention_f16_ws<DH>(&map_khi, &map_klo, &map_vhi, &map_vlo, a, sc, smem);
  else attention_tf32<DH>(&map_khi, &map_klo, &map_vhi, &map_vlo, a, smem);
}

template <int DH, bool F16, class T>
inline int attention_sm90_launch(const TcAttnArgs& a, const F16AttnScales& sc, const T* khi, const T* klo, int64_t ldk,
                                 const T* vthi, const T* vtlo, int64_t ldvt, cudaStream_t stream) {
  using namespace tca;
  using C = Cfg<DH, F16>;
  CUtensorMap mkh, mkl, mvh, mvl;
  int rc;
  if ((rc = tc::make_tmap_2d(&mkh, khi, (uint64_t)a.batch * a.nk, (uint64_t)a.d, (uint64_t)ldk, C::BNK)) != OG_OK) return rc;
  if ((rc = tc::make_tmap_2d(&mkl, klo, (uint64_t)a.batch * a.nk, (uint64_t)a.d, (uint64_t)ldk, C::BNK)) != OG_OK) return rc;
  if ((rc = tc::make_tmap_2d(&mvh, vthi, (uint64_t)a.batch * a.d, (uint64_t)a.nk, (uint64_t)ldvt, DH)) != OG_OK) return rc;
  if ((rc = tc::make_tmap_2d(&mvl, vtlo, (uint64_t)a.batch * a.d, (uint64_t)a.nk, (uint64_t)ldvt, DH)) != OG_OK) return rc;
  if ((rc = smem_opt_in<attention_sm90_kernel<DH, F16>>(C::SMEM_BYTES, true)) != OG_OK) return rc;   // the GEMMs' configuration
  return launch("attention_sm90_kernel", attention_sm90_kernel<DH, F16>, LaunchAttr::pdl, dim3(cdiv(a.nq, BM), a.num_heads, a.batch),
                dim3(C::THREADS), C::SMEM_BYTES, stream, mkh, mkl, mvh, mvl, a, sc);
}

inline bool attention_tc_eligible(int head_dim, int64_t ldq, int64_t ldk, int64_t ldvt, int64_t ldo) {
  return (head_dim == 32 || head_dim == 64) && ldq % 2 == 0 && ldk % 4 == 0 && ldvt % 4 == 0 && ldo % 2 == 0;
}
// khi/klo: tf32 [batch*nk, ldk];  vthi/vtlo: tf32 [batch*d, ldvt]  (ld in floats, multiples of 4)
inline int attention_tc_launch(const TcAttnArgs& a, const float* khi, const float* klo, int64_t ldk, const float* vthi,
                               const float* vtlo, int64_t ldvt, int head_dim, cudaStream_t stream) {
  const F16AttnScales none{nullptr, nullptr, nullptr, nullptr, 0};
  if (head_dim == 64) return attention_sm90_launch<64, false>(a, none, khi, klo, ldk, vthi, vtlo, ldvt, stream);
  if (head_dim == 32) return attention_sm90_launch<32, false>(a, none, khi, klo, ldk, vthi, vtlo, ldvt, stream);
  return fail(OG_EUNSUPPORTED, "attention_tc: head_dim %d not in {32, 64}", head_dim);
}

inline bool attention_f16_eligible(int head_dim, int64_t ldq, int64_t ldk, int64_t ldvt, int64_t ldo) {
  return head_dim == 64 && ldq % 2 == 0 && ldk % 8 == 0 && ldvt % 8 == 0 && ldo % 2 == 0;
}
// khi/klo: fp16 [batch*nk, ldk];  vthi/vtlo: fp16 [batch*d, ldvt]  (ld in elements, multiples of 8)
inline int attention_f16_launch(const TcAttnArgs& a, const F16AttnScales& sc, const __half* khi, const __half* klo, int64_t ldk,
                                const __half* vthi, const __half* vtlo, int64_t ldvt, int head_dim, cudaStream_t stream) {
  if (head_dim != 64) return fail(OG_EUNSUPPORTED, "attention_f16: head_dim %d != 64", head_dim);
  if (!sc.q_amax || !sc.k_scale || !sc.v_scale) return fail(OG_EINVAL, "attention_f16: operand scales missing");
  return attention_sm90_launch<64, true>(a, sc, khi, klo, ldk, vthi, vtlo, ldvt, stream);
}

}  // namespace og
