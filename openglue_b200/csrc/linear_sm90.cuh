// Hopper (sm_90a) tensor-core GEMM with fp32-grade accuracy from hi/lo operand pairs:
//     Y = epi(alpha * [A|A2] . B^T + bias),   A.B ~= A_lo.B_hi + A_hi.B_lo + A_hi.B_hi
// Two operand forms share one main loop:
//   3xTF32 (TcLinearArgs):  B_hi / B_lo are tf32-exact fp32 tensors; A is split into tf32 hi / lo in registers.
//   3xFP16 (F16LinearArgs): B_hi / B_lo are fp16 with a power-of-two weight scale sW (w_meta[0]); A is scaled on the fly by
//                           sA = f16_scale_for(max of the producers' amax slots) and split into fp16 hi / lo; alpha / (sA sW)
//                           undoes both scales exactly (see tc_common.cuh for the range argument).
// Persistent and warp-specialized: min(tiles, SMs) CTAs walk the 128 x 128 output tiles in a static schedule (tile = blockIdx.x +
// i gridDim.x over (batch item, row tile, column tile), column tile fastest, so the CTAs resident at one time share each A row
// block through L2).  Warpgroup 0 is the producer: it gives its registers back (setmaxnreg) and one thread stages, per K block
// (32 tf32 or 64 fp16 elements), the raw fp32 A tile and the B_hi / B_lo tiles (128-byte swizzled rows) by TMA into a ring of
// mbarrier-guarded stages, running ahead across tile boundaries so the next tile's first stages load during the epilogue.
// Warpgroups 1 and 2 own 64 rows of a tile each: a warp reads its A fragment out of shared memory and splits it into hi / lo
// registers, and the warpgroup issues wgmma with A from registers and B from shared memory.  The two consumers take turns to
// issue (a ping-pong over two named barriers), and each splits the A fragment of block kb + 1 while its wgmmas of block kb run,
// so the splits, folds and epilogues of one consumer run under the other's MMAs.  The wgmma accumulator holds at most CHUNK K
// blocks (K = 64 tf32 / 128 fp16) before it is folded into a register accumulator with round-to-nearest adds, so long
// reductions are not carried by the tensor core's own accumulation alone.
#pragma once
#include "tc_common.cuh"
#include <algorithm>
#include <type_traits>

namespace og {

struct TcLinearArgs {
  const float* A;  int64_t lda;  int64_t strideA;
  const float* A2; int64_t lda2; int64_t strideA2;
  int k1, k2;
  int b_rows_per_batch;                 // B tile row offset per batch item (0: B shared by the batch)
  const float* bias;
  int rows, nout, batch;
  float alpha;
  int relu;
  const float* R; int64_t ldr; int64_t strideR;
  const float* rscale;
  float* Y;   float* Yhi;  float* Ylo;  int64_t ldy;  int64_t strideY;     // row-major outputs (any may be null)
  float* Yt;  float* Ythi; float* Ytlo; int64_t ldyt; int64_t strideYt;    // transposed outputs [nout, rows]
};

// Output kinds of the fp16 form: F16_Y = fp32 Y [batch, rows, cols] (bias / ReLU / residual, amax tracking; Q in the forward
// pass), F16_K = row-major fp16 hi / lo [batch, rows, cols] (K operand of the attention kernel), F16_VT = transposed fp16 hi / lo
// [batch, cols, rows] (V^T operand).  The fp16 kinds' halves are written with a scale that the kernel publishes in their slot.
enum F16Kind { F16_Y, F16_K, F16_VT, F16_KINDS };
struct F16Out { float* y; __half *hi, *lo; int64_t ld, stride; float* scale; };   // y: F16_Y; hi, lo, scale: fp16 kinds

// A launch writes the run of kinds kind0 .. kind0 + nkinds - 1 from ONE product of A with B (with nkinds > 1: the stacked
// weights of several projections of the same A, Q | K | V or K | V).  The i-th kind of the run is output columns
// [i kind_cols, (i + 1) kind_cols), with its own weight scale / norm bound at w_meta + 4 i; the kind of a tile is
// kind0 + n0 / kind_cols.  A single output is nkinds = 1 with kind_cols = nout.
struct F16LinearArgs {
  const float* A;  int64_t lda;  int64_t strideA;
  const float* A2; int64_t lda2; int64_t strideA2;
  int k1, k2;
  int b_rows_per_batch;                 // B tile row offset per batch item (0: B shared by the batch)
  const float* bias;
  int rows, nout, batch;
  float alpha;
  int relu;
  const float* R; int64_t ldr; int64_t strideR;          // fp32 residual (F16_Y)
  F16Out out[F16_KINDS];                // indexed by kind; only the run's entries are read
  int kind0, nkinds, kind_cols;
  const float* amax_in[3];              // device scalars bounding |A| and |A2| (null entries ignored; at least one required)
  const float* w_meta;                  // device {scale of the pre-split B, max_n ||B_n||_1, max |bias|}
  float* amax_out;                      // optional: max |Y| (atomicMax; zeroed by the caller)
  int swap_halves;                      // debug: pack A with element 2c in the HIGH half (probe of the register operand layout)
};

namespace tcf {
constexpr int BM = 128, BN = 128, THREADS = 384;         // TMA producer warpgroup + two consumer warpgroups
template <bool F16> struct Cfg {
  static constexpr int KB = F16 ? 64 : 32;                // K elements per block: one 128-byte row of B
  static constexpr int A_BOXES = F16 ? 2 : 1;             // [128 rows x 32 fp32] TMA boxes of A per block
  static constexpr int A_BYTES = A_BOXES * BM * 128;
  static constexpr int B_TILE = BN * 128;                 // B_hi (or B_lo) part of a stage
  static constexpr int STAGE = A_BYTES + 2 * B_TILE;
  static constexpr int STAGES = F16 ? 3 : 4;              // 192 KB
  static constexpr int CHUNK = 2;                         // K blocks per wgmma accumulator chunk
  // fp16 form: an output staging buffer per consumer, one 64-row x 64-column half of its tile (fp32, or fp16 hi + lo)
  static constexpr int STAGING = F16 ? 64 * 64 * 4 : 0;
  static constexpr int SMEM_BYTES = 1024 + STAGES * STAGE + 2 * STAGING + 128;
  // The GEMMs and the attention kernel run in the 228 KB shared-memory configuration (cudaFuncAttributePreferredSharedMemory-
  // Carveout, set at launch): a neighbour in another configuration would make the SMs switch between kernels.
  static_assert(SMEM_BYTES <= OG_SMEM_OPTIN_MAX, "dynamic shared memory of one block");
};
constexpr int EPI = 3;                                    // named barriers EPI + consumer: one consumer's epilogue (ids 1, 2: TURN)
// output tile `tile` of the static schedule: column tile fastest, then row tile, then batch item
__host__ __device__ __forceinline__ void tile_origin(int tile, int tiles_n, int tiles_m, int& n0, int& m0, int& bz) {
  const int rt = tile / tiles_n;
  n0 = (tile - rt * tiles_n) * BN;
  bz = rt / tiles_m;
  m0 = (rt - bz * tiles_m) * BM;
}
}  // namespace tcf

// fp32 element (r, c) of a [rows x 32] fp32 tile written by TMA with the 128-byte swizzle
__device__ __forceinline__ const float* sw128_f32(const uint8_t* tile, int r, int c) {
  return reinterpret_cast<const float*>(tile + r * 128 + ((((c >> 2) ^ (r & 7))) << 4) + (c & 3) * 4);
}

// Output tensor maps of the fp16 form, one per output tensor of the run's kinds (box: 32 fp32 or 64 fp16 elements x 64 rows x 1,
// 128-byte swizzle; cols = kind_cols): hi[k] stores kind k's Y or hi halves, lo[k - 1] the lo halves of the fp16 kind k.
// tma = 0: the base, a stride or the row length of some output is not a multiple of 16 bytes, and the staged boxes are stored
// by the consumer's threads (out_copy_box).
struct OutMaps {
  CUtensorMap hi[F16_KINDS], lo[F16_KINDS - 1];
  int tma;
};

// byte offset of 16-byte chunk `chunk` of row `r` in a box of 128-byte rows written with the 128-byte swizzle
__device__ __forceinline__ int sw128_chunk(int r, int chunk) { return r * 128 + ((chunk ^ (r & 7)) << 4); }

// The box at `box` ([64 rows x 128 bytes], 128-byte swizzle) to T elements base[bz * bstride + (o0 + o) * ld + i0 + i] with
// o0 + o < olim and i0 + i < ilim, by the 128 threads of one consumer (tid).
template <class T>
__device__ __forceinline__ void out_copy_box(const uint8_t* box, T* base, int64_t ld, int64_t bstride, int bz, int i0, int o0, int ilim,
                                             int olim, int tid) {
  constexpr int NI = 128 / sizeof(T);
  for (int idx = tid; idx < 64 * NI; idx += 128) {
    const int o = idx / NI, i = idx - o * NI;
    if (o0 + o >= olim || i0 + i >= ilim) continue;
    const int b = i * (int)sizeof(T);
    base[(int64_t)bz * bstride + (int64_t)(o0 + o) * ld + i0 + i] =
        *reinterpret_cast<const T*>(box + sw128_chunk(o, b >> 4) + (b & 15));
  }
}

template <class Args>
__global__ void __launch_bounds__(tcf::THREADS, 1) linear_sm90_kernel(const __grid_constant__ CUtensorMap map_a,
                                                                      const __grid_constant__ CUtensorMap map_a2,
                                                                      const __grid_constant__ CUtensorMap map_bhi,
                                                                      const __grid_constant__ CUtensorMap map_blo,
                                                                      const __grid_constant__ OutMaps om, Args a) {
  using namespace tcf;
  using namespace tc;
  constexpr bool F16 = std::is_same<Args, F16LinearArgs>::value;
  using C = Cfg<F16>;
  constexpr int S = C::STAGES;
  constexpr int TURN = 1;                                    // named barriers TURN + consumer
  launch_dependents();
  extern __shared__ uint8_t og_lin_smem_raw[];
  uint8_t* smem = align_smem_1024(og_lin_smem_raw);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + S * C::STAGE + 2 * C::STAGING);
  uint64_t* empty = full + S;
  volatile uint32_t* timeout_flag = reinterpret_cast<uint32_t*>(empty + S);   // a consumer's wait on `full` timed out

  const int K = a.k1 + a.k2, nkb = cdiv(K, C::KB);
  const int tiles_n = cdiv(a.nout, BN), tiles_m = cdiv(a.rows, BM), ntiles = tiles_n * tiles_m * a.batch;
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    for (int i = 0; i < S; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }
    *timeout_flag = 0;
    fence_barrier_init();
    prefetch_tensormap(&map_a); prefetch_tensormap(&map_a2);
    prefetch_tensormap(&map_bhi); prefetch_tensormap(&map_blo);
    if constexpr (F16) {
#pragma unroll
      for (int k = 0; k < F16_KINDS; ++k)                   // the run's maps
        if (om.tma && k >= a.kind0 && k < a.kind0 + a.nkinds) { prefetch_tensormap(&om.hi[k]); if (k) prefetch_tensormap(&om.lo[k - 1]); }
    }
  }
  __syncthreads();
  grid_dependency_wait();                                    // A, the amax slots and the residual come from previous kernels

  if (wg == 0) {                                             // ---- producer
    setmaxnreg_dec<24>();
    if (threadIdx.x == 0) {
      uint32_t it = 0;                                       // K blocks staged so far (over all tiles of this CTA)
      for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        int n0, m0, bz;
        tile_origin(tile, tiles_n, tiles_m, n0, m0, bz);
        const int abz = a.strideA ? bz : 0, a2bz = a.strideA2 ? bz : 0;
        const int brow = n0 + bz * a.b_rows_per_batch;
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int s = it % S;
          if (it >= S) mbar_wait(&empty[s], (it / S - 1) & 1);
          uint8_t* st = smem + s * C::STAGE;
          mbar_arrive_expect_tx(&full[s], C::STAGE);         // out-of-bounds box parts arrive as zeros and count in full
#pragma unroll
          for (int j = 0; j < C::A_BOXES; ++j) {
            const int k = kb * C::KB + 32 * j;
            if (k < a.k1 || !a.A2) tma_load_3d(st + j * BM * 128, &map_a, &full[s], k, m0, abz);
            else                   tma_load_3d(st + j * BM * 128, &map_a2, &full[s], k - a.k1, m0, a2bz);
          }
          tma_load_2d(st + C::A_BYTES, &map_bhi, &full[s], kb * C::KB, brow);
          tma_load_2d(st + C::A_BYTES + C::B_TILE, &map_blo, &full[s], kb * C::KB, brow);
        }
      }
      mbar_wait(&empty[(it - 1) % S], ((it - 1) / S) & 1);   // both consumers are done with the last stage
      if (*timeout_flag) asm volatile("trap;");
    }
    return;
  }
  // ---- consumers.  Their waits on `full` are bounded without a trap (mbar_wait_flag): a trap anywhere after setmaxnreg.inc
  // makes ptxas allocate the whole kernel at its launch-bound register count, with spills and serialized wgmmas.  A timeout is
  // handed to the producer thread, which traps after the last release.
  setmaxnreg_inc<240>();
  const int c = wg - 1, tid = threadIdx.x & 127, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int r0 = c * 64 + warp * 16 + g;                     // tile rows of this thread: r0, r0 + 8

  // operand scales of the fp16 form (every thread derives the same values from the same device scalars)
  float s_a = 1.f, amax_a = 0.f;
  if constexpr (F16) {
#pragma unroll
    for (int i = 0; i < 3; ++i) if (a.amax_in[i]) amax_a = fmaxf(amax_a, __ldcg(a.amax_in[i]));
    s_a = f16_scale_for(amax_a);
    if (blockIdx.x == 0 && threadIdx.x == 128) {             // one thread of the grid publishes the fp16 kinds' output scales
#pragma unroll
      for (int k = F16_K; k < F16_KINDS; ++k) {
        if (k < a.kind0 || k >= a.kind0 + a.nkinds) continue;
        const float* wm = a.w_meta + 4 * (k - a.kind0);
        *a.out[k].scale = f16_out_scale_for(a.alpha, amax_a, __ldg(wm + 1), __ldg(wm + 2));
      }
    }
  }

  float racc[64], acc[64];
  uint32_t ahi0[4][4], alo0[4][4], ahi1[4][4], alo1[4][4];  // A fragments of two K blocks: split one while the other's wgmmas run
  uint32_t it = 0, timed_out = 0;

  // waits for stage `it_` and splits this warp's A fragment of it
  auto split_a = [&](uint32_t it_, uint32_t (&ahi)[4][4], uint32_t (&alo)[4][4]) {
    const int s = it_ % S;
    mbar_wait_flag(&full[s], (it_ / S) & 1, timed_out);
    const uint8_t* st = smem + s * C::STAGE;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      if constexpr (F16) {
        const uint8_t* box = st + (kk >> 1) * BM * 128;
        const int col = (kk & 1) * 16 + 2 * t;
#pragma unroll
        for (int q = 0; q < 4; ++q) {                        // q: (row r0 | r0 + 8) x (column col | col + 8)
          const float2 v = *reinterpret_cast<const float2*>(sw128_f32(box, r0 + (q & 1) * 8, col + (q >> 1) * 8));
          split_f16x2(v.x * s_a, v.y * s_a, ahi[kk][q], alo[kk][q]);
          if (a.swap_halves) { ahi[kk][q] = __byte_perm(ahi[kk][q], 0, 0x1032); alo[kk][q] = __byte_perm(alo[kk][q], 0, 0x1032); }
        }
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) split_tf32(*sw128_f32(st, r0 + (q & 1) * 8, 8 * kk + t + (q >> 1) * 4), ahi[kk][q], alo[kk][q]);
      }
    }
  };

  // consumer 0 takes the first turn; consumer 1 skips its last hand-over, so both barriers end balanced
  if (c == 1) named_bar_arrive(TURN + 0, 256);
#pragma unroll 1
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    int n0, m0, bz;
    tile_origin(tile, tiles_n, tiles_m, n0, m0, bz);
    const bool last_tile = tile + (int)gridDim.x >= ntiles;
#pragma unroll
    for (int i = 0; i < 64; ++i) racc[i] = 0.f;

    // one K block in this consumer's turn: its wgmmas from (ahi, alo), then the split of the next block into (nhi, nlo)
    auto mma_block = [&](int kb, const uint32_t (&ahi)[4][4], const uint32_t (&alo)[4][4], uint32_t (&nhi)[4][4],
                         uint32_t (&nlo)[4][4]) {
      const int s = it % S;
      const bool last = last_tile && kb == nkb - 1;
      if (last && timed_out) *timeout_flag = 1;              // published before the turn barrier, which orders it before the last release
      const uint32_t bhi = smem_u32(smem + s * C::STAGE + C::A_BYTES), blo = bhi + C::B_TILE;
      named_bar_sync(TURN + c, 256);
      fence_operands(acc);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint64_t dhi = make_wgdesc_sw128(bhi + kk * 32), dlo = make_wgdesc_sw128(blo + kk * 32);
        const int acc0 = (kb % C::CHUNK != 0 || kk) ? 1 : 0;
        if constexpr (F16) {
          wgmma_f16_m64n128(acc, alo[kk], dhi, acc0);
          wgmma_f16_m64n128(acc, ahi[kk], dlo, 1);
          wgmma_f16_m64n128(acc, ahi[kk], dhi, 1);
        } else {
          wgmma_tf32_m64n128(acc, alo[kk], dhi, acc0);
          wgmma_tf32_m64n128(acc, ahi[kk], dlo, 1);
          wgmma_tf32_m64n128(acc, ahi[kk], dhi, 1);
        }
      }
      wgmma_commit();
      if (!(last && c == 1)) named_bar_arrive(TURN + (c ^ 1), 256);
      if (kb + 1 < nkb) split_a(it + 1, nhi, nlo);
      wgmma_wait<0>();
      fence_operands(acc);
      if (tid == 0) mbar_arrive(&empty[s]);                  // this warpgroup's reads of the stage are done
      if (kb % C::CHUNK == C::CHUNK - 1 || kb == nkb - 1) {
#pragma unroll
        for (int i = 0; i < 64; ++i) racc[i] += acc[i];
      }
      ++it;
    };
    split_a(it, ahi0, alo0);
#pragma unroll 1
    for (int kb = 0; kb < nkb; kb += 2) {
      mma_block(kb, ahi0, alo0, ahi1, alo1);
      if (kb + 1 < nkb) mma_block(kb + 1, ahi1, alo1, ahi0, alo0);
    }

    // ---- epilogue: thread holds rows r0 / r0 + 8, columns n0 + 8j + 2t (+1), j = 0..15.  fp16 form: each 64-column half of
    // the consumer's 64 x 128 outputs is computed into its staging buffer and stored from there by TMA, so the consumer goes on
    // to the next tile's MMAs while the copy engine writes the tile; before it writes the buffer again, it waits for the reads of
    // the previous stores.
    if constexpr (F16) {
      // the tile's place in the run (n0 / kind_cols without a division: n0 < nout <= 3 kind_cols), and its kind
      const int kidx = (n0 >= a.kind_cols) + (n0 >= 2 * a.kind_cols), kind = a.kind0 + kidx;
      const float* wm = a.w_meta + 4 * kidx;
      const float alpha_t = a.alpha / (s_a * __ldg(wm));
      const float sos = kind != F16_Y ? f16_out_scale_for(a.alpha, amax_a, __ldg(wm + 1), __ldg(wm + 2)) : 1.f;
      float tmax = 0.f;
      uint8_t* stg = smem + S * C::STAGE + c * C::STAGING;   // two boxes of 64 rows x 128 bytes
      const int rl = warp * 16 + g;                          // rows r0 / r0 + 8 within the consumer's 64
      // the outputs by constant indices: a run-time index into the parameters would copy them to local memory
      const F16Out &oy = a.out[F16_Y], &ok = a.out[F16_K], &ovt = a.out[F16_VT];
      const int orow = m0 + 64 * c, bzy = oy.stride ? bz : 0, bzk = ok.stride ? bz : 0, bzt = ovt.stride ? bz : 0, cols = a.kind_cols;
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const int oc = n0 - kidx * cols + 64 * hf;           // first column of this half in its output
        // the half's values are computed in registers first, so that the wait for the previous stores' reads overlaps them
        auto buffer_free = [&] {
          if (tid == 0) bulk_wait_read<0>();
          named_bar_sync(EPI + c, 128);
        };
        if (kind == F16_Y) {
          float2 yv[2][8];
          // Every load of the half is issued before its first store: the compiler may not move a load across a store to a
          // pointer that could alias it, and loads interleaved with the stores expose one memory latency per 8-column block.
          // R may be Y: the half's residual is read before any of it is stored.
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int grow = m0 + r0 + 8 * h;
            const float* rrow = a.R && grow < a.rows ? a.R + (int64_t)bz * a.strideR + (int64_t)grow * a.ldr : nullptr;
            const int jh = 8 * hf;
            // bias and residual of columns n0 + 8 (jh + i / 2) + 2t + (i % 2)
            float bv[16], rv[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              const int col = n0 + 8 * (jh + (i >> 1)) + 2 * t + (i & 1);
              const bool in = col < a.nout;
              bv[i] = a.bias && in ? __ldg(a.bias + col) : 0.f;
              rv[i] = rrow && in ? rrow[col] : 0.f;
            }
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int j = jh + jj;
              const int col = n0 + 8 * j + 2 * t;
              const bool two = col + 1 < a.nout;
              float y0 = fmaf(racc[4 * j + 2 * h], alpha_t, bv[2 * jj]);
              float y1 = two ? fmaf(racc[4 * j + 2 * h + 1], alpha_t, bv[2 * jj + 1]) : 0.f;
              if (a.relu) { y0 = fmaxf(y0, 0.f); y1 = fmaxf(y1, 0.f); }
              if (a.R) {
                y0 += rv[2 * jj];
                if (two) y1 += rv[2 * jj + 1];
              }
              if (grow < a.rows && col < a.nout) tmax = fmaxf(tmax, fmaxf(fabsf(y0), fabsf(y1)));
              yv[h][jj] = make_float2(y0, y1);
            }
          }
          buffer_free();
#pragma unroll
          for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)                     // box jj / 4 holds columns 32 (jj / 4) .. + 31 of the half
              *reinterpret_cast<float2*>(stg + (jj >> 2) * 8192 + sw128_chunk(rl + 8 * h, 2 * (jj & 3) + (t >> 1)) + (t & 1) * 8) = yv[h][jj];
          }
        } else {
          // fp16 hi / lo operands (box 0: hi, box 1: lo): every element is computed (also rows / columns past the tensor, which
          // are not stored), then written as 8 x 8 matrices (h, jj) by stmatrix, four per instruction
          uint32_t hv[2][8], lv[2][8];                         // [row r0 | r0 + 8][jj]: columns n0 + 8 (8 hf + jj) + 2t, +1
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = 8 * hf + jj;
            const int col = n0 + 8 * j + 2 * t;
            const bool two = col + 1 < a.nout;
            const float b0 = a.bias && col < a.nout ? __ldg(a.bias + col) : 0.f;
            const float b1 = a.bias && two ? __ldg(a.bias + col + 1) : 0.f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float y0 = fmaf(racc[4 * j + 2 * h], alpha_t, b0);
              float y1 = two ? fmaf(racc[4 * j + 2 * h + 1], alpha_t, b1) : 0.f;
              if (a.relu) { y0 = fmaxf(y0, 0.f); y1 = fmaxf(y1, 0.f); }
              split_f16x2(y0 * sos, y1 * sos, hv[h][jj], lv[h][jj]);
            }
          }
          buffer_free();
          const int m = lane >> 3, k = lane & 7;               // this lane addresses row k of matrix m: h = m % 2, jj = 2q + m / 2
          const uint32_t stg_u = smem_u32(stg);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const uint32_t rh[4] = {hv[0][2 * q], hv[1][2 * q], hv[0][2 * q + 1], hv[1][2 * q + 1]};
            const uint32_t rlo[4] = {lv[0][2 * q], lv[1][2 * q], lv[0][2 * q + 1], lv[1][2 * q + 1]};
            if (kind == F16_K) {                               // row: keypoint; 16-byte chunk: 8 columns
              const uint32_t ad = stg_u + sw128_chunk(warp * 16 + 8 * (m & 1) + k, 2 * q + (m >> 1));
              stmatrix_x4(ad, rh); stmatrix_x4(ad + 8192, rlo);
            } else {                                           // V^T, row: column (channel); 16-byte chunk: 8 keypoints
              const uint32_t ad = stg_u + sw128_chunk(8 * (2 * q + (m >> 1)) + k, 2 * warp + (m & 1));
              stmatrix_x4_trans(ad, rh); stmatrix_x4_trans(ad + 8192, rlo);
            }
          }
        }
        fence_proxy_async();
        named_bar_sync(EPI + c, 128);
        if (om.tma) {
          if (tid == 0) {
            if (kind == F16_Y) { tma_store_3d(&om.hi[F16_Y], stg, oc, orow, bzy); tma_store_3d(&om.hi[F16_Y], stg + 8192, oc + 32, orow, bzy); }
            else if (kind == F16_K) { tma_store_3d(&om.hi[F16_K], stg, oc, orow, bzk); tma_store_3d(&om.lo[0], stg + 8192, oc, orow, bzk); }
            else { tma_store_3d(&om.hi[F16_VT], stg, orow, oc, bzt); tma_store_3d(&om.lo[1], stg + 8192, orow, oc, bzt); }
            bulk_commit();
          }
        } else if (kind == F16_Y) {
          out_copy_box(stg, oy.y, oy.ld, oy.stride, bz, oc, orow, cols, a.rows, tid);
          out_copy_box(stg + 8192, oy.y, oy.ld, oy.stride, bz, oc + 32, orow, cols, a.rows, tid);
        } else if (kind == F16_K) {
          out_copy_box(stg, ok.hi, ok.ld, ok.stride, bz, oc, orow, cols, a.rows, tid);
          out_copy_box(stg + 8192, ok.lo, ok.ld, ok.stride, bz, oc, orow, cols, a.rows, tid);
        } else {
          out_copy_box(stg, ovt.hi, ovt.ld, ovt.stride, bz, orow, oc, a.rows, cols, tid);
          out_copy_box(stg + 8192, ovt.lo, ovt.ld, ovt.stride, bz, orow, oc, a.rows, cols, tid);
        }
      }
      if (kind == F16_Y && a.amax_out) {
        tmax = warp_max(tmax);
        if (lane == 0 && tmax > 0.f) atomic_amax(a.amax_out, tmax);
      }
    } else {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int grow = m0 + r0 + 8 * h;
        if (grow >= a.rows) continue;
        const float* rrow = a.R ? a.R + (int64_t)bz * a.strideR + (int64_t)grow * a.ldr : nullptr;
        const int64_t yoff = (int64_t)bz * a.strideY + (int64_t)grow * a.ldy;
        const int64_t ytoff = (int64_t)bz * a.strideYt + grow;
#pragma unroll
        for (int jh = 0; jh < 16; jh += 8) {
          // loads first, as in the fp16 form: bias, rscale and residual of columns n0 + 8 (jh + i / 2) + 2t + (i % 2)
          float bv[16], sv[16], rv[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const int col = n0 + 8 * (jh + (i >> 1)) + 2 * t + (i & 1);
            const bool in = col < a.nout;
            bv[i] = a.bias && in ? __ldg(a.bias + col) : 0.f;
            sv[i] = rrow && a.rscale && in ? __ldg(a.rscale + col) : 0.f;
            rv[i] = rrow && in ? rrow[col] : 0.f;
          }
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = jh + jj;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = n0 + 8 * j + 2 * t + e;
              if (col >= a.nout) continue;
              float v = racc[4 * j + 2 * h + e] * a.alpha;
              if (a.bias) v += bv[2 * jj + e];
              if (a.relu) v = fmaxf(v, 0.f);
              if (rrow) { const float r = rv[2 * jj + e]; v = a.rscale ? fmaf(sv[2 * jj + e], r, v) : (v + r); }
              uint32_t vh = 0, vl = 0;
              if (a.Yhi || a.Ythi) split_tf32(v, vh, vl);
              if (a.Y) a.Y[yoff + col] = v;
              if (a.Yhi) { a.Yhi[yoff + col] = __uint_as_float(vh); a.Ylo[yoff + col] = __uint_as_float(vl); }
              const int64_t o = ytoff + (int64_t)col * a.ldyt;
              if (a.Yt) a.Yt[o] = v;
              if (a.Ythi) { a.Ythi[o] = __uint_as_float(vh); a.Ytlo[o] = __uint_as_float(vl); }
            }
          }
        }
      }
    }
  }
  // the outputs' stores have read the staging buffers (which live as long as the CTA) and are complete before the CTA exits
  if constexpr (F16) { if (tid == 0) bulk_wait<0>(); }
}

template <class Args, class BT>
inline int linear_sm90_launch(const Args& a, const BT* Bhi, const BT* Blo, int64_t ldb, int64_t b_total_rows, cudaStream_t stream) {
  using namespace tcf;
  constexpr bool F16 = std::is_same<Args, F16LinearArgs>::value;
  using C = Cfg<F16>;
  const int K = a.k1 + a.k2;
  CUtensorMap ma, ma2, mh, ml;
  int rc;
  if ((rc = tc::make_tmap_3d(&ma, a.A, a.strideA ? a.batch : 1, a.rows, a.k1, a.lda, a.strideA, BM)) != OG_OK) return rc;
  if (a.A2) { if ((rc = tc::make_tmap_3d(&ma2, a.A2, a.strideA2 ? a.batch : 1, a.rows, a.k2, a.lda2, a.strideA2, BM)) != OG_OK) return rc; }
  else ma2 = ma;
  if ((rc = tc::make_tmap_2d(&mh, Bhi, (uint64_t)b_total_rows, (uint64_t)K, (uint64_t)ldb, BN)) != OG_OK) return rc;
  if ((rc = tc::make_tmap_2d(&ml, Blo, (uint64_t)b_total_rows, (uint64_t)K, (uint64_t)ldb, BN)) != OG_OK) return rc;
  OutMaps om;
  memset(&om, 0, sizeof(om));
  if constexpr (F16) {
    // TMA stores need 16-byte aligned outputs with strides in multiples of 16 bytes, and they clip a box at the end of a row only
    // to a multiple of 16 bytes (measured on H100: a row of 334 fp32 had two more elements written).  Any other layout is
    // stored by the threads.
    om.tma = 1;
    for (int k = a.kind0; k < a.kind0 + a.nkinds && om.tma; ++k) {
      const F16Out& o = a.out[k];
      const int rows = k == F16_VT ? a.kind_cols : a.rows, cols = k == F16_VT ? a.rows : a.kind_cols;
      const auto map = [&](CUtensorMap* m, const auto* p) {
        const int64_t esz = sizeof(*p);
        return aligned16(p) && o.ld * esz % 16 == 0 && (a.batch == 1 || o.stride * esz % 16 == 0) && cols * esz % 16 == 0 &&
               tc::make_tmap_3d(m, p, a.batch, rows, cols, o.ld, o.stride, 64) == OG_OK;
      };
      om.tma = k == F16_Y ? map(&om.hi[k], o.y) : map(&om.hi[k], o.hi) && map(&om.lo[k - 1], o.lo);
    }
  }
  if ((rc = smem_opt_in<linear_sm90_kernel<Args>>(C::SMEM_BYTES, true)) != OG_OK) return rc;
  const int tiles = cdiv(a.nout, BN) * cdiv(a.rows, BM) * a.batch;
  const int sms = device_info().ok ? device_info().sm_count : 132;
  // persistent: each CTA walks tiles blockIdx.x + i gridDim.x
  return launch("linear_sm90_kernel", linear_sm90_kernel<Args>, LaunchAttr::pdl, dim3(std::min(tiles, sms)), dim3(THREADS), C::SMEM_BYTES,
                stream, ma, ma2, mh, ml, om, a);
}
// The two operand forms, instantiated next to the template: where the kernels sit in the binary (and so a cuobjdump -sass
// comparison of two builds) does not depend on where the host code first launches them.
template int linear_sm90_launch(const TcLinearArgs&, const float*, const float*, int64_t, int64_t, cudaStream_t);
template int linear_sm90_launch(const F16LinearArgs&, const __half*, const __half*, int64_t, int64_t, cudaStream_t);

// Bhi/Blo: [b_total_rows, K] row-major fp32 (tf32-exact values), row stride ldb.  A concatenated second operand needs k1 % 32 == 0
// (a K block comes from one of the two tensors).
inline bool linear_sm90_eligible(const TcLinearArgs& a, const float* Bhi, const float* Blo, int64_t ldb) {
  const int K = a.k1 + a.k2;
  return K >= 32 && a.k1 % 4 == 0 && a.k2 % 4 == 0 && a.lda % 4 == 0 && a.strideA % 4 == 0 && aligned16(a.A) &&
         (!a.A2 || (a.k1 % 32 == 0 && a.lda2 % 4 == 0 && a.strideA2 % 4 == 0 && aligned16(a.A2))) && ldb % 4 == 0 && aligned16(Bhi) && aligned16(Blo);
}

inline bool linear_sm90_eligible(const F16LinearArgs& a, const __half* Bh, const __half* Bl, int64_t ldb) {
  const int K = a.k1 + a.k2;
  if (!(K >= 64 && a.k1 % 4 == 0 && a.k2 % 4 == 0 && a.lda % 4 == 0 && a.strideA % 4 == 0 && aligned16(a.A) && ldb % 8 == 0 && aligned16(Bh) && aligned16(Bl))) return false;
  if (a.A2 && (a.k1 % 32 != 0 || a.lda2 % 4 != 0 || a.strideA2 % 4 != 0 || !aligned16(a.A2))) return false;
  if (!a.w_meta || !(a.amax_in[0] || a.amax_in[1] || a.amax_in[2])) return false;
  if (a.nkinds < 1 || a.kind0 < 0 || a.kind0 + a.nkinds > F16_KINDS || a.nout != a.nkinds * a.kind_cols) return false;
  if (a.nkinds > 1 && (a.kind_cols % tcf::BN != 0 || a.relu)) return false;
  if (a.R && (a.kind0 != F16_Y || a.nkinds > 1)) return false;    // the residual belongs to Y
  for (int k = a.kind0; k < a.kind0 + a.nkinds; ++k) {
    const F16Out& o = a.out[k];
    if (k == F16_Y && !(o.y && o.ld % 2 == 0 && o.stride % 2 == 0 && aligned16(o.y))) return false;
    if (k == F16_K && !(o.hi && o.lo && o.ld % 2 == 0 && o.stride % 2 == 0 && aligned16(o.hi) && aligned16(o.lo))) return false;
    if (k != F16_Y && !(o.hi && o.lo && o.scale)) return false;
  }
  return true;
}

// ---------------------------------------------------------------------------------------------------------------------
// pack-time / set-up kernels
// elementwise x -> (hi, lo) tf32 split of a flat buffer (weights at pack time)
__global__ void __launch_bounds__(256) split_tf32_kernel(const float* __restrict__ src, float* __restrict__ hi,
                                                          float* __restrict__ lo, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    uint32_t h, l;
    tc::split_tf32(src[i], h, l);
    hi[i] = __uint_as_float(h); lo[i] = __uint_as_float(l);
  }
}
// amax of a flat fp32 buffer into a device slot (the GNN's input activations come out of the CUDA-core encoder layers)
__global__ void __launch_bounds__(256) amax_kernel(const float* __restrict__ x, int64_t n, float* __restrict__ slot) {
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(__ldg(x + i)));
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0 && m > 0.f) tc::atomic_amax(slot, m);
}
// weight tensor [rows, cols] (+ bias [rows]) -> meta = {scale, max_n ||W_n||_1, max |b|}; one warp per row, atomics on
// non-negative floats (order independent); meta must be zeroed first.  meta[0] temporarily holds amax(W).
__global__ void __launch_bounds__(256) weight_meta_kernel(const float* __restrict__ w, const float* __restrict__ bias, int rows, int cols,
                                                          float* __restrict__ meta) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  float mx = 0.f, l1 = 0.f;
  for (int c = lane; c < cols; c += 32) { const float v = fabsf(__ldg(w + (int64_t)row * cols + c)); mx = fmaxf(mx, v); l1 += v; }
  mx = warp_max(mx); l1 = warp_sum(l1);
  if (lane == 0) {
    tc::atomic_amax(meta, mx); tc::atomic_amax(meta + 1, l1 * 1.0001f);           // 1.0001: the sum itself is rounded
    if (bias) tc::atomic_amax(meta + 2, fabsf(__ldg(bias + row)));
  }
}
// x -> hi / lo halves with the tensor's scale (meta[0] holds amax(W) on entry; finish_meta_kernel then replaces it by the scale)
__global__ void __launch_bounds__(256) split_f16_kernel(const float* __restrict__ src, __half* __restrict__ hi, __half* __restrict__ lo,
                                                        int64_t n, const float* __restrict__ amax) {
  const float s = tc::f16_scale_for(__ldg(amax));
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const float x = src[i] * s;
    const __half h = __float2half_rn(x);
    hi[i] = h; lo[i] = __float2half_rn(x - __half2float(h));
  }
}
__global__ void finish_meta_kernel(float* meta) { meta[0] = tc::f16_scale_for(meta[0]); }

}  // namespace og
