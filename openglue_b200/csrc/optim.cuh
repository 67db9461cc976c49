// The optimiser step of the reference's training loop (train.py / train_cached.py / pretrain_homography.py under Lightning):
//   clip_grad_norm_(params, max_norm) -> Adam.step() -> StepLR(step_size=1, gamma).step()
// with torch's foreach (non-capturable) Adam arithmetic, every scalar derived on the device so the step has no host sync.
//
// Two kernels over a table of parameter segments (og_optim_segment), each cut into OPT_TILE-element tiles numbered across
// the table (segment s owns tiles tile0 .. tile0 + cdiv(numel, OPT_TILE) - 1):
//   optim_norm_kernel    fixed grid of OPT_NORM_CTAS CTAs; CTA c sums g^2 in fp64 over tiles c, c + OPT_NORM_CTAS, ...; the last
//                        CTA to finish sums the partials in CTA order (deterministic, no float atomics), writes the norm and the
//                        clip coefficient to the state block, advances every segment's step count and derives its Adam scalars;
//   optim_update_kernel  launched with PDL after it: one fused pass per element (clip, m, v, p), then lr <- lr * gamma.
// A nullable `skip` (int32 on the device, og_clip_adam_step_guarded) skips the step when it reads non-zero: the norm kernel writes
// nothing, the update kernel only zeroes the gradients (parameters, moments, step counts, lr and sched_steps keep their bits).
// A null `skip` or *skip == 0 is the step above, bit for bit.
// HBM-bound: the norm reads 4 B per parameter, the update reads p, g, m, v and writes p, m, v (and g where clipping changes it).
#pragma once
#include "common.cuh"
#include "tc_common.cuh"

namespace og {

constexpr int OPT_THREADS = 256;
constexpr int OPT_VEC_PER_THREAD = 2;                                   // float4 per thread per tile
constexpr int64_t OPT_TILE = OG_OPTIM_TILE;
static_assert(OPT_TILE == OPT_THREADS * OPT_VEC_PER_THREAD * 4, "tile = threads x float4 x vectors");
constexpr int OPT_NORM_CTAS = 264;                                      // fixed: the reduction order does not depend on the GPU

struct OptHyper {
  double beta1, beta2, eps, max_norm, lr_gamma;
};

// Workspace: fp64 partial sums [OPT_NORM_CTAS], then {step_size, bc2_sqrt} per segment.
inline int64_t optim_workspace_bytes(int nseg) { return (int64_t)OPT_NORM_CTAS * 8 + (int64_t)nseg * 8; }

// Index of the segment that owns global tile t (tile0 ascending).
__device__ __forceinline__ int optim_find_segment(const og_optim_segment* segs, int nseg, int64_t t) {
  int lo = 0, hi = nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (segs[mid].tile0 <= t) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// Adam's bias-correction scalars for a step count, as torch's non-capturable path computes them with Python floats
// (bc1 = 1 - beta1**step, bc2_sqrt = (1 - beta2**step)**0.5, step_size = -lr / bc1), rounded to fp32 once, as the foreach
// kernels receive them.
__device__ __forceinline__ float2 adam_scalars(float step, double lr, double beta1, double beta2) {
  const double s = (double)step;
  const double bc1 = __dsub_rn(1.0, pow(beta1, s));
  const double bc2 = __dsub_rn(1.0, pow(beta2, s));
  const double step_size = -__ddiv_rn(lr, bc1);
  return make_float2((float)step_size, (float)__dsqrt_rn(bc2));
}

// clip_grad_norm_: clip_coef = max_norm / (norm + 1e-6), evaluated as torch's Tensor.__rtruediv__ does (reciprocal, then
// multiply), clamped at 1 by torch.clamp(max=1) (a NaN stays NaN).
__device__ __forceinline__ float clip_coefficient(float norm, double max_norm) {
  const float c = __fmul_rn(__frcp_rn(__fadd_rn(norm, 1e-6f)), (float)max_norm);
  return isnan(c) ? c : fminf(c, 1.f);
}

__global__ void __launch_bounds__(OPT_THREADS) optim_norm_kernel(const og_optim_segment* __restrict__ segs, int nseg, int64_t ntiles,
                                                                 OptHyper h, og_optim_state* state, double* partial, float2* scal,
                                                                 const int* skip) {
  tc::launch_dependents();                                    // the update kernel's CTAs may become resident; they wait for us
  if (skip && *skip) return;                                  // a skipped step: no norm, no step count, the counter stays 0
  __shared__ double red[OPT_THREADS / 32];
  __shared__ bool last;
  double acc = 0.0;
  for (int64_t t = blockIdx.x; t < ntiles; t += OPT_NORM_CTAS) {
    const og_optim_segment& s = segs[optim_find_segment(segs, nseg, t)];
    const int64_t base = (t - s.tile0) * OPT_TILE;
    const int64_t n = s.numel;
    const float* g = s.grad;
    if (aligned16(g)) {
#pragma unroll
      for (int k = 0; k < OPT_VEC_PER_THREAD; ++k) {
        const int64_t i = base + (int64_t)(k * OPT_THREADS + threadIdx.x) * 4;
        if (i + 4 <= n) {
          const float4 x = __ldg(reinterpret_cast<const float4*>(g + i));
          acc += (double)x.x * x.x; acc += (double)x.y * x.y; acc += (double)x.z * x.z; acc += (double)x.w * x.w;
        } else {
          for (int64_t j = i; j < n; ++j) { const double x = g[j]; acc += x * x; }
        }
      }
    } else {
      for (int k = 0; k < OPT_VEC_PER_THREAD * 4; ++k) {
        const int64_t i = base + (int64_t)k * OPT_THREADS + threadIdx.x;
        if (i < n) { const double x = g[i]; acc += x * x; }
      }
    }
  }
  const double tot = cta_sum<OPT_THREADS>(acc, red);
  if (threadIdx.x == 0) {
    partial[blockIdx.x] = tot;
    last = last_cta_arrive(&state->counter);
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  double p = 0.0;
  for (int c = threadIdx.x; c < OPT_NORM_CTAS; c += OPT_THREADS) p += __ldcg(partial + c);
  const double sumsq = cta_sum<OPT_THREADS>(p, red);
  if (threadIdx.x == 0) {
    const float norm = (float)sqrt(sumsq);
    state->grad_norm = norm;
    state->clip_coef = clip_coefficient(norm, h.max_norm);
    state->counter = 0;                                       // ready for the next call (and graph replay)
  }
  const double lr = state->lr;                                // the update kernel decays it after every CTA has read the scalars
  for (int i = threadIdx.x; i < nseg; i += OPT_THREADS) {
    float* sp = segs[i].step;
    const float step = __fadd_rn(*sp, 1.f);                   // torch: _foreach_add_(state_steps, 1) on fp32 step tensors
    *sp = step;
    scal[i] = adam_scalars(step, lr, h.beta1, h.beta2);
  }
}

// One element of clip -> Adam, with the rounding points of torch's foreach sequence (FMA contractions as its sm_90 kernels
// have them: lerp's small-weight branch m + w (g - m) and addcmul / addcdiv's a + s * x are single FFMAs).
struct AdamElt {
  float coef, w1, beta2, w2, eps, step_size, bc2_sqrt;
  __device__ __forceinline__ void operator()(float& p, float& g, float& m, float& v) const {
    g = __fmul_rn(g, coef);                                   // _foreach_mul_(grads, clip_coef_clamped)
    m = __fmaf_rn(__fsub_rn(g, m), w1, m);                    // _foreach_lerp_(exp_avgs, grads, 1 - beta1)
    v = __fmul_rn(v, beta2);                                  // _foreach_mul_(exp_avg_sqs, beta2)
    v = __fmaf_rn(__fmul_rn(g, g), w2, v);                    // _foreach_addcmul_(exp_avg_sqs, grads, grads, 1 - beta2)
    const float d = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2_sqrt), eps);   // sqrt, div_(bc2_sqrt), add_(eps)
    p = __fmaf_rn(__fdiv_rn(m, d), step_size, p);             // _foreach_addcdiv_(params, exp_avgs, denom, step_size)
  }
};

__global__ void __launch_bounds__(OPT_THREADS) optim_update_kernel(const og_optim_segment* __restrict__ segs, int nseg, int64_t ntiles,
                                                                   OptHyper h, og_optim_state* state, const float2* __restrict__ scal,
                                                                   const int* skip) {
  tc::grid_dependency_wait();                                 // the norm kernel has completed: coefficient, steps and scalars are final
  if (skip && *skip) {                                        // a skipped step leaves zero gradients and nothing else
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
      const og_optim_segment& s = segs[optim_find_segment(segs, nseg, t)];
      const int64_t base = (t - s.tile0) * OPT_TILE, end = min(base + OPT_TILE, s.numel);
      for (int64_t j = base + threadIdx.x; j < end; j += OPT_THREADS) s.grad[j] = 0.f;
    }
    return;
  }
  AdamElt op;
  op.coef = state->clip_coef;
  op.w1 = (float)(1.0 - h.beta1);
  op.beta2 = (float)h.beta2;
  op.w2 = (float)(1.0 - h.beta2);
  op.eps = (float)h.eps;
  const bool write_g = op.coef != 1.f;                        // g * 1 == g: the write-back would store the same bits
  for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int si = optim_find_segment(segs, nseg, t);
    const og_optim_segment& s = segs[si];
    const float2 sc = scal[si];
    op.step_size = sc.x; op.bc2_sqrt = sc.y;
    const int64_t base = (t - s.tile0) * OPT_TILE;
    const int64_t n = s.numel;
    float *P = s.param, *G = s.grad, *M = s.exp_avg, *V = s.exp_avg_sq;
    if (aligned16(P) && aligned16(G) && aligned16(M) && aligned16(V)) {
      float4 p[OPT_VEC_PER_THREAD], g[OPT_VEC_PER_THREAD], m[OPT_VEC_PER_THREAD], v[OPT_VEC_PER_THREAD];
      int64_t idx[OPT_VEC_PER_THREAD];
#pragma unroll
      for (int k = 0; k < OPT_VEC_PER_THREAD; ++k) {
        idx[k] = base + (int64_t)(k * OPT_THREADS + threadIdx.x) * 4;
        if (idx[k] + 4 <= n) {
          p[k] = *reinterpret_cast<const float4*>(P + idx[k]);
          g[k] = *reinterpret_cast<const float4*>(G + idx[k]);
          m[k] = *reinterpret_cast<const float4*>(M + idx[k]);
          v[k] = *reinterpret_cast<const float4*>(V + idx[k]);
        }
      }
#pragma unroll
      for (int k = 0; k < OPT_VEC_PER_THREAD; ++k) {
        if (idx[k] + 4 <= n) {
          op(p[k].x, g[k].x, m[k].x, v[k].x); op(p[k].y, g[k].y, m[k].y, v[k].y);
          op(p[k].z, g[k].z, m[k].z, v[k].z); op(p[k].w, g[k].w, m[k].w, v[k].w);
          *reinterpret_cast<float4*>(P + idx[k]) = p[k];
          *reinterpret_cast<float4*>(M + idx[k]) = m[k];
          *reinterpret_cast<float4*>(V + idx[k]) = v[k];
          if (write_g) *reinterpret_cast<float4*>(G + idx[k]) = g[k];
        } else {
          for (int64_t j = idx[k]; j < n; ++j) {
            float pj = P[j], gj = G[j], mj = M[j], vj = V[j];
            op(pj, gj, mj, vj);
            P[j] = pj; M[j] = mj; V[j] = vj;
            if (write_g) G[j] = gj;
          }
        }
      }
    } else {
      for (int k = 0; k < OPT_VEC_PER_THREAD * 4; ++k) {
        const int64_t j = base + (int64_t)k * OPT_THREADS + threadIdx.x;
        if (j < n) {
          float pj = P[j], gj = G[j], mj = M[j], vj = V[j];
          op(pj, gj, mj, vj);
          P[j] = pj; M[j] = mj; V[j] = vj;
          if (write_g) G[j] = gj;
        }
      }
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {                  // StepLR(step_size=1).step()
    state->lr = __dmul_rn(state->lr, h.lr_gamma);
    state->sched_steps += 1;
  }
}

inline unsigned optim_update_grid(int64_t ntiles) {
  const int sms = device_info().ok ? device_info().sm_count : 132;
  return (unsigned)std::min<int64_t>(ntiles, (int64_t)sms * 8);
}

inline int optim_step_launch(const og_optim_segment* segs, int nseg, int64_t ntiles, const OptHyper& h, og_optim_state* state,
                             void* ws, const int* skip, cudaStream_t stream) {
  double* partial = static_cast<double*>(ws);
  float2* scal = reinterpret_cast<float2*>(partial + OPT_NORM_CTAS);
  int rc = OG_LAUNCH(optim_norm_kernel, OPT_NORM_CTAS, OPT_THREADS, 0, stream, segs, nseg, ntiles, h, state, partial, scal, skip);
  if (rc != OG_OK) return rc;
  return launch("optim_update_kernel", optim_update_kernel, LaunchAttr::pdl, dim3(optim_update_grid(ntiles)), dim3(OPT_THREADS), 0,
                stream, segs, nseg, ntiles, h, state, (const float2*)scal, skip);
}

// Test path of the device-derived scalars: the lr schedule of steps 1 .. n (lr_out[k] = the lr step k + 1 uses, one thread,
// in order) and each step's fp32 {step_size, bc2_sqrt} from it, through the same functions as the fused step.
__global__ void adam_lr_chain_kernel(int64_t n, double lr, double gamma, double* lr_out) {
  for (int64_t k = 0; k < n; ++k) { lr_out[k] = lr; lr = __dmul_rn(lr, gamma); }
}
__global__ void adam_scalars_kernel(int64_t n, const double* lr_at, double beta1, double beta2, float* step_size, float* bc2_sqrt) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
    const float2 s = adam_scalars((float)(k + 1), lr_at[k], beta1, beta2);
    step_size[k] = s.x; bc2_sqrt[k] = s.y;
  }
}

}  // namespace og
