// Shared helpers for the openglue_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <math_constants.h>
#include <limits.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <stdlib.h>
#include <utility>
#include "../../include/openglue_b200.h"

namespace og {

// thread-local error message (og_last_error)
inline char* err_buf() { static thread_local char buf[512] = {0}; return buf; }
inline int fail(int code, const char* fmt, ...) {
  va_list ap; va_start(ap, fmt); vsnprintf(err_buf(), 512, fmt, ap); va_end(ap);
  return code;
}
#define OG_CHECK_ARG(cond, ...) do { if (!(cond)) return og::fail(OG_EINVAL, __VA_ARGS__); } while (0)
#define OG_CUDA(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) \
  return og::fail(OG_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)

// Kernels this thread has enqueued through launch() (og_last_forward_launches); og_superglue_forward resets it when it starts.
inline int& launch_counter() { static thread_local int c = 0; return c; }

// OG_PDL=0 turns the programmatic dependent launches (LaunchAttr::pdl) into plain launches.
inline int& pdl_mode() {
  static int v = [] { const char* e = getenv("OG_PDL"); return e ? atoi(e) : 1; }();
  return v;
}

enum class LaunchAttr { none, pdl, cooperative };

// Enqueues kernel(args...) on `stream` over `grid` x `block` with `smem` bytes of dynamic shared memory and the launch attribute
// `attr`, and counts it in launch_counter().  Every kernel of the library is launched here.  A failed launch is reported as
// "launch of <name> failed" and its error is cleared, so that it does not surface later in an unrelated cudaGetLastError.
template <class... Params, class... Args>
inline int launch(const char* name, void (*kernel)(Params...), LaunchAttr attr, dim3 grid, dim3 block, size_t smem,
                  cudaStream_t stream, Args&&... args) {
  cudaLaunchAttribute at[1] = {};
  if (attr == LaunchAttr::pdl) {
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
  } else if (attr == LaunchAttr::cooperative) {
    at[0].id = cudaLaunchAttributeCooperative;
    at[0].val.cooperative = 1;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cfg.attrs = at;
  cfg.numAttrs = (attr == LaunchAttr::cooperative || (attr == LaunchAttr::pdl && pdl_mode())) ? 1 : 0;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    return fail(OG_ECUDA, "launch of %s failed: %s", name, cudaGetErrorString(e));
  }
  ++launch_counter();
  return OG_OK;
}
// launch() without an attribute, named after the kernel expression
#define OG_LAUNCH(kernel, ...) og::launch(#kernel, kernel, og::LaunchAttr::none, __VA_ARGS__)

// Per-device state (a process may drive several GPUs: MatchingCore(device=...), .to(dev)): the capability cache and the
// "function attribute already set" flags (smem_opt_in) are indexed by the CURRENT device, never process-global.
constexpr int OG_MAX_DEVICES = 64;
inline int current_device() { int dev = 0; if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= OG_MAX_DEVICES) dev = 0; return dev; }

struct DeviceInfo { int sm_count = 0, cc_major = 0, cc_minor = 0; bool ok = false, probed = false; };
inline const DeviceInfo& device_info() {
  static DeviceInfo info[OG_MAX_DEVICES];          // immutable once probed (a benign race writes identical values)
  const int dev = current_device();
  DeviceInfo& d = info[dev];
  if (!d.probed) {
    DeviceInfo t; t.probed = true;
    int real = 0;
    cudaDeviceProp p;
    if (cudaGetDevice(&real) == cudaSuccess && cudaGetDeviceProperties(&p, real) == cudaSuccess) {
      t.sm_count = p.multiProcessorCount; t.cc_major = p.major; t.cc_minor = p.minor; t.ok = true;
    }
    d = t;
  }
  return d;
}
// Dynamic shared memory one block may opt in to on sm_90 (cudaDevAttrMaxSharedMemoryPerBlockOptin: 227 KB of the SM's 228 KB)
constexpr size_t OG_SMEM_OPTIN_MAX = 227 * 1024;
// Opts Kernel in to `bytes` of dynamic shared memory, once per device.  The flag is keyed on the kernel itself (every template
// instantiation has its own) and set only after the call succeeded, so a failed opt-in is retried on the next launch.
// max_carveout: the kernel prefers the largest shared-memory configuration of the SM (228 KB on sm_90) even where it needs less,
// so that it does not switch the SMs' configuration against neighbours that need it.
template <auto Kernel>
inline int smem_opt_in(int bytes, bool max_carveout = false) {
  static bool done[OG_MAX_DEVICES] = {};
  bool& d = done[current_device()];
  if (!d) {
    OG_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    if (max_carveout) OG_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
    d = true;
  }
  return OG_OK;
}

__host__ __device__ inline int64_t align_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }
__host__ __device__ inline int cdiv(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// The length of sequence b of a batch with capacity cap: cap, or in a padded batch (len non-null) its own length len[b], clamped
// into [1, cap]
__device__ __forceinline__ int padded_length(const int* len, int b, int cap) {
  return len ? min(max(__ldg(len + b), 1), cap) : cap;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
template <class T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// Sum of v over a CTA of THREADS threads in a fixed order: a warp butterfly, then thread 0 adds the warp totals in warp order.
// Valid in thread 0.  red: shared, THREADS / 32 slots; the __syncthreads() before it is written lets consecutive calls reuse it.
template <int THREADS, class T>
__device__ __forceinline__ T cta_sum(T v, T* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  T t = 0;
  if (threadIdx.x == 0) for (int w = 0; w < THREADS / 32; ++w) t += red[w];
  return t;
}

// The last CTA of a grid finishes a reduction: every CTA stores its partial, then its thread 0 calls last_cta_arrive(), which
// fences that store device-wide before it arrives on `counter` and returns whether every other CTA has already arrived.  The
// last CTA fences again before any of its threads reads the partials; last_cta_sum() does both for one thread.  `counter`
// starts at 0; resetting it for the next launch is the caller's.
__device__ __forceinline__ bool last_cta_arrive(unsigned int* counter) {
  __threadfence();
  return atomicAdd(counter, 1u) == gridDim.x - 1;
}
// partial[0 .. n) summed in index order (deterministic), by one thread of the last CTA
template <class T>
__device__ __forceinline__ T last_cta_sum(const T* partial, int n) {
  __threadfence();
  T t = 0;
  for (int p = 0; p < n; ++p) t += __ldcg(partial + p);
  return t;
}

// The smallest power of two >= x (1 for x <= 1): the length of a bitonic sort of x keys
__host__ __device__ __forceinline__ int pow2_ceil(int x) {
  int n = 1;
  while (n < x) n <<= 1;
  return n;
}
// CTA-wide bitonic sort of positions [0, n2), n2 a power of two, into the order of before(lo, hi): "the element at position lo
// goes first".  swap(lo, hi) exchanges two positions.  Every thread of the CTA calls it; one __syncthreads() per stride.
// THREADS: the CTA's size where every launch uses that constant (the compiler then unrolls the loop), or 0: blockDim.x.
template <int THREADS = 0, class Before, class Swap>
__device__ __forceinline__ void cta_bitonic_sort(int n2, Before before, Swap swap) {
  for (int size = 2; size <= n2; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = threadIdx.x; t < (n2 >> 1); t += THREADS ? THREADS : blockDim.x) {
        const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
        if (before(lo, hi) != ((lo & size) == 0)) swap(lo, hi);
      }
      __syncthreads();
    }
}
// Top-k order (torch.topk, the reference's nms_keypoints): the higher score first, on equal scores the lower index
__device__ __forceinline__ bool topk_before(float a, int ia, float b, int ib) { return a > b || (a == b && ia < ib); }

// Shared-memory top-k sort of scores[0 .. cnt): key / val [pow2_ceil(cnt)] receive the scores and their indices in top-k order,
// padded with (-inf, INT_MAX).  Every thread of the CTA calls it; THREADS as for cta_bitonic_sort.  CTA_TOPK_MAX keys at most
// (cta_topk_smem).
constexpr int CTA_TOPK_MAX = 16384;
template <int THREADS>
__device__ __forceinline__ void cta_topk_sort(const float* scores, int cnt, float* key, int* val) {
  const int n2 = pow2_ceil(cnt);
  for (int j = threadIdx.x; j < n2; j += THREADS ? THREADS : blockDim.x) {
    key[j] = j < cnt ? scores[j] : -CUDART_INF_F;
    val[j] = j < cnt ? j : INT_MAX;
  }
  __syncthreads();
  cta_bitonic_sort<THREADS>(n2, [&](int lo, int hi) { return topk_before(key[lo], val[lo], key[hi], val[hi]); },
                   [&](int lo, int hi) {
                     const float k0 = key[lo], k1 = key[hi];
                     const int v0 = val[lo], v1 = val[hi];
                     key[lo] = k1; key[hi] = k0; val[lo] = v1; val[hi] = v0;
                   });
}
// Host side of cta_topk_sort for Kernel: refuses more than CTA_TOPK_MAX keys (the error message is too_many % (max_count,
// CTA_TOPK_MAX)), opts Kernel in to the capacity's shared memory and sets *bytes to what a sort of max_count keys needs (key and
// val back to back).
template <auto Kernel>
inline int cta_topk_smem(int max_count, const char* too_many, size_t* bytes) {
  if (max_count > CTA_TOPK_MAX) return fail(OG_EUNSUPPORTED, too_many, max_count, CTA_TOPK_MAX);
  *bytes = (size_t)pow2_ceil(max_count) * 8;
  return smem_opt_in<Kernel>(CTA_TOPK_MAX * 8);
}
// One step of an ordered (stable) compaction by one CTA: every thread holds one element of a chunk, in thread order, flagged by
// `on`.  Returns the element's output slot (meaningful where `on`): `base` + the number of flagged elements before it in the
// chunk; then advances the shared running count `base` by the chunk's total.  Ballot per warp, a serial scan of the warp totals
// (`warp_tot`: shared, one int per warp).  Called by every thread of the CTA.
__device__ __forceinline__ int cta_ordered_slot(bool on, int* warp_tot, int& base) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned bal = __ballot_sync(0xffffffffu, on);
  if (lane == 0) warp_tot[warp] = __popc(bal);
  __syncthreads();
  int before = 0;
  for (int w = 0; w < warp; ++w) before += warp_tot[w];
  const int pos = base + before + __popc(bal & ((1u << lane) - 1u));
  __syncthreads();
  if (threadIdx.x == blockDim.x - 1) base = pos + (on ? 1 : 0);
  __syncthreads();
  return pos;
}

__device__ __forceinline__ float ex2_approx(float x) {
  float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y;
}
__device__ __forceinline__ float lg2_approx(float x) {
  float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y;
}

}  // namespace og
