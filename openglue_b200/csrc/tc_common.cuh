// sm_90a primitives used by the tensor-core kernels: mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA with the
// A operand in registers and B in shared memory), wgmma shared-memory descriptors, tf32 / fp16 hi/lo splits.
// Descriptor bit layouts follow the PTX ISA (wgmma matrix descriptor).
#pragma once
#include <string.h>
#include "common.cuh"
#include <cuda.h>
#include <cuda_fp16.h>
#include <type_traits>

namespace og {
namespace tc {

// ----------------------------------------------------------------------------- addresses
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
// 1024-byte alignment of the dynamic shared-memory block (128-byte swizzled TMA tiles), computed as an OFFSET from the
// __shared__ symbol: rounding the pointer up through uintptr_t hides the address space from the compiler and every
// shared-memory access of the kernel becomes a generic LD.E / ST.E with 64-bit address arithmetic (61 + 58 of them in the
// fp16 attention kernel, on the softmax chain's critical path) instead of LDS / STS.
__device__ __forceinline__ uint8_t* align_smem_1024(uint8_t* raw) {
  const uint32_t b = smem_u32(raw);
  return raw + (((b + 1023u) & ~1023u) - b);
}

// ----------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {          // generic-proxy writes -> visible to async proxy
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (the launch fails with an error) instead of hanging the GPU.  Call-free on purpose: a kernel
// whose wgmma chain crosses a function call (such as a device printf) has every wgmma serialized by ptxas (warning C7510).
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 24)) asm volatile("trap;");
  }
}
// The same bound without the trap, for code after setmaxnreg.inc: a trap anywhere in that code makes ptxas allocate the whole
// kernel at its launch-bound register count (spills, serialized wgmmas).  A timeout sets `timed_out` and returns, and later
// waits return at once; the caller hands the flag to a role that may trap.
__device__ __forceinline__ void mbar_wait_flag(uint64_t* bar, uint32_t parity, uint32_t& timed_out) {
  if (timed_out || mbar_try_wait(bar, parity)) return;
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 24)) { timed_out = 1; return; }
  }
}

// ----------------------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// Stores of a shared-memory box to global memory through a tensor map (the parts of the box outside the tensor are not
// written).  The writes to the box must be made visible to the async proxy first (fence_proxy_async, then a barrier among the
// writing threads).  The stores of one thread are grouped by bulk_commit: bulk_wait_read<N> returns once at most N groups still
// read shared memory (the box may then be written again), bulk_wait<N> once at most N groups are still incomplete.
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, const void* smem_src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }

// Four 8 x 8 matrices of 16-bit elements from the mma fragment layout (lane l holds row l / 4, elements 2 (l % 4), +1 of matrix
// i in r[i]) to shared memory: lane l gives the address of row l % 8 of matrix l / 8 (16 bytes).  trans: the rows written are the
// matrices' columns.
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[0]), "r"(r[1]), "r"(r[2]), "r"(r[3])
               : "memory");
}
__device__ __forceinline__ void stmatrix_x4_trans(uint32_t addr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[0]), "r"(r[1]), "r"(r[2]), "r"(r[3])
               : "memory");
}

// ----------------------------------------------------------------------------- programmatic dependent launch
// Kernels launched with LaunchAttr::pdl (cudaLaunchAttributeProgrammaticStreamSerialization) may become resident while the
// previous kernel of the stream is still draining: launch_dependents (issued at the very top) lets the NEXT kernel's CTAs take
// an SM as soon as this kernel's CTA leaves it, and grid_dependency_wait blocks until the PREVIOUS kernel has completed and
// flushed its writes.  Everything before the wait (barrier init, tensor-map prefetch) overlaps the previous kernel's tail.
__device__ __forceinline__ void launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void grid_dependency_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ----------------------------------------------------------------------------- warp specialization
// setmaxnreg moves registers between the warpgroups of a CTA (every warp of the warpgroup executes it; N a multiple of 8 in
// [24, 256]): a TMA producer warpgroup gives registers back, consumer warpgroups take them for larger fragments.
template <int N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
// Named barriers among `count` threads of whole warps (id 0 is __syncthreads): arrive does not wait, sync waits until `count`
// threads have arrived or synced on `id`.
__device__ __forceinline__ void named_bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id, int count) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// ----------------------------------------------------------------------------- wgmma
// Shared-memory matrix descriptor for a K-major operand tile stored as rows of 128 bytes with the 128-byte swizzle (what TMA
// writes with CU_TENSOR_MAP_SWIZZLE_128B and a 128-byte-wide box; the tile base 1024-byte aligned):
//   [0,14) start >> 4   [16,30) LBO >> 4 (=1, unused for swizzled K-major)   [32,46) SBO >> 4 (1024 B between 8-row groups)
//   [62,64) layout = 1 (SWIZZLE_128B).  A K step of 32 bytes inside the 128-byte row advances the start address by 32.
__device__ __forceinline__ uint64_t make_wgdesc_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Pins accumulator registers in place around an asynchronous wgmma chain (before the first wgmma and after wgmma_wait): the
// compiler may neither move them between the wgmma and the wait nor read them before the wait (CUTLASS's
// warpgroup_fence_operand).
template <int N> __device__ __forceinline__ void fence_operands(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D (+)= A . B over one warpgroup: D is 64 x N fp32 (thread t of warp w holds rows 16w + t/4 (+8), columns 8j + 2(t%4) (+1) in
// d[4j .. 4j+3]); A is the 16 x K slice of warp w in registers (the mma.sync m16n8k8 / m16n8k16 fragment layout); B is K-major in
// shared memory (descriptor).  accumulate = 0 overwrites D.
__device__ __forceinline__ void wgmma_tf32_m64n32(float (&d)[16], const uint32_t (&a)[4], uint64_t bdesc, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_tf32_m64n64(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_tf32_m64n128(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_f16_m64n32(float (&d)[16], const uint32_t (&a)[4], uint64_t bdesc, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_f16_m64n64(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_f16_m64n128(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}

// ----------------------------------------------------------------------------- tf32 split
// x = hi + lo (+ <= 2^-23 |x|):  hi = rna_tf32(x), lo = rna_tf32(x - hi).  Both are tf32-exact, so the
// tensor core's own truncation of the low mantissa bits never bites.
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(x));
  const float r = x - __uint_as_float(hi);
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(r));
}

// ----------------------------------------------------------------------------- fp16 hi/lo operands ("3xFP16", kind::f16)
// fp16 has tf32's 10 explicit mantissa bits at twice the MMA rate and half the operand bytes; what it lacks is range
// (2^-14 normal .. 65504).  Every operand tensor therefore carries a power-of-two scale that puts a bound on max|x| into
// [2^14, 2^15): hi = fp16(x s), lo = fp16(x s - hi).  |lo| <= 2^-11 |hi| stays a normal half for |x s| >= 2^-3 and is
// otherwise resolved to the subnormal spacing 2^-24, so the pair represents x s to max(2^-22 |x s|, 2^-25): 40 bits below the bound.
// Products of halves are exact in fp32; the scales are undone exactly in the epilogue (powers of two).

// power-of-two scale for a tensor whose magnitudes are bounded by `bound` (>= 0): bound * scale in [2^14, 2^15)
__host__ __device__ __forceinline__ float f16_scale_for(float bound) {
#ifdef __CUDA_ARCH__
  uint32_t e = (__float_as_uint(bound) >> 23) & 0xffu;
#else
  uint32_t bits; memcpy(&bits, &bound, 4); uint32_t e = (bits >> 23) & 0xffu;
#endif
  e = e < 87u ? 87u : (e > 187u ? 187u : e);                 // |bound| outside 2^-40 .. 2^60: clamp (all-zero tensors, garbage)
  const uint32_t sb = (268u - e) << 23;                        // 2^(14 - (e - 127))
#ifdef __CUDA_ARCH__
  return __uint_as_float(sb);
#else
  float r; memcpy(&r, &sb, 4); return r;
#endif
}
// scale of a GEMM's fp16 output y = alpha (A . W_n) + b_n, written before its maximum is known: from the bound
// |y| <= |alpha| amax(A) max_n ||W_n||_1 + max |b| (the bias is added after alpha, so it is not scaled by it)
__host__ __device__ __forceinline__ float f16_out_scale_for(float alpha, float a_amax, float w_l1, float b_max) {
  return f16_scale_for(fmaf(fabsf(alpha) * a_amax, w_l1, b_max));
}
// two already-scaled values -> packed hi halves and packed lo halves (element 0 in the low 16 bits)
__device__ __forceinline__ void split_f16x2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(x0, x1);
  const float2 f = __half22float2(h);
  const __half2 l = __floats2half2_rn(x0 - f.x, x1 - f.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
// non-negative float max through its bit pattern (amax tracking; the slot is zeroed at the start of a forward pass)
__device__ __forceinline__ void atomic_amax(float* slot, float v) { atomicMax(reinterpret_cast<unsigned int*>(slot), __float_as_uint(v)); }

// ----------------------------------------------------------------------------- host: tensor maps
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess) return (PFN_encodeTiled) nullptr;
    return (PFN_encodeTiled)p;
  }();
  return fn;
}

// Tensor map of a T tensor (float or __half) [batch, rows, cols] with row stride ld and batch stride bstride (in elements),
// in boxes of one 128-byte row (32 fp32 or 64 fp16 elements) x box_rows x 1, 128-byte swizzle; box parts outside the tensor load
// as zeros and are not stored.  rank 2 describes [rows, cols] alone; rank 3 with batch <= 1 or bstride == 0 has one batch item.
template <class T>
inline int make_tmap(CUtensorMap* map, int rank, const T* base, uint64_t batch, uint64_t rows, uint64_t cols, uint64_t ld,
                     uint64_t bstride, uint32_t box_rows) {
  static_assert(std::is_same<T, float>::value || std::is_same<T, __half>::value, "fp32 or fp16 tensor");
  constexpr bool F32 = std::is_same<T, float>::value;
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) return fail(OG_ECUDA, "cuTensorMapEncodeTiled entry point not available");
  if (batch <= 1 || bstride == 0) { batch = 1; bstride = rows * ld; }
  cuuint64_t dims[3] = {cols, rows, batch};
  cuuint64_t strides[2] = {ld * sizeof(T), bstride * sizeof(T)};
  cuuint32_t box[3] = {128 / sizeof(T), box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(map, F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<T*>(base), dims,
                  strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(OG_ECUDA, "cuTensorMapEncodeTiled (%dd %s) failed (%d): rows=%llu cols=%llu ld=%llu", rank,
                                     F32 ? "fp32" : "fp16", (int)r, (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld);
  return OG_OK;
}
// [rows, cols], loaded with tma_load_2d
template <class T>
inline int make_tmap_2d(CUtensorMap* map, const T* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  return make_tmap(map, 2, base, 1, rows, cols, ld, 0, box_rows);
}
// [batch, rows, cols], loaded with tma_load_3d or stored with tma_store_3d
template <class T>
inline int make_tmap_3d(CUtensorMap* map, const T* base, uint64_t batch, uint64_t rows, uint64_t cols, uint64_t ld, uint64_t bstride,
                        uint32_t box_rows) {
  return make_tmap(map, 3, base, batch, rows, cols, ld, bstride, box_rows);
}

}  // namespace tc
}  // namespace og
