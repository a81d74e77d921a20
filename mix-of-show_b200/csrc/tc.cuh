// tc.cuh — sm_90a primitives used by every tensor-core kernel in this library:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma descriptors (wgmma.cuh holds the MMA wrappers).
// Inline PTX only; no CUTLASS/CuTe dependency.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "wgmma.cuh"

namespace mos {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ------------------------------------------------------------------ programmatic dependent launch (PDL)
// Every kernel of the library is launched with cudaLaunchAttributeProgrammaticStreamSerialization: it may start while
// its predecessor in the stream is still running, does its private prologue (smem carve-up, barrier init), then
// pdl_wait() blocks until the predecessor has completed and flushed its writes.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  // make generic-proxy smem writes visible to the async proxy (wgmma / TMA reads)
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (CUDA error) instead of hanging the GPU.
// The timeout path traps without a message on purpose: printf is a function call, and a call anywhere in a kernel that
// issues wgmma makes ptxas serialise every wgmma of that kernel (warning C7510; a __noinline__ helper is a call too).
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();  // ~2 s at 2 GHz
  }
}

// try_wait with a suspend-time hint: the hardware may park the thread (no issue slots used) until the phase completes
// or `ns` nanoseconds pass, so that a polling single-thread role (the TMA producer) does not take issue slots from the
// math warps it shares a scheduler with.
__device__ __forceinline__ bool mbar_try_wait_hint(uint64_t* bar, uint32_t parity, uint32_t ns) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(ns)
      : "memory");
  return ok != 0;
}
// Bounded wait built on it; the clock is only consulted every 1024 polls.  Traps without a message, as mbar_wait does.
__device__ __forceinline__ void mbar_wait_hint(uint64_t* bar, uint32_t parity, uint32_t ns = 2000) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = 0;
  uint32_t n = 0;
  while (!mbar_try_wait_hint(bar, parity, ns)) {
    if ((++n & 1023u) == 0) {
      const long long t = clock64();
      if (t0 == 0) t0 = t;
      if (t - t0 > 4000000000LL) __trap();
    }
  }
}

// ------------------------------------------------------------------ TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], "
      "[%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, "
      "%6}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// shared -> global tensor stores (bulk-group completion); out-of-bounds box elements are not written
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2,
                                             int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// every committed bulk store has finished reading its shared-memory source (the buffer may be overwritten)
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// every committed bulk store has completed its global writes
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// multicast variants: the tile lands at the same smem offset (and signals the same mbarrier offset) in every CTA of
// the cluster selected by `mask`
__device__ __forceinline__ void tma_load_2d_mc(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                               uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, "
      "{%4, %5}], [%2], %3;" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "h"(mask), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d_mc(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                               int c2, int c3, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, "
      "{%4, %5, %6, %7}], [%2], %3;" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "h"(mask), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ------------------------------------------------------------------ thread-block clusters
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ------------------------------------------------------------------ wgmma shared-memory descriptor
// K-major operand tile in shared memory, rows of 64 16-bit elements (=128 B), SWIZZLE_128B, 8-row groups 1024 B apart
// (sm_90 matrix descriptor: start[0,14) LBO[16,30) SBO[32,46) base offset[49,52) layout[62,64) = 1 for SWIZZLE_128B).
// The tile must start on a 1024-byte boundary; +2 in the start field advances 16 elements (32 B) along K inside the atom.
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>(1) << 16;            // LBO (unused for swizzled K-major)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;    // SBO: 8 rows * 128 B
  d |= static_cast<uint64_t>(1) << 62;            // SWIZZLE_128B
  return d;
}

// ------------------------------------------------------------------ small math helpers
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 t = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(t);
}
// 16-bit storage (activations and packed weights) is bf16 (training) or fp16 (sampling: 3 more mantissa bits, which is what
// keeps the classifier-free-guidance difference c - u accurate); F16 = the codec.
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  __half2 t = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float2 unpack_f16x2(uint32_t u) {
  __half2 t = *reinterpret_cast<__half2*>(&u);
  return __half22float2(t);
}
template <bool F16>
__device__ __forceinline__ uint32_t pack16x2(float lo, float hi) {
  return F16 ? pack_f16x2(lo, hi) : pack_bf16x2(lo, hi);
}
template <bool F16>
__device__ __forceinline__ float2 unpack16x2(uint32_t u) {
  return F16 ? unpack_f16x2(u) : unpack_bf16x2(u);
}
template <bool F16>
__device__ __forceinline__ uint16_t cvt16(float v) {
  if (F16) return __half_as_ushort(__float2half_rn(v));
  return __bfloat16_as_ushort(__float2bfloat16(v));
}
template <bool F16>
__device__ __forceinline__ float ld16(const __nv_bfloat16* p) {   // 16-bit storage is typed __nv_bfloat16* throughout
  const uint16_t u = *reinterpret_cast<const uint16_t*>(p);
  return F16 ? __half2float(__ushort_as_half(u)) : __bfloat162float(__ushort_as_bfloat16(u));
}
// Accumulator fragment (wgmma.cuh) of columns [16k, 16k + 16), d = &acc[8k] -> the A register fragment of one k16 step
template <bool F16>
__device__ __forceinline__ void frag_to_a(const float* d, uint32_t (&a)[4]) {
  a[0] = pack16x2<F16>(d[0], d[1]);
  a[1] = pack16x2<F16>(d[2], d[3]);
  a[2] = pack16x2<F16>(d[4], d[5]);
  a[3] = pack16x2<F16>(d[6], d[7]);
}
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float silu(float x) { return x / (1.0f + __expf(-x)); }

}  // namespace mos
