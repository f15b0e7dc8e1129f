// vsb200 -- shared device helpers: PTX wrappers for mbarrier / TMA / wgmma (sm_90a).
// No CUTLASS: every instruction the kernels rely on is spelled out here.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

// ---- element type of this translation unit -------------------------------------------------------------------------
// Every kernel file is compiled twice: as is (bf16: OpenSora, CogVideoX-5b) and with -DVSB_HALF (IEEE fp16: the dtype the
// reference runs CogVideoX-2b and Latte in, pipeline_cogvideox.py:138-139, pipeline_latte.py:201).  The fp16 twin lives
// in namespace vsbh and exports every kernel entry with the suffix _f16 (same signatures).  `bf16` below is therefore
// "the 16-bit storage type of this build"; fp32 accumulation, rounding points and tile schedules are identical.
#ifdef VSB_HALF
#define vsb vsbh
#define VSB_API(name) name##_f16
#define VSB_MMA_T "f16"
#define VSB_ONE_BITS 0x3C00  // 1.0
#define VSB_TMAP_DTYPE 1
#else
#define VSB_API(name) name
#define VSB_MMA_T "bf16"
#define VSB_ONE_BITS 0x3F80  // 1.0
#define VSB_TMAP_DTYPE 0
#endif

namespace vsb {

#ifdef VSB_HALF
typedef __half bf16;
typedef __half2 elem2;
__device__ __forceinline__ float2 e2_to_float2(elem2 v) { return __half22float2(v); }
__device__ __forceinline__ elem2 floats_to_e2(float lo, float hi) { return __floats2half2_rn(lo, hi); }
__device__ __forceinline__ bf16 float_to_e(float x) { return __float2half_rn(x); }
__device__ __forceinline__ float e_to_float(bf16 x) { return __half2float(x); }
#else
typedef __nv_bfloat16 bf16;
typedef __nv_bfloat162 elem2;
__device__ __forceinline__ float2 e2_to_float2(elem2 v) { return __bfloat1622float2(v); }
__device__ __forceinline__ elem2 floats_to_e2(float lo, float hi) { return __floats2bfloat162_rn(lo, hi); }
__device__ __forceinline__ bf16 float_to_e(float x) { return __float2bfloat16_rn(x); }
__device__ __forceinline__ float e_to_float(bf16 x) { return __bfloat162float(x); }
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

// round-to-nearest-even float -> bf16 -> float (the rounding point of an eager bf16 op)
__device__ __forceinline__ float rbf(float x) { return e_to_float(float_to_e(x)); }

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  elem2 v = floats_to_e2(lo, hi);  // .x = lo (low 16 bits), .y = hi
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  elem2 v = *reinterpret_cast<elem2*>(&u);
  return e2_to_float2(v);
}

// ------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
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
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Spin with a watchdog: a protocol bug traps (kernel error) instead of hanging the GPU box.
#ifndef VSB_WATCHDOG_CYCLES
#define VSB_WATCHDOG_CYCLES 400000000ll  // ~0.2 s at 2 GHz: far beyond any legitimate wait inside one kernel
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > VSB_WATCHDOG_CYCLES) {
      if ((threadIdx.x & 31) == 0)
        printf("vsb200: mbarrier watchdog block=(%d,%d,%d) warp=%d bar=%u parity=%u\n", blockIdx.x, blockIdx.y,
               blockIdx.z, threadIdx.x >> 5, smem_u32(bar), parity);
      __trap();
    }
  }
}
// Same watchdog without the printf: a function call between wgmma.mma_async and its wait makes ptxas serialize the
// warpgroup MMAs, so the GEMM consumers wait with this one.
__device__ __forceinline__ void mbar_wait_quiet(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > VSB_WATCHDOG_CYCLES) __trap();
  }
}

// ------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_load_5d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], "
      "[%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3,
                                             int c4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA): operands in shared memory, fp32 accumulators in registers; wrappers in wgmma.cuh
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kPending>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory");
}
// Shared-memory matrix descriptor of a K-major tile written by TMA with SWIZZLE_128B: rows of 128 bytes (64 16-bit
// elements), 8-row groups 1024 bytes apart (stride byte offset), leading byte offset unused, layout 1 = 128B swizzle.
// Advancing K by 16 elements inside the swizzle atom adds 32 bytes to the start address.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr) {
  return uint64_t((saddr >> 4) & 0x3FFF) | (uint64_t(1) << 16) | (uint64_t(1024 >> 4) << 32) | (uint64_t(1) << 62);
}
// General form: leading / stride byte offsets and layout (1 = 128B, 2 = 64B, 3 = 32B swizzle).  For a K-major tile the stride
// byte offset is the distance between 8-row groups; for an MN-major tile (rows along K, the N extent contiguous inside the
// swizzle span) it is the distance between 8-row groups along K, and the leading byte offset the distance between swizzle
// spans along N (unused when N fits in one span).
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo, uint32_t layout) {
  return uint64_t((saddr >> 4) & 0x3FFF) | (uint64_t((lbo >> 4) & 0x3FFF) << 16) | (uint64_t((sbo >> 4) & 0x3FFF) << 32) |
         (uint64_t(layout) << 62);
}

// named barrier among a subset of warps (ids 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

}  // namespace vsb
