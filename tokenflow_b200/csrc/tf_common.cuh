// tokenflow_b200 — shared device/host helpers for the sm_90a kernels.
//
// Thin inline-PTX wrappers for the Hopper primitives the kernels use: mbarrier, TMA
// (cp.async.bulk.tensor) and wgmma (shared-memory matrix descriptors, fences, commit / wait; the
// MMA wrappers themselves are in tf_wgmma.cuh).  Bit layouts follow the PTX ISA "matrix descriptor"
// table of the asynchronous warpgroup MMA section.
#pragma once

#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace tf {

// ------------------------------------------------------------------------------------------
// error plumbing (host)
// ------------------------------------------------------------------------------------------
void set_last_error(const char* fmt, ...);
int  check_cuda(cudaError_t e, const char* what);   // 0 = ok, else sets last error and returns nonzero

enum Status : int {
  TF_OK = 0,
  TF_ERR_INVALID_ARGUMENT = 1,
  TF_ERR_CUDA = 2,
  TF_ERR_UNSUPPORTED = 3,
  TF_ERR_DRIVER = 4,
};

// cuTensorMapEncodeTiled resolved through cudaGetDriverEntryPoint (no link-time libcuda dependency,
// so the library also loads on a box without a driver).
CUresult encode_tiled(CUtensorMap* map, CUtensorMapDataType dtype, uint32_t rank, const void* base,
                      const uint64_t* dims, const uint64_t* strides_bytes /* rank-1 */,
                      const uint32_t* box, CUtensorMapSwizzle swizzle);

int sm_count();   // cached multiprocessor count of the current device

#ifdef __CUDACC__
// ------------------------------------------------------------------------------------------
// small device utilities
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }

// ------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug becomes a trap (launch error reported to the host) instead of a
// hung GPU.  No legal wait in these kernels lasts longer than a few milliseconds; the bound is 2 s
// of wall clock (%globaltimer, sampled every 2048 failed polls).
__device__ __forceinline__ uint64_t global_timer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  uint64_t t0 = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 2047u) == 0) {
      const uint64_t now = global_timer_ns();
      if (t0 == 0) t0 = now;
      if (now - t0 > 2000000000ull) __trap();   // no printf here: a call inside the loop serialises wgmma
    }
  }
}

// ------------------------------------------------------------------------------------------
// TMA (bulk tensor copies global -> shared, completion on an mbarrier)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
      "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
      "r"(c2), "r"(c3)
      : "memory");
}

// ------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA): shared-memory descriptors, fences, commit / wait
// ------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor, 128-byte swizzle, tile rows of exactly 128 bytes (64 x 16-bit):
//   bits [0,14)  start address >> 4        bits [16,30) leading byte offset >> 4
//   bits [32,46) stride byte offset >> 4   bits [49,52) base offset = 0 (tiles are 1024-byte aligned)
//   bits [62,64) layout: 1 = SWIZZLE_128B
// K-major operand  : rows (M or N index) are 128 B apart inside an 8-row group, groups are SBO apart
//                    (1024 B for a dense tile); LBO is unused for swizzled K-major (encoded as 1).  The
//                    k-th 16-element slice of a 64-wide chunk starts 32*k bytes into the tile.
// MN-major operand : 64 MN-elements are contiguous (one 128 B row), consecutive K indices are 128 B
//                    apart inside a group of 8, groups of 8 K are SBO apart (1024 B dense), and the
//                    next 64 MN-elements start LBO bytes further.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
// Orders register accesses of the accumulators before the wgmma that follows (whole warpgroup).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kPending>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory");
}
// Keeps the compiler from moving accesses of an accumulator register across wgmma issue / wait.
template <int N>
__device__ __forceinline__ void reg_fence(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}

// ------------------------------------------------------------------------------------------
// misc math
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_f16x2_rn(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));   // d = {hi: first src, lo: second src}
  return r;
}
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
#endif  // __CUDACC__

}  // namespace tf
