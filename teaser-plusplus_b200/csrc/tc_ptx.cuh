// Thin inline-PTX wrappers for the sm_90a features the tensor-core graph kernel uses:
// mbarrier, 1-D bulk async copy (TMA engine, SASS UBLKCP), warpgroup MMA (wgmma.mma_async kind tf32, SASS HGMMA) with
// both operands in shared memory and the accumulators in registers.  No CUTLASS dependency; field layouts follow the
// PTX ISA's shared-memory matrix descriptor table.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace tzr {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier -----------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  // suspend-time hint (ns): the thread sleeps in hardware until the phase completes or the hint expires, instead of
  // returning to a spin loop after the (short) default limit
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity), "r"(0x989680u)
      : "memory");
  return ok != 0;
}
// Spins until the phase with the given parity has completed.  try_wait suspends the thread in hardware for a
// bounded time, so this is not a hot spin.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---- bulk async copy global -> shared (TMA engine), completion on an mbarrier ------------------------
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src_gmem, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src_gmem), "r"(bytes), "r"(bar)
               : "memory");
}

// ---- named barrier over a subset of the CTA's warps -------------------------------------------------
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ---- descriptors -----------------------------------------------------------------------------------
// Shared-memory matrix descriptor, K-major operand, no swizzle ("interleave"): the operand is a grid of 8-row x
// 16-byte core matrices (rows 16 B apart inside a core matrix);
//   leading byte offset (bits 16-29, >>4) = distance between the two 16-byte K-chunks of one K=8 (tf32) step,
//   stride  byte offset (bits 32-45, >>4) = distance between consecutive 8-row groups,
//   base offset (bits 49-51) = 0, layout type (bits 62-63) = 0 (no swizzle).
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFFu);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  return d;
}

// ---- warpgroup MMA ---------------------------------------------------------------------------------
// Keeps the compiler from moving accesses of an accumulator register across the asynchronous MMA.
__device__ __forceinline__ void acc_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D (+)= A[smem] * B[smem]^T, one K = 8 step of tf32, M = 64 (this warpgroup's rows), N = 64; issued by all 128 threads
// of the warpgroup.  Thread t holds D rows 16 (t/32) + (t%32)/4 (+8), columns 8 i + 2 (t%4) (+1): d[4i + 2r + c].
__device__ __forceinline__ void wgmma_m64n64k8_tf32(float (&d)[32], uint64_t a_desc, uint64_t b_desc, bool accumulate) {
  const uint32_t acc = accumulate ? 1u : 0u;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a_desc), "l"(b_desc), "r"(acc)
      : "memory");
}

}  // namespace tc
}  // namespace tzr
