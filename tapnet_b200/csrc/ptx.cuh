// Inline-PTX wrappers for the Hopper (sm_90a) async machinery used by the GEMM kernels:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA with shared-memory operands).
#pragma once
#include <cuda.h>
#include <stdint.h>

namespace tapir {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ----------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)
               : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}

// Bounded wait: a pipeline bug must surface as a trap (an error the host can report), never
// as a hung GPU.  ~4e9 cycles is ~2 s at 1.9 GHz, far beyond any legitimate wait here.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int* err_flag, int code) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0x3ff) == 0 && (clock64() - t0) > 4000000000LL) {
      if (err_flag != nullptr) atomicExch(err_flag, code);
      __threadfence_system();
      __trap();
    }
  }
}

// ----------------------------------------------------------------------------- named barriers
// bar.sync waits until `count` threads (whole warps) have reached barrier `id`; bar.arrive counts
// the calling warp towards it without waiting.  Id 0 is __syncthreads().
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t count) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ----------------------------------------------------------------------------- registers
// Moves registers between warpgroups of a running CTA: every warp of the warpgroup executes the
// same instruction; .dec returns registers to the CTA's pool, .inc waits until the pool has them.
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}

// ----------------------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3),
      "r"(c4)
      : "memory");
}
// Makes this thread's generic-proxy shared-memory writes visible to later TMA (async-proxy) reads.
__device__ __forceinline__ void fence_proxy_async_shared() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// Shared (address `src`) -> global tile store, tracked in this thread's bulk async-groups.
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// Waits until at most N of this thread's bulk groups have not finished reading their source.
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
// Waits until at most N of this thread's bulk groups are incomplete (their writes not yet done).
template <int N>
__device__ __forceinline__ void bulk_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// Four 8 x 8 b16 matrices to shared memory: register i holds matrix i in the mma fragment layout
// (lane l: row l / 4, columns 2 (l % 4) + {0, 1}); lanes 8 i .. 8 i + 7 give its eight row addresses.
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1),
               "r"(r2), "r"(r3)
               : "memory");
}

// ----------------------------------------------------------------------------- wgmma
__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
// Waits until at most N committed wgmma groups of this warpgroup are still pending.
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Keeps the accumulator registers live across the asynchronous MMAs (no reordering around them).
template <int R>
__device__ __forceinline__ void reg_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D (64 x N, fp32, wgmma fragment layout) (+)= A (64 x 16) * B (N x 16)^T, both bf16 K-major;
// N / 2 accumulator registers per thread.
#define TAPIR_F8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), \
                    "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define TAPIR_R10(a) "%" #a "0, %" #a "1, %" #a "2, %" #a "3, %" #a "4, %" #a "5, %" #a "6, %" #a "7, " \
                     "%" #a "8, %" #a "9, "
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, " TAPIR_R10(1) TAPIR_R10(2) "%30, %31}, "
      "%32, %33, p, 1, 1, 0, 0;\n}\n"
      : TAPIR_F8(0), TAPIR_F8(8), TAPIR_F8(16), TAPIR_F8(24)
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, " TAPIR_R10(1) TAPIR_R10(2) TAPIR_R10(3) TAPIR_R10(4)
      TAPIR_R10(5) "%60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n}\n"
      : TAPIR_F8(0), TAPIR_F8(8), TAPIR_F8(16), TAPIR_F8(24), TAPIR_F8(32), TAPIR_F8(40), TAPIR_F8(48),
        TAPIR_F8(56)
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
#undef TAPIR_F8
#undef TAPIR_R10

// Shared-memory matrix descriptor (sm_90 wgmma) for a K-major operand tile whose rows are 128
// bytes (64 bf16) laid out by TMA with CU_TENSOR_MAP_SWIZZLE_128B: 8-row x 128 B swizzle atoms,
// consecutive atoms `sbo_bytes` apart (1024 for a dense tile); LBO is unused for swizzled
// K-major (canonical 1); layout type 1 = 128B swizzle (bits 62-63).  Advancing K by 16 bf16
// inside the swizzle row is +32 B of start address (+2 in the 16-byte units of bits 0-13).
// The hardware applies the 128B swizzle from the absolute shared-memory address bits, as TMA
// does when it writes the tile, so a view whose first row sits any number of 128-byte rows into
// its 1024-byte pattern (the halo-patch convolution) needs no base offset (bits 49-51 stay 0).
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t saddr, uint32_t sbo_bytes = 1024) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(sbo_bytes >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

}  // namespace ptx
}  // namespace tapir
