// Hand-written sm_90a PTX wrappers: mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA) and its shared-memory
// matrix descriptor.  No CuTe / CUTLASS: everything here is inline PTX plus the bit layout of the descriptor word.
//
// Replaces (on the reference side) the Ampere-era PTX macro sets
//   kernels/hgemm/mma/basic/hgemm_mma_stage.cu:L29-51   (cp.async / ldmatrix / mma.sync m16n8k16)
//   kernels/flash-attn/utils/utils.h:L32-59              (same set for the attention kernels)
//   ffpa-attn-mma/include/cuffpa/{mma,cp_async}.cuh
#pragma once
#include <cstdint>
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

namespace b200k {

#ifndef B200K_SPIN_LIMIT_CYCLES
// A protocol bug in an mbarrier pipeline shows up as a hang.  Every spin-wait below gives up after this many
// SM cycles (~5 s), prints which barrier it was waiting on (mbar_wait_nocall: does not print) and traps, so a bug
// becomes a CUDA error instead of a dead GPU box.  The check is only reached after a failed try_wait (slow path).
#define B200K_SPIN_LIMIT_CYCLES (10LL * 1000 * 1000 * 1000)
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// Moves registers between the warpgroups of a CTA: every warp of the warpgroup executes it, N is a multiple of 8 in
// [24, 256], and the CTA's total stays within what it was launched with.
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}

// ---------------------------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// generic-proxy writes (st.shared) -> visible to the async proxy (TMA store, wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t"
      "}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok;
}
static __device__ __noinline__ void mbar_timeout_trap(uint32_t bar, uint32_t parity) {
  printf("[b200k] mbarrier wait timed out: block (%d,%d) thread %d bar 0x%x parity %u\n", blockIdx.x, blockIdx.y,
         threadIdx.x, bar, parity);
  __trap();
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > B200K_SPIN_LIMIT_CYCLES) mbar_timeout_trap(bar, parity);
  }
}
// The same wait with no function call in it: on timeout it traps inline, without the message.  ptxas serialises every
// wgmma of a kernel that contains a call (info C7510: each MMA then waits for the previous one to finish), and the
// printf behind mbar_wait is such a call.  A kernel that overlaps wgmma must use this wait for every barrier it waits on.
__device__ __forceinline__ void mbar_wait_nocall(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > B200K_SPIN_LIMIT_CYCLES) asm volatile("trap;");
  }
}

// ---------------------------------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// L2 cache-policy words (createpolicy fractional encodings; same constants every TMA user passes)
constexpr uint64_t kPolicyEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kPolicyEvictFirst = 0x12F0000000000000ull;

__device__ __forceinline__ void tma_load_2d(uint32_t dst_smem, const CUtensorMap* m, uint32_t bar, int32_t c0,
                                            int32_t c1, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(dst_smem),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "l"(policy)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst_smem, const CUtensorMap* m, uint32_t bar, int32_t c0,
                                            int32_t c1, int32_t c2, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4, %5}], [%2], %6;" ::"r"(dst_smem),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "l"(policy)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t src_smem, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(src_smem), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {  // smem source may be overwritten afterwards
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {  // global writes are complete
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// Four 8x8 16-bit matrices to shared memory: lanes 8i .. 8i+7 give the row addresses of matrix i, and register i of
// lane l holds row l / 4, columns 2 (l % 4) and 2 (l % 4) + 1 of matrix i (the wgmma accumulator fragment, packed).
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1), "r"(r2),
               "r"(r3)
               : "memory");
}

// ---------------------------------------------------------------------------------------------- wgmma
// Shared-memory matrix descriptor (64 bit):
//   [0,14)  start address >> 4        [16,30) leading-dim byte offset >> 4 (LBO)
//   [32,46) stride-dim byte offset >> 4 (SBO)      [49,52) base offset = 0      [62,64) swizzle: 1 = 128B
// Canonical layouts with 128B swizzle (one TMA box row = 128 bytes, boxes 1024-byte aligned):
//   K-major  (row = M/N index, 128 B of K per row): groups of 8 rows at SBO = 1024 B, LBO unused; a K step of 32 bytes
//            is +32 B on the start address.
//   MN-major (row = K index, 64 M/N elements per row): 8 K-rows form a 1024 B atom, the next 8 K-rows at SBO = 1024 B,
//            the next 64 M/N elements at LBO; a K step of 16 rows is +2048 B on the start address.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
  return uint64_t((smem_addr & 0x3FFFF) >> 4) | (uint64_t(lbo >> 4) << 16) | (uint64_t(sbo >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Pins accumulator registers in place around the asynchronous MMAs: the compiler must not move reads or writes of
// them across a wgmma_fence / wgmma_wait.
template <int N>
__device__ __forceinline__ void fence_regs(float* d) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// An m64nN wgmma has N / 2 fp32 accumulators per thread, operands %0 .. %(N/2 - 1).  B200K_ACC<N> is their "+f"
// constraint list and B200K_PH<N> their placeholders, both built from 32-register groups.  The operands after them
// (descriptors or A registers, scale-d, transpose immediates) are numbered from N / 2 on, so each (form, N) spells its
// own tail; the element type only changes the type token.
#define B200K_ACC8(i) \
  "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define B200K_ACC32(i) B200K_ACC8(i), B200K_ACC8(i + 8), B200K_ACC8(i + 16), B200K_ACC8(i + 24)
#define B200K_ACC64 B200K_ACC32(0)
#define B200K_ACC128 B200K_ACC64, B200K_ACC32(32)
#define B200K_ACC192 B200K_ACC128, B200K_ACC32(64)
#define B200K_ACC256 B200K_ACC192, B200K_ACC32(96)
#define B200K_PH64 \
  "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
  "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
#define B200K_PH128 \
  B200K_PH64 ", %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, " \
  "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define B200K_PH192 \
  B200K_PH128 ", %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, " \
  "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95"
#define B200K_PH256 \
  B200K_PH192 ", %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, " \
  "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
// One instruction.  Predicate p is scale-d: 0 overwrites the accumulators, 1 adds to them.
#define B200K_WGMMA(shape, type, acc, scale, ops) \
  "{\n.reg .pred p;\nsetp.ne.b32 p, " scale ", 0;\n" \
  "wgmma.mma_async.sync.aligned." shape ".f32." type " {" acc "}, " ops ";\n}\n"
#define B200K_SS(type, n, scale, ops) \
  asm volatile(B200K_WGMMA("m64n" #n "k16", type, B200K_PH##n, scale, ops) \
               : B200K_ACC##n \
               : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB))
#define B200K_RS(type, n, scale, ops) \
  asm volatile(B200K_WGMMA("m64n" #n "k16", type, B200K_PH##n, scale, ops) \
               : B200K_ACC##n \
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d), "n"(TB))
// `op` with the 16-bit type token of the enclosing template's DT
#define B200K_F16_OR_BF16(op, ...) \
  if constexpr (DT == 0) \
    op("f16.f16", __VA_ARGS__); \
  else \
    op("bf16.bf16", __VA_ARGS__)

// d[0, N/2) = A * B, plus d when scale_d != 0, for one 64 x N x k tile, A and B in shared memory (descriptors da, db).
// DT: 0 f16, 1 bf16 (k16; TA / TB = 1 reads that operand MN-major), 2 tf32 (k8, N = 256, K-major operands only).
template <int DT, int N, int TA, int TB>
__device__ __forceinline__ void wgmma_ss(float* d, uint64_t da, uint64_t db, int scale_d) {
  static_assert(N == 64 || N == 128 || N == 256, "wgmma_ss: N must be 64, 128 or 256");
  static_assert(DT == 0 || DT == 1 || (DT == 2 && N == 256 && TA == 0 && TB == 0),
                "wgmma_ss: f16 / bf16, or tf32 with N = 256 and K-major operands");
  if constexpr (DT == 2) {
    asm volatile(B200K_WGMMA("m64n256k8", "tf32.tf32", B200K_PH256, "%130", "%128, %129, p, 1, 1")
                 : B200K_ACC256
                 : "l"(da), "l"(db), "r"(scale_d));
  } else if constexpr (N == 64) {
    B200K_F16_OR_BF16(B200K_SS, 64, "%34", "%32, %33, p, 1, 1, %35, %36");
  } else if constexpr (N == 128) {
    B200K_F16_OR_BF16(B200K_SS, 128, "%66", "%64, %65, p, 1, 1, %67, %68");
  } else {
    B200K_F16_OR_BF16(B200K_SS, 256, "%130", "%128, %129, p, 1, 1, %131, %132");
  }
}
// d[0, N/2) = A * B, plus d when scale_d != 0, for one 64 x N x 16 tile, A from registers (four packed 16-bit pairs per
// thread, the layout of an accumulator fragment) and B in shared memory (descriptor db; TB = 1 reads it MN-major).
// DT: 0 f16, 1 bf16.
template <int DT, int N, int TB>
__device__ __forceinline__ void wgmma_rs(float* d, const uint32_t* a, uint64_t db, int scale_d) {
  static_assert(N == 64 || N == 128 || N == 192 || N == 256, "wgmma_rs: N must be 64, 128, 192 or 256");
  static_assert(DT == 0 || DT == 1, "wgmma_rs: f16 or bf16");
  if constexpr (N == 64) {
    B200K_F16_OR_BF16(B200K_RS, 64, "%37", "{%32, %33, %34, %35}, %36, p, 1, 1, %38");
  } else if constexpr (N == 128) {
    B200K_F16_OR_BF16(B200K_RS, 128, "%69", "{%64, %65, %66, %67}, %68, p, 1, 1, %70");
  } else if constexpr (N == 192) {
    B200K_F16_OR_BF16(B200K_RS, 192, "%101", "{%96, %97, %98, %99}, %100, p, 1, 1, %102");
  } else {
    B200K_F16_OR_BF16(B200K_RS, 256, "%133", "{%128, %129, %130, %131}, %132, p, 1, 1, %134");
  }
}
#undef B200K_ACC8
#undef B200K_ACC32
#undef B200K_ACC64
#undef B200K_ACC128
#undef B200K_ACC192
#undef B200K_ACC256
#undef B200K_PH64
#undef B200K_PH128
#undef B200K_PH192
#undef B200K_PH256
#undef B200K_WGMMA
#undef B200K_SS
#undef B200K_RS
#undef B200K_F16_OR_BF16

// ---------------------------------------------------------------------------------------------- small helpers
__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ uint32_t pack_bf162(float lo, float hi) {
  __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

}  // namespace b200k
