// Helpers shared by the HBM-bound support kernels (support_kernels.cu, support_kernels2.cu): CTA size, warp / group
// reductions, the deterministic grid reduction and its workspace, grid sizing, the single-instruction exp path and the
// 16-byte row I/O packers.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cstdint>

#include "abi_common.cuh"

namespace b200k {

constexpr int kThreads = 256;

template <typename A>  // float or int
__device__ __forceinline__ A warp_sum(A v) {
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, m));
  return v;
}
// Reduction over a group of R threads (R = 32 .. 256, power of two, groups are R-aligned inside the CTA).
template <int R, bool IS_MAX>
__device__ __forceinline__ float group_reduce(float v, float* smem /* kThreads/32 floats */) {
  v = IS_MAX ? warp_max(v) : warp_sum(v);
  if constexpr (R > 32) {
    constexpr int W = R / 32;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();  // smem may still be read from a previous reduction
    if (lane == 0) smem[warp] = v;
    __syncthreads();
    const int g0 = (warp / W) * W;
    float r = smem[g0];
#pragma unroll
    for (int i = 1; i < W; ++i) r = IS_MAX ? fmaxf(r, smem[g0 + i]) : r + smem[g0 + i];
    v = r;
  }
  return v;
}

inline int grid_for(int64_t work_items, int per_block, int sm_count, int waves) {
  int64_t blocks = (work_items + per_block - 1) / per_block;
  int64_t cap = int64_t(sm_count) * waves;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return int(blocks);
}
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Workspace of the deterministic two-level reductions (b200k_reduce_workspace_bytes): kReduceMaxBlocks 4-byte partials,
// then 256 bytes holding the ticket counter (and, 128 bytes in, the whole-tensor softmax total).  Every entry point
// that uses the ticket zeroes it on its own stream first, so a caller may pass any (uninitialised) device buffer and
// an aborted launch cannot poison the next call.
constexpr int kReduceMaxBlocks = 2048;
constexpr size_t kReduceWorkspace = kReduceMaxBlocks * sizeof(float) + 256;
__host__ __device__ inline unsigned int* reduce_ticket(void* ws) {
  return reinterpret_cast<unsigned int*>(static_cast<char*>(ws) + kReduceMaxBlocks * sizeof(float));
}
inline float* softmax_total(void* ws) { return reinterpret_cast<float*>(reinterpret_cast<char*>(reduce_ticket(ws)) + 128); }
inline int zero_ticket(void* ws, cudaStream_t s) {
  B200K_CHECK_CUDA(cudaMemsetAsync(reduce_ticket(ws), 0, 256, s));
  return B200K_OK;
}
// Grid of a reduction over `nvec` 16-byte vectors: four per thread per CTA, at most 8 CTAs per SM and one partial each.
inline int reduce_grid(int64_t nvec, int sm_count) {
  const int grid = grid_for(nvec, kThreads * 4, sm_count, 8);
  return grid < kReduceMaxBlocks ? grid : kReduceMaxBlocks;
}

// Finishes a sum over the whole grid into *out, the same bits whatever order the CTAs run in: each CTA stores its sum
// as partial blockIdx.x, and the last CTA to take a ticket adds the partials in a fixed order and resets the ticket.
// Every thread of every CTA calls it with its own partial.
template <typename A>  // float or int
__device__ __forceinline__ void grid_sum(A v, A* out, void* workspace) {
  A* partials = reinterpret_cast<A*>(workspace);
  unsigned int* ticket = reduce_ticket(workspace);
  __shared__ A s_part[kThreads / 32];
  __shared__ bool s_last;
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) s_part[warp] = v;
  __syncthreads();
  if (warp == 0) {
    A r = (lane < kThreads / 32) ? s_part[lane] : A(0);
    r = warp_sum(r);
    if (lane == 0) {
      partials[blockIdx.x] = r;
      __threadfence();
      s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
    }
  }
  __syncthreads();
  if (s_last) {
    __threadfence();
    // thread t adds partials t, t + 256, ..., then a fixed tree
    A r = 0;
    for (int i = threadIdx.x; i < int(gridDim.x); i += kThreads) r += reinterpret_cast<volatile A*>(partials)[i];
    r = warp_sum(r);
    __syncthreads();
    if (lane == 0) s_part[warp] = r;
    __syncthreads();
    if (threadIdx.x == 0) {
      A t = 0;
      for (int i = 0; i < kThreads / 32; ++i) t += s_part[i];
      *out = t;
      *ticket = 0;  // leave the workspace ready for the next call
    }
  }
}

// e^(x - m) as ex2.approx.ftz(x * log2e - m * log2e): one FFMA and one MUFU.EX2.  (__expf / expf add a denormal-range
// test and two predicated multiplies per element, which made the f16 softmax instruction-bound; results below 2^-126
// flush to zero, the relative error is the 2^-22 of the MUFU unit either way.)
constexpr float kLog2e = 1.4426950408889634f;
__device__ __forceinline__ float exp_sub(float x, float m_log2e) {
  float y;
  const float t = fmaf(x, kLog2e, -m_log2e);
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(t));
  return y;
}

// 16-byte packs of a row <-> fp32 registers
template <typename T>
struct RowIO;
template <>
struct RowIO<float> {
  static constexpr int N = 4;
  __device__ static void unpack(uint4 u, float* f) {
    float4 v = *reinterpret_cast<float4*>(&u);
    f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
  }
  __device__ static uint4 pack(const float* f) {
    float4 v = make_float4(f[0], f[1], f[2], f[3]);
    return *reinterpret_cast<uint4*>(&v);
  }
};
template <>
struct RowIO<__half> {
  static constexpr int N = 8;
  __device__ static void unpack(uint4 u, float* f) {
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float2 v = __half22float2(h[i]);
      f[2 * i] = v.x; f[2 * i + 1] = v.y;
    }
  }
  __device__ static uint4 pack(const float* f) {
    uint4 u;
    __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
    return u;
  }
};

}  // namespace b200k
