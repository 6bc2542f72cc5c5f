// HBM-roofline support kernels for H100: elementwise add, all-reduce sum, softmax, RMS norm, layer norm, RoPE,
// histogram, embedding gather.  Coalesced 128-bit accesses, warp-shuffle reductions, grids sized from the SM count, one
// pass over HBM wherever the row fits in registers.  No tensor cores (none of this is GEMM shaped).
//
// Replaces (reference file:line)
//   kernels/elementwise/elementwise.cu:L24-168      kernels/reduce/block_all_reduce.cu:L42-686
//   kernels/softmax/softmax.cu:L102-391             kernels/rms-norm/rms_norm.cu:L53-366
//   kernels/layer-norm/layer_norm.cu:L48-419        kernels/rope/rope.cu:L20-69
//   kernels/histogram/histogram.cu:L18-48           kernels/embedding/embedding.cu:L16-78
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include <climits>

#include "abi_common.cuh"
#include "support_common.cuh"

namespace b200k {

// ============================================================================================ elementwise add
template <typename T>
struct Vec16;  // 16-byte vector of T
template <>
struct Vec16<float> {
  static constexpr int N = 4;
  __device__ static uint4 add(uint4 a, uint4 b) {
    float4 x = *reinterpret_cast<float4*>(&a), y = *reinterpret_cast<float4*>(&b);
    float4 r = make_float4(x.x + y.x, x.y + y.y, x.z + y.z, x.w + y.w);
    return *reinterpret_cast<uint4*>(&r);
  }
  __device__ static float add1(float a, float b) { return a + b; }
};
template <>
struct Vec16<__half> {
  static constexpr int N = 8;
  __device__ static uint4 add(uint4 a, uint4 b) {
    uint4 r;
    const __half2* x = reinterpret_cast<const __half2*>(&a);
    const __half2* y = reinterpret_cast<const __half2*>(&b);
    __half2* z = reinterpret_cast<__half2*>(&r);
#pragma unroll
    for (int i = 0; i < 4; ++i) z[i] = __hadd2(x[i], y[i]);
    return r;
  }
  __device__ static __half add1(__half a, __half b) { return __hadd(a, b); }
};
template <>
struct Vec16<__nv_bfloat16> {
  static constexpr int N = 8;
  __device__ static uint4 add(uint4 a, uint4 b) {
    uint4 r;
    const __nv_bfloat162* x = reinterpret_cast<const __nv_bfloat162*>(&a);
    const __nv_bfloat162* y = reinterpret_cast<const __nv_bfloat162*>(&b);
    __nv_bfloat162* z = reinterpret_cast<__nv_bfloat162*>(&r);
#pragma unroll
    for (int i = 0; i < 4; ++i) z[i] = __hadd2(x[i], y[i]);
    return r;
  }
  __device__ static __nv_bfloat16 add1(__nv_bfloat16 a, __nv_bfloat16 b) { return __hadd(a, b); }
};

template <typename T>
__global__ void __launch_bounds__(kThreads) elementwise_add_vec_kernel(const T* __restrict__ a, const T* __restrict__ b,
                                                                        T* __restrict__ c, int64_t n) {
  using V = Vec16<T>;
  const int64_t nvec = n / V::N;
  const uint4* av = reinterpret_cast<const uint4*>(a);
  const uint4* bv = reinterpret_cast<const uint4*>(b);
  uint4* cv = reinterpret_cast<uint4*>(c);
  const int64_t stride = int64_t(gridDim.x) * kThreads;
  int64_t i = int64_t(blockIdx.x) * kThreads + threadIdx.x;
  // 4 independent 16-byte loads per operand in flight per thread
  for (; i + 3 * stride < nvec; i += 4 * stride) {
    uint4 x0 = __ldcs(av + i), x1 = __ldcs(av + i + stride), x2 = __ldcs(av + i + 2 * stride),
          x3 = __ldcs(av + i + 3 * stride);
    uint4 y0 = __ldcs(bv + i), y1 = __ldcs(bv + i + stride), y2 = __ldcs(bv + i + 2 * stride),
          y3 = __ldcs(bv + i + 3 * stride);
    __stcs(cv + i, V::add(x0, y0));
    __stcs(cv + i + stride, V::add(x1, y1));
    __stcs(cv + i + 2 * stride, V::add(x2, y2));
    __stcs(cv + i + 3 * stride, V::add(x3, y3));
  }
  for (; i < nvec; i += stride) __stcs(cv + i, V::add(__ldcs(av + i), __ldcs(bv + i)));
  // scalar tail (n not a multiple of the pack)
  if (blockIdx.x == 0 && threadIdx.x < n - nvec * V::N) {
    const int64_t j = nvec * V::N + threadIdx.x;
    c[j] = V::add1(a[j], b[j]);
  }
}
template <typename T>
__global__ void __launch_bounds__(kThreads) elementwise_add_scalar_kernel(const T* __restrict__ a,
                                                                           const T* __restrict__ b, T* __restrict__ c,
                                                                           int64_t n) {
  const int64_t stride = int64_t(gridDim.x) * kThreads;
  for (int64_t i = int64_t(blockIdx.x) * kThreads + threadIdx.x; i < n; i += stride)
    c[i] = Vec16<T>::add1(a[i], b[i]);
}
template <typename T>
static int launch_add(const void* a, const void* b, void* c, int64_t n, cudaStream_t s, const DeviceInfo& di) {
  if (aligned16(a) && aligned16(b) && aligned16(c)) {
    const int grid = grid_for(n / Vec16<T>::N, kThreads * 4, di.sm_count, 8);
    elementwise_add_vec_kernel<T><<<grid, kThreads, 0, s>>>(static_cast<const T*>(a), static_cast<const T*>(b),
                                                            static_cast<T*>(c), n);
  } else {
    const int grid = grid_for(n, kThreads, di.sm_count, 16);
    elementwise_add_scalar_kernel<T><<<grid, kThreads, 0, s>>>(static_cast<const T*>(a), static_cast<const T*>(b),
                                                               static_cast<T*>(c), n);
  }
  B200K_CHECK_CUDA(cudaGetLastError());
  return B200K_OK;
}

// ============================================================================================ all-reduce sum
// Two-level deterministic reduction: every CTA writes one partial, the last CTA to finish (ticket counter) adds the
// partials in index order.  The reference finishes with atomicAdd(float) in arrival order instead.

template <int DT>
struct Loader;  // sum of one 16-byte pack as float (or int for i8), optional half-precision pack sum
template <>
struct Loader<B200K_F32> {
  using acc_t = float;
  static constexpr int N = 4;
  using elem_t = float;
  template <bool ACC16>
  __device__ static float pack(uint4 u) {
    float4 v = *reinterpret_cast<float4*>(&u);
    return (v.x + v.y) + (v.z + v.w);
  }
  __device__ static float one(const float* p) { return *p; }
};
template <>
struct Loader<B200K_F16> {
  using acc_t = float;
  static constexpr int N = 8;
  using elem_t = __half;
  template <bool ACC16>
  __device__ static float pack(uint4 u) {
    const __half2* h = reinterpret_cast<const __half2*>(&u);
    if constexpr (ACC16) {  // pack summed in half, like block_all_reduce_sum_f16x8_pack_f16 (block_all_reduce.cu:L270-300)
      __half2 s = __hadd2(__hadd2(h[0], h[1]), __hadd2(h[2], h[3]));
      return __half2float(__hadd(s.x, s.y));
    } else {
      float2 a = __half22float2(h[0]), b = __half22float2(h[1]), c = __half22float2(h[2]), d = __half22float2(h[3]);
      return ((a.x + a.y) + (b.x + b.y)) + ((c.x + c.y) + (d.x + d.y));
    }
  }
  __device__ static float one(const __half* p) { return __half2float(*p); }
};
template <>
struct Loader<B200K_BF16> {
  using acc_t = float;
  static constexpr int N = 8;
  using elem_t = __nv_bfloat16;
  template <bool ACC16>
  __device__ static float pack(uint4 u) {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
    if constexpr (ACC16) {
      __nv_bfloat162 s = __hadd2(__hadd2(h[0], h[1]), __hadd2(h[2], h[3]));
      return __bfloat162float(__hadd(s.x, s.y));
    } else {
      float2 a = __bfloat1622float2(h[0]), b = __bfloat1622float2(h[1]), c = __bfloat1622float2(h[2]),
             d = __bfloat1622float2(h[3]);
      return ((a.x + a.y) + (b.x + b.y)) + ((c.x + c.y) + (d.x + d.y));
    }
  }
  __device__ static float one(const __nv_bfloat16* p) { return __bfloat162float(*p); }
};
template <__nv_fp8_interpretation_t KIND>
struct Fp8Loader {
  using acc_t = float;
  static constexpr int N = 16;
  using elem_t = uint8_t;
  template <bool ACC16>
  __device__ static float pack(uint4 u) {
    const __nv_fp8x2_storage_t* p = reinterpret_cast<const __nv_fp8x2_storage_t*>(&u);
    if constexpr (ACC16) {  // the reference only has f16-accumulating fp8 variants (block_all_reduce.cu:L520-600)
      __half2 s = __half2(__nv_cvt_fp8x2_to_halfraw2(p[0], KIND));
#pragma unroll
      for (int i = 1; i < 8; ++i) s = __hadd2(s, __half2(__nv_cvt_fp8x2_to_halfraw2(p[i], KIND)));
      return __half2float(__hadd(s.x, s.y));
    } else {
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float2 f = __half22float2(__half2(__nv_cvt_fp8x2_to_halfraw2(p[i], KIND)));
        acc += f.x + f.y;
      }
      return acc;
    }
  }
  __device__ static float one(const uint8_t* p) { return __half2float(__half(__nv_cvt_fp8_to_halfraw(*p, KIND))); }
};
template <>
struct Loader<B200K_FP8_E4M3> : Fp8Loader<__NV_E4M3> {};
template <>
struct Loader<B200K_FP8_E5M2> : Fp8Loader<__NV_E5M2> {};
template <>
struct Loader<B200K_I8> {
  using acc_t = int;
  static constexpr int N = 16;
  using elem_t = int8_t;
  template <bool ACC16>
  __device__ static int pack(uint4 u) {
    // 4 x dp4a with a vector of ones: exact int32 sum of 16 int8
    return __dp4a(int(u.x), 0x01010101, __dp4a(int(u.y), 0x01010101, __dp4a(int(u.z), 0x01010101, __dp4a(int(u.w), 0x01010101, 0))));
  }
  __device__ static int one(const int8_t* p) { return int(*p); }
};

template <int DT, bool ACC16, bool EXP /* sum exp(x) instead of x: softmax mode 0 */>
__global__ void __launch_bounds__(kThreads) reduce_sum_kernel(const void* __restrict__ xin, void* __restrict__ out,
                                                              int64_t n, void* __restrict__ workspace, bool vec_ok) {
  using L = Loader<DT>;
  using A = typename L::acc_t;
  using E = typename L::elem_t;
  const E* x = reinterpret_cast<const E*>(xin);
  A acc = 0;
  const int64_t stride = int64_t(gridDim.x) * kThreads;
  int64_t tail_from = 0;
  if (vec_ok) {
    const int64_t nvec = n / L::N;
    const uint4* xv = reinterpret_cast<const uint4*>(xin);
    int64_t i = int64_t(blockIdx.x) * kThreads + threadIdx.x;
    if constexpr (EXP) {
      for (; i < nvec; i += stride) {
        uint4 u = __ldcs(xv + i);
        float4 v = *reinterpret_cast<float4*>(&u);
        acc += (exp_sub(v.x, 0.f) + exp_sub(v.y, 0.f)) + (exp_sub(v.z, 0.f) + exp_sub(v.w, 0.f));
      }
    } else {
      A a0 = 0, a1 = 0, a2 = 0, a3 = 0;
      for (; i + 3 * stride < nvec; i += 4 * stride) {
        uint4 u0 = __ldcs(xv + i), u1 = __ldcs(xv + i + stride), u2 = __ldcs(xv + i + 2 * stride),
              u3 = __ldcs(xv + i + 3 * stride);
        a0 += L::template pack<ACC16>(u0);
        a1 += L::template pack<ACC16>(u1);
        a2 += L::template pack<ACC16>(u2);
        a3 += L::template pack<ACC16>(u3);
      }
      for (; i < nvec; i += stride) a0 += L::template pack<ACC16>(__ldcs(xv + i));
      acc = (a0 + a1) + (a2 + a3);
    }
    tail_from = nvec * L::N;
  }
  for (int64_t j = tail_from + int64_t(blockIdx.x) * kThreads + threadIdx.x; j < n; j += stride) {
    if constexpr (EXP) acc += exp_sub(float(L::one(x + j)), 0.f);
    else acc += L::one(x + j);
  }
  grid_sum<A>(acc, static_cast<A*>(out), workspace);
}

template <int DT, bool EXP>
static int launch_reduce(const void* x, void* out, int64_t n, int acc_f16, void* ws, cudaStream_t s,
                         const DeviceInfo& di) {
  const int grid = reduce_grid(n / Loader<DT>::N, di.sm_count);
  const bool vec_ok = aligned16(x);
  // fp16 accumulation exists for the 16-bit and fp8 inputs only: no f32, int8 or exp-sum kernel is built with it
  constexpr bool kAcc16 = !EXP && DT != B200K_F32 && DT != B200K_I8;
  if (kAcc16 && acc_f16) reduce_sum_kernel<DT, kAcc16, false><<<grid, kThreads, 0, s>>>(x, out, n, ws, vec_ok);
  else reduce_sum_kernel<DT, false, EXP><<<grid, kThreads, 0, s>>>(x, out, n, ws, vec_ok);
  B200K_CHECK_CUDA(cudaGetLastError());
  return B200K_OK;
}

// ============================================================================================ row kernels
// One row is owned by R threads (R = 32, 128 or 256; 256/R rows per CTA).  Each thread keeps up to 32 elements of the
// row in registers (4 or 8 16-byte vectors), so x is read once and y written once.  Rows longer than 32*R fall back
// to re-reading x from L2/HBM.  Softmax sums exp(x - max) (the safe one finds the max first), RMS norm sums x^2, layer
// norm sums x for the mean and then (x - mean)^2, like the reference (layer_norm.cu:L62-72).
enum RowOp { OP_SOFTMAX = 0, OP_SAFE_SOFTMAX = 1, OP_RMSNORM = 2, OP_RMSNORM_ACC16 = 3, OP_LAYERNORM = 4 };

struct RowParams {
  float g, eps;
  int eps_inside_k;
  float b;             // layer norm: bias
  const float* total;  // softmax mode 0: precomputed sum of exp over the whole tensor
};

template <typename T, int R, int OP>
__global__ void __launch_bounds__(kThreads) row_kernel(const T* __restrict__ x, T* __restrict__ y, int64_t rows, int H,
                                                       RowParams prm) {
  using IO = RowIO<T>;
  constexpr int VN = IO::N;
  constexpr int MAXV = 32 / VN;  // vectors cached per thread
  constexpr int ROWS = kThreads / R;
  __shared__ float s_red[kThreads / 32];
  const int sub = threadIdx.x / R, t = threadIdx.x % R;
  const int nvec = H / VN;
  const bool cached = nvec <= MAXV * R;
  for (int64_t row = int64_t(blockIdx.x) * ROWS + sub; row < ((rows + ROWS - 1) / ROWS) * ROWS;
       row += int64_t(gridDim.x) * ROWS) {
    const bool live = row < rows;  // keep whole CTA in the loop: group_reduce uses __syncthreads when R > 32
    const uint4* xv = reinterpret_cast<const uint4*>(x + (live ? row : 0) * int64_t(H));
    uint4* yv = reinterpret_cast<uint4*>(y + (live ? row : 0) * int64_t(H));
    float v[MAXV * VN];
    float m = -INFINITY, s = 0.f;
    float ml2 = 0.f;   // m * log2(e) for the safe softmax, 0 for the plain one
    float mean = 0.f;  // layer norm: the row sum, then its mean
    if (cached) {
#pragma unroll
      for (int i = 0; i < MAXV; ++i) {
        const int vi = t + i * R;
        if (live && vi < nvec) {
          IO::unpack(__ldcs(xv + vi), v + i * VN);
        } else {
#pragma unroll
          for (int e = 0; e < VN; ++e) v[i * VN + e] = (OP == OP_SAFE_SOFTMAX) ? -INFINITY : 0.f;
        }
      }
      if constexpr (OP == OP_SAFE_SOFTMAX) {
#pragma unroll
        for (int e = 0; e < MAXV * VN; ++e) m = fmaxf(m, v[e]);
        m = group_reduce<R, true>(m, s_red);
        ml2 = m * kLog2e;
      }
      if constexpr (OP == OP_SAFE_SOFTMAX || OP == OP_SOFTMAX) {
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
          const bool in = (t + i * R) < nvec;
#pragma unroll
          for (int e = 0; e < VN; ++e) {
            float ex = in ? exp_sub(v[i * VN + e], ml2) : 0.f;
            v[i * VN + e] = ex;
            s += ex;
          }
        }
      } else if constexpr (OP == OP_RMSNORM_ACC16) {
        __half hs = __float2half(0.f);
#pragma unroll
        for (int e = 0; e < MAXV * VN; ++e) {
          __half h = __float2half(v[e]);
          hs = __hfma(h, h, hs);
        }
        s = __half2float(hs);
      } else if constexpr (OP == OP_LAYERNORM) {
#pragma unroll
        for (int e = 0; e < MAXV * VN; ++e) mean += v[e];
      } else {
#pragma unroll
        for (int e = 0; e < MAXV * VN; ++e) s = fmaf(v[e], v[e], s);
      }
    } else {
      // long rows: stream x twice (three times for safe softmax and layer norm)
      if constexpr (OP == OP_SAFE_SOFTMAX) {
        for (int vi = t; live && vi < nvec; vi += R) {
          float f[VN];
          IO::unpack(xv[vi], f);
#pragma unroll
          for (int e = 0; e < VN; ++e) m = fmaxf(m, f[e]);
        }
        m = group_reduce<R, true>(m, s_red);
        ml2 = m * kLog2e;
      }
      for (int vi = t; live && vi < nvec; vi += R) {
        float f[VN];
        IO::unpack(xv[vi], f);
#pragma unroll
        for (int e = 0; e < VN; ++e) {
          if constexpr (OP == OP_SAFE_SOFTMAX || OP == OP_SOFTMAX) s += exp_sub(f[e], ml2);
          else if constexpr (OP == OP_LAYERNORM) mean += f[e];
          else s = fmaf(f[e], f[e], s);
        }
      }
    }
    if constexpr (OP == OP_LAYERNORM) {  // s = sum of (x - mean)^2, with the centred row kept in registers
      mean = group_reduce<R, false>(mean, s_red) / float(H);
      if (cached) {
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
          const bool in = (t + i * R) < nvec;
#pragma unroll
          for (int e = 0; e < VN; ++e) {
            const float d = in ? v[i * VN + e] - mean : 0.f;
            v[i * VN + e] = d;
            s = fmaf(d, d, s);
          }
        }
      } else {
        for (int vi = t; live && vi < nvec; vi += R) {
          float f[VN];
          IO::unpack(xv[vi], f);
#pragma unroll
          for (int e = 0; e < VN; ++e) s = fmaf(f[e] - mean, f[e] - mean, s);
        }
      }
    }
    if (!(OP == OP_SOFTMAX && prm.total != nullptr)) s = group_reduce<R, false>(s, s_red);
    float scale;
    if constexpr (OP == OP_SOFTMAX || OP == OP_SAFE_SOFTMAX) {
      scale = 1.0f / ((OP == OP_SOFTMAX && prm.total != nullptr) ? *prm.total : s);
    } else {
      const float denom = prm.eps_inside_k ? s / (float(H) + prm.eps) : s / float(H) + prm.eps;
      scale = rsqrtf(denom) * prm.g;
    }
    if (cached) {
#pragma unroll
      for (int i = 0; i < MAXV; ++i) {
        const int vi = t + i * R;
        if (live && vi < nvec) {
          float o[VN];
#pragma unroll
          for (int e = 0; e < VN; ++e) {
            if constexpr (OP == OP_LAYERNORM) o[e] = fmaf(v[i * VN + e], scale, prm.b);
            else o[e] = v[i * VN + e] * scale;
          }
          __stcs(yv + vi, IO::pack(o));
        }
      }
    } else {
      for (int vi = t; live && vi < nvec; vi += R) {
        float f[VN];
        IO::unpack(xv[vi], f);
#pragma unroll
        for (int e = 0; e < VN; ++e) {
          if constexpr (OP == OP_SAFE_SOFTMAX || OP == OP_SOFTMAX) f[e] = exp_sub(f[e], ml2) * scale;
          else if constexpr (OP == OP_LAYERNORM) f[e] = fmaf(f[e] - mean, scale, prm.b);
          else f[e] = f[e] * scale;
        }
        yv[vi] = IO::pack(f);
      }
    }
  }
}

// Generic fallback (row length not a multiple of the pack, or unaligned): one CTA per row, scalar accesses.
template <typename T, int OP>
__global__ void __launch_bounds__(kThreads) row_kernel_scalar(const T* __restrict__ x, T* __restrict__ y, int64_t rows,
                                                              int H, RowParams prm) {
  __shared__ float s_red[kThreads / 32];
  for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
    const T* xr = x + row * int64_t(H);
    T* yr = y + row * int64_t(H);
    float m = -INFINITY, s = 0.f, mean = 0.f;
    if constexpr (OP == OP_SAFE_SOFTMAX) {
      for (int i = threadIdx.x; i < H; i += kThreads) m = fmaxf(m, float(xr[i]));
      m = group_reduce<kThreads, true>(m, s_red);
    } else if constexpr (OP == OP_LAYERNORM) {
      float sum = 0.f;
      for (int i = threadIdx.x; i < H; i += kThreads) sum += float(xr[i]);
      mean = group_reduce<kThreads, false>(sum, s_red) / float(H);
    }
    const float ml2 = (OP == OP_SAFE_SOFTMAX) ? m * kLog2e : 0.f;
    for (int i = threadIdx.x; i < H; i += kThreads) {
      const float f = float(xr[i]);
      if constexpr (OP == OP_SAFE_SOFTMAX || OP == OP_SOFTMAX) s += exp_sub(f, ml2);
      else if constexpr (OP == OP_LAYERNORM) s = fmaf(f - mean, f - mean, s);
      else s = fmaf(f, f, s);
    }
    if (!(OP == OP_SOFTMAX && prm.total != nullptr)) s = group_reduce<kThreads, false>(s, s_red);
    float scale;
    if constexpr (OP == OP_SOFTMAX || OP == OP_SAFE_SOFTMAX) {
      scale = 1.0f / ((OP == OP_SOFTMAX && prm.total != nullptr) ? *prm.total : s);
    } else {
      const float denom = prm.eps_inside_k ? s / (float(H) + prm.eps) : s / float(H) + prm.eps;
      scale = rsqrtf(denom) * prm.g;
    }
    for (int i = threadIdx.x; i < H; i += kThreads) {
      float f = float(xr[i]);
      if constexpr (OP == OP_SAFE_SOFTMAX || OP == OP_SOFTMAX) f = exp_sub(f, ml2) * scale;
      else if constexpr (OP == OP_LAYERNORM) f = fmaf(f - mean, scale, prm.b);
      else f = f * scale;
      yr[i] = T(f);
    }
    __syncthreads();
  }
}

template <typename T, int OP>
static int launch_row(const void* x, void* y, int64_t rows, int64_t H, RowParams prm, cudaStream_t s,
                      const DeviceInfo& di) {
  const T* xp = static_cast<const T*>(x);
  T* yp = static_cast<T*>(y);
  constexpr int VN = RowIO<T>::N;
  if (H % VN == 0 && aligned16(x) && aligned16(y)) {
    if (H <= 32 * 32) {
      const int grid = grid_for(rows, kThreads / 32, di.sm_count, 16);
      row_kernel<T, 32, OP><<<grid, kThreads, 0, s>>>(xp, yp, rows, int(H), prm);
    } else if (H <= 32 * 128) {
      const int grid = grid_for(rows, kThreads / 128, di.sm_count, 16);
      row_kernel<T, 128, OP><<<grid, kThreads, 0, s>>>(xp, yp, rows, int(H), prm);
    } else {
      const int grid = grid_for(rows, 1, di.sm_count, 16);
      row_kernel<T, 256, OP><<<grid, kThreads, 0, s>>>(xp, yp, rows, int(H), prm);
    }
  } else {
    const int grid = grid_for(rows, 1, di.sm_count, 16);
    row_kernel_scalar<T, OP><<<grid, kThreads, 0, s>>>(xp, yp, rows, int(H), prm);
  }
  B200K_CHECK_CUDA(cudaGetLastError());
  return B200K_OK;
}

// ============================================================================================ RoPE (f32)
// sin / cos of an fp32 angle of any size (positions reach 10^5): subtract k * 2 pi with a three-constant Cody-Waite
// split (exact products for |k| < 2^15), then MUFU.SIN / MUFU.COS on [-pi, pi] (absolute error ~5e-7).  The libdevice
// sincosf costs ~45 instructions per call, which made the textbook path instruction-bound (4.4 TB/s).
__device__ __forceinline__ void sincos_reduced(float a, float* sn, float* cs) {
  const float k = rintf(a * 0.15915494309189535f);
  float r = fmaf(k, -6.28125f, a);                 // 2 pi = 6.28125 + 1.9353071795864769e-3 (+ rounding term)
  r = fmaf(k, -1.9350051879882812e-3f, r);
  r = fmaf(k, -3.0199159819580696e-7f, r);
  *sn = __sinf(r);
  *cs = __cosf(r);
}

constexpr int kRopeMaxPairs = 8192;  // inverse-frequency table in shared memory (hidden <= 16384)
__global__ void __launch_bounds__(kThreads) rope_f32_kernel(const float* __restrict__ x, float* __restrict__ out,
                                                            int64_t seq_len, int hidden, bool quirk, bool vec) {
  const int pairs = hidden / 2;
  __shared__ float s_inv_freq[kRopeMaxPairs];
  // inverse frequency theta^(-2p/hidden) evaluated in double, once per CTA: at position 8191 an fp32 exponent costs
  // ~5e-3 rad.  Rows longer than the table fall back to computing it per element.
  const double neg2_log2theta_over_h = -2.0 * 13.287712379549449 / double(hidden);  // log2(10000)
  const bool table = !quirk && pairs <= kRopeMaxPairs;
  if (table) {
    for (int p = threadIdx.x; p < pairs; p += kThreads) s_inv_freq[p] = float(exp2(double(p) * neg2_log2theta_over_h));
    __syncthreads();
  }
  auto inv_freq = [&](int p) -> float {
    return table ? s_inv_freq[p] : float(exp2(double(p) * neg2_log2theta_over_h));
  };
  if (vec) {
    // One float4 = two neighbouring pairs.  Rows are walked without any per-element division: a CTA takes
    // ROWS = max(1, kThreads / per_row) rows at a time, a thread the float4s j, j + kThreads, ... of its row, up to
    // four loads in flight.
    const int per_row = hidden / 4;
    const int tpr = per_row < kThreads ? per_row : kThreads;  // threads per row
    const int rows_per_cta = kThreads / tpr;
    const int sub = threadIdx.x / tpr, j0 = threadIdx.x - sub * tpr;
    if (sub >= rows_per_cta) return;
    for (int64_t pos = int64_t(blockIdx.x) * rows_per_cta + sub; pos < seq_len; pos += int64_t(gridDim.x) * rows_per_cta) {
      const float4* xr = reinterpret_cast<const float4*>(x + pos * int64_t(hidden));
      float4* orow = reinterpret_cast<float4*>(out + pos * int64_t(hidden));
      float sq, cq;
      if (quirk) sincos_reduced(float(pos), &sq, &cq);
      for (int jb = j0; jb < per_row; jb += 4 * tpr) {
        float4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (jb + u * tpr < per_row) v[u] = __ldcs(xr + jb + u * tpr);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int j = jb + u * tpr;
          if (j >= per_row) break;
          float s0, c0, s1, c1;
          if (quirk) {
            s0 = s1 = sq;
            c0 = c1 = cq;
          } else {
            sincos_reduced(float(pos) * inv_freq(2 * j), &s0, &c0);
            sincos_reduced(float(pos) * inv_freq(2 * j + 1), &s1, &c1);
          }
          float4 o;
          o.x = v[u].x * c0 - v[u].y * s0;
          o.y = v[u].x * s0 + v[u].y * c0;
          o.z = v[u].z * c1 - v[u].w * s1;
          o.w = v[u].z * s1 + v[u].w * c1;
          __stcs(orow + j, o);
        }
      }
    }
  } else {
    const int64_t total = seq_len * int64_t(pairs);
    for (int64_t i = int64_t(blockIdx.x) * kThreads + threadIdx.x; i < total; i += int64_t(gridDim.x) * kThreads) {
      const int64_t pos = i / pairs;
      const int p = int(i - pos * pairs);
      const float x1 = x[pos * hidden + 2 * p], x2 = x[pos * hidden + 2 * p + 1];
      float sn, cs;
      sincos_reduced(quirk ? float(pos) : float(pos) * inv_freq(p), &sn, &cs);
      out[pos * hidden + 2 * p] = x1 * cs - x2 * sn;
      out[pos * hidden + 2 * p + 1] = x1 * sn + x2 * cs;
    }
  }
}

// ============================================================================================ histogram / max
__global__ void init_i32_kernel(int* p, int v) { *p = v; }

__global__ void __launch_bounds__(kThreads) max_i32_kernel(const int* __restrict__ a, int64_t n, int* __restrict__ out) {
  int m = INT_MIN;
  for (int64_t i = int64_t(blockIdx.x) * kThreads + threadIdx.x; i < n; i += int64_t(gridDim.x) * kThreads)
    m = max(m, a[i]);
#pragma unroll
  for (int k = 16; k >= 1; k >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, k));
  __shared__ int s[kThreads / 32];
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < kThreads / 32; ++i) m = max(m, s[i]);
    atomicMax(out, m);
  }
}

constexpr int kSmemBins = 8192;
// Per-CTA shared-memory bins merged with global atomics at the end (SMEM), or global atomics only (huge bin counts).
// Four 16-byte loads in flight per thread.  Measured at 128 Mi random 8-bit values: 5.2-5.5 TB/s; giving every lane its
// own copy of the bins (conflict-free banks) or more CTAs per SM did not move it (4.0-5.5 TB/s over the settings tried).
template <bool SMEM>
__global__ void __launch_bounds__(kThreads) histogram_i32_kernel(const int* __restrict__ a, int64_t n,
                                                                 int* __restrict__ hist, int nbins, bool vec) {
  __shared__ int s_hist[SMEM ? kSmemBins : 1];
  if constexpr (SMEM) {
    for (int i = threadIdx.x; i < nbins; i += kThreads) s_hist[i] = 0;
    __syncthreads();
  }
  auto bump = [&](int v) {
    if (unsigned(v) < unsigned(nbins)) {
      if constexpr (SMEM) atomicAdd(&s_hist[v], 1);
      else atomicAdd(&hist[v], 1);
    }
  };
  const int64_t stride = int64_t(gridDim.x) * kThreads;
  int64_t done = 0;
  if (vec) {
    const int64_t nvec = n / 4;
    const int4* av = reinterpret_cast<const int4*>(a);
    for (int64_t i = int64_t(blockIdx.x) * kThreads + threadIdx.x; i < nvec; i += 4 * stride) {
      int4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u)
        v[u] = (i + u * stride < nvec) ? __ldcs(av + i + u * stride) : make_int4(-1, -1, -1, -1);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        bump(v[u].x); bump(v[u].y); bump(v[u].z); bump(v[u].w);
      }
    }
    done = nvec * 4;
  }
  for (int64_t i = done + int64_t(blockIdx.x) * kThreads + threadIdx.x; i < n; i += stride) bump(a[i]);
  if constexpr (SMEM) {
    __syncthreads();
    for (int i = threadIdx.x; i < nbins; i += kThreads) {
      const int c = s_hist[i];
      if (c) atomicAdd(&hist[i], c);
    }
  }
}

// ============================================================================================ embedding
// One warp per output row, 16-byte chunks; rows with an out-of-range index are written as zeros.
__global__ void __launch_bounds__(kThreads) embedding_kernel(const int* __restrict__ idx, const uint8_t* __restrict__ w,
                                                             uint8_t* __restrict__ out, int64_t n, int64_t rows,
                                                             int64_t row_bytes, bool vec) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int64_t i = int64_t(blockIdx.x) * (kThreads / 32) + warp; i < n; i += int64_t(gridDim.x) * (kThreads / 32)) {
    const int r = idx[i];
    const bool ok = r >= 0 && r < rows;
    const uint8_t* src = w + (ok ? int64_t(r) : 0) * row_bytes;
    uint8_t* dst = out + i * row_bytes;
    if (vec) {
      const int64_t nv = row_bytes / 16;
      for (int64_t c = lane; c < nv; c += 32) {
        uint4 v = ok ? __ldg(reinterpret_cast<const uint4*>(src) + c) : make_uint4(0, 0, 0, 0);
        __stcs(reinterpret_cast<uint4*>(dst) + c, v);
      }
    } else {
      for (int64_t c = lane; c < row_bytes / 2; c += 32) {
        uint16_t v = ok ? reinterpret_cast<const uint16_t*>(src)[c] : uint16_t(0);
        reinterpret_cast<uint16_t*>(dst)[c] = v;
      }
    }
  }
}

}  // namespace b200k

// ================================================================================================ C ABI
using namespace b200k;

extern "C" int b200k_elementwise_add(const void* a, const void* b, void* c, int64_t n, int dtype, void* stream) {
  if (!a || !b || !c) return set_error(B200K_EARG, "b200k_elementwise_add: null pointer");
  if (n < 0) return set_error(B200K_ESHAPE, "b200k_elementwise_add: n < 0");
  if (n == 0) return B200K_OK;
  DeviceInfo di;
  int rc = get_device_info(&di);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  switch (dtype) {
    case B200K_F32: return launch_add<float>(a, b, c, n, s, di);
    case B200K_F16: return launch_add<__half>(a, b, c, n, s, di);
    case B200K_BF16: return launch_add<__nv_bfloat16>(a, b, c, n, s, di);
    default: return set_error(B200K_EDTYPE, "b200k_elementwise_add: dtype %d not supported (f32, f16, bf16)", dtype);
  }
}

extern "C" size_t b200k_reduce_workspace_bytes(void) { return kReduceWorkspace; }

extern "C" int b200k_block_all_reduce_sum(const void* x, void* out, int64_t n, int dtype, int acc_f16, void* workspace,
                                          void* stream) {
  if (!x || !out || !workspace) return set_error(B200K_EARG, "b200k_block_all_reduce_sum: null pointer");
  if (n < 0) return set_error(B200K_ESHAPE, "b200k_block_all_reduce_sum: n < 0");
  DeviceInfo di;
  int rc = get_device_info(&di);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if ((rc = zero_ticket(workspace, s))) return rc;
  switch (dtype) {
    case B200K_F32: return launch_reduce<B200K_F32, false>(x, out, n, 0, workspace, s, di);
    case B200K_F16: return launch_reduce<B200K_F16, false>(x, out, n, acc_f16, workspace, s, di);
    case B200K_BF16: return launch_reduce<B200K_BF16, false>(x, out, n, acc_f16, workspace, s, di);
    case B200K_FP8_E4M3: return launch_reduce<B200K_FP8_E4M3, false>(x, out, n, acc_f16, workspace, s, di);
    case B200K_FP8_E5M2: return launch_reduce<B200K_FP8_E5M2, false>(x, out, n, acc_f16, workspace, s, di);
    case B200K_I8: return launch_reduce<B200K_I8, false>(x, out, n, 0, workspace, s, di);
    default: return set_error(B200K_EDTYPE, "b200k_block_all_reduce_sum: dtype %d not supported", dtype);
  }
}

extern "C" int b200k_softmax(const void* x, void* y, int64_t S, int64_t H, int dtype, int mode, void* workspace,
                             void* stream) {
  if (!x || !y) return set_error(B200K_EARG, "b200k_softmax: null pointer");
  if (S < 0 || H < 1 || H > INT32_MAX) return set_error(B200K_ESHAPE, "b200k_softmax: bad shape [%lld,%lld]", (long long)S, (long long)H);
  if (S == 0) return B200K_OK;
  if (mode < 0 || mode > 3) return set_error(B200K_EARG, "b200k_softmax: mode %d not in 0..3", mode);
  DeviceInfo di;
  int rc = get_device_info(&di);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  RowParams prm = {1.f, 0.f, 0, 0.f, nullptr};
  if (mode == 0) {
    if (dtype != B200K_F32) return set_error(B200K_EDTYPE, "b200k_softmax: whole-tensor mode is f32 only (as in the reference)");
    if (!workspace) return set_error(B200K_EARG, "b200k_softmax: mode 0 needs a workspace");
    // total = sum(exp(x)) over the whole tensor (deterministic two-level reduction), then y = exp(x) / total.
    float* total = softmax_total(workspace);
    if ((rc = zero_ticket(workspace, s))) return rc;
    if ((rc = launch_reduce<B200K_F32, true>(x, total, S * H, 0, workspace, s, di))) return rc;
    prm.total = total;
    return launch_row<float, OP_SOFTMAX>(x, y, S, H, prm, s, di);
  }
  if (dtype == B200K_F32) {
    return mode == 1 ? launch_row<float, OP_SOFTMAX>(x, y, S, H, prm, s, di)
                     : launch_row<float, OP_SAFE_SOFTMAX>(x, y, S, H, prm, s, di);
  } else if (dtype == B200K_F16) {
    return mode == 1 ? launch_row<__half, OP_SOFTMAX>(x, y, S, H, prm, s, di)
                     : launch_row<__half, OP_SAFE_SOFTMAX>(x, y, S, H, prm, s, di);
  }
  return set_error(B200K_EDTYPE, "b200k_softmax: dtype %d not supported (f32, f16)", dtype);
}

extern "C" int b200k_rms_norm(const void* x, void* y, int64_t N, int64_t K, float g, float eps, int dtype, int acc_f16,
                              int eps_inside_k, void* stream) {
  if (!x || !y) return set_error(B200K_EARG, "b200k_rms_norm: null pointer");
  if (N < 0 || K < 1 || K > INT32_MAX) return set_error(B200K_ESHAPE, "b200k_rms_norm: bad shape [%lld,%lld]", (long long)N, (long long)K);
  if (N == 0) return B200K_OK;
  DeviceInfo di;
  int rc = get_device_info(&di);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  RowParams prm = {g, eps, eps_inside_k, 0.f, nullptr};
  if (dtype == B200K_F32) return launch_row<float, OP_RMSNORM>(x, y, N, K, prm, s, di);
  if (dtype == B200K_F16)
    return acc_f16 ? launch_row<__half, OP_RMSNORM_ACC16>(x, y, N, K, prm, s, di)
                   : launch_row<__half, OP_RMSNORM>(x, y, N, K, prm, s, di);
  return set_error(B200K_EDTYPE, "b200k_rms_norm: dtype %d not supported (f32, f16)", dtype);
}

extern "C" int b200k_layer_norm(const void* x, void* y, int64_t N, int64_t K, float g, float b, float eps, int dtype,
                                int eps_inside_k, void* stream) {
  if (!x || !y) return set_error(B200K_EARG, "b200k_layer_norm: null pointer");
  if (N < 1 || K < 1 || K > INT32_MAX) return set_error(B200K_ESHAPE, "b200k_layer_norm: need N >= 1, 1 <= K < 2^31");
  DeviceInfo di;
  int rc = get_device_info(&di);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const RowParams prm = {g, eps, eps_inside_k, b, nullptr};
  switch (dtype) {
    case B200K_F32: return launch_row<float, OP_LAYERNORM>(x, y, N, K, prm, s, di);
    case B200K_F16: return launch_row<__half, OP_LAYERNORM>(x, y, N, K, prm, s, di);
    default: return set_error(B200K_EDTYPE, "b200k_layer_norm: dtype %d not supported (f32, f16)", dtype);
  }
}

extern "C" int b200k_rope_f32(const void* x, void* out, int64_t seq_len, int64_t hidden, int ref_quirk, void* stream) {
  if (!x || !out) return set_error(B200K_EARG, "b200k_rope_f32: null pointer");
  if (seq_len < 0 || hidden < 2 || (hidden & 1) || hidden > INT32_MAX)
    return set_error(B200K_ESHAPE, "b200k_rope_f32: hidden must be even and >= 2 (got %lld)", (long long)hidden);
  if (seq_len == 0) return B200K_OK;
  DeviceInfo di;
  int rc = get_device_info(&di);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool vec = (hidden % 4 == 0) && aligned16(x) && aligned16(out);
  int grid;
  if (vec) {
    const int per_row = int(hidden / 4), tpr = per_row < kThreads ? per_row : kThreads;
    grid = grid_for(seq_len, kThreads / tpr, di.sm_count, 8);  // the kernel walks rows, kThreads / tpr rows per CTA
  } else {
    grid = grid_for(seq_len * (hidden / 2), kThreads, di.sm_count, 16);
  }
  rope_f32_kernel<<<grid, kThreads, 0, s>>>(static_cast<const float*>(x), static_cast<float*>(out), seq_len,
                                            int(hidden), ref_quirk != 0, vec);
  B200K_CHECK_CUDA(cudaGetLastError());
  return B200K_OK;
}

extern "C" int b200k_max_i32(const void* a, int64_t n, void* out_max, void* stream) {
  if (!a || !out_max) return set_error(B200K_EARG, "b200k_max_i32: null pointer");
  if (n < 1) return set_error(B200K_ESHAPE, "b200k_max_i32: n must be >= 1");
  DeviceInfo di;
  int rc = get_device_info(&di);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  init_i32_kernel<<<1, 1, 0, s>>>(static_cast<int*>(out_max), INT_MIN);
  max_i32_kernel<<<grid_for(n, kThreads * 4, di.sm_count, 8), kThreads, 0, s>>>(static_cast<const int*>(a), n,
                                                                               static_cast<int*>(out_max));
  B200K_CHECK_CUDA(cudaGetLastError());
  return B200K_OK;
}

extern "C" int b200k_histogram_i32(const void* a, int64_t n, void* hist, int64_t nbins, void* stream) {
  if (!hist || (!a && n > 0)) return set_error(B200K_EARG, "b200k_histogram_i32: null pointer");
  if (n < 0 || nbins < 1 || nbins > INT32_MAX) return set_error(B200K_ESHAPE, "b200k_histogram_i32: bad n/nbins");
  DeviceInfo di;
  int rc = get_device_info(&di);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200K_CHECK_CUDA(cudaMemsetAsync(hist, 0, size_t(nbins) * sizeof(int), s));
  if (n == 0) return B200K_OK;
  const bool vec = aligned16(a);
  const int grid = grid_for(n, kThreads * 16, di.sm_count, 4);
  if (nbins <= kSmemBins)
    histogram_i32_kernel<true><<<grid, kThreads, 0, s>>>(static_cast<const int*>(a), n, static_cast<int*>(hist), int(nbins), vec);
  else
    histogram_i32_kernel<false><<<grid, kThreads, 0, s>>>(static_cast<const int*>(a), n, static_cast<int*>(hist), int(nbins), vec);
  B200K_CHECK_CUDA(cudaGetLastError());
  return B200K_OK;
}

extern "C" int b200k_embedding(const void* idx, const void* weight, void* out, int64_t n, int64_t rows, int64_t emb,
                               int dtype, void* stream) {
  if (!idx || !weight || !out) return set_error(B200K_EARG, "b200k_embedding: null pointer");
  if (n < 0 || rows < 1 || emb < 1) return set_error(B200K_ESHAPE, "b200k_embedding: bad shape");
  if (n == 0) return B200K_OK;
  int esize;
  if (dtype == B200K_F32) esize = 4;
  else if (dtype == B200K_F16 || dtype == B200K_BF16) esize = 2;
  else return set_error(B200K_EDTYPE, "b200k_embedding: dtype %d not supported (f32, f16, bf16)", dtype);
  DeviceInfo di;
  int rc = get_device_info(&di);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int64_t row_bytes = emb * esize;
  const bool vec = (row_bytes % 16 == 0) && aligned16(weight) && aligned16(out);
  const int grid = grid_for(n, kThreads / 32, di.sm_count, 32);
  embedding_kernel<<<grid, kThreads, 0, s>>>(static_cast<const int*>(idx), static_cast<const uint8_t*>(weight),
                                             static_cast<uint8_t*>(out), n, rows, row_bytes, vec);
  B200K_CHECK_CUDA(cudaGetLastError());
  return B200K_OK;
}
