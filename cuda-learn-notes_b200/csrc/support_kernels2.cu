// HBM-roofline support kernels, second set (SURVEY.md section 8f-3): the seven activations, dot product, matrix
// transposes, GEMV (layer norm, also of this set, is an op of the row kernel in support_kernels.cu).  Same recipe as
// support_kernels.cu: coalesced 128-bit accesses, several independent loads in flight per thread, grids sized from the
// SM count, fp32 math on f16 I/O, no tensor cores.
//
// Replaces (reference file:line)
//   kernels/relu/relu.cu:L21-97              kernels/sigmoid/sigmoid.cu:L24-136        kernels/gelu/gelu.cu:L38-163
//   kernels/swish/swish.cu:L20-97            kernels/elu/elu.cu:L35-120                kernels/hardswish/hardswish.cu:L36-140
//   kernels/hardshrink/hardshrink.cu:L33-135 kernels/dot-product/dot_product.cu:L20-184
//   kernels/mat-transpose/mat_transpose.cu:L20-278   kernels/sgemv/sgemv.cu:L20-104    kernels/hgemv/hgemv.cu:L24-108
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <climits>

#include "abi_common.cuh"
#include "support_common.cuh"

namespace b200k {

// ============================================================================================ activations
__device__ __forceinline__ float rcp_fast(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Input clamp of the reference's sigmoid / gelu kernels (sigmoid.cu:L19-22, gelu.cu:L19-22): the f32 kernels limit x
// to +-88.3762626647949, the f16 kernels to [-9.704060527839234, 11.089866488461016] (both as rounded by their type).
template <typename T>
__device__ __forceinline__ float ref_clamp(float x) {
  if constexpr (sizeof(T) == 4) return fminf(fmaxf(x, -88.3762626647949f), 88.3762626647949f);
  else return fminf(fmaxf(x, -9.703125f), 11.09375f);  // the two bounds after rounding to fp16
}

template <typename T, int OP, bool CLAMP>
__device__ __forceinline__ float act(float x) {
  if constexpr (OP == B200K_ACT_RELU) {
    return fmaxf(x, 0.f);
  } else if constexpr (OP == B200K_ACT_SIGMOID) {
    if constexpr (CLAMP) x = ref_clamp<T>(x);
    return rcp_fast(1.0f + exp_sub(-x, 0.f));
  } else if constexpr (OP == B200K_ACT_GELU) {
    // tanh approximation: 0.5 x (1 + tanh(u)), u = sqrt(2/pi) (x + 0.044715 x^3), with e = exp(2u)
    if constexpr (CLAMP) x = ref_clamp<T>(x);
    const float u = 0.7978845608028654f * fmaf(0.044715f * x, x * x, x);
    const float e = exp_sub(2.0f * u, 0.f);
    const float t = rcp_fast(e + 1.0f);
    // (1 + tanh u) / 2 = 1 - 1/(e+1) = e/(e+1): the first form for u >= 0 (e may be +inf), the second for u < 0 (no
    // cancellation when e is tiny)
    return x * (u >= 0.f ? 1.0f - t : e * t);
  } else if constexpr (OP == B200K_ACT_SWISH) {
    return x * rcp_fast(1.0f + exp_sub(-x, 0.f));
  } else if constexpr (OP == B200K_ACT_ELU) {
    return x > 0.f ? x : exp_sub(x, 0.f) - 1.0f;  // alpha = 1 (elu.cu:L19)
  } else if constexpr (OP == B200K_ACT_HARDSWISH) {
    return x >= 3.f ? x : (x <= -3.f ? 0.f : x * (x + 3.f) * (1.0f / 6.0f));
  } else {  // HARDSHRINK, lambda = 0.5 (hardshrink.cu:L19)
    return (x > 0.5f || x < -0.5f) ? x : 0.f;
  }
}

template <typename T, int OP, bool CLAMP>
__global__ void __launch_bounds__(kThreads) activation_kernel(const T* __restrict__ x, T* __restrict__ y, int64_t n,
                                                              bool vec) {
  using IO = RowIO<T>;
  constexpr int VN = IO::N;
  const int64_t stride = int64_t(gridDim.x) * kThreads;
  int64_t done = 0;
  if (vec) {
    // A CTA walks chunks of 4 * kThreads consecutive 16-byte vectors; inside a full chunk the four loads of a thread are
    // at compile-time offsets from one base pointer (no per-load index arithmetic or bounds test).
    const int64_t nvec = n / VN;
    constexpr int64_t CH = 4 * kThreads;
    for (int64_t base = int64_t(blockIdx.x) * CH; base < nvec; base += int64_t(gridDim.x) * CH) {
      const uint4* xv = reinterpret_cast<const uint4*>(x) + base + threadIdx.x;
      uint4* yv = reinterpret_cast<uint4*>(y) + base + threadIdx.x;
      const bool full = base + CH <= nvec;
      const int64_t left = nvec - base - threadIdx.x;  // vectors from this thread's first one to the end
      uint4 u[4];
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (full || k * kThreads < left) u[k] = __ldcs(xv + k * kThreads);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (!full && k * kThreads >= left) break;
        float f[VN];
        IO::unpack(u[k], f);
#pragma unroll
        for (int e = 0; e < VN; ++e) f[e] = act<T, OP, CLAMP>(f[e]);
        __stcs(yv + k * kThreads, IO::pack(f));
      }
    }
    done = nvec * VN;
  }
  for (int64_t i = done + int64_t(blockIdx.x) * kThreads + threadIdx.x; i < n; i += stride)
    y[i] = T(act<T, OP, CLAMP>(float(x[i])));
}

template <typename T, int OP>
static int launch_act2(const void* x, void* y, int64_t n, bool clamp, cudaStream_t s, const DeviceInfo& di) {
  const bool vec = aligned16(x) && aligned16(y);
  const int grid = grid_for(vec ? n / RowIO<T>::N : n, kThreads * 4, di.sm_count, 8);
  const T* xp = static_cast<const T*>(x);
  T* yp = static_cast<T*>(y);
  auto kernel = activation_kernel<T, OP, false>;
  // only sigmoid and gelu have a clamp, and the f32 sigmoid one at +-88.4 cannot change a flush-to-zero fp32 result:
  // skip its two instructions per value
  if constexpr ((OP == B200K_ACT_SIGMOID && sizeof(T) == 2) || OP == B200K_ACT_GELU)
    if (clamp) kernel = activation_kernel<T, OP, true>;
  kernel<<<grid, kThreads, 0, s>>>(xp, yp, n, vec);
  B200K_CHECK_CUDA(cudaGetLastError());
  return B200K_OK;
}
template <typename T>
static int launch_act(const void* x, void* y, int64_t n, int op, bool clamp, cudaStream_t s, const DeviceInfo& di) {
  switch (op) {
    case B200K_ACT_RELU: return launch_act2<T, B200K_ACT_RELU>(x, y, n, clamp, s, di);
    case B200K_ACT_SIGMOID: return launch_act2<T, B200K_ACT_SIGMOID>(x, y, n, clamp, s, di);
    case B200K_ACT_GELU: return launch_act2<T, B200K_ACT_GELU>(x, y, n, clamp, s, di);
    case B200K_ACT_SWISH: return launch_act2<T, B200K_ACT_SWISH>(x, y, n, clamp, s, di);
    case B200K_ACT_ELU: return launch_act2<T, B200K_ACT_ELU>(x, y, n, clamp, s, di);
    case B200K_ACT_HARDSWISH: return launch_act2<T, B200K_ACT_HARDSWISH>(x, y, n, clamp, s, di);
    case B200K_ACT_HARDSHRINK: return launch_act2<T, B200K_ACT_HARDSHRINK>(x, y, n, clamp, s, di);
    default: return set_error(B200K_EARG, "b200k_activation: unknown op %d", op);
  }
}

// ============================================================================================ dot product
// Deterministic two-level reduction (grid_sum), as in b200k_block_all_reduce_sum; the reference finishes with
// atomicAdd(float) in arrival order (dot_product.cu:L52,L76).
template <typename T>
__global__ void __launch_bounds__(kThreads) dot_kernel(const T* __restrict__ a, const T* __restrict__ b,
                                                       float* __restrict__ out, int64_t n, void* __restrict__ workspace,
                                                       bool vec) {
  using IO = RowIO<T>;
  constexpr int VN = IO::N;
  const int64_t stride = int64_t(gridDim.x) * kThreads;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  int64_t done = 0;
  if (vec) {
    const int64_t nvec = n / VN;
    const uint4* av = reinterpret_cast<const uint4*>(a);
    const uint4* bv = reinterpret_cast<const uint4*>(b);
    for (int64_t i = int64_t(blockIdx.x) * kThreads + threadIdx.x; i < nvec; i += 4 * stride) {
      uint4 ua[4], ub[4];
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (i + k * stride < nvec) {
          ua[k] = __ldcs(av + i + k * stride);
          ub[k] = __ldcs(bv + i + k * stride);
        }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (i + k * stride >= nvec) break;
        float fa[VN], fb[VN];
        IO::unpack(ua[k], fa);
        IO::unpack(ub[k], fb);
#pragma unroll
        for (int e = 0; e < VN; ++e) acc[k] = fmaf(fa[e], fb[e], acc[k]);
      }
    }
    done = nvec * VN;
  }
  for (int64_t i = done + int64_t(blockIdx.x) * kThreads + threadIdx.x; i < n; i += stride)
    acc[0] = fmaf(float(a[i]), float(b[i]), acc[0]);
  grid_sum<float>((acc[0] + acc[1]) + (acc[2] + acc[3]), out, workspace);
}

template <typename T>
static int launch_dot(const void* a, const void* b, void* out, int64_t n, void* ws, cudaStream_t s,
                      const DeviceInfo& di) {
  dot_kernel<T><<<reduce_grid(n / RowIO<T>::N, di.sm_count), kThreads, 0, s>>>(
      static_cast<const T*>(a), static_cast<const T*>(b), static_cast<float*>(out), n, ws, aligned16(a) && aligned16(b));
  B200K_CHECK_CUDA(cudaGetLastError());
  return B200K_OK;
}

// ============================================================================================ transposes
// y[b][N,M] = x[b][M,N]^T through a 64 x 64 shared-memory tile (each row padded by one 32-bit word: conflict-free both
// ways); a warp reads and writes whole tile rows.  The reference's 13 fp32 entry points differ only in their index
// arithmetic (mat_transpose.cu:L29-278).  The batched 16-bit form serves the drop-in `*_swizzle_qkv` attention entry
// points for head dims above 128, which receive V as [B,H,D,N] while the FFPA kernel consumes [B,H,N,D].
constexpr int kTile = 64;
template <typename T>  // float, or uint16_t for any 16-bit type
__global__ void __launch_bounds__(kThreads) transpose_kernel(const T* __restrict__ x, T* __restrict__ y, int M, int N,
                                                             int tiles_m, int tiles_n, int64_t tiles) {
  __shared__ T tile[kTile][kTile + 4 / sizeof(T)];
  const int64_t per_batch = int64_t(tiles_m) * tiles_n;
  for (int64_t tidx = blockIdx.x; tidx < tiles; tidx += gridDim.x) {
    const int64_t b = tidx / per_batch;
    const int t = int(tidx - b * per_batch);
    const int m0 = (t / tiles_n) * kTile, n0 = (t % tiles_n) * kTile;
    const T* xb = x + b * int64_t(M) * N;
    T* yb = y + b * int64_t(M) * N;
    const int tx = threadIdx.x % kTile, ty = threadIdx.x / kTile;  // 64 x 4
#pragma unroll 4
    for (int r = ty; r < kTile; r += kThreads / kTile) {
      const int m = m0 + r, nn = n0 + tx;
      if (m < M && nn < N) tile[r][tx] = __ldcs(xb + int64_t(m) * N + nn);
    }
    __syncthreads();
#pragma unroll 4
    for (int r = ty; r < kTile; r += kThreads / kTile) {
      const int nn = n0 + r, m = m0 + tx;
      if (nn < N && m < M) __stcs(yb + int64_t(nn) * M + m, tile[tx][r]);
    }
    __syncthreads();
  }
}

// fp32 with M % 4 == 0, N % 4 == 0 and 16-byte aligned bases: 16-byte loads and stores, all four loads of a thread in
// flight
__global__ void __launch_bounds__(kThreads) transpose_f32x4_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                                   int M, int N, int tiles_n, int64_t tiles) {
  __shared__ float tile[kTile][kTile + 1];
  for (int64_t tidx = blockIdx.x; tidx < tiles; tidx += gridDim.x) {
    const int tm = int(tidx / tiles_n), tn = int(tidx - int64_t(tm) * tiles_n);
    const int m0 = tm * kTile, n0 = tn * kTile;
    float4 v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int idx = threadIdx.x + k * kThreads, r = idx >> 4, c = (idx & 15) * 4;
      if (m0 + r < M && n0 + c < N) v[k] = __ldcs(reinterpret_cast<const float4*>(x + int64_t(m0 + r) * N + n0 + c));
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int idx = threadIdx.x + k * kThreads, r = idx >> 4, c = (idx & 15) * 4;
      tile[r][c] = v[k].x; tile[r][c + 1] = v[k].y; tile[r][c + 2] = v[k].z; tile[r][c + 3] = v[k].w;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int idx = threadIdx.x + k * kThreads, r = idx >> 4, c = (idx & 15) * 4;  // r: column of x, c: row of x
      if (n0 + r < N && m0 + c < M)
        __stcs(reinterpret_cast<float4*>(y + int64_t(n0 + r) * M + m0 + c),
               make_float4(tile[c][r], tile[c + 1][r], tile[c + 2][r], tile[c + 3][r]));
    }
    __syncthreads();
  }
}

// Tiles of a batch of M x N matrices and the grid that walks them, one tile per CTA per pass.
struct TileGrid {
  int tiles_m, tiles_n;
  int64_t tiles;
  int grid;
};
static TileGrid tile_grid(int64_t batch, int64_t M, int64_t N, const DeviceInfo& di) {
  const int tiles_m = int((M + kTile - 1) / kTile), tiles_n = int((N + kTile - 1) / kTile);
  const int64_t tiles = batch * tiles_m * tiles_n;
  return {tiles_m, tiles_n, tiles, grid_for(tiles, 1, di.sm_count, 16)};
}

// ============================================================================================ GEMV
// y[m] = sum_k A[m,k] x[k]: one warp per row, 16-byte loads of the row (streamed) and of x (re-read by every warp, L1 /
// L2 resident), fp32 accumulation, shuffle reduction.  HBM-bound on A.  The reference's k32 / k128 / k16 entry points
// are the same product with different thread mappings (sgemv.cu:L32-104, hgemv.cu:L34-108; hgemv accumulates in half).
template <typename T>
__global__ void __launch_bounds__(kThreads) gemv_kernel(const T* __restrict__ a, const T* __restrict__ x, T* __restrict__ y,
                                                        int64_t M, int K, bool vec) {
  using IO = RowIO<T>;
  constexpr int VN = IO::N;
  const int lane = threadIdx.x & 31;
  const int64_t warps = int64_t(gridDim.x) * (kThreads / 32);
  for (int64_t m = int64_t(blockIdx.x) * (kThreads / 32) + (threadIdx.x >> 5); m < M; m += warps) {
    const T* row = a + m * int64_t(K);
    float acc[2] = {0.f, 0.f};
    int done = 0;
    if (vec) {
      const int nvec = K / VN;
      const uint4* rv = reinterpret_cast<const uint4*>(row);
      const uint4* xv = reinterpret_cast<const uint4*>(x);
      for (int i = lane; i < nvec; i += 64) {
        uint4 u0 = __ldcs(rv + i), u1;
        const bool two = i + 32 < nvec;
        if (two) u1 = __ldcs(rv + i + 32);
        float fa[VN], fx[VN];
        IO::unpack(u0, fa);
        IO::unpack(__ldg(xv + i), fx);
#pragma unroll
        for (int e = 0; e < VN; ++e) acc[0] = fmaf(fa[e], fx[e], acc[0]);
        if (two) {
          IO::unpack(u1, fa);
          IO::unpack(__ldg(xv + i + 32), fx);
#pragma unroll
          for (int e = 0; e < VN; ++e) acc[1] = fmaf(fa[e], fx[e], acc[1]);
        }
      }
      done = nvec * VN;
    }
    for (int k = done + lane; k < K; k += 32) acc[0] = fmaf(float(row[k]), float(x[k]), acc[0]);
    const float r = warp_sum(acc[0] + acc[1]);
    if (lane == 0) y[m] = T(r);
  }
}

}  // namespace b200k

// ================================================================================================ C ABI
using namespace b200k;

extern "C" int b200k_activation(const void* x, void* y, int64_t n, int dtype, int op, int ref_clamp, void* stream) {
  if ((!x || !y) && n > 0) return set_error(B200K_EARG, "b200k_activation: null pointer");
  if (n < 0) return set_error(B200K_ESHAPE, "b200k_activation: n < 0");
  if (n == 0) return B200K_OK;
  DeviceInfo di;
  int rc = get_device_info(&di);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  switch (dtype) {
    case B200K_F32: return launch_act<float>(x, y, n, op, ref_clamp != 0, s, di);
    case B200K_F16: return launch_act<__half>(x, y, n, op, ref_clamp != 0, s, di);
    default: return set_error(B200K_EDTYPE, "b200k_activation: dtype %d not supported (f32, f16)", dtype);
  }
}

extern "C" int b200k_dot_prod(const void* a, const void* b, void* out, int64_t n, int dtype, void* workspace,
                              void* stream) {
  if (!out || !workspace || ((!a || !b) && n > 0)) return set_error(B200K_EARG, "b200k_dot_prod: null pointer");
  if (n < 0) return set_error(B200K_ESHAPE, "b200k_dot_prod: n < 0");
  DeviceInfo di;
  int rc = get_device_info(&di);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype != B200K_F32 && dtype != B200K_F16)
    return set_error(B200K_EDTYPE, "b200k_dot_prod: dtype %d not supported (f32, f16)", dtype);
  if ((rc = zero_ticket(workspace, s))) return rc;
  return dtype == B200K_F32 ? launch_dot<float>(a, b, out, n, workspace, s, di)
                            : launch_dot<__half>(a, b, out, n, workspace, s, di);
}

extern "C" int b200k_mat_transpose_f32(const void* x, void* y, int64_t M, int64_t N, void* stream) {
  if (!x || !y) return set_error(B200K_EARG, "b200k_mat_transpose_f32: null pointer");
  if (M < 1 || N < 1 || M > INT32_MAX || N > INT32_MAX)
    return set_error(B200K_ESHAPE, "b200k_mat_transpose_f32: need 1 <= M, N < 2^31");
  DeviceInfo di;
  int rc = get_device_info(&di);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const TileGrid g = tile_grid(1, M, N, di);
  const float* xp = static_cast<const float*>(x);
  float* yp = static_cast<float*>(y);
  if (M % 4 == 0 && N % 4 == 0 && aligned16(x) && aligned16(y))
    transpose_f32x4_kernel<<<g.grid, kThreads, 0, s>>>(xp, yp, int(M), int(N), g.tiles_n, g.tiles);
  else
    transpose_kernel<float><<<g.grid, kThreads, 0, s>>>(xp, yp, int(M), int(N), g.tiles_m, g.tiles_n, g.tiles);
  B200K_CHECK_CUDA(cudaGetLastError());
  return B200K_OK;
}

extern "C" int b200k_transpose_u16_batched(const void* x, void* y, int64_t batch, int64_t M, int64_t N, void* stream) {
  if (!x || !y) return set_error(B200K_EARG, "b200k_transpose_u16_batched: null pointer");
  if (batch < 1 || M < 1 || N < 1 || M > INT32_MAX || N > INT32_MAX)
    return set_error(B200K_ESHAPE, "b200k_transpose_u16_batched: need batch >= 1, 1 <= M, N < 2^31");
  DeviceInfo di;
  int rc = get_device_info(&di);
  if (rc) return rc;
  const TileGrid g = tile_grid(batch, M, N, di);
  transpose_kernel<uint16_t><<<g.grid, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint16_t*>(x), static_cast<uint16_t*>(y), int(M), int(N), g.tiles_m, g.tiles_n, g.tiles);
  B200K_CHECK_CUDA(cudaGetLastError());
  return B200K_OK;
}

extern "C" int b200k_gemv(const void* a, const void* x, void* y, int64_t M, int64_t K, int dtype, void* stream) {
  if (!a || !x || !y) return set_error(B200K_EARG, "b200k_gemv: null pointer");
  if (M < 1 || K < 1 || K > INT32_MAX) return set_error(B200K_ESHAPE, "b200k_gemv: need M >= 1, 1 <= K < 2^31");
  DeviceInfo di;
  int rc = get_device_info(&di);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int grid = grid_for(M, kThreads / 32, di.sm_count, 8);
  if (dtype == B200K_F32) {
    const bool vec = (K % 4 == 0) && aligned16(a) && aligned16(x);
    gemv_kernel<float><<<grid, kThreads, 0, s>>>(static_cast<const float*>(a), static_cast<const float*>(x),
                                                 static_cast<float*>(y), M, int(K), vec);
  } else if (dtype == B200K_F16) {
    const bool vec = (K % 8 == 0) && aligned16(a) && aligned16(x);
    gemv_kernel<__half><<<grid, kThreads, 0, s>>>(static_cast<const __half*>(a), static_cast<const __half*>(x),
                                                  static_cast<__half*>(y), M, int(K), vec);
  } else {
    return set_error(B200K_EDTYPE, "b200k_gemv: dtype %d not supported (f32, f16)", dtype);
  }
  B200K_CHECK_CUDA(cudaGetLastError());
  return B200K_OK;
}
