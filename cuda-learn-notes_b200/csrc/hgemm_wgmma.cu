// GEMM on Hopper (sm_90a): C[M,N] = A[M,K] * B[K,N], fp32 accumulation in registers (wgmma), operands brought into
// 128B-swizzled shared memory by TMA through a 4-stage mbarrier ring.
//
// One CTA computes a 128 x 256 tile of C: warpgroup 0 is the producer (one thread issues the TMA loads), warpgroups 1
// and 2 each own 64 rows of the tile and issue m64n256 wgmma instructions straight from shared memory.  A consumer
// keeps one k-block of MMAs in flight and hands the stage before it back to the producer; that overlap exists in the
// machine code only while the kernel contains no function call, hence mbar_wait_nocall.  128 x 256 x 64 (16-bit) or
// x 32 (fp32) per stage = 48 KB, 4 stages = 192 KB of the 227 KB a block may use on H100.
//
// Operand storage: K-major tiles (A [M,K], B^T [N,K]) and, for 16-bit types, MN-major tiles (A^T [K,M], B [K,N]) are
// consumed in place through the transpose bits of wgmma.  TF32 wgmma reads K-major operands only, so an fp32 B stored
// [K,N] is transposed into a stream-ordered scratch buffer first.
#include "abi_common.cuh"
#include "ptx.cuh"

namespace b200k {

namespace gemm {
constexpr int BM = 128, BN = 256, STAGES = 4, THREADS = 384, GROUP_M = 16;
}

template <int DT_, bool A_MN_, bool B_MN_>  // DT: 0 f16, 1 bf16, 2 tf32 (fp32 storage)
struct GemmCfg {
  static constexpr int DT = DT_;
  static constexpr bool A_MN = A_MN_, B_MN = B_MN_;
  static constexpr int ES = DT == 2 ? 4 : 2;
  static constexpr int BK = 128 / ES;  // one 128-byte swizzle row of K
  static constexpr int KSTEP = DT == 2 ? 8 : 16;
  static constexpr int A_BYTES = gemm::BM * BK * ES;
  static constexpr int B_BYTES = gemm::BN * BK * ES;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int SMEM_BYTES = gemm::STAGES * STAGE_BYTES + 1024 + 2 * gemm::STAGES * 8;
  static_assert(!(DT == 2 && (A_MN || B_MN)), "tf32 wgmma reads K-major operands only");
};

template <class Cfg>
__device__ __forceinline__ void gemm_mma_kblock(float* d, uint32_t sA, uint32_t sB, int cw) {
  constexpr int STEPS = Cfg::BK / Cfg::KSTEP;
#pragma unroll
  for (int k = 0; k < STEPS; ++k) {
    // A: this warpgroup's 64 rows.  K-major: rows at 128 B; MN-major: its own 64-column box, K rows at 128 B.
    const uint64_t da = Cfg::A_MN ? wgmma_desc(sA + cw * 64 * Cfg::BK * Cfg::ES + k * 2048, 64 * Cfg::BK * Cfg::ES, 1024)
                                  : wgmma_desc(sA + cw * 64 * 128 + k * 32, 16, 1024);
    const uint64_t db = Cfg::B_MN ? wgmma_desc(sB + k * 2048, 64 * Cfg::BK * Cfg::ES, 1024) : wgmma_desc(sB + k * 32, 16, 1024);
    if constexpr (Cfg::DT == 2) {
      wgmma_ss_tf32_n256(d, da, db, 1);
    } else if constexpr (Cfg::DT == 1) {
      wgmma_ss_bf16_n256<Cfg::A_MN ? 1 : 0, Cfg::B_MN ? 1 : 0>(d, da, db, 1);
    } else {
      wgmma_ss_f16_n256<Cfg::A_MN ? 1 : 0, Cfg::B_MN ? 1 : 0>(d, da, db, 1);
    }
  }
}

template <class Cfg>
__global__ void __launch_bounds__(gemm::THREADS, 1)
    hgemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, void* C, int M,
                       int N, int K, int tiles_m, int tiles_n) {
  using namespace gemm;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023) & ~1023u;
  const uint32_t full0 = base + STAGES * Cfg::STAGE_BYTES, empty0 = full0 + STAGES * 8;
  const int wg = threadIdx.x / 128;

  // grouped rasterisation: GROUP_M row tiles share each B column tile while it is in L2
  const int tile = blockIdx.x, width = GROUP_M * tiles_n, g = tile / width, first_m = g * GROUP_M;
  const int gsz = min(tiles_m - first_m, GROUP_M);
  const int tm = first_m + (tile % width) % gsz, tn = (tile % width) / gsz;
  const int nkb = (K + Cfg::BK - 1) / Cfg::BK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, 2);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    if (threadIdx.x == 0) {
      tma_prefetch_desc(&tmA);
      tma_prefetch_desc(&tmB);
      for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % STAGES;
        if (kb >= STAGES) mbar_wait_nocall(empty0 + 8 * s, ((kb / STAGES) - 1) & 1);
        const uint32_t bar = full0 + 8 * s, sA = base + s * Cfg::STAGE_BYTES, sB = sA + Cfg::A_BYTES;
        mbar_arrive_expect_tx(bar, Cfg::STAGE_BYTES);
        if constexpr (Cfg::A_MN) {
#pragma unroll
          for (int c = 0; c < BM / 64; ++c)
            tma_load_2d(sA + c * 64 * Cfg::BK * Cfg::ES, &tmA, bar, tm * BM + c * 64, kb * Cfg::BK, kPolicyEvictNormal);
        } else {
          tma_load_2d(sA, &tmA, bar, kb * Cfg::BK, tm * BM, kPolicyEvictNormal);
        }
        if constexpr (Cfg::B_MN) {
#pragma unroll
          for (int c = 0; c < BN / 64; ++c)
            tma_load_2d(sB + c * 64 * Cfg::BK * Cfg::ES, &tmB, bar, tn * BN + c * 64, kb * Cfg::BK, kPolicyEvictNormal);
        } else {
          tma_load_2d(sB, &tmB, bar, kb * Cfg::BK, tn * BN, kPolicyEvictNormal);
        }
      }
    }
    return;
  }

  const int cw = wg - 1;
  float d[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) d[i] = 0.f;
  for (int kb = 0; kb < nkb; ++kb) {
    const int s = kb % STAGES;
    mbar_wait_nocall(full0 + 8 * s, (kb / STAGES) & 1);
    const uint32_t sA = base + s * Cfg::STAGE_BYTES, sB = sA + Cfg::A_BYTES;
    fence_regs<128>(d);
    wgmma_fence();
    gemm_mma_kblock<Cfg>(d, sA, sB, cw);
    wgmma_commit();
    wgmma_wait<1>();  // the previous k-block's MMAs are done: its stage can be refilled
    fence_regs<128>(d);
    if (kb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(empty0 + 8 * ((kb - 1) % STAGES));
  }
  wgmma_wait<0>();
  fence_regs<128>(d);

  // epilogue: accumulator fragment -> global, clipped to [M, N].  Thread owns rows r0, r0 + 8 and column pairs 8j + 2q.
  const int lane = threadIdx.x & 31, warp = (threadIdx.x & 127) / 32;
  const int r0 = tm * BM + cw * 64 + warp * 16 + lane / 4;
  const int c0 = tn * BN + 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r0 + 8 * h;
    if (r >= M) continue;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int c = c0 + 8 * j;
      if (c >= N) continue;  // N is even, so c + 1 < N as well
      const float x = d[4 * j + 2 * h], y = d[4 * j + 2 * h + 1];
      const size_t off = size_t(r) * N + c;
      if constexpr (Cfg::DT == 2) {
        *reinterpret_cast<float2*>(static_cast<float*>(C) + off) = make_float2(x, y);
      } else if constexpr (Cfg::DT == 1) {
        *reinterpret_cast<uint32_t*>(static_cast<__nv_bfloat16*>(C) + off) = pack_bf162(x, y);
      } else {
        *reinterpret_cast<uint32_t*>(static_cast<__half*>(C) + off) = pack_half2(x, y);
      }
    }
  }
}

template <class Cfg>
static int launch_gemm(const void* A, const void* B, void* C, int64_t M, int64_t N, int64_t K, cudaStream_t s,
                       const DeviceInfo& di) {
  using namespace gemm;
  CUtensorMap tmA, tmB;
  int rc = Cfg::A_MN ? make_tmap_2d(&tmA, A, K, M, M, Cfg::BK, 64, Cfg::ES)
                     : make_tmap_2d(&tmA, A, M, K, K, BM, Cfg::BK, Cfg::ES);
  if (rc) return rc;
  rc = Cfg::B_MN ? make_tmap_2d(&tmB, B, K, N, N, Cfg::BK, 64, Cfg::ES) : make_tmap_2d(&tmB, B, N, K, K, BN, Cfg::BK, Cfg::ES);
  if (rc) return rc;
  const int64_t tiles_m = (M + BM - 1) / BM, tiles_n = (N + BN - 1) / BN;
  if (tiles_m * tiles_n > INT32_MAX) return set_error(B200K_ESHAPE, "GEMM too large: %lld tiles", (long long)(tiles_m * tiles_n));
  auto kern = hgemm_wgmma_kernel<Cfg>;
  if ((rc = ensure_dynamic_smem(reinterpret_cast<const void*>(kern), di.device, Cfg::SMEM_BYTES))) return rc;
  kern<<<unsigned(tiles_m * tiles_n), THREADS, Cfg::SMEM_BYTES, s>>>(tmA, tmB, C, int(M), int(N), int(K), int(tiles_m),
                                                                      int(tiles_n));
  B200K_CHECK_CUDA(cudaGetLastError());
  return B200K_OK;
}

template <int DT>
static int gemm_dispatch(const char* who, const void* A, const void* B, void* C, int64_t M, int64_t N, int64_t K,
                         int b_is_nk, int variant, void* stream, int a_is_km = 0) {
  constexpr int PACK = (DT == 2) ? 4 : 8;  // elements per 16 bytes
  if (!A || !B || !C) return set_error(B200K_EARG, "%s: null pointer", who);
  if (M < 1 || N < 1 || K < 1 || M > INT32_MAX || N > INT32_MAX || K > INT32_MAX)
    return set_error(B200K_ESHAPE, "%s: M,N,K must be in [1, 2^31) (got %lld,%lld,%lld)", who, (long long)M, (long long)N,
                     (long long)K);
  if ((K % PACK) || (N % PACK))
    return set_error(B200K_ESHAPE, "%s: K and N must be multiples of %d (16-byte rows), got K=%lld N=%lld", who, PACK,
                     (long long)K, (long long)N);
  if (a_is_km && DT == 2) return set_error(B200K_EDTYPE, "%s: A stored as [K,M] is built for f16 / bf16 only", who);
  if (a_is_km && (M % PACK))
    return set_error(B200K_ESHAPE, "%s: M must be a multiple of %d when A is stored as [K,M]", who, PACK);
  const int v = variant & 0xff;
  if (v < B200K_HGEMM_AUTO || v > B200K_HGEMM_2CTA_512x256)
    return set_error(B200K_EARG, "%s: variant %d unknown", who, v);
  DeviceInfo di;
  int rc = get_device_info(&di);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool nn = (b_is_nk == 0);
  if constexpr (DT == 2) {
    if (!nn) return launch_gemm<GemmCfg<2, false, false>>(A, B, C, M, N, K, s, di);
    // fp32 B stored [K,N]: transpose to [N,K] in a scratch buffer that lives on the stream
    void* bt = nullptr;
    B200K_CHECK_CUDA(cudaMallocAsync(&bt, size_t(K) * size_t(N) * 4, s));
    rc = b200k_mat_transpose_f32(B, bt, K, N, stream);
    if (!rc) rc = launch_gemm<GemmCfg<2, false, false>>(A, bt, C, M, N, K, s, di);
    cudaError_t e = cudaFreeAsync(bt, s);
    if (!rc && e != cudaSuccess) rc = set_error(B200K_ECUDA, "cudaFreeAsync failed: %s", cudaGetErrorString(e));
    return rc;
  } else {
    if (a_is_km)
      return nn ? launch_gemm<GemmCfg<DT, true, true>>(A, B, C, M, N, K, s, di)
                : launch_gemm<GemmCfg<DT, true, false>>(A, B, C, M, N, K, s, di);
    return nn ? launch_gemm<GemmCfg<DT, false, true>>(A, B, C, M, N, K, s, di)
              : launch_gemm<GemmCfg<DT, false, false>>(A, B, C, M, N, K, s, di);
  }
}

}  // namespace b200k

extern "C" int b200k_hgemm_f16(const void* A, const void* B, void* C, int64_t M, int64_t N, int64_t K, int b_is_nk,
                               int variant, void* stream) {
  return b200k::gemm_dispatch<0>("b200k_hgemm_f16", A, B, C, M, N, K, b_is_nk, variant, stream);
}

extern "C" int b200k_gemm_ex(const void* A, const void* B, void* C, int64_t M, int64_t N, int64_t K, int a_is_km, int b_is_nk,
                             int dtype, int variant, void* stream) {
  switch (dtype) {
    case B200K_F16: return b200k::gemm_dispatch<0>("b200k_gemm_ex(f16)", A, B, C, M, N, K, b_is_nk, variant, stream, a_is_km);
    case B200K_BF16: return b200k::gemm_dispatch<1>("b200k_gemm_ex(bf16)", A, B, C, M, N, K, b_is_nk, variant, stream, a_is_km);
    case B200K_F32: return b200k::gemm_dispatch<2>("b200k_gemm_ex(tf32)", A, B, C, M, N, K, b_is_nk, variant, stream, a_is_km);
    default: return b200k::set_error(B200K_EDTYPE, "b200k_gemm_ex: dtype %d not supported (f16, bf16, f32-as-tf32)", dtype);
  }
}

extern "C" int b200k_gemm(const void* A, const void* B, void* C, int64_t M, int64_t N, int64_t K, int b_is_nk, int dtype,
                          int variant, void* stream) {
  switch (dtype) {
    case B200K_F16: return b200k::gemm_dispatch<0>("b200k_gemm(f16)", A, B, C, M, N, K, b_is_nk, variant, stream);
    case B200K_BF16: return b200k::gemm_dispatch<1>("b200k_gemm(bf16)", A, B, C, M, N, K, b_is_nk, variant, stream);
    case B200K_F32: return b200k::gemm_dispatch<2>("b200k_gemm(tf32)", A, B, C, M, N, K, b_is_nk, variant, stream);
    default: return b200k::set_error(B200K_EDTYPE, "b200k_gemm: dtype %d not supported (f16, bf16, f32-as-tf32)", dtype);
  }
}
