// GEMM on Hopper (sm_90a): C[M,N] = A[M,K] * B[K,N], fp32 accumulation in registers (wgmma), operands brought into
// 128B-swizzled shared memory by TMA through a 4-stage mbarrier ring.
//
// One CTA computes a 128 x 256 tile of C: warpgroup 0 is the producer (one thread issues the TMA loads), warpgroups 1
// and 2 each own 64 rows of the tile and issue m64n256 wgmma instructions straight from shared memory.  A consumer
// keeps one k-block of MMAs in flight and hands the stage before it back to the producer; that overlap exists in the
// machine code only while the kernel contains no function call, hence mbar_wait_nocall.  128 x 256 x 64 (16-bit) or
// x 32 (fp32) per stage = 48 KB, 4 stages = 192 KB, plus 32 KB of epilogue staging, of the 227 KB a block may use.
// C leaves through that staging buffer and TMA stores.
//
// Operand storage: K-major tiles (A [M,K], B^T [N,K]) and, for 16-bit types, MN-major tiles (A^T [K,M], B [K,N]) are
// consumed in place through the transpose bits of wgmma.  TF32 wgmma reads K-major operands only, so an fp32 B stored
// [K,N] is transposed into a stream-ordered scratch buffer first.
#include "abi_common.cuh"
#include "ptx.cuh"

namespace b200k {

namespace gemm {
constexpr int BM = 128, BN = 256, STAGES = 4, THREADS = 384, GROUP_M = 16;
constexpr int STG_BYTES = 16384;  // epilogue staging per consumer warpgroup: two 64-row x 128-byte TMA boxes
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
  static constexpr int SMEM_BYTES = gemm::STAGES * STAGE_BYTES + 2 * gemm::STG_BYTES + 1024 + 2 * gemm::STAGES * 8;
  static_assert(!(DT == 2 && (A_MN || B_MN)), "tf32 wgmma reads K-major operands only");
  static_assert(SMEM_BYTES <= 232448, "more shared memory than an H100 block may use");
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
    wgmma_ss<Cfg::DT, 256, Cfg::A_MN, Cfg::B_MN>(d, da, db, 1);
  }
}

// Epilogue of one warpgroup: its 64 x 256 accumulators -> C through a 16 KB staging buffer, in column slices (two for
// 16-bit, four for fp32).  Each slice is two 64-row x 128-byte boxes in the 128B-swizzled layout of tmC; TMA clips the
// store to [M, N].  A slice is written only after the store of the one before it has read the buffer.
template <class Cfg>
__device__ __forceinline__ void gemm_store_tile(const float* d, const CUtensorMap* tmC, uint32_t stg, int cw, int row0,
                                                int col0) {
  constexpr int SLICES = Cfg::DT == 2 ? 4 : 2, JS = 32 / SLICES, JB = JS / 2;  // 8-column groups per slice / per box
  const int t = threadIdx.x & 127, lane = t & 31, warp = t / 32;
  const bool leader = t == 0;
#pragma unroll
  for (int sl = 0; sl < SLICES; ++sl) {
    if (leader) tma_store_wait_read<0>();
    named_bar_sync(1 + cw, 128);
    if constexpr (Cfg::DT == 2) {
      // thread owns rows r, r + 8 and column pair 8j + 2q: 8 bytes in 16-byte chunk 2 (j % 4) + q / 2
      const int q = lane & 3;
#pragma unroll
      for (int jj = 0; jj < JS; ++jj) {
        const int j = sl * JS + jj;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = warp * 16 + 8 * h + lane / 4;
          const int chunk = 2 * (jj % JB) + q / 2;
          const uint32_t a = stg + (jj / JB) * 8192 + r * 128 + ((chunk ^ (r & 7)) << 4) + (q & 1) * 8;
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(d[4 * j + 2 * h]), "f"(d[4 * j + 2 * h + 1])
                       : "memory");
        }
      }
    } else {
      // one stmatrix.x4 per two 8-column groups: matrices (rows +0, j), (rows +8, j), (rows +0, j+1), (rows +8, j+1)
      const int m = lane / 8, r = warp * 16 + 8 * (m & 1) + (lane & 7);
#pragma unroll
      for (int jj = 0; jj < JS; jj += 2) {
        const int j = sl * JS + jj, chunk = jj % JB + (m >> 1);
        const uint32_t a = stg + (jj / JB) * 8192 + r * 128 + ((chunk ^ (r & 7)) << 4);
        uint32_t p[4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
          p[i] = Cfg::DT == 1 ? pack_bf162(d[4 * j + 2 * i], d[4 * j + 2 * i + 1])
                              : pack_half2(d[4 * j + 2 * i], d[4 * j + 2 * i + 1]);
        stmatrix_x4(a, p[0], p[1], p[2], p[3]);
      }
    }
    fence_proxy_async_smem();
    named_bar_sync(1 + cw, 128);
    if (leader) {
      const int c = col0 + sl * (gemm::BN / SLICES);
      tma_store_2d(tmC, stg, c, row0);
      tma_store_2d(tmC, stg + 8192, c + 128 / Cfg::ES, row0);
      tma_store_commit();
    }
  }
}

template <class Cfg>
__global__ void __launch_bounds__(gemm::THREADS, 1)
    hgemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const __grid_constant__ CUtensorMap tmC, int K, int tiles_m, int tiles_n) {
  using namespace gemm;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023) & ~1023u;
  const uint32_t stg0 = base + STAGES * Cfg::STAGE_BYTES;
  const uint32_t full0 = stg0 + 2 * STG_BYTES, empty0 = full0 + STAGES * 8;
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

  const int cw = wg - 1, t = threadIdx.x & 127;
  const bool leader = t == 0;
  if (leader) tma_prefetch_desc(&tmC);
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
    if (kb > 0 && leader) mbar_arrive(empty0 + 8 * ((kb - 1) % STAGES));
  }
  wgmma_wait<0>();
  fence_regs<128>(d);
  gemm_store_tile<Cfg>(d, &tmC, stg0 + cw * STG_BYTES, cw, tm * BM + cw * 64, tn * BN);
  if (leader) tma_store_wait_all<0>();
}

template <class Cfg>
static int launch_gemm(const void* A, const void* B, void* C, int64_t M, int64_t N, int64_t K, cudaStream_t s,
                       const DeviceInfo& di) {
  using namespace gemm;
  // every operand is a contiguous row-major [rows, cols] array
  auto tmap = [](CUtensorMap* m, const void* p, int64_t rows, int64_t cols, uint32_t box_rows, uint32_t box_cols) {
    const uint64_t dims[2] = {uint64_t(cols), uint64_t(rows)}, strides[1] = {uint64_t(cols) * Cfg::ES};
    const uint32_t box[2] = {box_cols, box_rows};
    return make_tmap(m, p, Cfg::ES, 2, dims, strides, box);
  };
  CUtensorMap tmA, tmB, tmC;
  int rc = Cfg::A_MN ? tmap(&tmA, A, K, M, Cfg::BK, 64) : tmap(&tmA, A, M, K, BM, Cfg::BK);
  if (rc) return rc;
  rc = Cfg::B_MN ? tmap(&tmB, B, K, N, Cfg::BK, 64) : tmap(&tmB, B, N, K, BN, Cfg::BK);
  if (rc) return rc;
  if ((rc = tmap(&tmC, C, M, N, 64, 128 / Cfg::ES))) return rc;
  const int64_t tiles_m = (M + BM - 1) / BM, tiles_n = (N + BN - 1) / BN, tiles = tiles_m * tiles_n;
  if (tiles > INT32_MAX) return set_error(B200K_ESHAPE, "GEMM too large: %lld tiles", (long long)tiles);
  auto kern = hgemm_wgmma_kernel<Cfg>;
  if ((rc = ensure_dynamic_smem(reinterpret_cast<const void*>(kern), di.device, Cfg::SMEM_BYTES))) return rc;
  kern<<<unsigned(tiles), THREADS, Cfg::SMEM_BYTES, s>>>(tmA, tmB, tmC, int(K), int(tiles_m), int(tiles_n));
  B200K_CHECK_CUDA(cudaGetLastError());
  return B200K_OK;
}

template <int DT>
static int gemm_dispatch(const char* who, const void* A, const void* B, void* C, int64_t M, int64_t N, int64_t K,
                         int b_is_nk, int variant, void* stream, int a_is_km = 0) {
  constexpr int PACK = (DT == 2) ? 4 : 8;  // elements per 16 bytes
  if (!A || !B || !C) return set_error(B200K_EARG, "%s: null pointer", who);
  if (reinterpret_cast<uintptr_t>(C) & 15) return set_error(B200K_EALIGN, "%s: C (%p) must be 16-byte aligned", who, C);
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
