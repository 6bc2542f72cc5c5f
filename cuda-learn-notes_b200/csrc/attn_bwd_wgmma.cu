// Attention backward on Hopper (sm_90a), dense [B, H, N, D] or packed [tokens, H, D] with grouped K/V heads: dQ, dK and dV of O = softmax(Q K^T * scale) V from Q, K,
// V, O, dO and the forward's log-sum-exp (b200k_fa2_fwd_lse), the FlashAttention-2 algorithm with every output element
// summed in one thread's registers, so the result is deterministic without atomics.  Three kernels, in stream order:
//   prep    Delta_i = sum_d dO_id O_id and lse_i * log2 e into the workspace (bandwidth kernel, no tensor cores)
//   dK/dV   one CTA per (64-key tile, b * H + h); K and V resident, Q / dO tiles of 64 rows streamed through a TMA +
//           mbarrier ring.  One consumer warpgroup owns the 64 keys:
//             S^T = K Q_i^T, dP^T = V dO_i^T   wgmma_ss, K-major operands
//             P^T = 2^(S^T scale log2 e - lse_i log2 e), dS^T = P^T (dP^T - Delta_i), in registers
//             dV += P~^T dO_i, dK += dS~^T Q_i  wgmma_rs (the accumulator fragment of S^T / dP^T is the A fragment),
//                                               dO_i and Q_i read MN-major as V is in the forward's P V
//   dQ      one CTA per (128-row query tile, b * H + h), the forward's geometry and its AttnDense addressing; Q and dO
//           resident, K / V tiles of 64 keys streamed.  Two consumer warpgroups of 64 rows: S = Q K_j^T,
//           dP = dO V_j^T, P, dS, dQ += dS~ K_j (K read MN-major)
// P~ and dS~ are P and dS rounded to the 16-bit dtype.  S and dP are computed by both the dK/dV and the dQ kernel:
// 7 products where an atomic-dQ backward needs 5, the price of determinism.
// The dK/dV warpgroup holds dK, dV (2 x DP / 2 fp32) and S^T, dP^T (2 x 32): 192 at DP = 128, more than a 384-thread
// block gives a thread (168), so it runs one consumer warpgroup in a 256-thread block.
// Packed sequences (b200k_fa2_bwd_varlen) run the same three kernels: the prep also zero-fills the gradients of tokens
// outside every sequence, the dK/dV kernel takes BwdKeysPacked (a CTA owns 64 keys of one K/V head and loops over the
// query tiles of every query head of its group, so dK / dV sum over the group in registers), and the dQ kernel takes
// the forward's AttnPacked.
#include "attn_common.cuh"

#include <climits>
#include <cmath>

namespace b200k {

// The dK/dV kernel's config is AttnCfg<DT, DP, 1, 64, false> (BM = BN = 64, 256 threads), the dQ kernel's
// AttnCfg<DT, DP, 2, 64, false> (BM = 128 rows, BN = 64 keys, 384 threads).  DP is the head dim padded to whole 64-column
// chunks (64 for D = 32 / 64, 128 for D = 96 / 128); TMA zero-fills the padding.
constexpr int kBwdStages = 2;
template <class KvCfg>
using BwdQCfg = AttnCfg<KvCfg::DT, KvCfg::DV, 2, 64, false>;

// A packed gradient tensor viewed as [total, width] 32-bit words, and its cumulative sequence offsets.
struct BwdPackedGrad {
  void* p;
  const int* cu;
  long long total, width;
};

// Zeroes the rows of tokens outside every sequence (before cu[0], from cu[B] on), which no main kernel stores.
__device__ __forceinline__ void zero_outside(const BwdPackedGrad g, int B) {
  const long long lo = min(max((long long)__ldg(g.cu), 0ll), g.total), hi = min(max((long long)__ldg(g.cu + B), lo), g.total);
  const long long n = (lo + g.total - hi) * g.width, stride = (long long)gridDim.x * blockDim.x;
#pragma unroll 1  // an unrolled loop's 64-bit trip count would be a division: a call
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += stride)
    static_cast<uint32_t*>(g.p)[i < lo * g.width ? i : (hi - lo) * g.width + i] = 0u;
}

// Delta[row] = sum_d dO[row, d] O[row, d] and lse2[row] = lse[row] * log2 e, one row per quad of threads, 16-byte loads,
// each thread's products summed in column order, then across the quad in a fixed order.  PACKED: a row that sees no key
// (lse = -inf) gets lse2 = +inf, so its P is exactly 0 against a masked score too (2^(-inf + inf) would be NaN); then
// the zeros of dQ, dK and dV outside the B sequences.  The dense layout passes no sequences.
template <int DT, bool PACKED>
__global__ void __launch_bounds__(256) attn_bwd_prep_kernel(
    const uint16_t* __restrict__ O, const uint16_t* __restrict__ dO, const float* __restrict__ lse,
    float* __restrict__ delta, float* __restrict__ lse2, long long rows, int D, int B, const BwdPackedGrad dq,
    const BwdPackedGrad dk, const BwdPackedGrad dv) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const int t = threadIdx.x & 3, lane = threadIdx.x & 31;
  // the loop bound is the same for the whole warp (its first thread's index), so the shuffles see every lane
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i - lane < rows * 4; i += stride) {
    const long long row = i / 4;
    float acc = 0.f;
    if (row < rows)
      for (int v = t; v < D / 8; v += 4) {
        const uint4 a = __ldg(reinterpret_cast<const uint4*>(O + row * D) + v);
        const uint4 b = __ldg(reinterpret_cast<const uint4*>(dO + row * D) + v);
        const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          float2 x, y;
          if constexpr (DT == 0) {
            x = __half22float2(*reinterpret_cast<const __half2*>(&aw[k]));
            y = __half22float2(*reinterpret_cast<const __half2*>(&bw[k]));
          } else {
            x = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&aw[k]));
            y = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&bw[k]));
          }
          acc = fmaf(x.x, y.x, acc);
          acc = fmaf(x.y, y.y, acc);
        }
      }
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    if (row < rows && t == 0) {
      delta[row] = acc;
      const float l = lse[row];
      lse2[row] = PACKED && l == -INFINITY ? INFINITY : l * 1.4426950408889634f;
    }
  }
  if constexpr (PACKED) {
    zero_outside(dq, B);
    zero_outside(dk, B);
    zero_outside(dv, B);
  }
}

// What both main kernels take beyond their tensor maps.
struct BwdArgs {
  const float* lse2;   // [B * H * N] (packed: [total_q * H]) lse * log2 e
  const float* delta;  // the same rows
  void* dst[2];        // dK / dV kernel: dK, dV; dQ kernel: dQ
  int D;
  float scale_log2, scale;
};

// The addressing modes of the dK/dV kernel.  Each places CTA (x, y) = (key tile, y), loads its K / V tile and its query
// tiles, and gives the causal diagonal, the row statistics and the store row of a key.  `group` query heads share the
// CTA's K / V head.

// Dense: y = b * H + h.  Every key < N is stored: keys past seqlens_k (clamped to [1, N]) are masked, so they store
// zeros, and a key tile past it sees no query tile.  Rows past N (ragged N) have zero-filled Q and dO; lse2 = +inf
// there makes their P exactly 0.
template <class Cfg>
struct BwdKeysDense {
  static constexpr int group = 1;
  const int* seqlens;  // int32 [B] valid keys per batch, or null
  int N, H, causal;

  struct Cta { int bh, k0, kv_len, first, end; };
  __device__ __forceinline__ bool setup(Cta& c) const {
    c.bh = blockIdx.y;
    c.k0 = blockIdx.x * 64;
    c.kv_len = seqlens ? min(max(__ldg(seqlens + c.bh / H), 1), N) : N;
    // query tiles that see a key of this tile: all of them, from the one holding row k0 when causal; none past the length
    c.first = causal ? c.k0 / 64 : 0;
    c.end = c.k0 < c.kv_len ? (N + 63) / 64 : c.first;
    return true;
  }
  __device__ __forceinline__ void load_kv(const Cta& c, uint32_t dst, const CUtensorMap* tm, uint32_t bar,
                                          int chunk) const {
    tma_load_3d(dst, tm, bar, chunk * 64, c.k0, c.bh, kPolicyEvictFirst);
  }
  __device__ __forceinline__ void load_q(const Cta& c, int, int i, uint32_t dst, const CUtensorMap* tm, uint32_t bar,
                                         int chunk) const {
    tma_load_3d(dst, tm, bar, chunk * 64, i * 64, c.bh, kPolicyEvictNormal);
  }
  __device__ __forceinline__ int diag(const Cta&, int r) const { return r; }
  __device__ __forceinline__ void zero_q_tail(const Cta&, int, uint32_t) const {}
  __device__ __forceinline__ void row_stats(const BwdArgs& a, const Cta& c, int, int r, float& l2, float& dl) const {
    const size_t base = size_t(c.bh) * N;
    l2 = r < N ? __ldg(a.lse2 + base + r) : INFINITY;
    dl = r < N ? __ldg(a.delta + base + r) : 0.f;
  }
  __device__ __forceinline__ bool key_row(const Cta& c, int k, size_t& row) const {
    if (k >= N) return false;
    row = size_t(c.bh) * N + k;
    return true;
  }
};

// Packed (AttnPacked's layout): y = b * H_kv + K/V head; the CTA visits the query tiles of each query head
// h = K/V head * group + g of its group in turn, g ascending.  A key tile past Lk returns.  A query tile that runs past
// Lq reads the next sequence's rows: their lse2 is +inf, so their P and dS are 0, and zero_q_tail zeroes their Q and
// dO, which P^T and dS^T multiply.  Keys past Lk are masked and not
// stored.  Row r sees keys <= r + Lk - Lq under the causal mask.  The store reloads cu_k rather than keep it through the
// main loop.
template <class Cfg>
struct BwdKeysPacked {
  const int* cu_q;
  const int* cu_k;
  int H, H_kv, group, causal;

  struct Cta { int kvh, k0, kv_len, first, end, q_tok, q_len, shift; };  // q_tok: first query token; shift: Lk - Lq
  __device__ __forceinline__ bool setup(Cta& c) const {
    const int b = blockIdx.y / H_kv, k_tok = __ldg(cu_k + b);
    c.kvh = blockIdx.y % H_kv;
    c.k0 = blockIdx.x * 64;
    c.kv_len = __ldg(cu_k + b + 1) - k_tok;
    if (c.k0 >= c.kv_len) return false;
    c.q_tok = __ldg(cu_q + b);
    c.q_len = __ldg(cu_q + b + 1) - c.q_tok;
    c.shift = c.kv_len - c.q_len;
    // query tiles that see a key of this tile: from the one holding row k0 - shift when causal, to the last
    c.first = causal ? max(c.k0 - c.shift, 0) / 64 : 0;
    c.end = max((c.q_len + 63) / 64, c.first);
    return true;
  }
  __device__ __forceinline__ void load_kv(const Cta& c, uint32_t dst, const CUtensorMap* tm, uint32_t bar,
                                          int chunk) const {
    tma_load_3d(dst, tm, bar, chunk * 64, c.kvh, __ldg(cu_k + blockIdx.y / H_kv) + c.k0, kPolicyEvictFirst);
  }
  __device__ __forceinline__ void load_q(const Cta& c, int g, int i, uint32_t dst, const CUtensorMap* tm, uint32_t bar,
                                         int chunk) const {
    tma_load_3d(dst, tm, bar, chunk * 64, c.kvh * group + g, c.q_tok + i * 64, kPolicyEvictNormal);
  }
  __device__ __forceinline__ int diag(const Cta& c, int r) const { return r + c.shift; }
  // the Q and dO rows of query tile q0 past Lq, which S^T / dP^T hold as P^T = 0 columns that still multiply them
  __device__ __forceinline__ void zero_q_tail(const Cta& c, int q0, uint32_t sq) const {
    zero_tile_tail<Cfg>(c.q_len, q0, sq);
    zero_tile_tail<Cfg>(c.q_len, q0, sq + 64 * Cfg::DV * 2);
  }
  __device__ __forceinline__ void row_stats(const BwdArgs& a, const Cta& c, int g, int r, float& l2, float& dl) const {
    const size_t row = size_t(c.q_tok + r) * H + c.kvh * group + g;
    l2 = r < c.q_len ? __ldg(a.lse2 + row) : INFINITY;
    dl = r < c.q_len ? __ldg(a.delta + row) : 0.f;
  }
  __device__ __forceinline__ bool key_row(const Cta& c, int k, size_t& row) const {
    if (k >= c.kv_len) return false;
    row = size_t(__ldg(cu_k + blockIdx.y / H_kv) + k) * H_kv + c.kvh;
    return true;
  }
};

// dK, dV of one 64-key tile, placed and fed by Mode (BwdKeysDense or BwdKeysPacked).  Warpgroup 0 produces (one thread
// issues TMA), warpgroup 1 computes; thread rows (keys) k0 + 16 warp + lane / 4 and + 8, columns (queries)
// q0 + 8 j + 2 (lane % 4) + e.  The query tiles of the group's heads stream through one ring, head by head; dK and dV
// sum over all of them in this thread's registers.
template <class Cfg, class Mode>
__global__ void __launch_bounds__(Cfg::THREADS, 1)
    attn_bwd_dkdv_kernel(const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                         const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmdO,
                         const BwdArgs a, const Mode md) {
  static_assert(Cfg::NWG == 1 && Cfg::BM == 64 && Cfg::BN == 64, "dK/dV: one warpgroup of 64 keys, query tiles of 64");
  constexpr int DP = Cfg::DV, NC = DP / 64, TILE = 64 * DP * 2, ST = kBwdStages;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sK = (smem_u32(smem_raw) + 1023) & ~1023u, sV = sK + TILE, sQ = sV + TILE;  // stage s: Q, then dO
  const uint32_t kvbar = sQ + ST * 2 * TILE, full = kvbar + 8, empty = full + 8 * ST;

  typename Mode::Cta c;
  if (!md.setup(c)) return;
  const int k0 = c.k0, first = c.first, end = c.end;
  const int wg = threadIdx.x / 128;

  if (threadIdx.x == 0) {
    mbar_init(kvbar, 1);
    for (int s = 0; s < ST; ++s) {
      mbar_init(full + 8 * s, 1);
      mbar_init(empty + 8 * s, 1);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    if (threadIdx.x == 0 && first < end) {
      mbar_arrive_expect_tx(kvbar, 2 * TILE);
      for (int ch = 0; ch < NC; ++ch) {
        md.load_kv(c, sK + ch * 8192, &tmK, kvbar, ch);
        md.load_kv(c, sV + ch * 8192, &tmV, kvbar, ch);
      }
      for (int g = 0; g < md.group; ++g)
        for (int i = first; i < end; ++i) {
          const int n = g * (end - first) + i - first, s = n % ST;
          if (n >= ST) mbar_wait_nocall(empty + 8 * s, ((n / ST) - 1) & 1);
          mbar_arrive_expect_tx(full + 8 * s, 2 * TILE);
          const uint32_t q = sQ + s * 2 * TILE;
          for (int ch = 0; ch < NC; ++ch) {
            md.load_q(c, g, i, q + ch * 8192, &tmQ, full + 8 * s, ch);
            md.load_q(c, g, i, q + TILE + ch * 8192, &tmdO, full + 8 * s, ch);
          }
        }
    }
    return;
  }

  const int lane = threadIdx.x & 31, warp = (threadIdx.x & 127) / 32;
  const int key0 = k0 + warp * 16 + lane / 4;  // this thread's keys: key0 and key0 + 8
  float dk[DP / 2], dv[DP / 2];
#pragma unroll
  for (int i = 0; i < DP / 2; ++i) dk[i] = dv[i] = 0.f;
  if (first < end) mbar_wait_nocall(kvbar, 0);

  for (int g = 0; g < md.group; ++g)
    for (int i = first; i < end; ++i) {
      const int n = g * (end - first) + i - first, s = n % ST, q0 = i * 64;
      const uint32_t sq = sQ + s * 2 * TILE, sdo = sq + TILE;
      float st[32], dpt[32];
#pragma unroll
      for (int e = 0; e < 32; ++e) st[e] = dpt[e] = 0.f;
      mbar_wait_nocall(full + 8 * s, (n / ST) & 1);
      md.zero_q_tail(c, q0, sq);
      fence_regs<32>(st);
      fence_regs<32>(dpt);
      wgmma_fence();
#pragma unroll
      for (int ch = 0; ch < NC; ++ch)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_ss<Cfg::DT, 64, 0, 0>(st, wgmma_desc(sK + ch * 8192 + k * 32, 16, 1024),
                                      wgmma_desc(sq + ch * 8192 + k * 32, 16, 1024), 1);
#pragma unroll
      for (int ch = 0; ch < NC; ++ch)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_ss<Cfg::DT, 64, 0, 0>(dpt, wgmma_desc(sV + ch * 8192 + k * 32, 16, 1024),
                                      wgmma_desc(sdo + ch * 8192 + k * 32, 16, 1024), 1);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs<32>(st);
      fence_regs<32>(dpt);

      // masks: keys past the length, and (causal) keys after the query's diagonal.  A masked score becomes -inf (P = 0)
      // and its dP 0, so nothing a padded key holds reaches dS.
      if (k0 + 64 > c.kv_len || (md.causal && k0 + 63 > md.diag(c, q0))) {
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int key = key0 + 8 * h, q = q0 + 8 * j + 2 * (lane & 3) + e;
              if (key >= c.kv_len || (md.causal && key > md.diag(c, q))) {
                st[4 * j + 2 * h + e] = -INFINITY;
                dpt[4 * j + 2 * h + e] = 0.f;
              }
            }
      }
      uint32_t pa[4][4], da[4][4];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float l2[2], dl[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) md.row_stats(a, c, g, q0 + 8 * j + 2 * (lane & 3) + e, l2[e], dl[e]);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float p[2], ds[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            p[e] = ex2(fmaf(st[4 * j + 2 * h + e], a.scale_log2, -l2[e]));
            ds[e] = p[e] * (dpt[4 * j + 2 * h + e] - dl[e]);
          }
          pa[j / 2][(j & 1) * 2 + h] = pack_round<Cfg::DT>(p[0], p[1]);
          da[j / 2][(j & 1) * 2 + h] = pack_round<Cfg::DT>(ds[0], ds[1]);
        }
      }

      // dV += P~^T dO_i, dK += dS~^T Q_i over the tile's 64 queries
      fence_regs<DP / 2>(dv);
      fence_regs<DP / 2>(dk);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_rs<Cfg::DT, DP, 1>(dv, pa[kk], wgmma_desc(sdo + kk * 2048, 8192, 1024), 1);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_rs<Cfg::DT, DP, 1>(dk, da[kk], wgmma_desc(sq + kk * 2048, 8192, 1024), 1);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs<DP / 2>(dv);
      fence_regs<DP / 2>(dk);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)  // the A registers are read by the MMAs until the wait above
#pragma unroll
        for (int e = 0; e < 4; ++e) asm volatile("" : "+r"(pa[kk][e]), "+r"(da[kk][e])::"memory");
      if ((threadIdx.x & 127) == 0) mbar_arrive(empty + 8 * s);
    }

  // keys the mode does not store are skipped; tiles no query sees store the zeros they hold
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    size_t row;
    if (!md.key_row(c, key0 + 8 * h, row)) continue;
    store_o<Cfg>(a.dst[0], row, 0, a.D, dk, h, a.scale);
    store_o<Cfg>(a.dst[1], row, 0, a.D, dv, h, 1.f);
  }
}

// dQ of one query tile, placed and fed by the forward's addressing mode (AttnDense or AttnPacked) on CTA (query tile,
// 0, b * H + h); a packed tile past the sequence returns.
template <class Cfg, class Mode>
__global__ void __launch_bounds__(Cfg::THREADS, 1)
    attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmdO,
                       const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                       const BwdArgs a, const Mode md) {
  static_assert(Cfg::BN == 64 && !Cfg::V_DN, "dQ: KV tiles of 64 keys, V [N, D]");
  constexpr int BM = Cfg::BM, BN = Cfg::BN, DP = Cfg::DV, NC = DP / 64, ST = kBwdStages;
  constexpr int QB = BM * DP * 2, KB = Cfg::V_BYTES;  // a resident Q / dO tile, a streamed K / V tile
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sQ = (smem_u32(smem_raw) + 1023) & ~1023u, sdO = sQ + QB, sKV = sdO + QB;  // stage s: K, then V
  const uint32_t qbar = sKV + ST * 2 * KB, full = qbar + 8, empty = full + 8 * ST;

  typename Mode::Cta cta;
  if (!md.setup(cta)) return;
  const KvTiles kv = md.tiles(cta);
  const int wg = threadIdx.x / 128;

  if (threadIdx.x == 0) {
    mbar_init(qbar, 1);
    for (int s = 0; s < ST; ++s) {
      mbar_init(full + 8 * s, 1);
      mbar_init(empty + 8 * s, Cfg::NWG);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(qbar, 2 * NC * md.q_bytes());
      for (int c = 0; c < NC; ++c) {
        md.load_q(cta, sQ + c * BM * 128, &tmQ, qbar, c);
        md.load_q(cta, sdO + c * BM * 128, &tmdO, qbar, c);
      }
      for (int j = kv.first; j < kv.end; ++j) {
        const int n = j - kv.first, s = n % ST;
        if (n >= ST) mbar_wait_nocall(empty + 8 * s, ((n / ST) - 1) & 1);
        mbar_arrive_expect_tx(full + 8 * s, 2 * KB);
        const int key0 = md.kv_tile(cta, j);
        for (int c = 0; c < NC; ++c) md.load_k(cta, key0, sKV + s * 2 * KB + c * BN * 128, &tmK, full + 8 * s, c);
        md.load_v(cta, key0, sKV + s * 2 * KB + KB, &tmV, full + 8 * s);
      }
    }
    return;
  }

  const int cw = wg - 1, lane = threadIdx.x & 31, warp = (threadIdx.x & 127) / 32;
  const int row0 = cta.q0 + cw * 64 + warp * 16 + lane / 4;  // this thread's rows: row0 and row0 + 8
  // lse2 and Delta of the row the mode stores, or padding (+inf, 0) for a row it does not (past N or the sequence)
  float l2[2], dl[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    size_t row = 0;
    const bool in = md.out_row(cta, row0 + 8 * h, row);
    l2[h] = in ? __ldg(a.lse2 + row) : INFINITY;
    dl[h] = in ? __ldg(a.delta + row) : 0.f;
  }
  float dq[DP / 2];
#pragma unroll
  for (int i = 0; i < DP / 2; ++i) dq[i] = 0.f;
  mbar_wait_nocall(qbar, 0);

  for (int j = kv.first; j < kv.end; ++j) {
    const int n = j - kv.first, s = n % ST, k0 = j * BN;
    const uint32_t sk = sKV + s * 2 * KB, sv = sk + KB;
    float sa[BN / 2], dp[BN / 2];
#pragma unroll
    for (int e = 0; e < BN / 2; ++e) sa[e] = dp[e] = 0.f;
    mbar_wait_nocall(full + 8 * s, (n / ST) & 1);
    md.zero_kv_tail(cta, k0, sk);  // dQ += dS~ K_j multiplies the masked dS of 0 by the K rows past the length
    fence_regs<BN / 2>(sa);
    fence_regs<BN / 2>(dp);
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_ss<Cfg::DT, BN, 0, 0>(sa, wgmma_desc(sQ + c * BM * 128 + cw * 64 * 128 + k * 32, 16, 1024),
                                    wgmma_desc(sk + c * BN * 128 + k * 32, 16, 1024), 1);
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_ss<Cfg::DT, BN, 0, 0>(dp, wgmma_desc(sdO + c * BM * 128 + cw * 64 * 128 + k * 32, 16, 1024),
                                    wgmma_desc(sv + c * BN * 128 + k * 32, 16, 1024), 1);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<BN / 2>(sa);
    fence_regs<BN / 2>(dp);

    // the forward's masks: keys past the length, keys after the row's causal diagonal
    if (k0 + BN > cta.kv_len || (md.causal && k0 + BN - 1 > md.diag(cta, cta.q0 + cw * 64))) {
      const int diag[2] = {md.diag(cta, row0), md.diag(cta, row0 + 8)};
#pragma unroll
      for (int i = 0; i < BN / 8; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int key = k0 + 8 * i + 2 * (lane & 3) + e;
            if (key >= cta.kv_len || (md.causal && key > diag[h])) {
              sa[4 * i + 2 * h + e] = -INFINITY;
              dp[4 * i + 2 * h + e] = 0.f;
            }
          }
    }
    uint32_t da[BN / 16][4];
#pragma unroll
    for (int i = 0; i < BN / 8; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float ds[2];
#pragma unroll
        for (int e = 0; e < 2; ++e)
          ds[e] = ex2(fmaf(sa[4 * i + 2 * h + e], a.scale_log2, -l2[h])) * (dp[4 * i + 2 * h + e] - dl[h]);
        da[i / 2][(i & 1) * 2 + h] = pack_round<Cfg::DT>(ds[0], ds[1]);
      }

    // dQ += dS~ K_j
    fence_regs<DP / 2>(dq);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk)
      wgmma_rs<Cfg::DT, DP, 1>(dq, da[kk], wgmma_desc(sk + kk * 2048, BN * 128, 1024), 1);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<DP / 2>(dq);
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk)
#pragma unroll
      for (int e = 0; e < 4; ++e) asm volatile("" : "+r"(da[kk][e])::"memory");
    if ((threadIdx.x & 127) == 0) mbar_arrive(empty + 8 * s);
  }

#pragma unroll
  for (int h = 0; h < 2; ++h) md.store(cta, row0 + 8 * h, dq, h, a.scale, 0.f, 0.f, a.dst[0], a.D);
}

// Workspace: Delta, then lse * log2 e, fp32 [rows] each, each on a 256-byte boundary.
static size_t bwd_section(int64_t rows) { return (size_t(rows) * sizeof(float) + 255) & ~size_t(255); }

// Checks that the workspace holds both sections of `rows` rows, and fills `a` with them, D and the scale (scale <= 0
// means 1 / sqrt(D)).  Each main kernel's launch sets dst.
static int bwd_args(const char* fn, int64_t rows, int64_t D, float scale, void* workspace, size_t workspace_bytes,
                    BwdArgs& a) {
  const size_t need = 2 * bwd_section(rows);
  if (workspace_bytes < need)
    return set_error(B200K_EARG, "%s: %zu workspace bytes needed, %zu given", fn, need, workspace_bytes);
  a.delta = static_cast<const float*>(workspace);
  a.lse2 = reinterpret_cast<const float*>(static_cast<const uint8_t*>(workspace) + bwd_section(rows));
  a.dst[0] = a.dst[1] = nullptr;
  a.D = int(D);
  if (scale <= 0.f) scale = 1.0f / sqrtf(float(D));
  a.scale = scale;
  a.scale_log2 = scale * 1.4426950408889634f;
  return B200K_OK;
}

// The prep kernel's grid: a quad of threads per row, at most 2^20 blocks of 256.
static unsigned bwd_prep_blocks(long long rows) {
  const long long blocks = (rows * 4 + 255) / 256;
  return unsigned(blocks < (1 << 20) ? blocks : (1 << 20));
}

static int bwd_shape(const char* fn, int64_t B, int64_t H, int64_t N) {
  if (B < 1 || H < 1 || N < 1 || N > INT32_MAX || B * H > 65535)
    return set_error(B200K_ESHAPE, "%s: need B, H, N >= 1, N <= 2^31 - 1 and B * H <= 65535 (got B=%lld H=%lld N=%lld)",
                     fn, (long long)B, (long long)H, (long long)N);
  return B200K_OK;
}

// The configurations: dtype, and DP = 64 for D = 32 / 64, 128 for D = 96 / 128.  `run` gets the dK/dV kernel's.
template <class Run>
static int run_bwd_cfg(int dtype, int64_t D, Run run) {
  const bool narrow = D <= 64;
  if (dtype == B200K_BF16) return narrow ? run(AttnCfg<1, 64, 1, 64, false>()) : run(AttnCfg<1, 128, 1, 64, false>());
  return narrow ? run(AttnCfg<0, 64, 1, 64, false>()) : run(AttnCfg<0, 128, 1, 64, false>());
}

template <class Kern, class Mode>
static int bwd_launch(Kern kern, dim3 grid, int threads, int smem, cudaStream_t s, const DeviceInfo& di, const char* fn,
                      const CUtensorMap (&tm)[4], const BwdArgs& a, const Mode& md) {
  if (smem > di.max_smem_optin)
    return set_error(B200K_ESHAPE, "%s: %d bytes of shared memory needed, device allows %d", fn, smem, di.max_smem_optin);
  int rc = ensure_dynamic_smem(reinterpret_cast<const void*>(kern), di.device, smem);
  if (rc) return rc;
  kern<<<grid, threads, smem, s>>>(tm[0], tm[1], tm[2], tm[3], a, md);
  B200K_CHECK_CUDA(cudaGetLastError());
  return B200K_OK;
}

constexpr int kBwdBars = 8 * (1 + 2 * kBwdStages);
template <int DP>
constexpr int dkdv_smem() { return 1024 + (2 + 2 * kBwdStages) * 64 * DP * 2 + kBwdBars; }
template <class QCfg>
constexpr int dq_smem() { return 1024 + 2 * QCfg::BM * QCfg::DV * 2 + 2 * kBwdStages * QCfg::V_BYTES + kBwdBars; }

// The main kernels of both layouts: the dK/dV kernel under `km` on `kv_grid`, reading K, V, Q, dO through maps of
// 64-row boxes (kv_t), then the dQ kernel under `qm` on `q_grid`, reading Q, dO in 128-row boxes (q_t) and the same
// K, V.  The prep kernel goes first: its launch makes the device's primary context current on the calling thread,
// which the tensor-map encoder (a driver call) needs.  torch runs a backward on an autograd thread of its own, where
// no CUDA runtime call may have run yet.
template <class KvCfg, class KvMode, class QMode>
static int bwd_main(const char* fn, const AttnTensor (&kv_t)[4], const AttnTensor (&q_t)[2], const KvMode& km,
                    dim3 kv_grid, const QMode& qm, dim3 q_grid, BwdArgs a, void* dQ, void* dK, void* dV, cudaStream_t s,
                    const DeviceInfo& di) {
  using QCfg = BwdQCfg<KvCfg>;
  CUtensorMap kv_tm[4], q_tm[4];
  int rc;
  for (int i = 0; i < 4; ++i)
    if ((rc = attn_tmap(&kv_tm[i], kv_t[i]))) return rc;
  for (int i = 0; i < 2; ++i)
    if ((rc = attn_tmap(&q_tm[i], q_t[i]))) return rc;
  q_tm[2] = kv_tm[0];
  q_tm[3] = kv_tm[1];
  a.dst[0] = dK;
  a.dst[1] = dV;
  rc = bwd_launch(attn_bwd_dkdv_kernel<KvCfg, KvMode>, kv_grid, KvCfg::THREADS, dkdv_smem<KvCfg::DV>(), s, di, fn, kv_tm,
                  a, km);
  if (rc) return rc;
  a.dst[0] = dQ;
  a.dst[1] = nullptr;
  return bwd_launch(attn_bwd_dq_kernel<QCfg, QMode>, q_grid, QCfg::THREADS, dq_smem<QCfg>(), s, di, fn, q_tm, a, qm);
}

}  // namespace b200k

extern "C" int b200k_fa2_bwd_workspace_bytes(int64_t B, int64_t H, int64_t N, size_t* bytes) {
  using namespace b200k;
  if (!bytes) return set_error(B200K_EARG, "b200k_fa2_bwd_workspace_bytes: null pointer");
  const int rc = bwd_shape("b200k_fa2_bwd_workspace_bytes", B, H, N);
  if (rc) return rc;
  *bytes = 2 * bwd_section(B * H * N);
  return B200K_OK;
}

extern "C" int b200k_fa2_bwd(const void* Q, const void* K, const void* V, const void* O, const float* lse, const void* dO,
                             void* dQ, void* dK, void* dV, int64_t B, int64_t H, int64_t N, int64_t D, float scale,
                             int dtype, int causal, const int* seqlens_k, void* workspace, size_t workspace_bytes,
                             void* stream) {
  using namespace b200k;
  const char* fn = "b200k_fa2_bwd";
  if (!Q || !K || !V || !O || !lse || !dO || !dQ || !dK || !dV || !workspace)
    return set_error(B200K_EARG, "%s: null pointer", fn);
  if (dtype != B200K_F16 && dtype != B200K_BF16) return set_error(B200K_EDTYPE, "%s: dtype %d not supported (f16, bf16)", fn, dtype);
  int rc = check_headdim(fn, D);
  if (rc || (rc = bwd_shape(fn, B, H, N))) return rc;
  if ((rc = check_align(fn, {{Q, "Q", 16}, {K, "K", 16}, {V, "V", 16}, {O, "O", 16}, {dO, "dO", 16},
                             {workspace, "workspace", 16}, {dQ, "dQ", 4}, {dK, "dK", 4}, {dV, "dV", 4}, {lse, "lse", 4},
                             {seqlens_k, "seqlens_k", 4}})))
    return rc;
  const int64_t BH = B * H, rows = BH * N;
  BwdArgs a;
  if ((rc = bwd_args(fn, rows, D, scale, workspace, workspace_bytes, a))) return rc;
  DeviceInfo di;
  if ((rc = get_device_info(&di))) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  return run_bwd_cfg(dtype, D, [&](auto cfg) {
    using KvCfg = decltype(cfg);
    using QCfg = BwdQCfg<KvCfg>;
    attn_bwd_prep_kernel<KvCfg::DT, false><<<bwd_prep_blocks(rows), 256, 0, s>>>(
        static_cast<const uint16_t*>(O), static_cast<const uint16_t*>(dO), lse, const_cast<float*>(a.delta),
        const_cast<float*>(a.lse2), rows, int(D), 0, {}, {}, {});
    B200K_CHECK_CUDA(cudaGetLastError());
    const AttnTensor kv_t[4] = {{K, BH, N, D, 1, 64}, {V, BH, N, D, 1, 64}, {Q, BH, N, D, 1, 64}, {dO, BH, N, D, 1, 64}};
    const AttnTensor q_t[2] = {{Q, BH, N, D, 1, QCfg::BM}, {dO, BH, N, D, 1, QCfg::BM}};
    const BwdKeysDense<KvCfg> km = {seqlens_k, int(N), int(H), causal ? 1 : 0};
    const AttnDense<QCfg> qm = {seqlens_k, int(N), int(H), causal ? 1 : 0};
    return bwd_main<KvCfg>(fn, kv_t, q_t, km, dim3(unsigned((N + 63) / 64), unsigned(BH)), qm,
                           dim3(unsigned((N + QCfg::BM - 1) / QCfg::BM), 1, unsigned(BH)), a, dQ, dK, dV, s, di);
  });
}

// The checks b200k_fa2_bwd_varlen shares with its workspace query.
static int bwd_varlen_shape(const char* fn, int64_t B, int64_t max_q, int64_t max_k, int64_t total_q, int64_t total_k,
                            int64_t H, int64_t H_kv) {
  using namespace b200k;
  if (B < 1 || H < 1 || H_kv < 1 || H % H_kv != 0)
    return set_error(B200K_ESHAPE, "%s: need B, H, H_kv >= 1 and H %% H_kv == 0 (got B=%lld H=%lld H_kv=%lld)", fn,
                     (long long)B, (long long)H, (long long)H_kv);
  if (total_q > INT32_MAX || total_k > INT32_MAX || max_q < 1 || max_q > total_q || max_k < 1 || max_k > total_k)
    return set_error(B200K_ESHAPE,
                     "%s: need 1 <= max_seqlen_q <= total_q <= 2^31 - 1 and 1 <= max_seqlen_k <= total_k <= 2^31 - 1 "
                     "(got max_seqlen_q=%lld total_q=%lld max_seqlen_k=%lld total_k=%lld)",
                     fn, (long long)max_q, (long long)total_q, (long long)max_k, (long long)total_k);
  if (B > 65535 || H > 65535 || B * H > 65535)
    return set_error(B200K_ESHAPE, "%s: B * H = %lld CTAs per query tile, the grid allows 65535", fn,
                     (long long)B * (long long)H);
  return B200K_OK;
}

extern "C" int b200k_fa2_bwd_varlen_workspace_bytes(int64_t total_q, int64_t H, size_t* bytes) {
  using namespace b200k;
  if (!bytes) return set_error(B200K_EARG, "b200k_fa2_bwd_varlen_workspace_bytes: null pointer");
  if (total_q < 1 || total_q > INT32_MAX || H < 1 || H > 65535)
    return set_error(B200K_ESHAPE,
                     "b200k_fa2_bwd_varlen_workspace_bytes: need 1 <= total_q <= 2^31 - 1 and 1 <= H <= 65535 "
                     "(got total_q=%lld H=%lld)",
                     (long long)total_q, (long long)H);
  *bytes = 2 * bwd_section(total_q * H);
  return B200K_OK;
}

// The packed layout: the maps over (D, heads, tokens), grids sized by the longest sequences.
extern "C" int b200k_fa2_bwd_varlen(const void* Q, const void* K, const void* V, const void* O, const float* lse,
                                    const void* dO, void* dQ, void* dK, void* dV, const int* cu_seqlens_q,
                                    const int* cu_seqlens_k, int64_t B, int64_t max_seqlen_q, int64_t max_seqlen_k,
                                    int64_t total_q, int64_t total_k, int64_t H, int64_t H_kv, int64_t D, float scale,
                                    int dtype, int causal, void* workspace, size_t workspace_bytes, void* stream) {
  using namespace b200k;
  const char* fn = "b200k_fa2_bwd_varlen";
  if (!Q || !K || !V || !O || !lse || !dO || !dQ || !dK || !dV || !cu_seqlens_q || !cu_seqlens_k || !workspace)
    return set_error(B200K_EARG, "%s: null pointer", fn);
  if (dtype != B200K_F16 && dtype != B200K_BF16) return set_error(B200K_EDTYPE, "%s: dtype %d not supported (f16, bf16)", fn, dtype);
  int rc = check_headdim(fn, D);
  if (rc || (rc = bwd_varlen_shape(fn, B, max_seqlen_q, max_seqlen_k, total_q, total_k, H, H_kv))) return rc;
  if ((rc = check_align(fn, {{Q, "Q", 16}, {K, "K", 16}, {V, "V", 16}, {O, "O", 16}, {dO, "dO", 16},
                             {workspace, "workspace", 16}, {dQ, "dQ", 4}, {dK, "dK", 4}, {dV, "dV", 4}, {lse, "lse", 4},
                             {cu_seqlens_q, "cu_seqlens_q", 4}, {cu_seqlens_k, "cu_seqlens_k", 4}})))
    return rc;
  const int64_t rows = total_q * H;
  BwdArgs a;
  if ((rc = bwd_args(fn, rows, D, scale, workspace, workspace_bytes, a))) return rc;
  DeviceInfo di;
  if ((rc = get_device_info(&di))) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  return run_bwd_cfg(dtype, D, [&](auto cfg) {
    using KvCfg = decltype(cfg);
    using QCfg = BwdQCfg<KvCfg>;
    const BwdPackedGrad gq = {dQ, cu_seqlens_q, total_q, H * D / 2}, gk = {dK, cu_seqlens_k, total_k, H_kv * D / 2},
                        gv = {dV, cu_seqlens_k, total_k, H_kv * D / 2};
    attn_bwd_prep_kernel<KvCfg::DT, true><<<bwd_prep_blocks(rows), 256, 0, s>>>(
        static_cast<const uint16_t*>(O), static_cast<const uint16_t*>(dO), lse, const_cast<float*>(a.delta),
        const_cast<float*>(a.lse2), rows, int(D), int(B), gq, gk, gv);
    B200K_CHECK_CUDA(cudaGetLastError());
    const AttnTensor kv_t[4] = {{K, total_k, H_kv, D, 64, 1}, {V, total_k, H_kv, D, 64, 1}, {Q, total_q, H, D, 64, 1},
                                {dO, total_q, H, D, 64, 1}};
    const AttnTensor q_t[2] = {{Q, total_q, H, D, QCfg::BM, 1}, {dO, total_q, H, D, QCfg::BM, 1}};
    const BwdKeysPacked<KvCfg> km = {cu_seqlens_q, cu_seqlens_k, int(H), int(H_kv), int(H / H_kv), causal ? 1 : 0};
    const AttnPacked<QCfg> qm = {cu_seqlens_q, cu_seqlens_k, int(H), int(H / H_kv), int(total_q), causal ? 1 : 0};
    return bwd_main<KvCfg>(fn, kv_t, q_t, km, dim3(unsigned((max_seqlen_k + 63) / 64), unsigned(B * H_kv)), qm,
                           dim3(unsigned((max_seqlen_q + QCfg::BM - 1) / QCfg::BM), 1, unsigned(B * H)), a, dQ, dK, dV,
                           s, di);
  });
}
