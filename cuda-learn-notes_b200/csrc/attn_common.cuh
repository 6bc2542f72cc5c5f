// What the attention forward (attn_fwd_wgmma.cu) and backward (attn_bwd_wgmma.cu) share: the kernel configuration, the
// fp32 -> 16-bit rounding of MMA operands and outputs, the dense [B, H, N, D] and packed [tokens, H, D] addressing, the
// tensor maps of Q / K / V,
// and the argument checks of the entry points.
#pragma once
#include "abi_common.cuh"
#include "ptx.cuh"

#include <initializer_list>

namespace b200k {

template <int DT_, int DV_, int NWG_, int BN_, bool V_DN_>  // DT: 0 f16, 1 bf16
struct AttnCfg {
  static constexpr int DT = DT_, DV = DV_, NWG = NWG_, BN = BN_;
  static constexpr bool V_DN = V_DN_;
  static constexpr int BM = 64 * NWG;
  static constexpr int THREADS = 128 * (NWG + 1);
  static constexpr int KSTAGES = 4, VSTAGES = 2;
  static constexpr int K_BYTES = BN * 128;  // BN keys x 64 head-dim columns
  static constexpr int V_BYTES = BN * DV * 2;
  static constexpr int BAR_BYTES = 8 * (1 + 2 * KSTAGES + 2 * VSTAGES);
  static int smem_bytes(int nqc) { return 1024 + nqc * BM * 128 + KSTAGES * K_BYTES + VSTAGES * V_BYTES + BAR_BYTES; }
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Two fp32 values -> packed 16-bit pair; `lo` / `hi` come back as the rounded values (so the row sum matches what the
// tensor core multiplies).
template <int DT>
__device__ __forceinline__ uint32_t pack_round(float& lo, float& hi) {
  if constexpr (DT == 0) {
    const __half2 h = __floats2half2_rn(lo, hi);
    const float2 f = __half22float2(h);
    lo = f.x;
    hi = f.y;
    return *reinterpret_cast<const uint32_t*>(&h);
  } else {
    const __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
    const float2 f = __bfloat1622float2(h);
    lo = f.x;
    hi = f.y;
    return *reinterpret_cast<const uint32_t*>(&h);
  }
}

// Row `row` of a 16-bit [rows, D] O from this thread's column pairs of accumulator row h (o[4 i + 2 h], o[4 i + 2 h + 1]
// hold columns dv0 + 8 i + 2 (lane % 4) and the next), times inv, clipped to D columns (D is even).
template <class Cfg>
__device__ __forceinline__ void store_o(void* O, size_t row, int dv0, int D, const float (&o)[Cfg::DV / 2], int h,
                                        float inv) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < Cfg::DV / 8; ++i) {
    const int c = dv0 + 8 * i + 2 * (lane & 3);
    if (c >= D) continue;
    float x = o[4 * i + 2 * h] * inv, y = o[4 * i + 2 * h + 1] * inv;
    *reinterpret_cast<uint32_t*>(static_cast<uint16_t*>(O) + row * size_t(D) + c) = pack_round<Cfg::DT>(x, y);
  }
}

// KV tiles [first, end) of a CTA: tile j holds keys [j * BN, (j + 1) * BN) of its sequence.
struct KvTiles { int first, end; };

// Zeroes the rows at and past `len` of the BN-row tile of rows [k0, k0 + BN) at `tile`, laid out as Cfg's V: DV / 64
// chunks of BN rows of 128 bytes (V [keys, D], a K tile, or the backward's Q and dO tiles), or with V_DN those keys'
// columns of BN / 64 sub-tiles of DV rows of 64 keys, 128B-swizzled (unit u of row d at unit u ^ (d % 8)).  Rows a call
// does not own may hold anything, and a masked P or dS of 0 times a NaN or Inf is NaN in the tensor core, so each mode
// zeroes the operand rows it multiplies by a masked 0.  All 128 * NWG consumer threads share the stores and meet at one
// barrier before any of them issues its wgmma; each reaches it in the same iteration, since the condition is the CTA's.
template <class Cfg>
__device__ __forceinline__ void zero_tile_tail(int len, int k0, uint32_t tile) {
  constexpr int N = 128 * Cfg::NWG;
  if (k0 + Cfg::BN <= len) return;
  const int r0 = len - k0;  // first row to zero, within the tile
  if constexpr (Cfg::V_DN) {
    constexpr int UNITS = Cfg::BN / 64 * Cfg::DV * 8;  // 16-byte units of the tile
    static_assert(UNITS % N == 0, "zero_tile_tail: every unit needs a thread");
#pragma unroll
    for (int k = 0; k < UNITS / N; ++k) {
      const int w = threadIdx.x % N + k * N, d = w / 8 % Cfg::DV, u = w % 8, key = w / (8 * Cfg::DV) * 64 + 8 * u;
      const uint32_t a = tile + w / (8 * Cfg::DV) * Cfg::DV * 128 + d * 128 + ((u ^ (d & 7)) << 4);
      if (key >= r0) {
        asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(a), "r"(0) : "memory");
      } else if (key + 8 > r0) {
#pragma unroll
        for (int e = 0; e < 8; ++e)
          if (key + e >= r0) asm volatile("st.shared.u16 [%0], %1;" ::"r"(a + 2 * e), "h"((unsigned short)0) : "memory");
      }
    }
  } else {
    const int words = (Cfg::BN - r0) * 8;  // 16-byte words per 64-column chunk
    auto zero = [&](int i, int w) {
      asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(tile + i * Cfg::BN * 128 + r0 * 128 + w * 16), "r"(0)
                   : "memory");
    };
#pragma unroll
    for (int i = 0; i < Cfg::DV / 64; ++i) {
      if constexpr (Cfg::NWG == 1) {
        for (int w = threadIdx.x % N; w < words; w += N) zero(i, w);
      } else {
        // Two consumer warpgroups already hold 168 registers, the most a 384-thread CTA allows; a fixed count of
        // predicated stores needs fewer live registers than the loop above, which would spill.
        static_assert(Cfg::BN * 8 % N == 0, "zero_tile_tail: every 16-byte word of a chunk needs a thread");
#pragma unroll
        for (int k = 0; k < Cfg::BN * 8 / N; ++k)
          if (threadIdx.x % N + k * N < words) zero(i, threadIdx.x % N + k * N);
      }
    }
  }
  fence_proxy_async_smem();  // generic-proxy stores -> the wgmma's operand reads
  named_bar_sync(1, N);
}

// [B, H, N, D], one 3-D map per tensor over (D, N, B * H); V stored [B, H, D, N] over (N, D, B * H).  CTA (x, y, z) =
// (query tile, O column slice, batch * H + head).  Rows are numbered within the head, so row r sees keys <= r under the
// causal mask.  The modes of the forward are described in attn_fwd_wgmma.cu; the backward's dQ kernel takes this one
// and AttnPacked.
template <class Cfg>
struct AttnDense {
  const int* seqlens;  // int32 [B] valid keys per batch, or null
  int N, H, causal;

  struct Cta { int bh, q0, dv0, kv_len; };
  __device__ __forceinline__ bool setup(Cta& c) const {
    c.bh = blockIdx.z;
    c.q0 = blockIdx.x * Cfg::BM;
    c.dv0 = blockIdx.y * Cfg::DV;
    c.kv_len = seqlens ? min(max(__ldg(seqlens + c.bh / H), 1), N) : N;
    return true;
  }
  __device__ __forceinline__ KvTiles tiles(const Cta& c) const {
    int nt = (c.kv_len + Cfg::BN - 1) / Cfg::BN;
    if (causal) nt = min(nt, (c.q0 + Cfg::BM - 1) / Cfg::BN + 1);
    return {0, nt};
  }
  __device__ __forceinline__ int q_bytes() const { return Cfg::BM * 128; }
  __device__ __forceinline__ void load_q(const Cta& c, uint32_t dst, const CUtensorMap* tm, uint32_t bar, int chunk) const {
    tma_load_3d(dst, tm, bar, chunk * 64, c.q0, c.bh, kPolicyEvictFirst);
  }
  __device__ __forceinline__ int kv_tile(const Cta&, int j) const { return j * Cfg::BN; }
  __device__ __forceinline__ void load_k(const Cta& c, int key0, uint32_t dst, const CUtensorMap* tm, uint32_t bar,
                                         int chunk) const {
    tma_load_3d(dst, tm, bar, chunk * 64, key0, c.bh, kPolicyEvictNormal);
  }
  __device__ __forceinline__ void load_v(const Cta& c, int key0, uint32_t dst, const CUtensorMap* tm, uint32_t bar) const {
    if constexpr (Cfg::V_DN) {
#pragma unroll
      for (int i = 0; i < Cfg::BN / 64; ++i)
        tma_load_3d(dst + i * Cfg::DV * 128, tm, bar, key0 + i * 64, c.dv0, c.bh, kPolicyEvictNormal);
    } else {
#pragma unroll
      for (int i = 0; i < Cfg::DV / 64; ++i)
        tma_load_3d(dst + i * Cfg::BN * 128, tm, bar, c.dv0 + i * 64, key0, c.bh, kPolicyEvictNormal);
    }
  }
  __device__ __forceinline__ int diag(const Cta&, int r) const { return r; }
  // keys past seqlens_k are the caller's padding; past N, TMA has zero-filled the tile, so a call without seqlens_k
  // (kv_len = N) does no extra work
  __device__ __forceinline__ void zero_kv_tail(const Cta& c, int k0, uint32_t tile) const {
    if (c.kv_len < N) zero_tile_tail<Cfg>(c.kv_len, k0, tile);
  }
  __device__ __forceinline__ bool out_row(const Cta& c, int r, size_t& row) const {
    if (r >= N) return false;
    row = size_t(c.bh) * N + r;
    return true;
  }
  __device__ __forceinline__ void store(const Cta& c, int r, const float (&o)[Cfg::DV / 2], int h, float inv, float,
                                        float, void* O, int D) const {
    size_t row;
    if (out_row(c, r, row)) store_o<Cfg>(O, row, c.dv0, D, o, h, inv);
  }
};

// Packed sequences: sequence b is tokens [cu_q[b], cu_q[b+1]) of Q / O ([total_q, H, D]) and [cu_k[b], cu_k[b+1]) of
// K / V ([total_k, H / group, D]); query head h reads K / V head h / group.  The maps are over (D, heads, tokens).  CTA
// (x, z) = (query tile of the sequence, b * H + head).  Rows are numbered within the sequence; row r sees keys <=
// r + Lk - Lq under the causal mask (bottom-right aligned).  Its epilogue stores rows of the sequence within tokens [0, total_q), and reloads cu_q
// rather than keep it in registers through the main loop.
template <class Cfg>
struct AttnPacked {
  static_assert(!Cfg::V_DN, "packed sequences take V as [tokens, heads, D]");
  const int* cu_q;
  const int* cu_k;
  int H, group, total_q, causal;

  struct Cta { int kv_head, q0, q_tok, k_tok, kv_len, shift; };  // q_tok, k_tok: first tokens; shift: Lk - Lq
  __device__ __forceinline__ bool setup(Cta& c) const {
    const int b = blockIdx.z / H;
    c.kv_head = blockIdx.z % H / group;
    c.q0 = blockIdx.x * Cfg::BM;
    c.q_tok = __ldg(cu_q + b);
    const int q_len = __ldg(cu_q + b + 1) - c.q_tok;
    if (c.q0 >= q_len) return false;
    c.k_tok = __ldg(cu_k + b);
    c.kv_len = __ldg(cu_k + b + 1) - c.k_tok;
    c.shift = c.kv_len - q_len;
    return true;
  }
  __device__ __forceinline__ KvTiles tiles(const Cta& c) const {
    int nt = (c.kv_len + Cfg::BN - 1) / Cfg::BN;
    const int last = c.q0 + c.shift + Cfg::BM - 1;  // can be negative: no key visible
    if (causal) nt = min(nt, last < 0 ? 0 : last / Cfg::BN + 1);
    return {0, nt};
  }
  __device__ __forceinline__ int q_bytes() const { return Cfg::BM * 128; }
  __device__ __forceinline__ void load_q(const Cta& c, uint32_t dst, const CUtensorMap* tm, uint32_t bar, int chunk) const {
    tma_load_3d(dst, tm, bar, chunk * 64, blockIdx.z % H, c.q_tok + c.q0, kPolicyEvictFirst);
  }
  __device__ __forceinline__ int kv_tile(const Cta& c, int j) const { return c.k_tok + j * Cfg::BN; }
  __device__ __forceinline__ void load_k(const Cta& c, int tok, uint32_t dst, const CUtensorMap* tm, uint32_t bar,
                                         int chunk) const {
    tma_load_3d(dst, tm, bar, chunk * 64, c.kv_head, tok, kPolicyEvictNormal);
  }
  __device__ __forceinline__ void load_v(const Cta& c, int tok, uint32_t dst, const CUtensorMap* tm, uint32_t bar) const {
#pragma unroll
    for (int i = 0; i < Cfg::DV / 64; ++i) load_k(c, tok, dst + i * Cfg::BN * 128, tm, bar, i);
  }
  __device__ __forceinline__ int diag(const Cta& c, int r) const { return r + c.shift; }
  // keys past Lk are the next sequence's tokens, or whatever lies past cu_k[B]
  __device__ __forceinline__ void zero_kv_tail(const Cta& c, int k0, uint32_t tile) const {
    zero_tile_tail<Cfg>(c.kv_len, k0, tile);
  }
  __device__ __forceinline__ bool out_row(const Cta&, int r, size_t& row) const {
    const int b = blockIdx.z / H, q_tok = __ldg(cu_q + b);
    if (r >= __ldg(cu_q + b + 1) - q_tok) return false;
    const long long tok = (long long)q_tok + r;
    if (tok < 0 || tok >= total_q) return false;
    row = size_t(tok) * H + blockIdx.z % H;
    return true;
  }
  __device__ __forceinline__ void store(const Cta& c, int r, const float (&o)[Cfg::DV / 2], int h, float inv, float,
                                        float, void* O, int D) const {
    size_t row;
    if (out_row(c, r, row)) store_o<Cfg>(O, row, 0, D, o, h, inv);
  }
};

// One contiguous [d2, d1, d0] tensor of `elem`-byte elements (2: f16 / bf16, 1: fp8) read through boxes
// [box2, box1, 128 / elem]: each box row is one 128-byte swizzle row.
struct AttnTensor {
  const void* p;
  int64_t d2, d1, d0;
  int box2, box1;
  int elem = 2;
};

static int attn_tmap(CUtensorMap* m, const AttnTensor& t) {
  const uint64_t e = uint64_t(t.elem);
  const uint64_t dims[3] = {uint64_t(t.d0), uint64_t(t.d1), uint64_t(t.d2)}, strides[2] = {e * dims[0], e * dims[0] * dims[1]};
  const uint32_t box[3] = {uint32_t(128 / t.elem), uint32_t(t.box1), uint32_t(t.box2)};
  return make_tmap(m, t.p, t.elem, 3, dims, strides, box);
}

static int check_headdim(const char* fn, int64_t D) {
  if (D != 32 && D != 64 && D != 96 && D != 128)
    return set_error(B200K_EHEADDIM, "headdim not support! (%s: D=%lld, supported 32/64/96/128)", fn, (long long)D);
  return B200K_OK;
}

// Alignment checks of the attention entry points, in order, before any CUDA call: the first pointer that is not a
// multiple of its byte count is B200K_EALIGN, named in the message.  Null pointers pass (each call checks those it
// needs).  The rules: Q, K, V, the caches, the new rows, cos / sin and workspaces 16 bytes (TMA maps, 16-byte loads
// and stores, fp32 partials); O 4 bytes (32-bit stores of column pairs); lse and the int32 arrays 4 bytes.
struct AlignRule {
  const void* p;
  const char* name;
  unsigned bytes;
};

static int check_align(const char* fn, std::initializer_list<AlignRule> rules) {
  for (const AlignRule& r : rules)
    if (reinterpret_cast<uintptr_t>(r.p) % r.bytes)
      return set_error(B200K_EALIGN, "%s: %s must be %u-byte aligned", fn, r.name, r.bytes);
  return B200K_OK;
}

}  // namespace b200k
