// Attention forward on Hopper (sm_90a): O = softmax(Q K^T * scale) V, FlashAttention-2 style online softmax, fp32
// statistics and accumulators in registers, wgmma for both products, TMA + mbarrier rings for Q / K / V.
//
// A CTA owns BM = 64 * NWG query rows and DV columns of O.  Warpgroup 0 is the producer (one thread issues TMA loads);
// each consumer warpgroup owns 64 query rows:
//   S  = Q K^T     wgmma m64nBNk16, both operands in shared memory, Q resident for the whole CTA, K streamed in
//                  64-column chunks of the head dim through a 4-deep ring (so any head dim up to 1024 fits)
//   P  = exp2(S * scale * log2 e - m)        the S accumulator fragment is, register for register, the A fragment
//                  of the next product, so P never goes through shared memory
//   O += P V       wgmma m64nDVk16 with A from registers, V tile (BN keys x DV columns) from a 2-deep ring; V stored
//                  [N,D] is an MN-major operand, V stored [D,N] a K-major one
// Head dims above 256 split O into ceil(D / 256) column slices, one per CTA (grid.y); each slice recomputes S.
// Ragged N and head dims that are not multiples of 64 are zero-filled by TMA (3-D maps: per head) and clipped on the
// store; padded keys are masked.  Causal CTAs stop at their diagonal tile.
// The layout is the kernel's one mode argument (AttnDense, AttnPacked for packed sequences with grouped K/V heads,
// AttnDecode): it places the CTA and its TMA boxes, cuts its KV tiles, gives its causal diagonals and stores its rows.
// In KV-cache decode a CTA owns the query rows of one K/V head (tokens x grouped heads packed into one 64-row tile),
// reads K / V through a page table, takes one split of the sequence's KV tiles, and writes either O or fp32 partials
// that attn_combine_kernel merges.  kvcache_append_kernel, launched before it, writes new K / V rows (K and Q
// optionally rotated) into the caches and the lengths the decode kernel reads.
#include "attn_common.cuh"

#include <climits>
#include <cmath>

namespace b200k {

template <int DT>
__device__ __forceinline__ float2 unpack2(uint32_t w) {
  if constexpr (DT == 0) return __half22float2(*reinterpret_cast<const __half2*>(&w));
  else return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w));
}

// The modes.  Each holds its layout's kernel arguments and provides: Cta, the CTA's coordinates, key count kv_len and
// first row q0 (its rows are q0 .. q0 + BM - 1 in the numbering diag and store take), which setup fills (false: no rows
// here; the CTA returns before any barrier exists); tiles, the KV tiles it visits; q_bytes and load_q, the bytes and the
// box of 64-column chunk c of Q; kv_tile, where KV tile j is, for load_k (chunk c of K) and load_v (all of V); diag,
// the causal diagonal (last key seen) of row r; zero_kv_tail, which zeroes the V rows of a tile past the CTA's key
// count (zero_tile_tail, attn_common.cuh; what the tile holds there is not the call's); out_row, whether row r
// is stored and to which row of O (viewed as [rows, D]); store, the epilogue of row r.  The dense and packed modes,
// AttnDense and AttnPacked, are in attn_common.cuh, which the backward shares.

// K / V read from caches [num_pages, page_size, H_kv, D] through a block table, for the modes that do (AttnDecode,
// AttnPackedPaged).  Key j of sequence seq is at slot j % page_size of page table[seq * pages_per_seq + j / page_size]
// (table null: contiguous cache, sequence seq at rows [seq * page_size, ...)).  A KV tile is BN / box_rows TMA boxes,
// one per page when pages are smaller than a tile.  M is the mode, which holds table, page_size, pages_per_seq,
// box_rows and oob (a row coordinate past the end of the cache maps: TMA zero-fills the box); kv_len is the sequence's
// key count, already clamped to its capacity pages_per_seq * page_size.
template <class Cfg>
struct PagedKv {
  // cache row of each box of a KV tile
  struct Rows { int row[Cfg::BN / 16]; };
  // A box past the sequence's last page reads outside the map, so the table is read only up to the length.
  template <class M>
  __device__ __forceinline__ static Rows tile(const M& m, int seq, int kv_len, int j) {
    Rows t;
#pragma unroll
    for (int i = 0; i < Cfg::BN / 16; ++i) {
      const int key = j * Cfg::BN + i * m.box_rows;
      if (i * m.box_rows >= Cfg::BN) break;
      if (!m.table) t.row[i] = seq * m.page_size + key;
      else if (key >= kv_len) t.row[i] = m.oob;
      else t.row[i] = __ldg(m.table + size_t(seq) * m.pages_per_seq + key / m.page_size) * m.page_size + key % m.page_size;
    }
    return t;
  }
  template <class M>
  __device__ __forceinline__ static void load_k(const M& m, int kvh, const Rows& t, uint32_t dst, const CUtensorMap* tm,
                                                uint32_t bar, int chunk) {
#pragma unroll
    for (int i = 0; i < Cfg::BN / 16; ++i) {
      if (i * m.box_rows >= Cfg::BN) break;
      tma_load_3d(dst + i * m.box_rows * 128, tm, bar, chunk * 64, kvh, t.row[i], kPolicyEvictNormal);
    }
  }
  template <class M>
  __device__ __forceinline__ static void load_v(const M& m, int kvh, const Rows& t, uint32_t dst, const CUtensorMap* tm,
                                                uint32_t bar) {
#pragma unroll
    for (int i = 0; i < Cfg::DV / 64; ++i) load_k(m, kvh, t, dst + i * Cfg::BN * 128, tm, bar, i);
  }
};

// KV-cache decode.  Q / O are [B, Lq, H, D]; the caches are paged as PagedKv describes.  CTA (x, y, z) = (split, token
// tile * nhb + head tile, b * H_kv + K/V head).  Its 64 rows are T tokens x hb heads of one group (row r = token r / hb,
// head r % hb); row r of token t sees keys <= t + Lk - Lq under the causal mask.  With more than one split (gridDim.x)
// the CTA writes O / l and the row's base-2 log-sum-exp to `part` / `lse` ([split][row][D], [split][row], row =
// (b * Lq + t) * H + h) instead of O.
template <class Cfg>
struct AttnDecode {
  static_assert(Cfg::NWG == 1 && !Cfg::V_DN, "decode: one consumer warpgroup, V [keys, heads, D]");
  const int *seqlens = nullptr, *table = nullptr;  // int32 [B] key counts, block table
  float *part = nullptr, *lse = nullptr;
  long long rows = 0;  // B * Lq * H
  int H = 1, causal = 0;
  int Lq = 1, group = 1, hb = 1, T = 1, nhb = 1;
  int page_size = 1, pages_per_seq = 1, box_rows = 1;
  int oob = 0;

  struct Cta { int q0, seq, kvh, t0, h0, kv_len, shift; };  // q0 = 0; t0, h0: first token and head; shift: Lk - Lq
  using KvRows = typename PagedKv<Cfg>::Rows;
  __device__ __forceinline__ bool setup(Cta& c) const {
    const int h_kv = H / group;
    c.q0 = 0;
    c.seq = blockIdx.z / h_kv;
    c.kvh = blockIdx.z % h_kv;
    c.t0 = (blockIdx.y / nhb) * T;
    c.h0 = c.kvh * group + (blockIdx.y % nhb) * hb;
    c.kv_len = min(max(__ldg(seqlens + c.seq), 0), pages_per_seq * page_size);
    c.shift = c.kv_len - Lq;
    return true;
  }
  // split s of gridDim.x takes tiles [s * nt / splits, (s + 1) * nt / splits) of this sequence; it may take none
  __device__ __forceinline__ KvTiles tiles(const Cta& c) const {
    int nt = (c.kv_len + Cfg::BN - 1) / Cfg::BN;
    if (causal) {  // the tile's last token sees keys <= its index + shift
      const int last = min(c.t0 + T, Lq) - 1 + c.shift;
      nt = min(nt, last < 0 ? 0 : last / Cfg::BN + 1);
    }
    return {int((long long)blockIdx.x * nt / gridDim.x), int((long long)(blockIdx.x + 1) * nt / gridDim.x)};
  }
  // the Q box is T tokens x hb heads; rows it reads past the sequence, the group or the tensor are computed and never
  // stored (zero-filled past the tensor, which TMA still counts in full)
  __device__ __forceinline__ int q_bytes() const { return T * hb * 128; }
  __device__ __forceinline__ void load_q(const Cta& c, uint32_t dst, const CUtensorMap* tm, uint32_t bar, int chunk) const {
    tma_load_3d(dst, tm, bar, chunk * 64, c.h0, c.seq * Lq + c.t0, kPolicyEvictFirst);
  }
  __device__ __forceinline__ KvRows kv_tile(const Cta& c, int j) const {
    return PagedKv<Cfg>::tile(*this, c.seq, c.kv_len, j);
  }
  __device__ __forceinline__ void load_k(const Cta& c, const KvRows& t, uint32_t dst, const CUtensorMap* tm, uint32_t bar,
                                         int chunk) const {
    PagedKv<Cfg>::load_k(*this, c.kvh, t, dst, tm, bar, chunk);
  }
  __device__ __forceinline__ void load_v(const Cta& c, const KvRows& t, uint32_t dst, const CUtensorMap* tm,
                                         uint32_t bar) const {
    PagedKv<Cfg>::load_v(*this, c.kvh, t, dst, tm, bar);
  }
  __device__ __forceinline__ int diag(const Cta& c, int r) const { return c.t0 + r / hb + c.shift; }
  __device__ __forceinline__ void zero_kv_tail(const Cta& c, int k0, uint32_t tile) const {
    zero_tile_tail<Cfg>(c.kv_len, k0, tile);
  }
  // the CTA's K/V head, from the grid rather than from Cta, so that no register holds it through the main loop
  __device__ __forceinline__ int kv_head() const { return blockIdx.z % (H / group); }
  // rows past the box, the sequence or the group are not stored
  __device__ __forceinline__ bool out_row(const Cta& c, int r, size_t& row) const {
    const int tt = r / hb, hh = r % hb;
    if (tt >= T || c.t0 + tt >= Lq || c.h0 - c.kvh * group + hh >= group) return false;
    row = (size_t(c.seq) * Lq + c.t0 + tt) * size_t(H) + c.h0 + hh;
    return true;
  }
  __device__ __forceinline__ void store(const Cta& c, int r, const float (&o)[Cfg::DV / 2], int h, float inv, float m,
                                        float l, void* O, int D) const {
    size_t row;
    if (!out_row(c, r, row)) return;
    if (gridDim.x == 1) return store_o<Cfg>(O, row, 0, D, o, h, inv);
    // one split of several: O / l in fp32 and the base-2 log-sum-exp (-inf: no key seen)
    const int lane = threadIdx.x & 31;
    float* dst = part + (size_t(blockIdx.x) * size_t(rows) + row) * size_t(D);
#pragma unroll
    for (int i = 0; i < Cfg::DV / 8; ++i) {
      const int col = 8 * i + 2 * (lane & 3);
      if (col >= D) continue;
      *reinterpret_cast<float2*>(dst + col) = make_float2(o[4 * i + 2 * h] * inv, o[4 * i + 2 * h + 1] * inv);
    }
    if ((lane & 3) == 0) lse[size_t(blockIdx.x) * size_t(rows) + row] = l > 0.f ? m + log2f(l) : -INFINITY;
  }
};

// Packed queries over paged caches.  Q / O, the grid, the causal diagonals and the stores are AttnPacked's; K / V are
// read through the block table as PagedKv describes.  Sequence b has Lk = cu_k[b + 1] - cu_k[b] keys, clamped to
// [0, pages_per_seq * page_size] (cu_k gives lengths only, no cache position).
template <class Cfg>
struct AttnPackedPaged : AttnPacked<Cfg> {
  const int* table;
  int page_size, pages_per_seq, box_rows, oob;

  using Cta = typename AttnPacked<Cfg>::Cta;
  using KvRows = typename PagedKv<Cfg>::Rows;
  __device__ __forceinline__ bool setup(Cta& c) const {
    if (!AttnPacked<Cfg>::setup(c)) return false;
    const int q_len = c.kv_len - c.shift;
    c.kv_len = min(max(c.kv_len, 0), pages_per_seq * page_size);
    c.shift = c.kv_len - q_len;
    return true;
  }
  __device__ __forceinline__ KvRows kv_tile(const Cta& c, int j) const {
    return PagedKv<Cfg>::tile(*this, blockIdx.z / this->H, c.kv_len, j);
  }
  __device__ __forceinline__ void load_k(const Cta& c, const KvRows& t, uint32_t dst, const CUtensorMap* tm, uint32_t bar,
                                         int chunk) const {
    PagedKv<Cfg>::load_k(*this, c.kv_head, t, dst, tm, bar, chunk);
  }
  __device__ __forceinline__ void load_v(const Cta& c, const KvRows& t, uint32_t dst, const CUtensorMap* tm,
                                         uint32_t bar) const {
    PagedKv<Cfg>::load_v(*this, c.kv_head, t, dst, tm, bar);
  }
  __device__ __forceinline__ int kv_head() const { return blockIdx.z % this->H / this->group; }
};

// A paged mode (AttnDecode, AttnPackedPaged) over fp8 caches: KVF is B200K_FP8_E4M3 or B200K_FP8_E5M2, k_scale /
// v_scale fp32 [H_kv] or null (1.0).  The producer warpgroup stages each KV tile's fp8 rows and converts them into the
// 16-bit K / V rings (fp8_produce), so the consumers run the 16-bit main loop unchanged; the scales enter through two
// hooks: k_scale[h] multiplies scale_log2, and v_scale[h] the epilogue's 1 / l.  V rows past the key count are written
// as zeros by the producer, so zero_kv_tail has nothing to do.
template <class Mode, int KVF>
struct Fp8Kv : Mode {
  static constexpr int KV_FP8 = KVF;
  const float *k_scale, *v_scale;

  using Cta = typename Mode::Cta;
  __device__ __forceinline__ float kv_scale_log2(float scale_log2) const {
    return k_scale ? scale_log2 * __ldg(k_scale + Mode::kv_head()) : scale_log2;
  }
  __device__ __forceinline__ float kv_out_scale(float inv) const {
    return v_scale ? inv * __ldg(v_scale + Mode::kv_head()) : inv;
  }
  __device__ __forceinline__ void zero_kv_tail(const Cta&, int, uint32_t) const {}
};

// The KV format of a mode: 0 for the 16-bit caches, else Fp8Kv's KVF (also through WithLse, which derives from it).
template <class M, class = void>
struct KvFormat {
  static constexpr int value = 0;
};
template <class M>
struct KvFormat<M, std::void_t<decltype(M::KV_FP8)>> {
  static constexpr int value = M::KV_FP8;
};

// Shared memory a mode adds to Cfg::smem_bytes: an fp8 mode's staging ring of two slots, each one BN-row fp8 tile of K
// and one of V (BN x 128 bytes each: columns past D are zero-filled by TMA), and the slots' two full barriers.
template <class Cfg, class Mode>
constexpr int kv_stage_bytes() {
  return KvFormat<Mode>::value ? 2 * 2 * Cfg::BN * 128 + 16 : 0;
}

// Two fp8 values (x: the first in the low byte) -> two 16-bit values of DT (the first in the low half), exactly:
// every e4m3 and e5m2 value is an f16 value, and every f16 value converts exactly to f32 and, from these formats,
// to bf16.
template <int DT, int KVF>
__device__ __forceinline__ uint32_t fp8x2_to_16(uint16_t x) {
  uint32_t h;
  if constexpr (KVF == B200K_FP8_E4M3) asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h) : "h"(x));
  else asm("cvt.rn.f16x2.e5m2x2 %0, %1;" : "=r"(h) : "h"(x));
  if constexpr (DT == 0) {
    return h;
  } else {
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&h));
    const __nv_bfloat162 b = __floats2bfloat162_rn(f.x, f.y);
    return *reinterpret_cast<const uint32_t*>(&b);
  }
}

// Columns [64 c, 64 c + 64) of row r of a staged fp8 tile (BN rows of 128 bytes, 128B-swizzled as TMA wrote them) into
// row r of a 16-bit chunk (BN rows of 64 columns, the layout TMA writes for the 16-bit caches), or zeros.  Row r's
// 16-byte unit u sits at unit u ^ (r % 8) of the row; eight threads with consecutive rows hit eight distinct units,
// so neither the loads nor the stores conflict on banks.
template <int DT, int KVF>
__device__ __forceinline__ void fp8_row_chunk(uint32_t src, uint32_t dst, int r, int c, bool zero) {
  const uint32_t sw = r & 7;
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    uint32_t w[4] = {0u, 0u, 0u, 0u}, y[8];
    if (!zero)
      asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
                   : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3])
                   : "r"(src + r * 128 + (((4 * c + u) ^ sw) << 4)));
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      y[2 * k] = fp8x2_to_16<DT, KVF>(uint16_t(w[k] & 0xFFFFu));
      y[2 * k + 1] = fp8x2_to_16<DT, KVF>(uint16_t(w[k] >> 16));
    }
#pragma unroll
    for (int h = 0; h < 2; ++h)
      asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(dst + r * 128 + (((2 * u + h) ^ sw) << 4)),
                   "r"(y[4 * h]), "r"(y[4 * h + 1]), "r"(y[4 * h + 2]), "r"(y[4 * h + 3])
                   : "memory");
  }
}

// The producer warpgroup of an fp8 mode.  Its thread 0 TMA-loads each KV tile's fp8 K and V rows (the mode's paged
// boxes, 128 fp8 columns wide) into staging slot n % 2 and, for the first two tiles, before the loop.  Per tile all 128
// threads wait for the slot, and thread t converts key row t: the nqc K chunks (each after its kempty), then
// fence.proxy.async and a named barrier, after which thread 0 arrives once on each chunk's kfull; then the DV / 64 V
// chunks (after vempty, zeros for keys at or past kv_len, whatever the cache holds there), the fence and the barrier,
// after which thread 0 arrives on vfull and refills the slot with tile n + 2.  No thread ever waits on itself: the
// slot's reads are done at the barrier.
template <class Cfg, class Mode>
__device__ __forceinline__ void fp8_produce(const Mode& md, const typename Mode::Cta& cta, KvTiles kv, int nqc, uint32_t sK,
                                            uint32_t sV, uint32_t sS, uint32_t kfull, uint32_t kempty, uint32_t vfull,
                                            uint32_t vempty, uint32_t sfull, const CUtensorMap* tmK,
                                            const CUtensorMap* tmV) {
  constexpr int KVF = KvFormat<Mode>::value, TILE = Cfg::BN * 128, KST = Cfg::KSTAGES, VST = Cfg::VSTAGES;
  const int r = threadIdx.x;
  auto stage = [&](int j) {
    const int ss = (j - kv.first) % 2;
    const auto rows = md.kv_tile(cta, j);
    mbar_arrive_expect_tx(sfull + 8 * ss, 2 * TILE);
    md.load_k(cta, rows, sS + ss * 2 * TILE, tmK, sfull + 8 * ss, 0);
    md.load_k(cta, rows, sS + ss * 2 * TILE + TILE, tmV, sfull + 8 * ss, 0);
  };
  if (r == 0)
    for (int j = kv.first; j < kv.end && j < kv.first + 2; ++j) stage(j);
  int kc = 0;
  for (int j = kv.first; j < kv.end; ++j) {
    const int n = j - kv.first;
    const uint32_t src = sS + (n % 2) * 2 * TILE;
    mbar_wait_nocall(sfull + 8 * (n % 2), (n / 2) & 1);
    for (int c = 0; c < nqc; ++c) {
      const int s = (kc + c) % KST;
      if (kc + c >= KST) mbar_wait_nocall(kempty + 8 * s, (((kc + c) / KST) - 1) & 1);
      fp8_row_chunk<Cfg::DT, KVF>(src, sK + s * Cfg::K_BYTES, r, c, false);
    }
    fence_proxy_async_smem();  // generic-proxy stores -> the wgmma's operand reads
    named_bar_sync(2, 128);
    if (r == 0)
      for (int c = 0; c < nqc; ++c) mbar_arrive(kfull + 8 * ((kc + c) % KST));
    kc += nqc;
    const int sv = n % VST;
    if (n >= VST) mbar_wait_nocall(vempty + 8 * sv, ((n / VST) - 1) & 1);
    const bool past = j * Cfg::BN + r >= cta.kv_len;
#pragma unroll
    for (int i = 0; i < Cfg::DV / 64; ++i)
      fp8_row_chunk<Cfg::DT, KVF>(src + TILE, sV + sv * Cfg::V_BYTES + i * Cfg::BN * 128, r, i, past);
    fence_proxy_async_smem();
    named_bar_sync(2, 128);
    if (r == 0) {
      mbar_arrive(vfull + 8 * sv);
      if (j + 2 < kv.end) stage(j + 2);
    }
  }
}

// A mode that also writes each stored row's natural-log log-sum-exp to `lse` (fp32, indexed like the rows of O): m is
// the row's final running max in base-2 units and l the sum of the rounded P that divides O, so O and lse describe
// one softmax.  A row that saw no key gets -inf.  Decode takes it only unsplit; split rows are merged by the combine.
template <class Mode>
struct WithLse : Mode {
  float* lse;
  template <int N>
  __device__ __forceinline__ void store(const typename Mode::Cta& c, int r, const float (&o)[N], int h, float inv,
                                        float m, float l, void* O, int D) const {
    Mode::store(c, r, o, h, inv, m, l, O, D);
    size_t row;
    if (Mode::out_row(c, r, row) && (threadIdx.x & 3) == 0) lse[row] = l > 0.f ? (m + log2f(l)) * 0.6931472f : -INFINITY;
  }
};

template <class Cfg, class Mode>
__global__ void __launch_bounds__(Cfg::THREADS, 1)
    attn_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                          const __grid_constant__ CUtensorMap tmV, void* O, int D, int nqc, float scale_log2,
                          const Mode md) {
  constexpr int BM = Cfg::BM, BN = Cfg::BN, DV = Cfg::DV, KST = Cfg::KSTAGES, VST = Cfg::VSTAGES;
  constexpr bool FP8 = KvFormat<Mode>::value != 0;
  static_assert(!FP8 || BN == 128, "fp8 caches: one producer thread per key of a tile");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sQ = (smem_u32(smem_raw) + 1023) & ~1023u;
  const uint32_t sK = sQ + nqc * BM * 128, sV = sK + KST * Cfg::K_BYTES;
  const uint32_t sS = sV + VST * Cfg::V_BYTES;  // fp8 staging ring (fp8 modes only)
  const uint32_t qbar = sS + (FP8 ? 2 * 2 * BN * 128 : 0);
  const uint32_t kfull = qbar + 8, kempty = kfull + 8 * KST, vfull = kempty + 8 * KST, vempty = vfull + 8 * VST;
  const uint32_t sfull = vempty + 8 * VST;  // fp8 staging slots' full barriers

  typename Mode::Cta cta;
  if (!md.setup(cta)) return;
  const KvTiles kv = md.tiles(cta);
  const int wg = threadIdx.x / 128;

  if (threadIdx.x == 0) {
    mbar_init(qbar, 1);
    for (int s = 0; s < KST; ++s) {
      mbar_init(kfull + 8 * s, 1);
      mbar_init(kempty + 8 * s, Cfg::NWG);
    }
    for (int s = 0; s < VST; ++s) {
      mbar_init(vfull + 8 * s, 1);
      mbar_init(vempty + 8 * s, Cfg::NWG);
    }
    if constexpr (FP8)
      for (int s = 0; s < 2; ++s) mbar_init(sfull + 8 * s, 1);
    fence_mbar_init();
  }
  __syncthreads();

  if constexpr (FP8) {
    // Two consumer warpgroups hold 168 registers, the most a 384-thread CTA allows, and ptxas spills their row sums at
    // that count once the converting producer shares the kernel.  The producer needs fewer: it runs on 80 and the
    // consumers on 208, within the CTA's 384 x 168.  (The values computed before the split must fit the producer's
    // count: at 56, ptxas spills them.)
    constexpr int PRODUCER_REGS = 80, CONSUMER_REGS = 208;
    static_assert(128 * PRODUCER_REGS + 256 * CONSUMER_REGS <= 384 * 168, "more registers than the CTA holds");
    if (wg == 0) {
      if constexpr (Cfg::NWG == 2) setmaxnreg_dec<PRODUCER_REGS>();
      if (threadIdx.x == 0) {
        mbar_arrive_expect_tx(qbar, nqc * md.q_bytes());
        for (int c = 0; c < nqc; ++c) md.load_q(cta, sQ + c * BM * 128, &tmQ, qbar, c);
      }
      fp8_produce<Cfg>(md, cta, kv, nqc, sK, sV, sS, kfull, kempty, vfull, vempty, sfull, &tmK, &tmV);
      return;
    }
    if constexpr (Cfg::NWG == 2) setmaxnreg_inc<CONSUMER_REGS>();
    scale_log2 = md.kv_scale_log2(scale_log2);
  } else if (wg == 0) {
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(qbar, nqc * md.q_bytes());
      for (int c = 0; c < nqc; ++c) md.load_q(cta, sQ + c * BM * 128, &tmQ, qbar, c);
      int kc = 0;
      for (int j = kv.first; j < kv.end; ++j) {
        const auto t = md.kv_tile(cta, j);
        for (int c = 0; c < nqc; ++c, ++kc) {
          const int s = kc % KST;
          if (kc >= KST) mbar_wait(kempty + 8 * s, ((kc / KST) - 1) & 1);
          mbar_arrive_expect_tx(kfull + 8 * s, Cfg::K_BYTES);
          md.load_k(cta, t, sK + s * Cfg::K_BYTES, &tmK, kfull + 8 * s, c);
        }
        const int n = j - kv.first, s = n % VST;
        if (n >= VST) mbar_wait(vempty + 8 * s, ((n / VST) - 1) & 1);
        mbar_arrive_expect_tx(vfull + 8 * s, Cfg::V_BYTES);
        md.load_v(cta, t, sV + s * Cfg::V_BYTES, &tmV, vfull + 8 * s);
      }
    }
    return;
  }

  // The fp8 modes wait without the timeout's printf: a kernel with a call in it keeps neither its setmaxnreg nor
  // unserialised wgmmas.  The 16-bit modes keep the wait they have always compiled with.
  auto wait = [](uint32_t bar, uint32_t parity) {
    if constexpr (FP8) mbar_wait_nocall(bar, parity);
    else mbar_wait(bar, parity);
  };
  const int cw = wg - 1, lane = threadIdx.x & 31, warp = (threadIdx.x & 127) / 32;
  const bool leader = (threadIdx.x & 127) == 0;
  const int row0 = cta.q0 + cw * 64 + warp * 16 + lane / 4;  // this thread's rows: row0 and row0 + 8
  float o[DV / 2];
#pragma unroll
  for (int i = 0; i < DV / 2; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  wait(qbar, 0);

  int kc = 0;
  for (int j = kv.first; j < kv.end; ++j) {
    const int n = j - kv.first;  // position in the rings
    // ---- S = Q K^T over the head dim, chunk by chunk
    float s_acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) s_acc[i] = 0.f;
    for (int c = 0; c < nqc; ++c, ++kc) {
      const int s = kc % KST;
      wait(kfull + 8 * s, (kc / KST) & 1);
      fence_regs<BN / 2>(s_acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t da = wgmma_desc(sQ + c * BM * 128 + cw * 64 * 128 + k * 32, 16, 1024);
        const uint64_t db = wgmma_desc(sK + s * Cfg::K_BYTES + k * 32, 16, 1024);
        wgmma_ss<Cfg::DT, BN, 0, 0>(s_acc, da, db, 1);
      }
      wgmma_commit();
      wgmma_wait<1>();
      fence_regs<BN / 2>(s_acc);
      if (c > 0 && leader) mbar_arrive(kempty + 8 * ((kc - 1) % KST));
    }
    wgmma_wait<0>();
    fence_regs<BN / 2>(s_acc);
    if (leader) mbar_arrive(kempty + 8 * ((kc - 1) % KST));

    // ---- masks: keys past the valid length, keys after the row's causal diagonal.  A tile that ends at or before the
    // diagonal of the warpgroup's first row needs no causal mask.
    const int k0 = j * BN;
    if (k0 + BN > cta.kv_len || (md.causal && k0 + BN - 1 > md.diag(cta, cta.q0 + cw * 64))) {
      const int diag[2] = {md.diag(cta, row0), md.diag(cta, row0 + 8)};
#pragma unroll
      for (int i = 0; i < BN / 8; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int key = k0 + 8 * i + 2 * (lane & 3) + e;
            if (key >= cta.kv_len || (md.causal && key > diag[h])) s_acc[4 * i + 2 * h + e] = -INFINITY;
          }
    }

    // ---- online softmax (a row lives in the 4 lanes of a quad)
    float alpha[2], mu[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) mx = fmaxf(mx, fmaxf(s_acc[4 * i + 2 * h], s_acc[4 * i + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m[h], mx * scale_log2);
      mu[h] = (m_new == -INFINITY) ? 0.f : m_new;
      alpha[h] = ex2(m[h] - mu[h]);
      m[h] = m_new;
      l[h] *= alpha[h];
    }
    uint32_t pa[BN / 16][4];
#pragma unroll
    for (int i = 0; i < BN / 8; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float p0 = ex2(fmaf(s_acc[4 * i + 2 * h], scale_log2, -mu[h]));
        float p1 = ex2(fmaf(s_acc[4 * i + 2 * h + 1], scale_log2, -mu[h]));
        pa[i / 2][(i & 1) * 2 + h] = pack_round<Cfg::DT>(p0, p1);
        l[h] += p0 + p1;
      }
#pragma unroll
    for (int i = 0; i < DV / 8; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        o[4 * i + 2 * h] *= alpha[h];
        o[4 * i + 2 * h + 1] *= alpha[h];
      }

    // ---- O += P V
    const int sv = n % VST;
    wait(vfull + 8 * sv, (n / VST) & 1);
    const uint32_t vb = sV + sv * Cfg::V_BYTES;
    md.zero_kv_tail(cta, k0, vb);
    fence_regs<DV / 2>(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk) {
      const uint64_t db = Cfg::V_DN ? wgmma_desc(vb + (kk / 4) * DV * 128 + (kk % 4) * 32, 16, 1024)
                                    : wgmma_desc(vb + kk * 2048, BN * 128, 1024);
      wgmma_rs<Cfg::DT, DV, Cfg::V_DN ? 0 : 1>(o, pa[kk], db, 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<DV / 2>(o);
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk)  // P registers are read by the MMAs until the wait above
#pragma unroll
      for (int e = 0; e < 4; ++e) asm volatile("" : "+r"(pa[kk][e])::"memory");
    if (leader) mbar_arrive(vempty + 8 * sv);
  }

  // ---- epilogue: O / l; rows that saw no key have l = 0 and store 0
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float t = l[h];
    t += __shfl_xor_sync(0xffffffffu, t, 1);
    t += __shfl_xor_sync(0xffffffffu, t, 2);
    if constexpr (FP8) md.store(cta, row0 + 8 * h, o, h, md.kv_out_scale(t > 0.f ? 1.f / t : 0.f), m[h], t, O, D);
    else md.store(cta, row0 + 8 * h, o, h, t > 0.f ? 1.f / t : 0.f, m[h], t, O, D);
  }
}

// The launch every mode shares: the shared-memory check, Q / K / V as tensor maps, then the kernel on `grid`.
// scale <= 0 means 1 / sqrt(D).
template <class Cfg, class Mode>
static int launch_attn(const AttnTensor (&qkv)[3], dim3 grid, void* O, int64_t D, float scale, const Mode& args,
                       cudaStream_t s, const DeviceInfo& di) {
  const int nqc = int((D + 63) / 64);
  const int smem = Cfg::smem_bytes(nqc) + kv_stage_bytes<Cfg, Mode>();
  if (smem > di.max_smem_optin)
    return set_error(B200K_ESHAPE, "attention: %d bytes of shared memory needed, device allows %d", smem, di.max_smem_optin);
  CUtensorMap tm[3];
  int rc;
  for (int i = 0; i < 3; ++i)
    if ((rc = attn_tmap(&tm[i], qkv[i]))) return rc;
  auto kern = attn_fwd_wgmma_kernel<Cfg, Mode>;
  if ((rc = ensure_dynamic_smem(reinterpret_cast<const void*>(kern), di.device, smem))) return rc;
  if (scale <= 0.f) scale = 1.0f / sqrtf(float(D));
  kern<<<grid, Cfg::THREADS, smem, s>>>(tm[0], tm[1], tm[2], O, int(D), nqc, scale * 1.4426950408889634f, args);
  B200K_CHECK_CUDA(cudaGetLastError());
  return B200K_OK;
}

// Dense [B, H, N, D]: one 3-D map per tensor over (D, N, B * H); V stored [B, H, D, N] over (N, D, B * H).
// `args` as it is, or with its lse written when `lse` is not null.
template <class Cfg, class Mode>
static int launch_mode(const AttnTensor (&qkv)[3], dim3 grid, void* O, int64_t D, float scale, const Mode& args,
                       float* lse, cudaStream_t s, const DeviceInfo& di) {
  if (lse) return launch_attn<Cfg>(qkv, grid, O, D, scale, WithLse<Mode>{args, lse}, s, di);
  return launch_attn<Cfg>(qkv, grid, O, D, scale, args, s, di);
}

// lse: null, or [B, H, N] fp32 (the D <= 128 configurations only).
template <class Cfg>
static int launch_dense(const void* Q, const void* K, const void* V, void* O, int64_t B, int64_t H, int64_t N, int64_t D,
                        float scale, const int* seqlens, int causal, float* lse, cudaStream_t s, const DeviceInfo& di) {
  const int64_t BH = B * H;
  AttnTensor v = {V, BH, N, D, 1, Cfg::BN};
  if (Cfg::V_DN) v = {V, BH, D, N, 1, Cfg::DV};
  const AttnTensor qkv[3] = {{Q, BH, N, D, 1, Cfg::BM}, {K, BH, N, D, 1, Cfg::BN}, v};
  const dim3 grid(unsigned((N + Cfg::BM - 1) / Cfg::BM), unsigned((D + Cfg::DV - 1) / Cfg::DV), unsigned(BH));
  const AttnDense<Cfg> args = {seqlens, int(N), int(H), causal ? 1 : 0};
  if constexpr (Cfg::DV <= 128) return launch_mode<Cfg>(qkv, grid, O, D, scale, args, lse, s, di);
  else return launch_attn<Cfg>(qkv, grid, O, D, scale, args, s, di);
}

// The D <= 128 configurations: BN = 128 keys per tile; O columns DV = 64 for D = 32 / 64, 128 for D = 96 / 128.  V
// stored [D, N] is built for fp16 only.
template <int NWG, bool V_DN, class Run>
static int run_attn_cfg(int dtype, int64_t D, Run run) {
  const bool narrow = D <= 64;
  if (dtype != B200K_BF16)
    return narrow ? run(AttnCfg<0, 64, NWG, 128, V_DN>()) : run(AttnCfg<0, 128, NWG, 128, V_DN>());
  if constexpr (V_DN) return set_error(B200K_EARG, "attention: the [B,H,D,N] V layout is built for fp16 only");
  else return narrow ? run(AttnCfg<1, 64, NWG, 128, false>()) : run(AttnCfg<1, 128, NWG, 128, false>());
}

// Merges `splits` partial attentions of each row over disjoint key sets: O[row] = sum_s 2^(t_s - max) part_s[row] /
// sum_s 2^(t_s - max), summed in ascending s, so the result does not depend on which part finished first.  A part with
// no key for the row has lse = -inf and adds nothing; a row no part saw a key for is 0.
//   Part = float     KV-cache decode with several splits: fp32 O / l partials, t_s = lse_s in base 2.  One thread per
//                    (row, column pair).
//   Part = uint16_t  b200k_attn_merge: DT partials, t_s = lse_s * log2(e) from a natural-log lse; a part with
//                    lse_s = -inf is skipped, so whatever its O holds (NaN included) never reaches the result.  One
//                    thread per (row, 8 columns).
// LSE: also write the merged natural-log lse of each row to lse_out ([rows]; -inf where no part saw a key).
template <int DT, class Part = float, bool LSE = false>
__global__ void attn_combine_kernel(const Part* __restrict__ part, const float* __restrict__ lse, void* O, long long rows,
                                    int D, int splits, float* __restrict__ lse_out = nullptr) {
  constexpr bool P16 = sizeof(Part) == 2;
  constexpr int VEC = P16 ? 8 : 2;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x, pairs = D / VEC;
  if (i >= rows * pairs) return;
  const long long row = i / pairs;
  const int c = VEC * int(i % pairs);
  auto t = [&](int s) { return P16 ? lse[s * rows + row] * 1.4426950f : lse[s * rows + row]; };
  float mx = -INFINITY;
  for (int s = 0; s < splits; ++s) mx = fmaxf(mx, t(s));
  float x[VEC] = {}, den = 0.f;
  if (mx != -INFINITY) {
    for (int s = 0; s < splits; ++s) {
      const float ts = t(s);
      if (P16 && ts == -INFINITY) continue;
      const float w = ex2(ts - mx);
      if constexpr (P16) {
        const uint4 p = *reinterpret_cast<const uint4*>(part + (s * rows + row) * D + c);
        const uint32_t pw[4] = {p.x, p.y, p.z, p.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = unpack2<DT>(pw[k]);
          x[2 * k] = fmaf(w, f.x, x[2 * k]);
          x[2 * k + 1] = fmaf(w, f.y, x[2 * k + 1]);
        }
      } else {
        const float2 p = *reinterpret_cast<const float2*>(part + (s * rows + row) * D + c);
        x[0] = fmaf(w, p.x, x[0]);
        x[1] = fmaf(w, p.y, x[1]);
      }
      den += w;
    }
  }
  const float inv = den > 0.f ? 1.f / den : 0.f;
  uint32_t out[VEC / 2];
#pragma unroll
  for (int k = 0; k < VEC / 2; ++k) {
    x[2 * k] *= inv;
    x[2 * k + 1] *= inv;
    out[k] = pack_round<DT>(x[2 * k], x[2 * k + 1]);
  }
  uint16_t* dst = static_cast<uint16_t*>(O) + row * D + c;
  if constexpr (P16) *reinterpret_cast<uint4*>(dst) = make_uint4(out[0], out[1], out[2], out[3]);
  else *reinterpret_cast<uint32_t*>(dst) = out[0];
  if constexpr (LSE)
    if (c == 0) lse_out[row] = den > 0.f ? (mx + log2f(den)) * 0.6931472f : -INFINITY;
}

// KV-cache append (b200k_fa2_fwd_kvcache_append), in front of the decode kernel.  New token i of sequence b goes to cache
// position p = max(cache_seqlens[b], 0) + i when p < capacity; lens_out[b] = that base + L_new is what the decode kernel
// reads as its lengths.  With rotary the first rotary_dim columns of each new K row are rotated at p and each Q row at
// base + t (causal) or base, into q_out.  cos / sin are [rotary_seqlen, rotary_dim / 2].
struct KvAppend {
  const uint16_t *q, *k_new, *v_new, *cos, *sin;
  uint16_t *q_out, *k_cache, *v_cache;
  const int *seqlens, *table;
  int* lens_out;
  long long kv_rows, q_rows;  // B * L_new * H_kv, B * Lq * H (rotary only, else 0)
  long long rotary_seqlen;
  int B, L_new, Lq, H, H_kv, D, page_size, pages_per_seq, rotary_dim, causal;
  const float *k_scale = nullptr, *v_scale = nullptr;  // fp8 caches: fp32 [H_kv] or null (1.0)
};

// Eight 16-bit values of DT -> eight fp8 bytes of KVF (the first in the low byte): cvt.rn.satfinite of
// float(x) / scale in IEEE fp32, so values past the format's largest finite value become it and NaN stays NaN.
template <int DT, int KVF>
__device__ __forceinline__ uint2 quantize8(uint4 x, float scale) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(&x);
  uint32_t out[2];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 f = unpack2<DT>(w[k]);
    const float lo = __fdiv_rn(f.x, scale), hi = __fdiv_rn(f.y, scale);
    uint16_t q;
    if constexpr (KVF == B200K_FP8_E4M3) asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(q) : "f"(hi), "f"(lo));
    else asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(q) : "f"(hi), "f"(lo));
    out[k / 2] = k & 1 ? out[k / 2] | (uint32_t(q) << 16) : uint32_t(q);
  }
  return make_uint2(out[0], out[1]);
}

// Pair (x0, x1) at position pos becomes (x0 c - x1 s, x0 s + x1 c) in fp32, rounded once.  The products are not left to
// contraction, so Q and K rows go through the same operations wherever this is inlined.
__device__ __forceinline__ float rot_lo(float x0, float x1, float c, float s) { return fmaf(x0, c, -__fmul_rn(x1, s)); }
__device__ __forceinline__ float rot_hi(float x0, float x1, float c, float s) { return fmaf(x0, s, __fmul_rn(x1, c)); }

// Rotates 16-byte vector v (columns 8v .. 8v + 7 < rotary_dim) of `row`.  Interleaved pairs (2j, 2j + 1) lie inside the
// vector; NeoX pairs (j, j + rotary_dim / 2) pair it with the whole vector rotary_dim / 2 columns away.
template <int DT, bool INTERLEAVED>
__device__ __forceinline__ uint4 rotate_vec(uint4 x, const uint16_t* row, int v, long long pos, const KvAppend& a) {
  const int half = a.rotary_dim / 2;
  const long long crow = pos < a.rotary_seqlen ? pos : a.rotary_seqlen - 1;
  const uint16_t* cs = a.cos + crow * half;
  const uint16_t* sn = a.sin + crow * half;
  uint32_t* w = reinterpret_cast<uint32_t*>(&x);
  if constexpr (INTERLEAVED) {
    const uint2 cw = __ldg(reinterpret_cast<const uint2*>(cs + 4 * v)), sw = __ldg(reinterpret_cast<const uint2*>(sn + 4 * v));
    const float2 c[2] = {unpack2<DT>(cw.x), unpack2<DT>(cw.y)}, s[2] = {unpack2<DT>(sw.x), unpack2<DT>(sw.y)};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 p = unpack2<DT>(w[k]);
      const float ck = k & 1 ? c[k / 2].y : c[k / 2].x, sk = k & 1 ? s[k / 2].y : s[k / 2].x;
      float lo = rot_lo(p.x, p.y, ck, sk), hi = rot_hi(p.x, p.y, ck, sk);
      w[k] = pack_round<DT>(lo, hi);
    }
  } else {
    const bool first = 8 * v < half;
    const int j0 = first ? 8 * v : 8 * v - half;
    const uint4 y = __ldg(reinterpret_cast<const uint4*>(row + (first ? 8 * v + half : j0)));
    const uint4 cv = __ldg(reinterpret_cast<const uint4*>(cs + j0)), sv = __ldg(reinterpret_cast<const uint4*>(sn + j0));
    const uint32_t* yw = reinterpret_cast<const uint32_t*>(&y);
    const uint32_t* cw = reinterpret_cast<const uint32_t*>(&cv);
    const uint32_t* sw = reinterpret_cast<const uint32_t*>(&sv);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 p = unpack2<DT>(w[k]), q = unpack2<DT>(yw[k]), c = unpack2<DT>(cw[k]), s = unpack2<DT>(sw[k]);
      // first half: this vector holds x0, the partner x1; second half: the partner holds x0
      float lo = first ? rot_lo(p.x, q.x, c.x, s.x) : rot_hi(q.x, p.x, c.x, s.x);
      float hi = first ? rot_lo(p.y, q.y, c.y, s.y) : rot_hi(q.y, p.y, c.y, s.y);
      w[k] = pack_round<DT>(lo, hi);
    }
  }
  return x;
}

// One thread per 16-byte vector: K rows, then V rows, then (rotary) Q rows; the first B threads also write lens_out.
// Cache slots are written only for positions below the capacity, and the block table is read only for those.  KVF: 0
// for 16-bit caches, or the fp8 format the vector is quantised to (quantize8, by the scale of its K/V head) after
// rotary, into one 8-byte store.
template <int DT, bool ROTARY, bool INTERLEAVED, int KVF>
__global__ void __launch_bounds__(256) kvcache_append_kernel(const KvAppend a) {
  const int vecs = a.D / 8;
  const long long tid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (tid < a.B) {
    const long long n = (long long)max(__ldg(a.seqlens + tid), 0) + a.L_new;
    a.lens_out[tid] = int(n < INT_MAX ? n : INT_MAX);
  }
  const long long cap = (long long)a.pages_per_seq * a.page_size;
  const long long total = (2 * a.kv_rows + a.q_rows) * vecs;
  for (long long i = tid; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long row = i / vecs;
    const int v = int(i - row * vecs);
    if (row < 2 * a.kv_rows) {
      const bool is_k = row < a.kv_rows;
      if (!is_k) row -= a.kv_rows;
      const long long b = row / ((long long)a.L_new * a.H_kv);
      const int tok = int((row / a.H_kv) % a.L_new), hk = int(row % a.H_kv);
      const long long p = (long long)max(__ldg(a.seqlens + b), 0) + tok;
      if (p >= cap) continue;
      const uint16_t* src = (is_k ? a.k_new : a.v_new) + row * a.D;
      uint4 x = __ldg(reinterpret_cast<const uint4*>(src) + v);
      if constexpr (ROTARY)
        if (is_k && 8 * v < a.rotary_dim) x = rotate_vec<DT, INTERLEAVED>(x, src, v, p, a);
      const long long page = a.table ? (long long)__ldg(a.table + b * a.pages_per_seq + p / a.page_size) : b;
      if constexpr (KVF == 0) {
        uint16_t* dst = (is_k ? a.k_cache : a.v_cache) + ((page * a.page_size + p % a.page_size) * a.H_kv + hk) * a.D;
        reinterpret_cast<uint4*>(dst)[v] = x;
      } else {
        const float* sc = is_k ? a.k_scale : a.v_scale;
        uint8_t* dst = reinterpret_cast<uint8_t*>(is_k ? a.k_cache : a.v_cache) +
                       ((page * a.page_size + p % a.page_size) * a.H_kv + hk) * a.D;
        reinterpret_cast<uint2*>(dst)[v] = quantize8<DT, KVF>(x, sc ? __ldg(sc + hk) : 1.f);
      }
    } else if constexpr (ROTARY) {
      row -= 2 * a.kv_rows;
      const long long b = row / ((long long)a.Lq * a.H);
      const int t = int((row / a.H) % a.Lq);
      const uint16_t* src = a.q + row * a.D;
      uint4 x = __ldg(reinterpret_cast<const uint4*>(src) + v);
      if (8 * v < a.rotary_dim)
        x = rotate_vec<DT, INTERLEAVED>(x, src, v, (long long)max(__ldg(a.seqlens + b), 0) + (a.causal ? t : 0), a);
      reinterpret_cast<uint4*>(a.q_out + row * a.D)[v] = x;
    }
  }
}

// One call of the KV-cache family as its entry point received it: decode (b200k_fa2_fwd_kvcache), append
// (b200k_fa2_fwd_kvcache_append), fp8 caches (b200k_fa2_kvcache_fp8), packed prefill over paged caches
// (b200k_fa2_varlen_paged, _fp8), or the shapes of a workspace query.  The fields follow the entry points' parameter
// order.  A cache holds num_pages pages of page_size keys; a sequence's capacity is pages_per_seq pages (a contiguous
// cache: B pages of S keys, one per sequence; a workspace query: one page of max_seqlen_k keys).
struct KvCall {
  const char* fn;               // the entry point, in messages
  const char* lse_fn = nullptr;  // the name lse's alignment message uses (decode, append, fp8)
  bool fp8 = false;     // b200k_fa2_kvcache_fp8: kv_dtype, the scales and lse are checked before the append part
  bool append = false;  // new K / V rows go into the caches before the decode
  bool rotary = false;  // ... rotated by cos / sin
  const void *Q = nullptr, *K_cache = nullptr, *V_cache = nullptr;
  void* O = nullptr;
  float* lse = nullptr;
  const int* cu_seqlens_q = nullptr;  // paged prefill
  const int* seqlens = nullptr;       // cache_seqlens [B], or cu_seqlens_k [B + 1] in paged prefill
  const int* table = nullptr;         // block table [B, pages_per_seq], or null
  const float *k_scale = nullptr, *v_scale = nullptr;
  int kv_dtype = 0;  // 0: caches in dtype; B200K_FP8_E4M3 / B200K_FP8_E5M2 (Fp8Kv)
  const void *K_new = nullptr, *V_new = nullptr;
  int64_t L_new = 0;
  const void *cos = nullptr, *sin = nullptr;
  int64_t rotary_seqlen = 0, rotary_dim = 0;
  int interleaved = 0;
  int64_t B = 0, Lq = 0, total_q = 0, H = 0, H_kv = 0, D = 0;  // paged prefill: Lq is max_seqlen_q
  int64_t num_pages = 0, page_size = 0, pages_per_seq = 0;
  float scale = 0.f;
  int dtype = 0, causal = 0;
  void* workspace = nullptr;
  size_t workspace_bytes = 0;
  void* stream = nullptr;

  int64_t capacity() const { return pages_per_seq * page_size; }
};

// Calls f with the cache format of kv_dtype as a std::integral_constant: B200K_FP8_E4M3, B200K_FP8_E5M2, or 0 for
// caches in the call's dtype.
template <class F>
static int with_kv_format(int kv_dtype, F&& f) {
  if (kv_dtype == B200K_FP8_E4M3) return f(std::integral_constant<int, B200K_FP8_E4M3>());
  if (kv_dtype == B200K_FP8_E5M2) return f(std::integral_constant<int, B200K_FP8_E5M2>());
  return f(std::integral_constant<int, 0>());
}

// Mode `m` over caches of format KVF: as it is for 0, else through Fp8Kv with the call's scales.
template <int KVF, class Mode>
static auto kv_mode(const Mode& m, const KvCall& c) {
  if constexpr (KVF == 0) return m;
  else return Fp8Kv<Mode, KVF>{m, c.k_scale, c.v_scale};
}

// Launch geometry and workspace of a decode call, with or without new rows.  The 64 rows of a CTA are T tokens x hb
// query heads of one K/V head's group of G; a group wider than 64 takes nhb head tiles.  The workspace, each section on
// a 256-byte boundary: with new rows, int32 lengths [B] at 0 and the rotated Q [B, Lq, H, D] (rotary only) at q; from
// part, the fp32 partials of a split call.
struct KvcacheGrid {
  int hb = 1, T = 1, nhb = 1, splits = 1;
  int64_t qtiles = 1;
  size_t q = 0, part = 0, bytes = 0;
};

// The split rule.  ctas = B * H_kv * q tiles * head tiles CTAs each stream one K/V head of one sequence.  When they fill
// 80 % of the SMs, one split.  Otherwise each sequence's KV tiles are split s ways, s at most 128 and at most one split
// per two KV tiles of the capacity (max_seqlen_k); of those, the fewest splits whose grid fills its last wave of SMs
// within 85 % of the best fill any allowed s reaches.  It depends on the shapes and the SM count only, never on the
// lengths in the cache, so a captured graph keeps a valid grid while they grow.
static int kvcache_splits(int64_t ctas, int64_t max_seqlen_k, int sm_count) {
  if (ctas * 5 >= int64_t(sm_count) * 4) return 1;
  const int64_t tiles = (max_seqlen_k + 127) / 128;
  const int max_s = int(tiles / 2 < 1 ? 1 : (tiles / 2 > 128 ? 128 : tiles / 2));
  auto fill = [&](int s) {
    const int64_t n = ctas * s, waves = (n + sm_count - 1) / sm_count;
    return double(n) / double(waves * sm_count);
  };
  double best = 0.0;
  for (int s = 1; s <= max_s; ++s) best = fill(s) > best ? fill(s) : best;
  for (int s = 1; s <= max_s; ++s)
    if (fill(s) >= 0.85 * best) return s;
  return 1;
}

// The one workspace rule: the calls and the three workspace queries all size it here.
static KvcacheGrid kvcache_grid(const KvCall& c, int sm_count) {
  auto up = [](size_t n) { return (n + 255) & ~size_t(255); };
  KvcacheGrid g;
  const int64_t G = c.H / c.H_kv;
  g.hb = int(G < 64 ? G : 64);
  g.T = 64 / g.hb;
  g.nhb = int((G + g.hb - 1) / g.hb);
  g.qtiles = (c.Lq + g.T - 1) / g.T;
  g.splits = kvcache_splits(c.B * c.H_kv * g.qtiles * g.nhb, c.capacity(), sm_count);
  if (c.append) {
    g.q = up(size_t(c.B) * sizeof(int));
    g.part = g.q + (c.rotary ? up(size_t(c.B * c.Lq * c.H) * size_t(c.D) * 2) : 0);
  }
  g.bytes = g.part;
  if (g.splits > 1) g.bytes += size_t(g.splits) * size_t(c.B * c.Lq * c.H) * size_t(c.D + 1) * sizeof(float);
  return g;
}

// Shape checks of the decode calls and their workspace queries (before any CUDA call).
static int kvcache_check(const KvCall& c) {
  const char* fn = c.fn;
  const int64_t B = c.B, Lq = c.Lq, H = c.H, H_kv = c.H_kv, max_seqlen_k = c.capacity();
  if (B < 1 || Lq < 1 || H < 1 || H_kv < 1 || max_seqlen_k < 1 || H % H_kv != 0 || H > INT32_MAX)
    return set_error(B200K_ESHAPE, "%s: need B, Lq, H, H_kv, key capacity >= 1 and H %% H_kv == 0 (got B=%lld Lq=%lld "
                     "H=%lld H_kv=%lld capacity=%lld)", fn, (long long)B, (long long)Lq, (long long)H, (long long)H_kv,
                     (long long)max_seqlen_k);
  if (max_seqlen_k > INT32_MAX || B > INT32_MAX / Lq)
    return set_error(B200K_ESHAPE, "%s: B * Lq and the key capacity must be <= 2^31 - 1", fn);
  const int64_t G = H / H_kv, hb = G < 64 ? G : 64, tiles = ((Lq + 64 / hb - 1) / (64 / hb)) * ((G + hb - 1) / hb);
  if (tiles > 65535 || B * H_kv > 65535)
    return set_error(B200K_ESHAPE, "%s: %lld (token, head) tiles and %lld (sequence, K/V head) pairs, the grid allows 65535 "
                     "each", fn, (long long)tiles, (long long)(B * H_kv));
  return B200K_OK;
}

// Page counts of a cache read through a block table, or of a contiguous one: cache rows and a sequence's capacity
// are int32.
static int check_page_counts(const KvCall& c) {
  if (c.num_pages < 1 || c.page_size < 1 || c.pages_per_seq < 1)
    return set_error(B200K_ESHAPE, "%s: need num_pages, page_size, pages_per_seq >= 1 (got %lld %lld %lld)", c.fn,
                     (long long)c.num_pages, (long long)c.page_size, (long long)c.pages_per_seq);
  if (c.num_pages > INT32_MAX / c.page_size || c.pages_per_seq > INT32_MAX / c.page_size)
    return set_error(B200K_ESHAPE, "%s: num_pages * page_size and pages_per_seq * page_size must be <= 2^31 - 1", c.fn);
  return B200K_OK;
}

// The pages a block table can name: a KV tile of 128 keys is one TMA box inside one page, or a whole number of pages.
static int check_page_size(const KvCall& c) {
  if (c.page_size != 16 && c.page_size != 32 && c.page_size != 64 && c.page_size % 128 != 0)
    return set_error(B200K_ESHAPE, "%s: page_size %lld (16, 32, 64 or a multiple of 128)", c.fn, (long long)c.page_size);
  return B200K_OK;
}

// The checks fp8 caches add: the cache format, and the scales' alignment.
static int fp8_args(const KvCall& c) {
  if (c.kv_dtype != B200K_FP8_E4M3 && c.kv_dtype != B200K_FP8_E5M2)
    return set_error(B200K_EDTYPE, "%s: kv_dtype %d not supported (fp8 e4m3, fp8 e5m2)", c.fn, c.kv_dtype);
  return check_align(c.fn, {{c.k_scale, "k_scale", 4}, {c.v_scale, "v_scale", 4}});
}

// Large head dims: O in column slices of DV = 192 or 256 (as few slices as possible, each a whole number of 64-column
// chunks).  DV = 192 runs two consumer warpgroups: it serves at most 9 Q chunks (D <= 576), whose 128 Q rows fit in
// shared memory next to the K and V rings on every sm_90 part (230 504 of 232 448 bytes at 9 chunks).  DV = 256 needs
// more registers than a 384-thread block can give each thread (168), so it runs one.
template <int DV>
static int launch_ffpa(const void* Q, const void* K, const void* V, void* O, int64_t B, int64_t H, int64_t N, int64_t D,
                       float scale, cudaStream_t s, const DeviceInfo& di) {
  return launch_dense<AttnCfg<0, DV, DV == 192 ? 2 : 1, 64, false>>(Q, K, V, O, B, H, N, D, scale, nullptr, 0, nullptr, s,
                                                                     di);
}

// The one check an lse output adds to an attention call (null: no lse).
static int check_lse(const char* fn, const float* lse) { return check_align(fn, {{lse, "lse", 4}}); }

// The checks of a decode, append or fp8 call, before any CUDA call.  The fp8 entry point checks its cache format and
// lse before the append part; the 16-bit ones check lse last.
static int kvcache_args(const KvCall& c) {
  const char* fn = c.fn;
  if (!c.Q || !c.K_cache || !c.V_cache || !c.O || !c.seqlens) return set_error(B200K_EARG, "%s: null pointer", fn);
  if (c.dtype != B200K_F16 && c.dtype != B200K_BF16)
    return set_error(B200K_EDTYPE, "%s: dtype %d not supported (f16, bf16)", fn, c.dtype);
  int rc = check_headdim(fn, c.D);
  if (rc || (rc = check_page_counts(c)) || (rc = kvcache_check(c))) return rc;
  if (c.table && (rc = check_page_size(c))) return rc;
  if (!c.table && (c.num_pages != c.B || c.pages_per_seq != 1))
    return set_error(B200K_ESHAPE, "%s: a contiguous cache (no block table) is num_pages = B pages of page_size = S keys, "
                     "pages_per_seq = 1 (got num_pages=%lld pages_per_seq=%lld)", fn, (long long)c.num_pages,
                     (long long)c.pages_per_seq);
  if ((rc = check_align(fn, {{c.Q, "Q", 16}, {c.K_cache, "K_cache", 16}, {c.V_cache, "V_cache", 16}, {c.O, "O", 4},
                             {c.seqlens, "cache_seqlens", 4}, {c.table, "block_table", 4}})))
    return rc;
  if (c.fp8 && ((rc = fp8_args(c)) || (rc = check_lse(c.lse_fn, c.lse)))) return rc;
  if (c.append) {
    if (!c.K_new || !c.V_new) return set_error(B200K_EARG, "%s: null K_new / V_new", fn);
    if (!c.cos != !c.sin) return set_error(B200K_EARG, "%s: rotary needs both rotary_cos and rotary_sin", fn);
    if (c.L_new < 1 || c.L_new > INT32_MAX || c.B > INT32_MAX / c.L_new)
      return set_error(B200K_ESHAPE, "%s: need L_new >= 1 and B * L_new <= 2^31 - 1 (got L_new=%lld)", fn,
                       (long long)c.L_new);
    if (c.cos && (c.rotary_dim < 16 || c.rotary_dim > c.D || c.rotary_dim % 16 != 0))
      return set_error(B200K_ESHAPE, "%s: rotary_dim %lld (a multiple of 16 in [16, D = %lld])", fn,
                       (long long)c.rotary_dim, (long long)c.D);
    if (c.cos && c.rotary_seqlen < c.capacity())
      return set_error(B200K_ESHAPE, "%s: rotary_seqlen %lld is below the cache capacity %lld", fn,
                       (long long)c.rotary_seqlen, (long long)c.capacity());
    rc = check_align(fn, {{c.K_new, "K_new", 16}, {c.V_new, "V_new", 16}, {c.cos, "rotary_cos", 16},
                          {c.sin, "rotary_sin", 16}, {c.workspace, "workspace", 16}});
  } else if (c.cos || c.sin) {
    return set_error(B200K_EARG, "%s: rotary_cos / rotary_sin rotate appended keys and need K_new / V_new", fn);
  } else {
    rc = check_align(fn, {{c.workspace, "workspace", 16}});
  }
  if (rc || c.fp8) return rc;
  return check_lse(c.lse_fn, c.lse);
}

// The append kernel of cache format KVF for the call's dtype and rotary options: one thread per 16-byte vector, at most
// 65535 blocks.
template <int KVF>
static int launch_append(const KvAppend& a, const KvCall& c, cudaStream_t s) {
  const long long items = (2 * a.kv_rows + a.q_rows) * (c.D / 8);
  const long long blocks = ((items > c.B ? items : c.B) + 255) / 256;
  const dim3 grid(unsigned(blocks < 65535 ? blocks : 65535));
  auto append = [&](auto kern) {
    kern<<<grid, 256, 0, s>>>(a);
    B200K_CHECK_CUDA(cudaGetLastError());
    return B200K_OK;
  };
  if (c.dtype == B200K_BF16)
    return !c.rotary ? append(kvcache_append_kernel<1, false, false, KVF>)
                     : c.interleaved ? append(kvcache_append_kernel<1, true, true, KVF>)
                                     : append(kvcache_append_kernel<1, true, false, KVF>);
  return !c.rotary ? append(kvcache_append_kernel<0, false, false, KVF>)
                   : c.interleaved ? append(kvcache_append_kernel<0, true, true, KVF>)
                                   : append(kvcache_append_kernel<0, true, false, KVF>);
}

// A decode, append or fp8 call: its checks, the workspace check, then the append kernel when the call has new rows, the
// decode kernel on the grid (Q read through a 3-D map), and the combine kernel when the call is split.  lse (null, or
// [B, Lq, H] fp32) is written by the decode kernel unsplit and by the combine kernel split.
static int kvcache_run(const KvCall& c) {
  int rc = kvcache_args(c);
  DeviceInfo di;
  if (rc || (rc = get_device_info(&di))) return rc;
  const KvcacheGrid g = kvcache_grid(c, di.sm_count);
  if (g.bytes > 0 && (!c.workspace || c.workspace_bytes < g.bytes))
    return set_error(B200K_EARG, "%s: %zu workspace bytes needed, %zu given", c.fn, g.bytes,
                     c.workspace ? c.workspace_bytes : size_t(0));
  cudaStream_t s = static_cast<cudaStream_t>(c.stream);
  uint8_t* ws = static_cast<uint8_t*>(c.workspace);
  return with_kv_format(c.kv_dtype, [&](auto kvf) {
    constexpr int KVF = decltype(kvf)::value;
    const void* Q = c.Q;
    const int* seqlens = c.seqlens;
    if (c.append) {
      // the append entry points take the caches writable
      const KvAppend a = {.q = static_cast<const uint16_t*>(c.Q), .k_new = static_cast<const uint16_t*>(c.K_new),
                          .v_new = static_cast<const uint16_t*>(c.V_new), .cos = static_cast<const uint16_t*>(c.cos),
                          .sin = static_cast<const uint16_t*>(c.sin),
                          .q_out = c.rotary ? reinterpret_cast<uint16_t*>(ws + g.q) : nullptr,
                          .k_cache = static_cast<uint16_t*>(const_cast<void*>(c.K_cache)),
                          .v_cache = static_cast<uint16_t*>(const_cast<void*>(c.V_cache)), .seqlens = c.seqlens,
                          .table = c.table, .lens_out = reinterpret_cast<int*>(ws), .kv_rows = c.B * c.L_new * c.H_kv,
                          .q_rows = c.rotary ? c.B * c.Lq * c.H : 0, .rotary_seqlen = c.rotary_seqlen,
                          .B = int(c.B), .L_new = int(c.L_new), .Lq = int(c.Lq), .H = int(c.H), .H_kv = int(c.H_kv),
                          .D = int(c.D), .page_size = int(c.page_size), .pages_per_seq = int(c.pages_per_seq),
                          .rotary_dim = c.rotary ? int(c.rotary_dim) : 0, .causal = c.causal ? 1 : 0,
                          .k_scale = c.k_scale, .v_scale = c.v_scale};
      if ((rc = launch_append<KVF>(a, c, s))) return rc;
      // kernel boundaries order the cache writes above before the decode kernel's TMA reads of the caches
      if (c.rotary) Q = a.q_out;
      seqlens = a.lens_out;
    }
    return run_attn_cfg<1, false>(c.dtype, c.D, [&](auto cfg) {
      using Cfg = decltype(cfg);
      const long long rows = c.B * c.Lq * c.H;
      float* part = g.splits > 1 ? reinterpret_cast<float*>(ws + g.part) : nullptr;
      // a tile is one box of BN cache rows, or BN / page_size boxes (one per page) when pages are smaller
      const AttnDecode<Cfg> d = {.seqlens = seqlens, .table = c.table, .part = part,
                                 .lse = part ? part + size_t(g.splits) * size_t(rows) * size_t(c.D) : nullptr,
                                 .rows = rows, .H = int(c.H), .causal = c.causal ? 1 : 0, .Lq = int(c.Lq),
                                 .group = int(c.H / c.H_kv), .hb = g.hb, .T = g.T, .nhb = g.nhb,
                                 .page_size = int(c.page_size), .pages_per_seq = int(c.pages_per_seq),
                                 .box_rows = c.table && c.page_size < Cfg::BN ? int(c.page_size) : Cfg::BN,
                                 .oob = int(c.num_pages * c.page_size)};
      const int elem = KVF ? 1 : 2;
      const AttnTensor qkv[3] = {{Q, c.B * c.Lq, c.H, c.D, g.T, g.hb},
                                 {c.K_cache, c.num_pages * c.page_size, c.H_kv, c.D, d.box_rows, 1, elem},
                                 {c.V_cache, c.num_pages * c.page_size, c.H_kv, c.D, d.box_rows, 1, elem}};
      const dim3 grid(unsigned(g.splits), unsigned(g.qtiles * g.nhb), unsigned(c.B * c.H_kv));
      const auto mode = kv_mode<KVF>(d, c);
      if (g.splits == 1) return launch_mode<Cfg>(qkv, grid, c.O, c.D, c.scale, mode, c.lse, s, di);
      if ((rc = launch_attn<Cfg>(qkv, grid, c.O, c.D, c.scale, mode, s, di))) return rc;
      const long long work = d.rows * (c.D / 2);
      const unsigned blocks = unsigned((work + 255) / 256);
      if (c.lse)
        attn_combine_kernel<Cfg::DT, float, true><<<blocks, 256, 0, s>>>(d.part, d.lse, c.O, d.rows, int(c.D), g.splits,
                                                                         c.lse);
      else
        attn_combine_kernel<Cfg::DT><<<blocks, 256, 0, s>>>(d.part, d.lse, c.O, d.rows, int(c.D), g.splits);
      B200K_CHECK_CUDA(cudaGetLastError());
      return B200K_OK;
    });
  });
}

// The workspace queries: the bytes a call of c's shapes needs on the current device.
static int kvcache_workspace_bytes(const KvCall& c, size_t* bytes) {
  if (!bytes) return set_error(B200K_EARG, "%s: null pointer", c.fn);
  int rc = check_headdim(c.fn, c.D);
  DeviceInfo di;
  if (rc || (rc = kvcache_check(c)) || (rc = get_device_info(&di))) return rc;
  *bytes = kvcache_grid(c, di.sm_count).bytes;
  return B200K_OK;
}

// Packed queries over paged caches (b200k_fa2_varlen_paged), and with kv_dtype and its scales, over fp8 pages.
static int varlen_paged(const KvCall& c) {
  const char* fn = c.fn;
  if (!c.Q || !c.K_cache || !c.V_cache || !c.O || !c.cu_seqlens_q || !c.seqlens || !c.table)
    return set_error(B200K_EARG, "%s: null pointer", fn);
  if (c.dtype != B200K_F16 && c.dtype != B200K_BF16)
    return set_error(B200K_EDTYPE, "%s: dtype %d not supported (f16, bf16)", fn, c.dtype);
  int rc = c.kv_dtype ? fp8_args(c) : B200K_OK;
  if (rc || (rc = check_headdim(fn, c.D))) return rc;
  if (c.B < 1 || c.H < 1 || c.H_kv < 1 || c.H % c.H_kv != 0)
    return set_error(B200K_ESHAPE, "%s: need B, H, H_kv >= 1 and H %% H_kv == 0 (got B=%lld H=%lld H_kv=%lld)", fn,
                     (long long)c.B, (long long)c.H, (long long)c.H_kv);
  if ((rc = check_page_counts(c)) || (rc = check_page_size(c))) return rc;
  if (c.total_q < 1 || c.total_q > INT32_MAX || c.Lq < 1 || c.Lq > c.total_q)
    return set_error(B200K_ESHAPE, "%s: need 1 <= total_q <= 2^31 - 1 and 1 <= max_seqlen_q <= total_q (got total_q=%lld "
                     "max_seqlen_q=%lld)", fn, (long long)c.total_q, (long long)c.Lq);
  if (c.B > 65535 || c.H > 65535 || c.B * c.H > 65535)
    return set_error(B200K_ESHAPE, "%s: B * H = %lld CTAs per query tile, the grid allows 65535", fn,
                     (long long)c.B * (long long)c.H);
  if ((rc = check_align(fn, {{c.Q, "Q", 16}, {c.K_cache, "K_cache", 16}, {c.V_cache, "V_cache", 16}, {c.O, "O", 4},
                             {c.lse, "lse", 4}, {c.cu_seqlens_q, "cu_seqlens_q", 4}, {c.seqlens, "cu_seqlens_k", 4},
                             {c.table, "block_table", 4}})))
    return rc;
  DeviceInfo di;
  if ((rc = get_device_info(&di))) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(c.stream);
  return with_kv_format(c.kv_dtype, [&](auto kvf) {
    constexpr int KVF = decltype(kvf)::value;
    return run_attn_cfg<2, false>(c.dtype, c.D, [&](auto cfg) {
      using Cfg = decltype(cfg);
      const int box_rows = c.page_size < Cfg::BN ? int(c.page_size) : Cfg::BN;
      const int64_t cache_rows = c.num_pages * c.page_size;
      const int elem = KVF ? 1 : 2;
      const AttnTensor qkv[3] = {{c.Q, c.total_q, c.H, c.D, Cfg::BM, 1},
                                 {c.K_cache, cache_rows, c.H_kv, c.D, box_rows, 1, elem},
                                 {c.V_cache, cache_rows, c.H_kv, c.D, box_rows, 1, elem}};
      const dim3 grid(unsigned((c.Lq + Cfg::BM - 1) / Cfg::BM), 1, unsigned(c.B * c.H));
      const AttnPackedPaged<Cfg> args = {
          {c.cu_seqlens_q, c.seqlens, int(c.H), int(c.H / c.H_kv), int(c.total_q), c.causal ? 1 : 0},
          c.table, int(c.page_size), int(c.pages_per_seq), box_rows, int(cache_rows)};
      return launch_mode<Cfg>(qkv, grid, c.O, c.D, c.scale, kv_mode<KVF>(args, c), c.lse, s, di);
    });
  });
}

}  // namespace b200k

extern "C" int b200k_fa2_fwd_f16(const void* Q, const void* K, const void* V, void* O, int64_t B, int64_t H, int64_t N,
                                 int64_t D, float scale, int v_is_dn, int variant, void* stream) {
  return b200k_fa2_fwd(Q, K, V, O, B, H, N, D, scale, v_is_dn, B200K_F16, 0, nullptr, variant, stream);
}

extern "C" int b200k_fa2_fwd(const void* Q, const void* K, const void* V, void* O, int64_t B, int64_t H, int64_t N,
                             int64_t D, float scale, int v_is_dn, int dtype, int causal, const int* seqlens_k, int variant,
                             void* stream) {
  return b200k_fa2_fwd_lse(Q, K, V, O, nullptr, B, H, N, D, scale, v_is_dn, dtype, causal, seqlens_k, variant, stream);
}

extern "C" int b200k_fa2_fwd_lse(const void* Q, const void* K, const void* V, void* O, float* lse, int64_t B, int64_t H,
                                 int64_t N, int64_t D, float scale, int v_is_dn, int dtype, int causal,
                                 const int* seqlens_k, int variant, void* stream) {
  using namespace b200k;
  (void)variant;  // one configuration per head dim on this architecture
  if (dtype != B200K_F16 && dtype != B200K_BF16)
    return set_error(B200K_EDTYPE, "b200k_fa2_fwd: dtype %d not supported (f16, bf16)", dtype);
  if (dtype == B200K_BF16 && v_is_dn)
    return set_error(B200K_EARG, "b200k_fa2_fwd: the [B,H,D,N] V layout is built for fp16 only");
  if (!Q || !K || !V || !O) return set_error(B200K_EARG, "b200k_fa2_fwd: null pointer");
  if (B < 1 || H < 1 || N < 1 || N > INT32_MAX || B * H > 65535)
    return set_error(B200K_ESHAPE, "b200k_fa2_fwd_f16: need B,H,N >= 1 and B*H <= 65535 (got B=%lld H=%lld N=%lld)",
                     (long long)B, (long long)H, (long long)N);
  int rc = check_headdim("b200k_fa2_fwd_f16", D);
  if (rc) return rc;
  if (v_is_dn && (N % 8))
    return set_error(B200K_ESHAPE, "b200k_fa2_fwd: V stored [B,H,D,N] needs N %% 8 == 0 (16-byte rows), got N=%lld",
                     (long long)N);
  if ((rc = check_align("b200k_fa2_fwd", {{Q, "Q", 16}, {K, "K", 16}, {V, "V", 16}, {O, "O", 4},
                                          {seqlens_k, "seqlens_k", 4}})) ||
      (rc = check_lse("b200k_fa2_fwd_lse", lse)))
    return rc;
  DeviceInfo di;
  if ((rc = get_device_info(&di))) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  auto run = [&](auto cfg) {
    return launch_dense<decltype(cfg)>(Q, K, V, O, B, H, N, D, scale, seqlens_k, causal, lse, s, di);
  };
  return v_is_dn ? run_attn_cfg<2, true>(dtype, D, run) : run_attn_cfg<2, false>(dtype, D, run);
}

extern "C" int b200k_fa2_fwd_varlen(const void* Q, const void* K, const void* V, void* O, const int* cu_seqlens_q,
                                    const int* cu_seqlens_k, int64_t B, int64_t max_seqlen_q, int64_t total_q,
                                    int64_t total_k, int64_t H, int64_t H_kv, int64_t D, float scale, int dtype,
                                    int causal, void* stream) {
  return b200k_fa2_fwd_varlen_lse(Q, K, V, O, nullptr, cu_seqlens_q, cu_seqlens_k, B, max_seqlen_q, total_q, total_k, H,
                                  H_kv, D, scale, dtype, causal, stream);
}

extern "C" int b200k_fa2_fwd_varlen_lse(const void* Q, const void* K, const void* V, void* O, float* lse,
                                        const int* cu_seqlens_q, const int* cu_seqlens_k, int64_t B, int64_t max_seqlen_q,
                                        int64_t total_q, int64_t total_k, int64_t H, int64_t H_kv, int64_t D, float scale,
                                        int dtype, int causal, void* stream) {
  using namespace b200k;
  if (!Q || !K || !V || !O || !cu_seqlens_q || !cu_seqlens_k)
    return set_error(B200K_EARG, "b200k_fa2_fwd_varlen: null pointer");
  if (dtype != B200K_F16 && dtype != B200K_BF16)
    return set_error(B200K_EDTYPE, "b200k_fa2_fwd_varlen: dtype %d not supported (f16, bf16)", dtype);
  int rc = check_headdim("b200k_fa2_fwd_varlen", D);
  if (rc) return rc;
  if (B < 1 || H < 1 || H_kv < 1 || H % H_kv != 0)
    return set_error(B200K_ESHAPE, "b200k_fa2_fwd_varlen: need B, H, H_kv >= 1 and H %% H_kv == 0 (got B=%lld H=%lld H_kv=%lld)",
                     (long long)B, (long long)H, (long long)H_kv);
  if (total_q < 1 || total_q > INT32_MAX || total_k < 1 || total_k > INT32_MAX || max_seqlen_q < 1 || max_seqlen_q > total_q)
    return set_error(B200K_ESHAPE,
                     "b200k_fa2_fwd_varlen: need 1 <= total_q, total_k <= 2^31 - 1 and 1 <= max_seqlen_q <= total_q "
                     "(got total_q=%lld total_k=%lld max_seqlen_q=%lld)",
                     (long long)total_q, (long long)total_k, (long long)max_seqlen_q);
  if (B > 65535 || H > 65535 || B * H > 65535)
    return set_error(B200K_ESHAPE, "b200k_fa2_fwd_varlen: B * H = %lld CTAs per query tile, the grid allows 65535",
                     (long long)B * (long long)H);
  if ((rc = check_align("b200k_fa2_fwd_varlen", {{Q, "Q", 16}, {K, "K", 16}, {V, "V", 16}, {O, "O", 4},
                                                 {cu_seqlens_q, "cu_seqlens_q", 4}, {cu_seqlens_k, "cu_seqlens_k", 4}})) ||
      (rc = check_lse("b200k_fa2_fwd_varlen_lse", lse)))
    return rc;
  DeviceInfo di;
  if ((rc = get_device_info(&di))) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  return run_attn_cfg<2, false>(dtype, D, [&](auto cfg) {
    using Cfg = decltype(cfg);
    const AttnTensor qkv[3] = {{Q, total_q, H, D, Cfg::BM, 1}, {K, total_k, H_kv, D, Cfg::BN, 1}, {V, total_k, H_kv, D, Cfg::BN, 1}};
    const dim3 grid(unsigned((max_seqlen_q + Cfg::BM - 1) / Cfg::BM), 1, unsigned(B * H));
    const AttnPacked<Cfg> args = {cu_seqlens_q, cu_seqlens_k, int(H), int(H / H_kv), int(total_q), causal ? 1 : 0};
    return launch_mode<Cfg>(qkv, grid, O, D, scale, args, lse, s, di);
  });
}

extern "C" int b200k_fa2_varlen_paged(const void* Q, const void* K_cache, const void* V_cache, void* O, float* lse,
                                      const int* cu_seqlens_q, const int* cu_seqlens_k, const int* block_table,
                                      int64_t B, int64_t max_seqlen_q, int64_t total_q, int64_t H, int64_t H_kv,
                                      int64_t D, int64_t num_pages, int64_t page_size, int64_t pages_per_seq,
                                      float scale, int dtype, int causal, void* stream) {
  return b200k::varlen_paged({.fn = "b200k_fa2_varlen_paged", .Q = Q, .K_cache = K_cache, .V_cache = V_cache, .O = O,
                              .lse = lse, .cu_seqlens_q = cu_seqlens_q, .seqlens = cu_seqlens_k, .table = block_table,
                              .B = B, .Lq = max_seqlen_q, .total_q = total_q, .H = H, .H_kv = H_kv, .D = D,
                              .num_pages = num_pages, .page_size = page_size, .pages_per_seq = pages_per_seq,
                              .scale = scale, .dtype = dtype, .causal = causal, .stream = stream});
}

extern "C" int b200k_fa2_varlen_paged_fp8(const void* Q, const void* K_cache, const void* V_cache, void* O, float* lse,
                                          const int* cu_seqlens_q, const int* cu_seqlens_k, const int* block_table,
                                          const float* k_scale, const float* v_scale, int kv_dtype, int64_t B,
                                          int64_t max_seqlen_q, int64_t total_q, int64_t H, int64_t H_kv, int64_t D,
                                          int64_t num_pages, int64_t page_size, int64_t pages_per_seq, float scale,
                                          int dtype, int causal, void* stream) {
  return b200k::varlen_paged({.fn = "b200k_fa2_varlen_paged_fp8", .Q = Q, .K_cache = K_cache, .V_cache = V_cache, .O = O,
                              .lse = lse, .cu_seqlens_q = cu_seqlens_q, .seqlens = cu_seqlens_k, .table = block_table,
                              .k_scale = k_scale, .v_scale = v_scale, .kv_dtype = kv_dtype, .B = B, .Lq = max_seqlen_q,
                              .total_q = total_q, .H = H, .H_kv = H_kv, .D = D, .num_pages = num_pages,
                              .page_size = page_size, .pages_per_seq = pages_per_seq, .scale = scale, .dtype = dtype,
                              .causal = causal, .stream = stream});
}

extern "C" int b200k_fa2_fwd_kvcache_workspace_bytes(int64_t B, int64_t Lq, int64_t H, int64_t H_kv, int64_t D,
                                                     int64_t max_seqlen_k, size_t* bytes) {
  return b200k::kvcache_workspace_bytes({.fn = "b200k_fa2_fwd_kvcache_workspace_bytes", .B = B, .Lq = Lq, .H = H,
                                         .H_kv = H_kv, .D = D, .page_size = max_seqlen_k, .pages_per_seq = 1},
                                        bytes);
}

extern "C" int b200k_fa2_fwd_kvcache(const void* Q, const void* K_cache, const void* V_cache, void* O,
                                     const int* cache_seqlens, const int* block_table, int64_t B, int64_t Lq, int64_t H,
                                     int64_t H_kv, int64_t D, int64_t num_pages, int64_t page_size, int64_t pages_per_seq,
                                     float scale, int dtype, int causal, void* workspace, size_t workspace_bytes,
                                     void* stream) {
  return b200k_fa2_fwd_kvcache_lse(Q, K_cache, V_cache, O, nullptr, cache_seqlens, block_table, B, Lq, H, H_kv, D,
                                   num_pages, page_size, pages_per_seq, scale, dtype, causal, workspace, workspace_bytes,
                                   stream);
}

extern "C" int b200k_fa2_fwd_kvcache_lse(const void* Q, const void* K_cache, const void* V_cache, void* O, float* lse,
                                         const int* cache_seqlens, const int* block_table, int64_t B, int64_t Lq,
                                         int64_t H, int64_t H_kv, int64_t D, int64_t num_pages, int64_t page_size,
                                         int64_t pages_per_seq, float scale, int dtype, int causal, void* workspace,
                                         size_t workspace_bytes, void* stream) {
  return b200k::kvcache_run({.fn = "b200k_fa2_fwd_kvcache", .lse_fn = "b200k_fa2_fwd_kvcache_lse", .Q = Q,
                             .K_cache = K_cache, .V_cache = V_cache, .O = O, .lse = lse, .seqlens = cache_seqlens,
                             .table = block_table, .B = B, .Lq = Lq, .H = H, .H_kv = H_kv, .D = D,
                             .num_pages = num_pages, .page_size = page_size, .pages_per_seq = pages_per_seq,
                             .scale = scale, .dtype = dtype, .causal = causal, .workspace = workspace,
                             .workspace_bytes = workspace_bytes, .stream = stream});
}

extern "C" int b200k_fa2_fwd_kvcache_append_workspace_bytes(int64_t B, int64_t Lq, int64_t H, int64_t H_kv, int64_t D,
                                                            int64_t max_seqlen_k, int rotary, size_t* bytes) {
  return b200k::kvcache_workspace_bytes({.fn = "b200k_fa2_fwd_kvcache_append_workspace_bytes", .append = true,
                                         .rotary = rotary != 0, .B = B, .Lq = Lq, .H = H, .H_kv = H_kv, .D = D,
                                         .page_size = max_seqlen_k, .pages_per_seq = 1},
                                        bytes);
}

extern "C" int b200k_fa2_fwd_kvcache_append(const void* Q, void* K_cache, void* V_cache, void* O, const int* cache_seqlens,
                                            const int* block_table, const void* K_new, const void* V_new, int64_t L_new,
                                            const void* rotary_cos, const void* rotary_sin, int64_t rotary_seqlen,
                                            int64_t rotary_dim, int rotary_interleaved, int64_t B, int64_t Lq, int64_t H,
                                            int64_t H_kv, int64_t D, int64_t num_pages, int64_t page_size,
                                            int64_t pages_per_seq, float scale, int dtype, int causal, void* workspace,
                                            size_t workspace_bytes, void* stream) {
  return b200k_fa2_fwd_kvcache_append_lse(Q, K_cache, V_cache, O, nullptr, cache_seqlens, block_table, K_new, V_new, L_new,
                                          rotary_cos, rotary_sin, rotary_seqlen, rotary_dim, rotary_interleaved, B, Lq, H,
                                          H_kv, D, num_pages, page_size, pages_per_seq, scale, dtype, causal, workspace,
                                          workspace_bytes, stream);
}

extern "C" int b200k_fa2_fwd_kvcache_append_lse(const void* Q, void* K_cache, void* V_cache, void* O, float* lse,
                                                const int* cache_seqlens, const int* block_table, const void* K_new,
                                                const void* V_new, int64_t L_new, const void* rotary_cos,
                                                const void* rotary_sin, int64_t rotary_seqlen, int64_t rotary_dim,
                                                int rotary_interleaved, int64_t B, int64_t Lq, int64_t H, int64_t H_kv,
                                                int64_t D, int64_t num_pages, int64_t page_size, int64_t pages_per_seq,
                                                float scale, int dtype, int causal, void* workspace,
                                                size_t workspace_bytes, void* stream) {
  return b200k::kvcache_run({.fn = "b200k_fa2_fwd_kvcache_append", .lse_fn = "b200k_fa2_fwd_kvcache_append_lse",
                             .append = true, .rotary = rotary_cos != nullptr, .Q = Q, .K_cache = K_cache,
                             .V_cache = V_cache, .O = O, .lse = lse, .seqlens = cache_seqlens, .table = block_table,
                             .K_new = K_new, .V_new = V_new, .L_new = L_new, .cos = rotary_cos, .sin = rotary_sin,
                             .rotary_seqlen = rotary_seqlen, .rotary_dim = rotary_dim, .interleaved = rotary_interleaved,
                             .B = B, .Lq = Lq, .H = H, .H_kv = H_kv, .D = D, .num_pages = num_pages,
                             .page_size = page_size, .pages_per_seq = pages_per_seq, .scale = scale, .dtype = dtype,
                             .causal = causal, .workspace = workspace, .workspace_bytes = workspace_bytes,
                             .stream = stream});
}

extern "C" int b200k_attn_merge(const void* O_parts, const float* lse_parts, void* O, float* lse, int64_t S, int64_t rows,
                                int64_t D, int dtype, void* stream) {
  using namespace b200k;
  if (!O_parts || !lse_parts || !O) return set_error(B200K_EARG, "b200k_attn_merge: null pointer");
  if (dtype != B200K_F16 && dtype != B200K_BF16)
    return set_error(B200K_EDTYPE, "b200k_attn_merge: dtype %d not supported (f16, bf16)", dtype);
  if (S < 1 || rows < 1 || D < 8 || D % 8 || S > INT32_MAX || D > INT32_MAX || rows > (int64_t(INT32_MAX) << 8) / (D / 8))
    return set_error(B200K_ESHAPE, "b200k_attn_merge: need S, rows >= 1, D %% 8 == 0 and rows * D / 8 < 2^39 (got S=%lld "
                     "rows=%lld D=%lld)", (long long)S, (long long)rows, (long long)D);
  const int rc = check_align("b200k_attn_merge", {{O_parts, "O_parts", 16}, {lse_parts, "lse_parts", 4}, {O, "O", 16},
                                                  {lse, "lse", 4}});
  if (rc) return rc;
  const long long work = rows * (D / 8);
  const unsigned blocks = unsigned((work + 255) / 256);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const uint16_t* parts = static_cast<const uint16_t*>(O_parts);
  auto merge = [&](auto kern) {
    kern<<<blocks, 256, 0, s>>>(parts, lse_parts, O, rows, int(D), int(S), lse);
    B200K_CHECK_CUDA(cudaGetLastError());
    return B200K_OK;
  };
  if (dtype == B200K_BF16)
    return lse ? merge(attn_combine_kernel<1, uint16_t, true>) : merge(attn_combine_kernel<1, uint16_t, false>);
  return lse ? merge(attn_combine_kernel<0, uint16_t, true>) : merge(attn_combine_kernel<0, uint16_t, false>);
}

extern "C" int b200k_ffpa_fwd_f16(const void* Q, const void* K, const void* V, void* O, int64_t B, int64_t H, int64_t N,
                                  int64_t D, float scale, int variant, void* stream) {
  using namespace b200k;
  if (D == 32 || D == 64 || D == 96 || D == 128) return b200k_fa2_fwd_f16(Q, K, V, O, B, H, N, D, scale, 0, variant, stream);
  if (!Q || !K || !V || !O) return set_error(B200K_EARG, "b200k_ffpa_fwd_f16: null pointer");
  // 160, 224, ... (D % 64 == 32) are the reference's ENABLE_FFPA_ALL_HEADDIM rungs (launch_templates.cuh:L483-552)
  if (D < 128 || D > 1024 || (D % 32) != 0)
    return set_error(B200K_EHEADDIM, "headdim not support! (b200k_ffpa_fwd_f16: D=%lld; supported 32 .. 1024 step 32)", (long long)D);
  if (B < 1 || H < 1 || N < 1 || N > INT32_MAX || B * H > 65535)
    return set_error(B200K_ESHAPE, "b200k_ffpa_fwd_f16: need B,H,N >= 1 and B*H <= 65535");
  int rc = check_align("b200k_ffpa_fwd_f16", {{Q, "Q", 16}, {K, "K", 16}, {V, "V", 16}, {O, "O", 4}});
  DeviceInfo di;
  if (rc || (rc = get_device_info(&di))) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int nqc = int((D + 63) / 64), slices = (nqc + 3) / 4, chunks = (nqc + slices - 1) / slices;
  return chunks == 3 ? launch_ffpa<192>(Q, K, V, O, B, H, N, D, scale, s, di)
                     : launch_ffpa<256>(Q, K, V, O, B, H, N, D, scale, s, di);
}

extern "C" int b200k_fa2_kvcache_fp8_workspace_bytes(int64_t B, int64_t Lq, int64_t H, int64_t H_kv, int64_t D,
                                                     int64_t max_seqlen_k, int append, int rotary, size_t* bytes) {
  return b200k::kvcache_workspace_bytes({.fn = "b200k_fa2_kvcache_fp8_workspace_bytes", .append = append != 0,
                                         .rotary = rotary != 0, .B = B, .Lq = Lq, .H = H, .H_kv = H_kv, .D = D,
                                         .page_size = max_seqlen_k, .pages_per_seq = 1},
                                        bytes);
}

extern "C" int b200k_fa2_kvcache_fp8(const void* Q, void* K_cache, void* V_cache, void* O, float* lse,
                                     const int* cache_seqlens, const int* block_table, const float* k_scale,
                                     const float* v_scale, int kv_dtype, const void* K_new, const void* V_new,
                                     int64_t L_new, const void* rotary_cos, const void* rotary_sin, int64_t rotary_seqlen,
                                     int64_t rotary_dim, int rotary_interleaved, int64_t B, int64_t Lq, int64_t H,
                                     int64_t H_kv, int64_t D, int64_t num_pages, int64_t page_size, int64_t pages_per_seq,
                                     float scale, int dtype, int causal, void* workspace, size_t workspace_bytes,
                                     void* stream) {
  return b200k::kvcache_run({.fn = "b200k_fa2_kvcache_fp8", .lse_fn = "b200k_fa2_kvcache_fp8", .fp8 = true,
                             .append = K_new || V_new, .rotary = rotary_cos != nullptr, .Q = Q, .K_cache = K_cache,
                             .V_cache = V_cache, .O = O, .lse = lse, .seqlens = cache_seqlens, .table = block_table,
                             .k_scale = k_scale, .v_scale = v_scale, .kv_dtype = kv_dtype, .K_new = K_new,
                             .V_new = V_new, .L_new = L_new, .cos = rotary_cos, .sin = rotary_sin,
                             .rotary_seqlen = rotary_seqlen, .rotary_dim = rotary_dim, .interleaved = rotary_interleaved,
                             .B = B, .Lq = Lq, .H = H, .H_kv = H_kv, .D = D, .num_pages = num_pages,
                             .page_size = page_size, .pages_per_seq = pages_per_seq, .scale = scale, .dtype = dtype,
                             .causal = causal, .workspace = workspace, .workspace_bytes = workspace_bytes,
                             .stream = stream});
}
