/* b200k.h — the C ABI of libb200k.so: H100-native (sm_90a) replacements for the hot paths of
 * DefTruth/CUDA-Learn-Notes.  Plain C: raw device pointers, sizes, a CUDA stream handle.  No torch types.
 *
 * Every entry point
 *   - takes DEVICE pointers owned by the caller (never allocates, keeps no state between calls),
 *   - enqueues its kernels on `stream` (a cudaStream_t passed as void*; NULL = legacy default stream, which is
 *     what the reference launches on) and returns without synchronising,
 *   - returns B200K_OK or a negative B200K_E* code; b200k_last_error() gives the message for the calling thread,
 *   - needs every pointer aligned to its element size (a precondition the caller keeps: torch tensors always do);
 *     where a call needs more, its comment says so.
 *
 * Each declaration cites the reference interface it replaces (paths relative to the reference repo root).
 * The Python side (cuda-learn-notes_b200/b200k/_loader.py) binds exactly these symbols with ctypes; the
 * reference-side stubs a maintainer would add are shown in INTEGRATION.md.
 */
#ifndef B200K_H_
#define B200K_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200K_OK 0
#define B200K_EDTYPE (-1)   /* unsupported dtype / pack enum                         */
#define B200K_ESHAPE (-2)   /* shape not supported (see each function)               */
#define B200K_EALIGN (-3)   /* pointer or row pitch below the alignment a call needs */
#define B200K_EHEADDIM (-4) /* head dim not supported ("headdim not support!")       */
#define B200K_ECUDA (-5)    /* a CUDA runtime / driver call failed                   */
#define B200K_EARCH (-6)    /* current device is not compute capability 9.0 (H100)   */
#define B200K_EARG (-7)     /* bad enum / null pointer                               */

#define B200K_ABI_VERSION 1

int b200k_abi_version(void);
const char* b200k_last_error(void);
/* Fills sm count and compute capability of the current device; B200K_EARCH if it is not sm_90. */
int b200k_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ------------------------------------------------------------------------------------------------ HGEMM
 * C[M,N] = A[M,K] * B, fp16 in / fp16 out, fp32 accumulation in registers (wgmma, 128 x 256 tiles, TMA-fed).
 *   b_is_nk = 0 ("NN"): B is [K,N] row-major           — replaces every NN entry point of
 *       kernels/hgemm/pybind/hgemm.cc:L58-107, flagship kernels/hgemm/mma/basic/hgemm_mma_stage.cu:L2380-2454
 *       (hgemm_mma_m16n8k16_mma2x4_warp4x4x2_stages_dsmem)
 *   b_is_nk = 1 ("TN"): B storage is B^T = [N,K] row-major — replaces
 *       kernels/hgemm/mma/basic/hgemm_mma_stage_tn.cu:L517 (…_dsmem_tn),
 *       kernels/hgemm/mma/swizzle/hgemm_mma_stage_tn_swizzle_x4.cu:L860, kernels/hgemm/cutlass/hgemm_mma_stage_tn_cute.cu:L522,
 *       kernels/hgemm/cublas/hgemm_cublas.cu:L63-84 (hgemm_cublas_tensor_op_tn)
 * All matrices contiguous row-major; M,N,K >= 1; K % 8 == 0 and N % 8 == 0 (16-byte row pitch for TMA).
 * A, B and C must be 16-byte aligned (C is written by TMA stores); an unaligned C returns B200K_EALIGN before any
 * CUDA call.  Ragged M/N/K (not multiples of the tile) are handled by TMA zero-fill / store clipping.
 * variant (low 8 bits): 0 .. 4, the B200K_HGEMM_* names below.  They are kept for source compatibility: every value
 *   runs the same 128 x 256 tile kernel, so all of them give the same bits.  Higher bits are ignored.
 */
#define B200K_HGEMM_AUTO 0
#define B200K_HGEMM_1CTA_128x256 1
#define B200K_HGEMM_2CTA_256x256 2
#define B200K_HGEMM_2CTA_256x128 3
#define B200K_HGEMM_2CTA_512x256 4
int b200k_hgemm_f16(const void* A, const void* B, void* C, int64_t M, int64_t N, int64_t K, int b_is_nk,
                    int variant, void* stream);

/* Same kernel for other operand types (SURVEY.md section 8f-4): dtype B200K_F16 (identical to b200k_hgemm_f16),
 * B200K_BF16 (bf16 in / bf16 out, fp32 accumulation), or B200K_F32 = TF32 tensor-core product of fp32 matrices with
 * fp32 output (wgmma .tf32: the operands' low 13 mantissa bits are ignored by the tensor core, fp32 accumulation) - the
 * H100 counterpart of kernels/sgemm/sgemm_wmma_tf32_stage.cu:L25-420 (sgemm_wmma_m16n16k8_*).
 * K and N must be multiples of 8 (16-bit types) or 4 (fp32).  TF32 wgmma reads K-major operands only, so an fp32 [K,N] B
 * is first transposed into a scratch buffer allocated on `stream` (cudaMallocAsync) and freed after the product.  That form
 * reads B only through the transpose, so its B needs only the 4-byte alignment of a float (A and C must still be 16-byte
 * aligned); the allocation and free are stream-ordered, so the call can be captured in a CUDA graph. */
int b200k_gemm(const void* A, const void* B, void* C, int64_t M, int64_t N, int64_t K, int b_is_nk, int dtype, int variant,
               void* stream);
/* All four storage cases (SURVEY.md 8(f)-4 "TN/NT"): a_is_km != 0 means A is stored transposed, [K,M] row-major (the BLAS
 * "NT" / "TT" cases; f16 and bf16; M % 8 == 0); b_is_nk as above.  Operands are consumed in place (MN-major wgmma
 * descriptors), no transpose pass.  b200k_gemm(...) == b200k_gemm_ex(..., a_is_km = 0, ...). */
int b200k_gemm_ex(const void* A, const void* B, void* C, int64_t M, int64_t N, int64_t K, int a_is_km, int b_is_nk, int dtype,
                  int variant, void* stream);

/* ------------------------------------------------------------------------------------------------ attention
 * O = softmax(Q K^T * scale) V, non-causal, Q/K/V/O [B,H,N,D] fp16 contiguous (V optionally [B,H,D,N]).
 *
 * b200k_fa2_fwd_f16 — FlashAttention-2 forward, D in {32, 64, 96, 128}; N % 128 == 0 is NOT required (ragged N
 *   is masked), N >= 1.  Replaces the 25(+3) entry points flash_attn_mma_stages_* of
 *   kernels/flash-attn/pybind/flash_attn.cc:L182-216, flagship
 *   kernels/flash-attn/mma/basic/flash_attn_mma_share_qkv.cu:L833-886 (…_split_q_shared_qkv).
 *   v_is_dn = 1: V is passed transposed as [B,H,D,N] (the *_swizzle_qkv entry points, flash_attn_mma.py:L378).
 *
 * b200k_ffpa_fwd_f16 — large-headdim forward (FFPA L1), D in {160 .. 1024 step 32} (and the small D above); the
 *   D % 64 == 32 rungs are the reference's ENABLE_FFPA_ALL_HEADDIM set (launch_templates.cuh:L483-552).
 *   Replaces ffpa_mma_acc_f16_L1 / ffpa_mma_acc_f32_L1, ffpa-attn-mma/csrc/pybind/ffpa_attn_api.cc:L8-17,
 *   launcher ffpa-attn-mma/csrc/cuffpa/launch_templates.cuh:L261-449.
 * scale <= 0 means 1/sqrt(D) (what both references hard-code).
 * variant: accepted for source compatibility and ignored; there is one configuration per head dim.  Both entry points run
 *   the same wgmma kernel (csrc/attn_fwd_wgmma.cu); head dims above 256 compute O in column slices of 192 or 256, each
 *   slice recomputing S = Q K^T.
 * Alignment (every attention call below states its own): Q, K, V 16 bytes, O 4 bytes.  A pointer below its rule is
 *   B200K_EALIGN, with the argument named in the message, before any CUDA call.
 */
int b200k_fa2_fwd_f16(const void* Q, const void* K, const void* V, void* O, int64_t B, int64_t H, int64_t N,
                      int64_t D, float scale, int v_is_dn, int variant, void* stream);
int b200k_ffpa_fwd_f16(const void* Q, const void* K, const void* V, void* O, int64_t B, int64_t H, int64_t N,
                       int64_t D, float scale, int variant, void* stream);
/* b200k_fa2_fwd — the same FA-2 kernel with the caller-facing options the reference lacks (SURVEY.md 8(f)-4):
 *   dtype      B200K_F16 or B200K_BF16 (Q, K, V, O and the P operand; statistics and accumulators stay fp32)
 *   causal     != 0: query row r attends keys <= r; KV tiles above the diagonal are skipped, not masked
 *   seqlens_k  NULL, or int32 device array [B]: keys >= seqlens_k[b] are masked for batch b (key-padding mask of the
 *              padded [B,H,N,D] layout; 1 <= seqlens_k[b] <= N; every query row is still computed)
 *   alignment  Q, K, V 16 bytes; O, seqlens_k 4 bytes
 * b200k_fa2_fwd_f16(...) == b200k_fa2_fwd(..., B200K_F16, 0, NULL, ...). */
int b200k_fa2_fwd(const void* Q, const void* K, const void* V, void* O, int64_t B, int64_t H, int64_t N, int64_t D,
                  float scale, int v_is_dn, int dtype, int causal, const int* seqlens_k, int variant, void* stream);
/* b200k_fa2_fwd_varlen — the same FA-2 kernel on packed variable-length sequences with grouped-query K/V heads (the
 * counterpart of flash-attn's flash_attn_varlen_func forward):
 *   layouts    Q, O [total_q, H, D]; K, V [total_k, H_kv, D]; contiguous, one dtype (B200K_F16 or B200K_BF16);
 *              D in {32, 64, 96, 128}; scale <= 0 means 1/sqrt(D)
 *   sequences  cu_seqlens_q, cu_seqlens_k: int32 device arrays [B + 1], non-decreasing, starting at 0.  Sequence b is
 *              query tokens [cu_seqlens_q[b], cu_seqlens_q[b+1]) and key tokens [cu_seqlens_k[b], cu_seqlens_k[b+1]);
 *              their lengths Lq and Lk may differ, and either may be 0
 *   heads      H % H_kv == 0; query head h reads K/V head h / (H / H_kv) (GQA; H_kv == 1 is MQA, H_kv == H is MHA), the
 *              grouping of torch.repeat_interleave and scaled_dot_product_attention(enable_gqa=True)
 *   causal     != 0: aligned bottom-right, query row r of a sequence sees key j iff j <= r + Lk - Lq (flash-attn >= 2.1);
 *              with Lq == Lk this is the causal mask of b200k_fa2_fwd
 *   zero rows  a row that sees no key (Lk == 0, or causal with r + Lk - Lq < 0) is written as 0
 *   no sync    max_seqlen_q (>= every Lq; a longer sequence is a caller error) sizes the grid, so the call never reads
 *              the lengths back to the host and can be captured in a CUDA graph.  Stores are clipped to tokens
 *              [0, total_q) whatever cu_seqlens holds; reads past total_k are zero-filled
 *   neighbours the last KV tile of a sequence also reads keys of the next one; they are masked to -inf, so with finite
 *              K/V each sequence's O has the same bits as when computed alone.  A non-finite V in a neighbouring
 *              sequence leaks through as 0 * Inf = NaN (the same contract as the padded keys of b200k_fa2_fwd)
 *   alignment  Q, K, V 16 bytes; O, cu_seqlens_q, cu_seqlens_k 4 bytes
 * Errors: B200K_EARG for a null pointer, B200K_EDTYPE, B200K_EHEADDIM, and B200K_ESHAPE unless B >= 1, H, H_kv >= 1,
 * H % H_kv == 0, 1 <= max_seqlen_q <= total_q, 1 <= total_q, total_k <= INT32_MAX and B * H <= 65535; then
 * B200K_EALIGN. */
int b200k_fa2_fwd_varlen(const void* Q, const void* K, const void* V, void* O, const int* cu_seqlens_q,
                         const int* cu_seqlens_k, int64_t B, int64_t max_seqlen_q, int64_t total_q, int64_t total_k,
                         int64_t H, int64_t H_kv, int64_t D, float scale, int dtype, int causal, void* stream);
/* b200k_fa2_fwd_kvcache — attention of the newest Lq query tokens of each sequence against its KV cache (decode,
 * speculative decoding): the forward of flash-attn's flash_attn_with_kvcache (b200k_fa2_fwd_kvcache_append below adds
 * its append / rotary step).  The
 * same FA-2 kernel in a decode mode: one CTA per (sequence, K/V head) reads each K/V byte once for all the query heads
 * of its group, and a long cache is split across CTAs (the split count is chosen by the library from the shapes and the
 * SM count) and merged by a second kernel in a fixed order, so the result is deterministic.
 *   Q, O           [B, Lq, H, D] contiguous; dtype B200K_F16 or B200K_BF16; D in {32, 64, 96, 128}; scale <= 0 -> 1/sqrt(D)
 *   K_cache, V_cache [num_pages, page_size, H_kv, D] contiguous, same dtype; H % H_kv == 0, query head h reads K/V head
 *                  h / (H / H_kv)
 *   block_table    NULL: contiguous cache [B, S, H_kv, D], passed as num_pages = B, page_size = S, pages_per_seq = 1
 *                  (sequence b owns page b).  Otherwise int32 device array [B, pages_per_seq]: key j of sequence b is
 *                  slot j % page_size of page block_table[b * pages_per_seq + j / page_size]; page_size is 16, 32, 64
 *                  or a multiple of 128.  Entries past ceil(Lk_b / page_size) are never read
 *   cache_seqlens  int32 device array [B]: sequence b has Lk_b keys, 0 <= Lk_b <= pages_per_seq * page_size
 *   causal         query token t of sequence b sees key j iff j <= t + Lk_b - Lq (the new tokens are the last Lq keys)
 *   zero rows      a row that sees no key is written as 0
 *   isolation      cache slots at or past Lk_b, and pages a sequence's table does not list, never affect O, whatever
 *                  they hold (NaN and Inf included): caches are allocated uninitialised and pages are recycled
 *   workspace      >= the bytes b200k_fa2_fwd_kvcache_workspace_bytes reports for the same shapes (may be NULL when
 *                  that is 0)
 *   no sync        nothing is read back to the host, so the call can be captured in a CUDA graph and replayed while
 *                  cache_seqlens and block_table change
 *   alignment      Q, K_cache, V_cache, workspace 16 bytes; O, cache_seqlens, block_table 4 bytes
 * Errors before any CUDA call: B200K_EARG (null pointer), B200K_EDTYPE, B200K_EHEADDIM, B200K_ESHAPE (counts < 1,
 * H % H_kv, page_size, num_pages * page_size or B * Lq > INT32_MAX, grid limits: at most 65535 (token, head) tiles of
 * 64 rows per K/V head and B * H_kv <= 65535; without a table num_pages must be B and pages_per_seq 1), B200K_EALIGN.
 * After the device query (the split count needs the SM count): B200K_EARG when workspace_bytes is below what the
 * workspace function reports. */
int b200k_fa2_fwd_kvcache(const void* Q, const void* K_cache, const void* V_cache, void* O, const int* cache_seqlens,
                          const int* block_table, int64_t B, int64_t Lq, int64_t H, int64_t H_kv, int64_t D,
                          int64_t num_pages, int64_t page_size, int64_t pages_per_seq, float scale, int dtype, int causal,
                          void* workspace, size_t workspace_bytes, void* stream);
/* Workspace the call above needs for these shapes (max_seqlen_k = pages_per_seq * page_size); 0 when it runs
 * unsplit.  Depends on the current device's SM count, so it can fail like any device query. */
int b200k_fa2_fwd_kvcache_workspace_bytes(int64_t B, int64_t Lq, int64_t H, int64_t H_kv, int64_t D,
                                          int64_t max_seqlen_k, size_t* bytes);
/* b200k_fa2_fwd_kvcache_append — b200k_fa2_fwd_kvcache with flash_attn_with_kvcache's append and rotary steps in the
 * same call: the new tokens' K / V rows are written into the cache, optionally with rotary embedding on K and Q, and the
 * attention then runs over each sequence's old keys plus the new ones.  One bandwidth kernel runs before the decode
 * kernel on `stream`; arguments shared with b200k_fa2_fwd_kvcache mean what they mean there, with every rule it checks.
 *   K_new, V_new   [B, L_new, H_kv, D] contiguous, Q's dtype, L_new >= 1 (it may differ from Lq).  With base_b =
 *                  max(cache_seqlens[b], 0), new token i of sequence b is written at cache position p = base_b + i (slot
 *                  p % page_size of page block_table[b * pages_per_seq + p / page_size], or row p of sequence b without
 *                  a table).  The caches are updated in place; cache_seqlens is NOT: the caller adds L_new afterwards
 *   attention      over Lk_b = base_b + L_new keys, with the causal rule of b200k_fa2_fwd_kvcache
 *   rotary         rotary_cos, rotary_sin: both NULL, or both [rotary_seqlen, rotary_dim / 2] in Q's dtype with
 *                  rotary_dim % 16 == 0, 16 <= rotary_dim <= D and rotary_seqlen >= pages_per_seq * page_size.  Pair j
 *                  at position p becomes (x0 c - x1 s, x0 s + x1 c), c = cos[p, j], s = sin[p, j], in fp32 rounded once.
 *                  rotary_interleaved != 0 pairs columns (2j, 2j + 1), otherwise (j, j + rotary_dim / 2) (GPT-NeoX).
 *                  New key i is rotated at base_b + i; query token t at base_b + t when causal, at base_b when not.  Only
 *                  the first rotary_dim columns of K and Q are rotated; the rest, and all of V, are copied bit for bit.
 *                  Q is not modified: the rotated Q goes to the workspace
 *   overflow       base_b + L_new > capacity is a caller error; nothing is then written at or past the capacity or
 *                  outside the sequence's listed pages, and O is the attention over the first capacity keys
 *   workspace      >= the bytes b200k_fa2_fwd_kvcache_append_workspace_bytes reports (never 0): int32 lengths [B], the
 *                  rotated Q [B, Lq, H, D] (rotary only), then the split region, each on a 256-byte boundary
 *   no sync        nothing is read back to the host; the call and the caller's cache_seqlens += L_new can be captured
 *                  together in a CUDA graph
 *   alignment      Q, K_cache, V_cache, K_new, V_new, rotary_cos, rotary_sin, workspace 16 bytes; O, cache_seqlens,
 *                  block_table 4 bytes
 * Errors before any CUDA call: those of b200k_fa2_fwd_kvcache; B200K_EARG when K_new or V_new is NULL or only one of
 * rotary_cos / rotary_sin is given; B200K_ESHAPE for L_new < 1, B * L_new > INT32_MAX, a bad rotary_dim or rotary_seqlen
 * below the capacity; B200K_EALIGN.  After the device query, still before the caches are written: B200K_EARG for a
 * missing or short workspace. */
int b200k_fa2_fwd_kvcache_append(const void* Q, void* K_cache, void* V_cache, void* O, const int* cache_seqlens,
                                 const int* block_table, const void* K_new, const void* V_new, int64_t L_new,
                                 const void* rotary_cos, const void* rotary_sin, int64_t rotary_seqlen,
                                 int64_t rotary_dim, int rotary_interleaved,
                                 int64_t B, int64_t Lq, int64_t H, int64_t H_kv, int64_t D,
                                 int64_t num_pages, int64_t page_size, int64_t pages_per_seq,
                                 float scale, int dtype, int causal, void* workspace, size_t workspace_bytes,
                                 void* stream);
/* Workspace the call above needs for these shapes (max_seqlen_k = pages_per_seq * page_size; rotary != 0 when
 * rotary_cos / rotary_sin are given).  Depends on the current device's SM count. */
int b200k_fa2_fwd_kvcache_append_workspace_bytes(int64_t B, int64_t Lq, int64_t H, int64_t H_kv, int64_t D,
                                                 int64_t max_seqlen_k, int rotary, size_t* bytes);

/* ------------------------------------------------------------------------------------------------ attention log-sum-exp
 * The four *_lse calls below are the calls above with `float* lse` inserted right after O; everything else, checks,
 * messages and return codes included, is the same, and lse == NULL is exactly the call without it (each call above is
 * its *_lse form with lse = NULL).  They also write the softmax log-sum-exp of each query row (flash-attn's
 * return_softmax_lse), so that attention results over disjoint key sets can be merged by b200k_attn_merge:
 *   definition  lse[row] = ln sum_j exp(scale * q_row . k_j) over exactly the keys the row sees (length, key padding,
 *               causal diagonal, cache length), fp32 in natural-log units.  The kernel forms it as
 *               (m + log2f(l)) * 0.6931472f, m the row's final running max in base-2 units and l the same sum of rounded
 *               P that divides O, so O and lse describe one softmax
 *   empty rows  a row that sees no key gets -inf, the log of an empty sum (flash-attn writes +inf): -inf is what makes
 *               such a part weigh nothing in a merge
 *   layout      O's shape without its last dim, contiguous fp32, 4-byte aligned: dense [B, H, N] (as flash-attn), packed
 *               [total_q, H], decode [B, Lq, H] (flash-attn uses [H, total_q] and [B, H, Lq]).  Every mode then has
 *               rows = numel(O) / D with lse[row] belonging to O's row `row`, the indexing b200k_attn_merge takes
 *   stores      lse is written for exactly the rows whose O is written (packed tokens outside every sequence are left
 *               untouched, like O)
 *   split       a split decode call writes the merged value (mx + log2f(den)) * ln 2 (or -inf) from its combine kernel;
 *               the result stays deterministic.  The workspace functions are unchanged: lse needs no workspace
 * D in {32, 64, 96, 128}; b200k_ffpa_fwd_f16 and b200k_fa2_fwd_f16 have no lse form.  Errors: those of the call without
 * lse, then B200K_EALIGN for an lse that is not 4-byte aligned (before any CUDA call).
 *   alignment  the pointers of the call without lse as that call states; lse 4 bytes */
int b200k_fa2_fwd_lse(const void* Q, const void* K, const void* V, void* O, float* lse, int64_t B, int64_t H, int64_t N,
                      int64_t D, float scale, int v_is_dn, int dtype, int causal, const int* seqlens_k, int variant,
                      void* stream);
/* Packed sequences (b200k_fa2_fwd_varlen): lse [total_q, H]. */
int b200k_fa2_fwd_varlen_lse(const void* Q, const void* K, const void* V, void* O, float* lse, const int* cu_seqlens_q,
                             const int* cu_seqlens_k, int64_t B, int64_t max_seqlen_q, int64_t total_q, int64_t total_k,
                             int64_t H, int64_t H_kv, int64_t D, float scale, int dtype, int causal, void* stream);
/* KV-cache decode (b200k_fa2_fwd_kvcache): lse [B, Lq, H]. */
int b200k_fa2_fwd_kvcache_lse(const void* Q, const void* K_cache, const void* V_cache, void* O, float* lse,
                              const int* cache_seqlens, const int* block_table, int64_t B, int64_t Lq, int64_t H,
                              int64_t H_kv, int64_t D, int64_t num_pages, int64_t page_size, int64_t pages_per_seq,
                              float scale, int dtype, int causal, void* workspace, size_t workspace_bytes, void* stream);
/* KV-cache decode with append (b200k_fa2_fwd_kvcache_append): lse [B, Lq, H], over the old keys plus the new ones. */
int b200k_fa2_fwd_kvcache_append_lse(const void* Q, void* K_cache, void* V_cache, void* O, float* lse,
                                     const int* cache_seqlens, const int* block_table, const void* K_new,
                                     const void* V_new, int64_t L_new, const void* rotary_cos, const void* rotary_sin,
                                     int64_t rotary_seqlen, int64_t rotary_dim, int rotary_interleaved,
                                     int64_t B, int64_t Lq, int64_t H, int64_t H_kv, int64_t D,
                                     int64_t num_pages, int64_t page_size, int64_t pages_per_seq,
                                     float scale, int dtype, int causal, void* workspace, size_t workspace_bytes,
                                     void* stream);
/* b200k_fa2_varlen_paged — b200k_fa2_fwd_varlen with K / V read from paged caches through a block table (flash-attn's
 * flash_attn_varlen_func with block_table): prefill of a prompt chunk after a cached prefix, chunked prefill, or a batch
 * of prompts of different lengths, without gathering the cached keys into a contiguous buffer.  The same kernel as the
 * packed call, 128 query rows per CTA, with the block-table addressing of b200k_fa2_fwd_kvcache:
 *   Q, O, lse      as b200k_fa2_fwd_varlen_lse: Q, O [total_q, H, D], sequence b is query tokens
 *                  [cu_seqlens_q[b], cu_seqlens_q[b+1]); lse NULL or fp32 [total_q, H].  Stores are clipped to tokens
 *                  [0, total_q), and tokens outside every sequence are left untouched
 *   K_cache, V_cache [num_pages, page_size, H_kv, D] contiguous, Q's dtype; H % H_kv == 0
 *   block_table    int32 device array [B, pages_per_seq] (required): key j of sequence b is slot j % page_size of page
 *                  block_table[b * pages_per_seq + j / page_size]; page_size is 16, 32, 64 or a multiple of 128.
 *                  Entries past ceil(Lk_b / page_size) are never read
 *   cu_seqlens_k   int32 device array [B + 1]: sequence b has Lk_b = cu_seqlens_k[b+1] - cu_seqlens_k[b] keys, clamped to
 *                  [0, pages_per_seq * page_size].  Only the differences are used
 *   causal         bottom-right as b200k_fa2_fwd_varlen: query row r sees key j iff j <= r + Lk_b - Lq_b
 *   isolation      cache slots at or past Lk_b, and pages the sequence's table row does not list, never affect O or lse,
 *                  whatever they hold (NaN and Inf included)
 *   bits           O and lse have the bits b200k_fa2_fwd_varlen_lse gives on K / V gathered through the table
 *   no sync        max_seqlen_q sizes the grid; nothing is read back to the host, so the call can be captured in a CUDA
 *                  graph and replayed while cu_seqlens and block_table change.  A decode step (Lq = 1) still takes a CTA
 *                  of 128 rows per query head: b200k_fa2_fwd_kvcache is the decode call
 *   alignment      Q, K_cache, V_cache 16 bytes; O, lse, cu_seqlens_q, cu_seqlens_k, block_table 4 bytes
 * Errors before any CUDA call: B200K_EARG for a null pointer (lse may be NULL), B200K_EDTYPE, B200K_EHEADDIM,
 * B200K_ESHAPE unless B, H, H_kv >= 1, H % H_kv == 0, num_pages, page_size, pages_per_seq >= 1 with num_pages * page_size
 * and pages_per_seq * page_size <= INT32_MAX, page_size as above, 1 <= max_seqlen_q <= total_q <= INT32_MAX and
 * B * H <= 65535; then B200K_EALIGN. */
int b200k_fa2_varlen_paged(const void* Q, const void* K_cache, const void* V_cache, void* O, float* lse,
                           const int* cu_seqlens_q, const int* cu_seqlens_k, const int* block_table, int64_t B,
                           int64_t max_seqlen_q, int64_t total_q, int64_t H, int64_t H_kv, int64_t D,
                           int64_t num_pages, int64_t page_size, int64_t pages_per_seq, float scale, int dtype,
                           int causal, void* stream);
/* ------------------------------------------------------------------------------------------------ fp8 KV caches
 * Decode (with or without append) and paged prefill over caches that hold K and V in 8-bit floats: twice the tokens in
 * the same memory, and half the bytes a decode step reads (vLLM's kv_cache_dtype "fp8" / "fp8_e5m2" with k_scale /
 * v_scale, flash-attn 3's descale_k / descale_v).  Everything not stated here is the 16-bit call's:
 *   kv_dtype     B200K_FP8_E4M3 (torch float8_e4m3fn) or B200K_FP8_E5M2 (torch float8_e5m2).  K_cache, V_cache are
 *                [num_pages, page_size, H_kv, D] (or contiguous [B, S, H_kv, D]) of 1-byte elements; Q, O, K_new, V_new,
 *                rotary_cos / rotary_sin stay in dtype (B200K_F16 or B200K_BF16); D in {32, 64, 96, 128}.  Page sizes,
 *                block table, lengths, causal rule, split rule, isolation, lse and "no sync" are the 16-bit calls'
 *   scales       k_scale, v_scale: NULL (1.0) or fp32 device arrays [H_kv]; the key of K/V head h is fp8 * k_scale[h]
 *                (vLLM's convention).  Device arrays, so a captured graph stays valid when the scales change
 *   arithmetic   every fp8 value converts exactly to dtype.  k_scale folds into the softmax exponent: the kernel's
 *                scale_log2 = (scale * log2 e) is multiplied once more, by k_scale[h], in fp32.  v_scale folds into
 *                the epilogue: O = dtype(o * ((1 / l) * v_scale[h])), and split partials carry the same factor.  lse
 *                is the log-sum-exp of the scaled scores
 *   bits         with NULL scales, O and lse have the bits of the 16-bit call on caches holding dtype(K8), dtype(V8);
 *                with power-of-two scales, on caches holding dtype(K8) * k_scale[h] and dtype(V8) * v_scale[h]
 *                (while those products are normal dtype values), since every step above is then an exact rescaling
 *   append       the byte stored for new element x is cvt.rn.satfinite(float(x16) / scale[h]) in the cache's format:
 *                x16 the 16-bit value b200k_fa2_fwd_kvcache_append would store (rotary included), the division IEEE
 *                fp32; values past the largest finite value become +-448 (e4m3) or +-57344 (e5m2), NaN stays NaN
 *   alignment    the 16-bit call's, and k_scale, v_scale 4 bytes
 * Errors before any CUDA call: those of the 16-bit call, B200K_EDTYPE for a kv_dtype other than the two above, and
 * B200K_EALIGN naming k_scale or v_scale. */
/* b200k_fa2_kvcache_fp8 — b200k_fa2_fwd_kvcache_lse over fp8 caches, and with K_new, V_new (both non-NULL)
 * b200k_fa2_fwd_kvcache_append_lse: L_new, rotary_* and the workspace then mean what they mean there.  K_new == V_new
 * == NULL is decode alone (L_new and the rotary sizes are ignored; rotary_cos / rotary_sin must be NULL, else
 * B200K_EARG).  lse may be NULL.  workspace: at least what b200k_fa2_kvcache_fp8_workspace_bytes reports. */
int b200k_fa2_kvcache_fp8(const void* Q, void* K_cache, void* V_cache, void* O, float* lse, const int* cache_seqlens,
                          const int* block_table, const float* k_scale, const float* v_scale, int kv_dtype,
                          const void* K_new, const void* V_new, int64_t L_new, const void* rotary_cos,
                          const void* rotary_sin, int64_t rotary_seqlen, int64_t rotary_dim, int rotary_interleaved,
                          int64_t B, int64_t Lq, int64_t H, int64_t H_kv, int64_t D, int64_t num_pages,
                          int64_t page_size, int64_t pages_per_seq, float scale, int dtype, int causal,
                          void* workspace, size_t workspace_bytes, void* stream);
/* Workspace b200k_fa2_kvcache_fp8 needs: append == 0, decode's (b200k_fa2_fwd_kvcache_workspace_bytes); otherwise
 * append's layout (b200k_fa2_fwd_kvcache_append_workspace_bytes with rotary).  Depends on the device's SM count. */
int b200k_fa2_kvcache_fp8_workspace_bytes(int64_t B, int64_t Lq, int64_t H, int64_t H_kv, int64_t D,
                                          int64_t max_seqlen_k, int append, int rotary, size_t* bytes);
/* b200k_fa2_varlen_paged_fp8 — b200k_fa2_varlen_paged over fp8 pages, with k_scale, v_scale and kv_dtype as above.
 * O and lse have the bits b200k_fa2_fwd_varlen_lse gives on K / V gathered through the table and dequantized (with
 * NULL or power-of-two scales). */
int b200k_fa2_varlen_paged_fp8(const void* Q, const void* K_cache, const void* V_cache, void* O, float* lse,
                               const int* cu_seqlens_q, const int* cu_seqlens_k, const int* block_table,
                               const float* k_scale, const float* v_scale, int kv_dtype, int64_t B,
                               int64_t max_seqlen_q, int64_t total_q, int64_t H, int64_t H_kv, int64_t D,
                               int64_t num_pages, int64_t page_size, int64_t pages_per_seq, float scale, int dtype,
                               int causal, void* stream);
/* b200k_attn_merge — the attention over the union of S disjoint key sets from the attention over each (cascade /
 * shared-prefix decode, chunked prefill, keys sharded across devices):
 *   inputs      O_parts [S, rows, D] in dtype (B200K_F16 or B200K_BF16), lse_parts [S, rows] fp32 natural log, as the
 *               *_lse calls write them; a dense [B, H, N, D] output is rows = B * H * N
 *   outputs     O [rows, D] in dtype; lse [rows] fp32 natural log, or NULL.  O must not overlap O_parts
 *   arithmetic  t_s = lse_s * 1.4426950f, mx = max_s t_s, w_s = 2^(t_s - mx) (ex2.approx.ftz); x = sum_s w_s O_s and
 *               den = sum_s w_s in fp32, in ascending s; O = dtype(x * (1 / den)), lse = (mx + log2f(den)) * ln 2
 *   empty parts a part with lse_s = -inf is skipped, so whatever its O holds (NaN included) never reaches the result; a
 *               row where every part is -inf gets O = 0 and lse = -inf
 *   guarantees  deterministic; no host sync, so the call can be captured in a CUDA graph.  The split-decode combine of
 *               b200k_fa2_fwd_kvcache is the same kernel on fp32 base-2 partials
 * Errors before any CUDA call: B200K_EARG for a null O_parts, lse_parts or O; B200K_EDTYPE; B200K_ESHAPE unless S,
 * rows >= 1 and D % 8 == 0 (every row a whole number of 16-byte vectors); B200K_EALIGN.
 *   alignment   O_parts, O 16 bytes (16-byte loads and stores); lse_parts, lse 4 bytes */
int b200k_attn_merge(const void* O_parts, const float* lse_parts, void* O, float* lse, int64_t S, int64_t rows, int64_t D,
                     int dtype, void* stream);

/* ------------------------------------------------------------------------------------------------ attention backward
 * b200k_fa2_bwd — the gradients of b200k_fa2_fwd (flash-attn's backward), dense layout:
 *   inputs      Q, K, V, O, dO [B, H, N, D] contiguous in dtype (B200K_F16 or B200K_BF16); lse [B, H, N] fp32, natural
 *               log, as b200k_fa2_fwd_lse wrote it for this O.  D in {32, 64, 96, 128}; scale <= 0 means 1/sqrt(D)
 *   contract    scale, causal and seqlens_k are those of the forward call that produced O and lse (not checked).  As in
 *               the forward, seqlens_k[b] is clamped to [1, N]
 *   outputs     dQ, dK, dV [B, H, N, D] in dtype, every element written once; nothing else outside the workspace is
 *               written.  dK and dV rows of keys no query sees (at or past seqlens_k[b]) are 0
 *   arithmetic  fp32 throughout: P = 2^(s * scale * log2 e - lse * log2 e), s = q . k from the tensor core;
 *               Delta_i = sum_d dO_id O_id from the 16-bit O and dO; dP_ij = dO_i . v_j; dS = P (dP - Delta);
 *               dV_j = sum_i P~_ij dO_i, dQ_i = scale sum_j dS~_ij k_j, dK_j = scale sum_i dS~_ij q_i, where P~ and dS~ are
 *               P and dS rounded to dtype (the tensor core's A operand); each output rounded once
 *   guarantees  deterministic (no atomics, no fp32 accumulation buffer: each output element is summed in one thread's
 *               registers), so two calls, or a call replayed from a CUDA graph, give the same bits.  No host sync
 *   workspace   >= b200k_fa2_bwd_workspace_bytes(B, H, N): the per-row Delta, then lse * log2 e, fp32 [B, H, N] each on
 *               a 256-byte boundary
 *   cost        S and dP are computed by both the dK/dV and the dQ kernel: 7 matrix products where an atomic-dQ backward
 *               needs 5
 *   alignment   Q, K, V, O, dO, workspace 16 bytes; dQ, dK, dV, lse, seqlens_k 4 bytes (32-bit stores and loads)
 * Errors, all before any CUDA call: B200K_EARG for a null pointer (seqlens_k may be NULL), B200K_EDTYPE,
 * B200K_EHEADDIM, B200K_ESHAPE unless B, H, N >= 1, N <= INT32_MAX and B * H <= 65535, B200K_EALIGN naming the
 * argument, then B200K_EARG for a workspace below the size above. */
int b200k_fa2_bwd(const void* Q, const void* K, const void* V, const void* O, const float* lse, const void* dO,
                  void* dQ, void* dK, void* dV, int64_t B, int64_t H, int64_t N, int64_t D, float scale, int dtype,
                  int causal, const int* seqlens_k, void* workspace, size_t workspace_bytes, void* stream);
/* Workspace bytes b200k_fa2_bwd needs for these shapes (no device query); B200K_ESHAPE as b200k_fa2_bwd. */
int b200k_fa2_bwd_workspace_bytes(int64_t B, int64_t H, int64_t N, size_t* bytes);

/* b200k_fa2_bwd_varlen — the gradients of b200k_fa2_fwd_varlen (flash-attn's varlen backward): packed sequences with
 * grouped-query K/V heads, the same kernels and arithmetic as b200k_fa2_bwd:
 *   inputs      Q, O, dO [total_q, H, D] and K, V [total_k, H_kv, D] contiguous in one dtype (B200K_F16 or B200K_BF16);
 *               lse [total_q, H] fp32 as b200k_fa2_fwd_varlen_lse wrote it (-inf for a row that sees no key).  D in
 *               {32, 64, 96, 128}; scale <= 0 means 1/sqrt(D)
 *   sequences   as b200k_fa2_fwd_varlen: sequence b is tokens [cu_seqlens_q[b], cu_seqlens_q[b+1]) of Q and
 *               [cu_seqlens_k[b], cu_seqlens_k[b+1]) of K / V; query head h reads K/V head h / (H / H_kv); causal is
 *               bottom-right (row r sees key j iff j <= r + Lk - Lq).  max_seqlen_q / max_seqlen_k size the grids, so
 *               nothing is read back to the host; a longer sequence is a caller error
 *   contract    scale, causal and cu_seqlens_* are those of the forward call that produced O and lse (not checked)
 *   outputs     dQ [total_q, H, D], dK, dV [total_k, H_kv, D], every element written once; nothing else outside the
 *               workspace is written.  dK and dV of K/V head k sum over the H / H_kv query heads of its group.  Rows are
 *               +0 for: dQ of a row that sees no key (Lk = 0, or causal with r + Lk - Lq < 0); dK, dV of a key no query
 *               sees (Lq = 0, or above every causal diagonal); tokens outside every sequence (before cu_seqlens[0] or at
 *               or past cu_seqlens[B]), whose gradient is 0
 *   arithmetic  b200k_fa2_bwd's (P and dS rounded to dtype before their products; dV = dtype(sum), dQ, dK =
 *               dtype(fp32(sum * scale))); the group sum runs query head ascending, then query tile ascending, in one
 *               thread's registers
 *   guarantees  deterministic (no atomics, no fp32 accumulation buffer) and no host sync (CUDA-graph capturable).  With
 *               H_kv = H and Lq = Lk = N for every sequence, the bits of b200k_fa2_bwd on the same data in the dense
 *               layout.  With finite inputs, each sequence's gradients have the bits of that sequence passed alone (a
 *               non-finite value in a neighbouring sequence can reach a row as 0 * Inf, as in the forward)
 *   workspace   >= b200k_fa2_bwd_varlen_workspace_bytes(total_q, H): Delta, then lse * log2 e, fp32 [total_q, H] each on
 *               a 256-byte boundary
 *   alignment   Q, K, V, O, dO, workspace 16 bytes; dQ, dK, dV, lse, cu_seqlens_q, cu_seqlens_k 4 bytes
 * Errors, all before any CUDA call: B200K_EARG for a null pointer, B200K_EDTYPE, B200K_EHEADDIM, B200K_ESHAPE unless
 * B, H, H_kv >= 1, H % H_kv == 0, 1 <= max_seqlen_q <= total_q <= INT32_MAX, 1 <= max_seqlen_k <= total_k <= INT32_MAX
 * and B * H <= 65535 (so B * H_kv <= 65535 too), B200K_EALIGN naming the argument, then B200K_EARG for a workspace
 * below the size above. */
int b200k_fa2_bwd_varlen(const void* Q, const void* K, const void* V, const void* O, const float* lse, const void* dO,
                         void* dQ, void* dK, void* dV, const int* cu_seqlens_q, const int* cu_seqlens_k, int64_t B,
                         int64_t max_seqlen_q, int64_t max_seqlen_k, int64_t total_q, int64_t total_k, int64_t H,
                         int64_t H_kv, int64_t D, float scale, int dtype, int causal, void* workspace,
                         size_t workspace_bytes, void* stream);
/* Workspace bytes b200k_fa2_bwd_varlen needs (no device query); B200K_ESHAPE unless 1 <= total_q <= INT32_MAX and
 * 1 <= H <= 65535. */
int b200k_fa2_bwd_varlen_workspace_bytes(int64_t total_q, int64_t H, size_t* bytes);

/* ------------------------------------------------------------------------------------------------ support kernels
 * HBM-roofline kernels (128-bit vectorised, warp-shuffle reductions, no tensor cores).  dtype enums: */
#define B200K_F32 0
#define B200K_F16 1
#define B200K_BF16 2
#define B200K_I8 3
#define B200K_FP8_E4M3 4
#define B200K_FP8_E5M2 5
#define B200K_I32 6

/* c = a + b, n elements.  kernels/elementwise/elementwise.cu:L24-168 (elementwise_add_{f32,f32x4,f16,f16x2,f16x8,f16x8_pack}). */
int b200k_elementwise_add(const void* a, const void* b, void* c, int64_t n, int dtype, void* stream);

/* out[0] = sum(x[0..n)).  `out` is a 1-element device buffer (f32, or i32 when dtype == B200K_I8) that this call
 * overwrites.  acc_f16 = 1 reproduces the reference's half-precision per-thread partial sums.
 * kernels/reduce/block_all_reduce.cu:L42-686, bindings L734-790 (block_all_reduce_sum_*).
 * Deterministic (fixed two-pass order) where the reference uses atomicAdd. `workspace`: >= b200k_reduce_workspace_bytes(). */
size_t b200k_reduce_workspace_bytes(void);
int b200k_block_all_reduce_sum(const void* x, void* out, int64_t n, int dtype, int acc_f16, void* workspace,
                               void* stream);

/* Row softmax over the last dim of x[S,H] -> y[S,H].  kernels/softmax/softmax.cu:L102-391, bindings L778-884.
 * mode 0: softmax over the WHOLE tensor (softmax_f32 / softmax_f32x4: one global sum, grid fence),
 * mode 1: per-token (per-row) softmax without max subtraction, mode 2: per-token safe softmax,
 * mode 3: per-token online safe softmax (same result as 2).  dtype F32 or F16 (f16 I/O, f32 math).
 * `workspace` (mode 0 only): >= b200k_reduce_workspace_bytes(). */
int b200k_softmax(const void* x, void* y, int64_t S, int64_t H, int dtype, int mode, void* workspace, void* stream);

/* y = x * rsqrt(mean(x^2) + eps) * g for each row of x[N,K]; scalar g.  kernels/rms-norm/rms_norm.cu:L53-366, L457-800.
 * eps_inside_k = 1 reproduces the reference's f16-input kernels, which compute rsqrt(sum/(K + eps)) (L164 etc.).
 * acc_f16 = 1: squares summed in half like the *_f16 variants. */
int b200k_rms_norm(const void* x, void* y, int64_t N, int64_t K, float g, float eps, int dtype, int acc_f16,
                   int eps_inside_k, void* stream);

/* Interleaved-pair rotary embedding on x[seq_len, hidden] f32, theta = 10000.  kernels/rope/rope.cu:L20-113.
 * ref_quirk = 1 reproduces the reference kernels' integer-division exponent (every pair rotates with frequency 1.0,
 * see SURVEY.md §8 a9); ref_quirk = 0 is the textbook formula of the script's naive_rope (rope.py:L71-91). */
int b200k_rope_f32(const void* x, void* out, int64_t seq_len, int64_t hidden, int ref_quirk, void* stream);

/* hist[v] += 1 for v in a[0..n) (int32 values in [0, nbins)); `hist` (int32[nbins]) is zeroed by this call.
 * kernels/histogram/histogram.cu:L18-72.  b200k_max_i32 gives max(a) (the reference sizes its output as max+1
 * through a host sync, L57-60); `out_max` is a 1-element int32 device buffer. */
int b200k_max_i32(const void* a, int64_t n, void* out_max, void* stream);
int b200k_histogram_i32(const void* a, int64_t n, void* hist, int64_t nbins, void* stream);

/* out[i,:] = weight[idx[i],:], idx int32[n], weight [rows, emb] f32 or f16.  kernels/embedding/embedding.cu:L16-119. */
int b200k_embedding(const void* idx, const void* weight, void* out, int64_t n, int64_t rows, int64_t emb, int dtype,
                    void* stream);

/* ------------------------------------------------------------------------------------------------ support kernels, set 2
 * (SURVEY.md section 8f-3: the remaining bandwidth kernels of the reference, same recipe as above.)
 *
 * y = f(x) elementwise over n values, dtype B200K_F32 or B200K_F16 (f16 I/O, f32 math).
 *   kernels/relu/relu.cu:L21-97, sigmoid/sigmoid.cu:L24-136, gelu/gelu.cu:L38-163 (tanh approximation), swish/swish.cu:L20-97,
 *   elu/elu.cu:L35-120 (alpha = 1), hardswish/hardswish.cu:L36-140, hardshrink/hardshrink.cu:L33-135 (lambda = 0.5); each
 *   family's six entry points (f32, f32x4, f16, f16x2, f16x8, f16x8_pack) map here.
 * ref_clamp = 1 reproduces the input clamp of the reference's sigmoid / gelu kernels: x limited to +-88.3762626647949
 *   (f32 kernels) or to [-9.703125, 11.09375] (f16 kernels: MIN_EXP_F16 / MAX_EXP_F16 as rounded to half) BEFORE the
 *   function, so the f16 gelu saturates at 11.09375 for large x.  ref_clamp = 0 is the plain function. */
#define B200K_ACT_RELU 0
#define B200K_ACT_SIGMOID 1
#define B200K_ACT_GELU 2
#define B200K_ACT_SWISH 3
#define B200K_ACT_ELU 4
#define B200K_ACT_HARDSWISH 5
#define B200K_ACT_HARDSHRINK 6
int b200k_activation(const void* x, void* y, int64_t n, int dtype, int op, int ref_clamp, void* stream);

/* y = (x - mean(x)) * rsqrt(v) * g + b for each row of x[N,K]; scalar g, b; dtype F32 or F16 (f32 math).
 * kernels/layer-norm/layer_norm.cu:L48-419, bindings L732-812.  eps_inside_k = 1 reproduces the reference:
 * v = sum((x-mean)^2) / (K + eps) (L69, L103, L187 ...); eps_inside_k = 0 is the textbook v = sum(..)/K + eps. */
int b200k_layer_norm(const void* x, void* y, int64_t N, int64_t K, float g, float b, float eps, int dtype,
                     int eps_inside_k, void* stream);

/* out[0] = sum_i a[i] * b[i] (f32 result, f32 accumulation; dtype F32 or F16).  kernels/dot-product/dot_product.cu:L20-184,
 * bindings L233-283.  Deterministic (fixed two-pass order) where the reference uses atomicAdd.  `out`: 1-element f32
 * device buffer; `workspace`: >= b200k_reduce_workspace_bytes(). */
int b200k_dot_prod(const void* a, const void* b, void* out, int64_t n, int dtype, void* workspace, void* stream);

/* y[N,M] = transpose(x[M,N]), fp32.  kernels/mat-transpose/mat_transpose.cu:L20-278 (13 entry points, L296-359). */
int b200k_mat_transpose_f32(const void* x, void* y, int64_t M, int64_t N, void* stream);

/* y[M] = A[M,K] x[K], dtype F32 or F16 (f32 accumulation; the reference's hgemv accumulates in half).
 * kernels/sgemv/sgemv.cu:L20-104 (sgemv_k32_f32, sgemv_k128_f32x4, sgemv_k16_f32), kernels/hgemv/hgemv.cu:L24-108. */
int b200k_gemv(const void* a, const void* x, void* y, int64_t M, int64_t K, int dtype, void* stream);
/* y[b][N,M] = x[b][M,N]^T for 16-bit elements (f16 / bf16), `batch` matrices back to back; exact.  Used by the drop-in
 * flash_attn_mma_stages_*_swizzle_qkv entry points for head dims above 128 (V arrives as [B,H,D,N], flash_attn.cc:L128-159). */
int b200k_transpose_u16_batched(const void* x, void* y, int64_t batch, int64_t M, int64_t N, void* stream);


#ifdef __cplusplus
}
#endif
#endif /* B200K_H_ */
