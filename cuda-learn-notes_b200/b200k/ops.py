"""Tensor-level host wrappers over the C ABI (include/b200k.h).

These are the single place where torch tensors are turned into raw pointers + sizes + the current CUDA stream.
Argument checks reproduce the reference bindings' behaviour and error strings
(kernels/hgemm/mma/basic/hgemm_mma_stage.cu:L2078-2087 CHECK_TORCH_TENSOR_DTYPE / _SHAPE,
kernels/flash-attn/utils/utils.h:L66-78, kernels/flash-attn/mma/basic/flash_attn_mma_share_qkv.cu:L860).

PyTorch is used for device memory and streams only; every computation happens in libb200k.so.
"""
from __future__ import annotations

import ctypes
import math
from typing import Optional

import torch

from . import _loader as L

_lib = L.lib

_DTYPE_ENUM = {
    torch.float32: L.F32,
    torch.float16: L.F16,
    torch.bfloat16: L.BF16,
    torch.int8: L.I8,
    torch.int32: L.I32,
}
if hasattr(torch, "float8_e4m3fn"):
    _DTYPE_ENUM[torch.float8_e4m3fn] = L.FP8_E4M3
    _DTYPE_ENUM[torch.float8_e5m2] = L.FP8_E5M2

_TH_NAME = {
    torch.float16: "torch::kHalf",
    torch.float32: "torch::kFloat32",
    torch.int32: "torch::kInt32",
    torch.bfloat16: "torch::kBFloat16",
    torch.int8: "torch::kInt8",
}


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def _stream(t: torch.Tensor) -> int:
    """The current CUDA stream of the tensor's device as a raw handle.  The private torch hook skips building a
    torch.cuda.Stream object (the wrapper's per-call cost matters for a 17 us GEMM); the public API is the fallback."""
    if _raw_stream is not None:
        return _raw_stream(t.device.index)
    return torch.cuda.current_stream(t.device).cuda_stream


def _check_dtype(t: torch.Tensor, dtype: torch.dtype) -> None:
    if t.dtype != dtype:
        # same message as the reference's CHECK_TORCH_TENSOR_DTYPE
        raise RuntimeError("values must be " + _TH_NAME.get(dtype, str(dtype)))


def _check_cuda_contig(*ts: torch.Tensor) -> None:
    dev = None
    for t in ts:
        if not t.is_cuda:
            raise RuntimeError("b200k: tensors must live on a CUDA device (there is no CPU path)")
        if not t.is_contiguous():
            raise RuntimeError("b200k: tensors must be contiguous")
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise RuntimeError("b200k: tensors must be on the same device")


class _DeviceGuard:
    """The reference launches on whatever device is current; we launch on the tensors' device."""

    def __init__(self, t: torch.Tensor):
        self.dev = t.device
        self.ctx = None

    def __enter__(self):
        if self.dev.index != torch.cuda.current_device():   # the common case switches nothing
            self.ctx = torch.cuda.device(self.dev)
            self.ctx.__enter__()

    def __exit__(self, *a):
        if self.ctx is not None:
            return self.ctx.__exit__(*a)
        return False


# ------------------------------------------------------------------------------------------------ HGEMM
def hgemm(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor, tn: bool = False, variant: int = L.HGEMM_AUTO) -> None:
    """c[M,N] = a[M,K] @ B (in place).  ``b`` has logical shape [K,N]; for ``tn`` its storage is B^T row-major
    (the reference's ``as_col_major``, kernels/hgemm/tools/utils.py:L135-140), i.e. it arrives as a [K,N]-shaped
    view whose memory is [N,K] contiguous."""
    _check_dtype(a, torch.float16)
    _check_dtype(b, torch.float16)
    _check_dtype(c, torch.float16)
    M, K = a.size(0), a.size(1)
    N = b.size(1)
    if b.size(0) != K or c.size(0) != M or c.size(1) != N:
        raise RuntimeError("Tensor size mismatch!")
    if tn:
        # Two spellings of "storage is B^T [N,K] row-major": the reference's as_col_major() returns a CONTIGUOUS
        # [K,N]-shaped tensor holding B^T's elements (tools/utils.py:L135-140); a strided view b = Bt.t() is the other.
        _check_cuda_contig(a, b if b.is_contiguous() else b.t(), c)
    else:
        _check_cuda_contig(a, b, c)
    with _DeviceGuard(a):
        L.check(_lib.b200k_hgemm_f16(a.data_ptr(), b.data_ptr(), c.data_ptr(), M, N, K, 1 if tn else 0, variant,
                                     _stream(a)))


def gemm(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor, tn: bool = False, variant: int = L.HGEMM_AUTO,
         a_km: bool = False) -> None:
    """c = a @ B for fp16, bf16 (fp32 accumulation) or fp32 operands (TF32 tensor-core product, fp32 accumulation and
    output); same layouts as :func:`hgemm`.  ``a_km``: ``a`` has logical shape [M,K] but its storage is A^T [K,M] row-major
    (pass ``At.t()`` of a contiguous ``At``) - the BLAS "NT"/"TT" cases, f16 / bf16."""
    if a_km:
        if a.dtype not in (torch.float16, torch.bfloat16):
            raise RuntimeError("values must be torch::kHalf or torch::kBFloat16")
        _check_dtype(b, a.dtype)
        _check_dtype(c, a.dtype)
        M, K, N = a.size(0), a.size(1), b.size(1)
        if b.size(0) != K or c.size(0) != M or c.size(1) != N:
            raise RuntimeError("Tensor size mismatch!")
        _check_cuda_contig(a.t(), (b if b.is_contiguous() else b.t()) if tn else b, c)
        with _DeviceGuard(a):
            L.check(_lib.b200k_gemm_ex(a.data_ptr(), b.data_ptr(), c.data_ptr(), M, N, K, 1, 1 if tn else 0,
                                       _DTYPE_ENUM[a.dtype], variant, _stream(a)))
        return
    if a.dtype not in (torch.float16, torch.bfloat16, torch.float32):
        raise RuntimeError("values must be torch::kHalf, torch::kBFloat16 or torch::kFloat32")
    _check_dtype(b, a.dtype)
    _check_dtype(c, a.dtype)
    M, K = a.size(0), a.size(1)
    N = b.size(1)
    if b.size(0) != K or c.size(0) != M or c.size(1) != N:
        raise RuntimeError("Tensor size mismatch!")
    if tn:
        _check_cuda_contig(a, b if b.is_contiguous() else b.t(), c)
    else:
        _check_cuda_contig(a, b, c)
    with _DeviceGuard(a):
        L.check(_lib.b200k_gemm(a.data_ptr(), b.data_ptr(), c.data_ptr(), M, N, K, 1 if tn else 0, _DTYPE_ENUM[a.dtype],
                                variant, _stream(a)))


# ------------------------------------------------------------------------------------------------ attention
FA2_HEADDIMS = (32, 64, 96, 128)


def _check_qkvo(q, k, v, o, v_is_dn=False, dtype=torch.float16):
    for t in (q, k, v, o):
        _check_dtype(t, dtype)
    if q.dim() != 4:
        raise RuntimeError("Tensor size mismatch!")
    B, H, N, D = q.shape
    vshape = (B, H, D, N) if v_is_dn else (B, H, N, D)
    if tuple(k.shape) != (B, H, N, D) or tuple(v.shape) != vshape or tuple(o.shape) != (B, H, N, D):
        raise RuntimeError("Tensor size mismatch!")
    _check_cuda_contig(q, k, v, o)
    return B, H, N, D


def _check_lse(lse: torch.Tensor, o: torch.Tensor) -> None:
    """``lse`` must be fp32 of o's shape without its last dim, contiguous, on o's device."""
    _check_dtype(lse, torch.float32)
    if tuple(lse.shape) != tuple(o.shape[:-1]):
        raise RuntimeError("Tensor size mismatch!")
    _check_cuda_contig(o, lse)


def fa2_fwd(q, k, v, o, scale: Optional[float] = None, v_is_dn: bool = False, variant: int = 0, causal: bool = False,
            seqlens_k: Optional[torch.Tensor] = None, lse: Optional[torch.Tensor] = None) -> None:
    """FA-2 forward, [B,H,N,D] fp16 (the reference's layout and dtype) or bf16.  ``causal`` and ``seqlens_k`` (int32 [B] on
    the device: valid keys per batch) are the caller-facing options of SURVEY 8(f)-4; the reference has neither.
    ``lse``: an fp32 [B, H, N] tensor that receives each row's softmax log-sum-exp (natural log; see :func:`attn_merge`)."""
    dt = q.dtype if q.dtype == torch.bfloat16 else torch.float16
    if lse is not None:
        _check_lse(lse, o)
    B, H, N, D = _check_qkvo(q, k, v, o, v_is_dn, dt)
    if D not in FA2_HEADDIMS:
        raise RuntimeError("headdim not support!")
    sl = 0
    if seqlens_k is not None:
        _check_dtype(seqlens_k, torch.int32)
        _check_cuda_contig(seqlens_k)
        if seqlens_k.numel() != B:
            raise RuntimeError("Tensor size mismatch!")
        sl = seqlens_k.data_ptr()
    with _DeviceGuard(q):
        L.check(_lib.b200k_fa2_fwd_lse(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(),
                                       lse.data_ptr() if lse is not None else None, B, H, N, D,
                                       float(scale) if scale else 0.0, 1 if v_is_dn else 0, _DTYPE_ENUM[dt],
                                       1 if causal else 0, sl, variant, _stream(q)))


def fa2_fwd_varlen(q, k, v, o, cu_seqlens_q: torch.Tensor, cu_seqlens_k: torch.Tensor, max_seqlen_q: int,
                   scale: Optional[float] = None, causal: bool = False, lse: Optional[torch.Tensor] = None, *,
                   block_table: Optional[torch.Tensor] = None, k_scale: Optional[torch.Tensor] = None,
                   v_scale: Optional[torch.Tensor] = None) -> None:
    """FA-2 forward on packed variable-length sequences (the forward of flash-attn's ``flash_attn_varlen_func``).
    q, o [total_q, H, D]; k, v [total_k, H_kv, D] with H % H_kv == 0 (query head h reads K/V head h // (H // H_kv));
    fp16 or bf16.  ``cu_seqlens_q`` / ``cu_seqlens_k``: int32 [B + 1] cumulative token offsets on the device.
    ``max_seqlen_q`` (a Python int, >= every query length) sizes the grid, so nothing is read back to the host.
    ``causal`` is aligned bottom-right (row r sees keys <= r + Lk - Lq); rows that see no key are 0.
    ``lse``: an fp32 [total_q, H] tensor that receives each row's softmax log-sum-exp (-inf for a row that sees no key);
    tokens outside every sequence are left untouched, like o.

    Paged K/V (prefill after a cached prefix, chunked prefill, prompts of mixed lengths): with an int32
    ``block_table`` [B, pages_per_seq], k and v are caches [num_pages, page_size, H_kv, D] and key j of sequence b is
    slot j % page_size of page block_table[b, j // page_size], as in flash-attn.  Sequence b then has
    Lk = cu_seqlens_k[b + 1] - cu_seqlens_k[b] keys, clamped to [0, pages_per_seq * page_size]; page_size is 16, 32, 64
    or a multiple of 128.  Cache slots past Lk and pages the table row does not list never affect o or lse, whatever
    they hold.  o and lse have the bits of the call without a table on k / v gathered through it.  Each query tile is
    128 rows, so for decode (one query token per sequence) :func:`fa2_fwd_kvcache` is the call to use.

    FP8 pages: with a ``block_table``, k and v may be ``torch.float8_e4m3fn`` or ``torch.float8_e5m2`` caches (one dtype
    for both), dequantized as fp8 * ``k_scale`` / ``v_scale`` (fp32 [H_kv] device tensors, or None for 1.0); see
    :func:`fa2_fwd_kvcache`.  o and lse then have the bits of the call on the gathered, dequantized K / V."""
    fp8 = _fp8_kv(k, v, k_scale, v_scale)
    if fp8 and block_table is None:
        raise RuntimeError("b200k: fp8 K / V are read from paged caches: pass block_table")
    dt = q.dtype if q.dtype == torch.bfloat16 else torch.float16
    for t in (q, o) if fp8 else (q, k, v, o):
        _check_dtype(t, dt)
    if block_table is not None:
        _fa2_fwd_varlen_paged(q, k, v, o, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, scale, causal, lse, block_table, dt,
                              fp8, k_scale, v_scale)
        return
    if q.dim() != 3 or k.dim() != 3:
        raise RuntimeError("Tensor size mismatch!")
    total_q, H, D = q.shape
    total_k, H_kv = k.size(0), k.size(1)
    if tuple(k.shape) != (total_k, H_kv, D) or tuple(v.shape) != tuple(k.shape) or tuple(o.shape) != tuple(q.shape):
        raise RuntimeError("Tensor size mismatch!")
    if H_kv < 1 or H % H_kv:
        raise RuntimeError("Tensor size mismatch!")
    if D not in FA2_HEADDIMS:
        raise RuntimeError("headdim not support!")
    _check_dtype(cu_seqlens_q, torch.int32)
    _check_dtype(cu_seqlens_k, torch.int32)
    B = cu_seqlens_q.numel() - 1
    if B < 1 or cu_seqlens_k.numel() != B + 1:
        raise RuntimeError("Tensor size mismatch!")
    if lse is not None:
        _check_lse(lse, o)
    _check_cuda_contig(q, k, v, o, cu_seqlens_q, cu_seqlens_k)
    with _DeviceGuard(q):
        L.check(_lib.b200k_fa2_fwd_varlen_lse(
            q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr() if lse is not None else None,
            cu_seqlens_q.data_ptr(), cu_seqlens_k.data_ptr(), B, int(max_seqlen_q), total_q, total_k, H, H_kv, D,
            float(scale) if scale else 0.0, _DTYPE_ENUM[dt], 1 if causal else 0, _stream(q)))


def _fa2_fwd_varlen_paged(q, k_cache, v_cache, o, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, scale, causal, lse,
                          block_table, dt, fp8, k_scale, v_scale) -> None:
    """:func:`fa2_fwd_varlen` with ``block_table``: the shape checks of the paged layout, for caches of either dtype,
    then b200k_fa2_varlen_paged, or b200k_fa2_varlen_paged_fp8 over fp8 pages."""
    if q.dim() != 3 or k_cache.dim() != 4:
        raise RuntimeError("Tensor size mismatch!")
    total_q, H, D = q.shape
    num_pages, page_size, H_kv = k_cache.size(0), k_cache.size(1), k_cache.size(2)
    if (tuple(k_cache.shape) != (num_pages, page_size, H_kv, D) or tuple(v_cache.shape) != tuple(k_cache.shape)
            or tuple(o.shape) != tuple(q.shape)):
        raise RuntimeError("Tensor size mismatch!")
    if H_kv < 1 or H % H_kv:
        raise RuntimeError("Tensor size mismatch!")
    if D not in FA2_HEADDIMS:
        raise RuntimeError("headdim not support!")
    _check_dtype(cu_seqlens_q, torch.int32)
    _check_dtype(cu_seqlens_k, torch.int32)
    _check_dtype(block_table, torch.int32)
    B = cu_seqlens_q.numel() - 1
    if B < 1 or cu_seqlens_k.numel() != B + 1 or block_table.dim() != 2 or block_table.size(0) != B:
        raise RuntimeError("Tensor size mismatch!")
    if not block_table.is_contiguous():  # the kernel reads row b at b * pages_per_seq
        raise RuntimeError("b200k: tensors must be contiguous")
    if lse is not None:
        _check_lse(lse, o)
    _check_cuda_contig(q, k_cache, v_cache, o, cu_seqlens_q, cu_seqlens_k, block_table)
    ks, vs = _fp8_scales(k_scale, v_scale, H_kv) if fp8 else (None, None)
    ptrs = (q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), o.data_ptr(), lse.data_ptr() if lse is not None else None,
            cu_seqlens_q.data_ptr(), cu_seqlens_k.data_ptr(), block_table.data_ptr())
    shapes = (B, int(max_seqlen_q), total_q, H, H_kv, D, num_pages, page_size, block_table.size(1),
              float(scale) if scale else 0.0, _DTYPE_ENUM[dt], 1 if causal else 0, _stream(q))
    with _DeviceGuard(q):
        if fp8:
            L.check(_lib.b200k_fa2_varlen_paged_fp8(*ptrs, ks, vs, _DTYPE_ENUM[k_cache.dtype], *shapes))
        else:
            L.check(_lib.b200k_fa2_varlen_paged(*ptrs, *shapes))


_FP8_KV = tuple(d for d in (getattr(torch, "float8_e4m3fn", None), getattr(torch, "float8_e5m2", None)) if d is not None)


def _fp8_kv(k_cache, v_cache, k_scale, v_scale) -> bool:
    """Whether a call reads fp8 caches.  Scales with 16-bit caches and caches of two different dtypes are refused."""
    fp8 = k_cache.dtype in _FP8_KV or v_cache.dtype in _FP8_KV
    if fp8 and k_cache.dtype != v_cache.dtype:
        raise RuntimeError("b200k: k_cache and v_cache must hold the same fp8 dtype (got %s and %s)"
                           % (k_cache.dtype, v_cache.dtype))
    if not fp8 and (k_scale is not None or v_scale is not None):
        raise RuntimeError("b200k: k_scale / v_scale dequantize fp8 caches; the caches are %s" % k_cache.dtype)
    return fp8


def _fp8_scales(k_scale, v_scale, H_kv: int) -> list:
    """The scale pointers (None for 1.0) after their checks: fp32 [H_kv], contiguous, on the device."""
    ptrs = []
    for t in (k_scale, v_scale):
        if t is None:
            ptrs.append(None)
            continue
        _check_dtype(t, torch.float32)
        if t.numel() != H_kv:
            raise RuntimeError("Tensor size mismatch!")
        _check_cuda_contig(t)
        ptrs.append(t.data_ptr())
    return ptrs


def fa2_fwd_kvcache_fp8_workspace_bytes(B: int, Lq: int, H: int, H_kv: int, D: int, max_seqlen_k: int,
                                        append: bool = False, rotary: bool = False) -> int:
    """Workspace bytes :func:`fa2_fwd_kvcache` needs over fp8 caches, with or without ``k`` / ``v``; queries the
    device."""
    n = ctypes.c_size_t(0)
    L.check(_lib.b200k_fa2_kvcache_fp8_workspace_bytes(B, Lq, H, H_kv, D, max_seqlen_k, 1 if append else 0,
                                                       1 if rotary else 0, ctypes.byref(n)))
    return n.value


def fa2_fwd_kvcache_workspace_bytes(B: int, Lq: int, H: int, H_kv: int, D: int, max_seqlen_k: int) -> int:
    """Workspace bytes :func:`fa2_fwd_kvcache` needs for these shapes (0 when it runs unsplit); queries the device."""
    n = ctypes.c_size_t(0)
    L.check(_lib.b200k_fa2_fwd_kvcache_workspace_bytes(B, Lq, H, H_kv, D, max_seqlen_k, ctypes.byref(n)))
    return n.value


def fa2_fwd_kvcache_append_workspace_bytes(B: int, Lq: int, H: int, H_kv: int, D: int, max_seqlen_k: int,
                                           rotary: bool) -> int:
    """Workspace bytes :func:`fa2_fwd_kvcache` needs with ``k`` / ``v`` for these shapes; queries the device."""
    n = ctypes.c_size_t(0)
    L.check(_lib.b200k_fa2_fwd_kvcache_append_workspace_bytes(B, Lq, H, H_kv, D, max_seqlen_k, 1 if rotary else 0,
                                                              ctypes.byref(n)))
    return n.value


def _kvcache_checks(q, k_cache, v_cache, o, cache_seqlens, block_table, lse, k, v, rotary_cos, rotary_sin, cache_dt):
    """The checks of :func:`fa2_fwd_kvcache` with caches of dtype cache_dt (q's, or an fp8 one); returns
    (B, Lq, H, H_kv, D, num_pages, page_size, pages_per_seq, append, rotary)."""
    dt = q.dtype if q.dtype == torch.bfloat16 else torch.float16
    for t, want in ((q, dt), (k_cache, cache_dt), (v_cache, cache_dt), (o, dt)):
        _check_dtype(t, want)
    if q.dim() != 4 or k_cache.dim() != 4:
        raise RuntimeError("Tensor size mismatch!")
    B, Lq, H, D = q.shape
    num_pages, page_size, H_kv = k_cache.size(0), k_cache.size(1), k_cache.size(2)
    if (tuple(k_cache.shape) != (num_pages, page_size, H_kv, D) or tuple(v_cache.shape) != tuple(k_cache.shape)
            or tuple(o.shape) != tuple(q.shape)):
        raise RuntimeError("Tensor size mismatch!")
    if H_kv < 1 or H % H_kv:
        raise RuntimeError("Tensor size mismatch!")
    if D not in FA2_HEADDIMS:
        raise RuntimeError("headdim not support!")
    _check_dtype(cache_seqlens, torch.int32)
    if cache_seqlens.numel() != B:
        raise RuntimeError("Tensor size mismatch!")
    tensors = [q, k_cache, v_cache, o, cache_seqlens]
    if block_table is None:
        if num_pages != B:
            raise RuntimeError("Tensor size mismatch!")
        pages_per_seq = 1
    else:
        _check_dtype(block_table, torch.int32)
        if block_table.dim() != 2 or block_table.size(0) != B:
            raise RuntimeError("Tensor size mismatch!")
        pages_per_seq = block_table.size(1)
        tensors.append(block_table)
    if lse is not None:
        _check_lse(lse, o)
    rotary = rotary_cos is not None or rotary_sin is not None
    append = k is not None or v is not None or rotary
    if append:
        if k is None or v is None:
            raise RuntimeError("b200k: append needs both k and v (rotary applies to appended keys)")
        if (rotary_cos is None) != (rotary_sin is None):
            raise RuntimeError("b200k: rotary needs both rotary_cos and rotary_sin")
        for t in (k, v):
            _check_dtype(t, dt)
        if k.dim() != 4 or k.size(0) != B or tuple(k.shape[2:]) != (H_kv, D) or tuple(v.shape) != tuple(k.shape):
            raise RuntimeError("Tensor size mismatch!")
        tensors += [k, v]
        if rotary:
            _check_dtype(rotary_cos, dt)
            _check_dtype(rotary_sin, dt)
            if rotary_cos.dim() != 2 or tuple(rotary_sin.shape) != tuple(rotary_cos.shape):
                raise RuntimeError("Tensor size mismatch!")
            tensors += [rotary_cos, rotary_sin]
    _check_cuda_contig(*tensors)
    return B, Lq, H, H_kv, D, num_pages, page_size, pages_per_seq, append, rotary


def fa2_fwd_kvcache(q, k_cache, v_cache, o, cache_seqlens: torch.Tensor, block_table: Optional[torch.Tensor] = None,
                    scale: Optional[float] = None, causal: bool = False, *, k: Optional[torch.Tensor] = None,
                    v: Optional[torch.Tensor] = None, rotary_cos: Optional[torch.Tensor] = None,
                    rotary_sin: Optional[torch.Tensor] = None, rotary_interleaved: bool = True,
                    lse: Optional[torch.Tensor] = None, k_scale: Optional[torch.Tensor] = None,
                    v_scale: Optional[torch.Tensor] = None) -> None:
    """Attention of the newest Lq query tokens of each sequence against its KV cache (flash-attn's
    ``flash_attn_with_kvcache``).  q, o [B, Lq, H, D], fp16 or bf16.  Caches
    [B, S, H_kv, D] without ``block_table``, or [num_pages, page_size, H_kv, D] with an int32 ``block_table``
    [B, pages_per_seq] (key j of sequence b is slot j % page_size of page block_table[b, j // page_size]).
    ``cache_seqlens``: int32 [B] key counts on the device.  ``causal``: token t sees keys <= t + Lk - Lq.  H % H_kv == 0
    (query head h reads K/V head h // (H // H_kv)).  Nothing is read back to the host, so the call can be captured in a
    CUDA graph; the workspace is allocated per call on the current stream.

    Append: ``k``, ``v`` [B, L_new, H_kv, D] are written into the caches in place at positions
    cache_seqlens[b] + i (through the table when paged), and the attention runs over cache_seqlens[b] + L_new keys.
    ``cache_seqlens`` itself is not updated; the caller adds L_new afterwards.  ``rotary_cos`` / ``rotary_sin``
    [rotary_seqlen, rotary_dim / 2] in q's dtype (rotary_dim a multiple of 16, at most D; rotary_seqlen at least the
    capacity) rotate the first rotary_dim columns of k and q: new key i at position cache_seqlens[b] + i, query token t
    at cache_seqlens[b] + t when causal and at cache_seqlens[b] when not.  ``rotary_interleaved`` pairs columns
    (2j, 2j + 1); otherwise (j, j + rotary_dim / 2), GPT-NeoX style.  q is not modified.

    ``lse``: an fp32 [B, Lq, H] tensor that receives each row's softmax log-sum-exp over the keys it sees (-inf for
    none), with or without ``k`` / ``v``.

    FP8 caches (vLLM's ``kv_cache_dtype="fp8"`` / ``"fp8_e5m2"``): k_cache and v_cache both ``torch.float8_e4m3fn``
    or both ``torch.float8_e5m2``.  The key of K/V head h is fp8 * ``k_scale[h]`` and its value fp8 * ``v_scale[h]``
    (fp32 [H_kv] device tensors, or None for 1.0; being tensors, they can change between replays of a captured graph).
    q, o, ``k`` / ``v`` and cos / sin stay fp16 or bf16; appended rows are stored as
    satfinite(float(x) / scale[h]) in the cache's format, after rotary.  With no scales, o and lse have the bits of the
    16-bit call on the dequantized caches; with power-of-two scales too, as long as the dequantized values are normal
    in q's dtype.  A scale with 16-bit caches, or caches of two dtypes, is a RuntimeError."""
    fp8 = _fp8_kv(k_cache, v_cache, k_scale, v_scale)
    dt = q.dtype if q.dtype == torch.bfloat16 else torch.float16
    B, Lq, H, H_kv, D, num_pages, page_size, pages_per_seq, append, rotary = _kvcache_checks(
        q, k_cache, v_cache, o, cache_seqlens, block_table, lse, k, v, rotary_cos, rotary_sin,
        k_cache.dtype if fp8 else dt)
    cos, sin = rotary_cos, rotary_sin
    ks, vs = _fp8_scales(k_scale, v_scale, H_kv) if fp8 else (None, None)
    capacity = pages_per_seq * page_size
    with _DeviceGuard(q):
        if fp8:
            nbytes = fa2_fwd_kvcache_fp8_workspace_bytes(B, Lq, H, H_kv, D, capacity, append, rotary)
        elif append:
            nbytes = fa2_fwd_kvcache_append_workspace_bytes(B, Lq, H, H_kv, D, capacity, rotary)
        else:
            nbytes = fa2_fwd_kvcache_workspace_bytes(B, Lq, H, H_kv, D, capacity)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=q.device) if nbytes else None
        ptrs = (q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), o.data_ptr(),
                lse.data_ptr() if lse is not None else None, cache_seqlens.data_ptr(),
                block_table.data_ptr() if block_table is not None else None)
        new = (k.data_ptr() if append else None, v.data_ptr() if append else None, k.size(1) if append else 0,
               cos.data_ptr() if rotary else None, sin.data_ptr() if rotary else None, cos.size(0) if rotary else 0,
               2 * cos.size(1) if rotary else 0, 1 if rotary_interleaved else 0)
        shapes = (B, Lq, H, H_kv, D, num_pages, page_size, pages_per_seq, float(scale) if scale else 0.0,
                  _DTYPE_ENUM[dt], 1 if causal else 0, ws.data_ptr() if ws is not None else None, nbytes, _stream(q))
        if fp8:
            L.check(_lib.b200k_fa2_kvcache_fp8(*ptrs, ks, vs, _DTYPE_ENUM[k_cache.dtype], *new, *shapes))
        elif append:
            L.check(_lib.b200k_fa2_fwd_kvcache_append_lse(*ptrs, *new, *shapes))
        else:
            L.check(_lib.b200k_fa2_fwd_kvcache_lse(*ptrs, *shapes))


def attn_merge(o_parts: torch.Tensor, lse_parts: torch.Tensor, o: torch.Tensor,
               lse: Optional[torch.Tensor] = None) -> None:
    """o (and lse) = the attention over the union of S disjoint key sets, from the attention over each: o_parts
    [S, *o.shape] in o's dtype (fp16 or bf16) and lse_parts [S, *o.shape[:-1]] fp32, as the ``lse=`` outputs of
    :func:`fa2_fwd`, :func:`fa2_fwd_varlen` and :func:`fa2_fwd_kvcache` give them.  Parts are weighted by
    exp(lse_s - max) in fp32 and summed in ascending s (deterministic); a part with lse = -inf is skipped, and a row with
    no part left is 0 with lse -inf.  ``lse`` (fp32, o.shape[:-1]) receives the merged log-sum-exp.  o must not overlap
    o_parts; o.shape[-1] must be a multiple of 8."""
    if o.dtype not in (torch.float16, torch.bfloat16):
        raise RuntimeError("values must be torch::kHalf or torch::kBFloat16")
    _check_dtype(o_parts, o.dtype)
    _check_dtype(lse_parts, torch.float32)
    if o.dim() < 1 or o_parts.dim() != o.dim() + 1 or tuple(o_parts.shape[1:]) != tuple(o.shape):
        raise RuntimeError("Tensor size mismatch!")
    S, D = o_parts.size(0), o.size(-1)
    if tuple(lse_parts.shape) != (S,) + tuple(o.shape[:-1]):
        raise RuntimeError("Tensor size mismatch!")
    if lse is not None:
        _check_lse(lse, o)
    _check_cuda_contig(o_parts, lse_parts, o)
    with _DeviceGuard(o):
        L.check(_lib.b200k_attn_merge(o_parts.data_ptr(), lse_parts.data_ptr(), o.data_ptr(),
                                      lse.data_ptr() if lse is not None else None, S, o.numel() // D if D else 0, D,
                                      _DTYPE_ENUM[o.dtype], _stream(o)))


def fa2_bwd_workspace_bytes(B: int, H: int, N: int) -> int:
    """Workspace bytes :func:`fa2_bwd` needs for these shapes."""
    n = ctypes.c_size_t(0)
    L.check(_lib.b200k_fa2_bwd_workspace_bytes(B, H, N, ctypes.byref(n)))
    return n.value


def fa2_bwd(q, k, v, o, lse, do, dq, dk, dv, scale: Optional[float] = None, causal: bool = False,
            seqlens_k: Optional[torch.Tensor] = None) -> None:
    """Gradients of :func:`fa2_fwd` (dense [B, H, N, D], fp16 or bf16) into dq, dk, dv: o and ``lse`` (fp32 [B, H, N])
    are what ``fa2_fwd(q, k, v, o, scale, causal=causal, seqlens_k=seqlens_k, lse=lse)`` wrote, ``do`` the gradient of
    o.  ``scale``, ``causal`` and ``seqlens_k`` must be the forward's.  Deterministic (no atomics), and nothing is read
    back to the host, so the call can be captured in a CUDA graph; the workspace is allocated per call on the current
    stream."""
    dt = q.dtype if q.dtype == torch.bfloat16 else torch.float16
    for t in (q, k, v, o, do, dq, dk, dv):
        _check_dtype(t, dt)
    if q.dim() != 4 or any(tuple(t.shape) != tuple(q.shape) for t in (k, v, o, do, dq, dk, dv)):
        raise RuntimeError("Tensor size mismatch!")
    B, H, N, D = q.shape
    if D not in FA2_HEADDIMS:
        raise RuntimeError("headdim not support!")
    tensors = [q, k, v, o, lse, do, dq, dk, dv]
    sl = None
    if seqlens_k is not None:
        _check_dtype(seqlens_k, torch.int32)
        if seqlens_k.numel() != B:
            raise RuntimeError("Tensor size mismatch!")
        tensors.append(seqlens_k)
        sl = seqlens_k.data_ptr()
    _check_lse(lse, o)
    _check_cuda_contig(*tensors)
    with _DeviceGuard(q):
        nbytes = fa2_bwd_workspace_bytes(B, H, N)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=q.device)
        L.check(_lib.b200k_fa2_bwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(), do.data_ptr(),
                                   dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), B, H, N, D,
                                   float(scale) if scale else 0.0, _DTYPE_ENUM[dt], 1 if causal else 0, sl,
                                   ws.data_ptr(), nbytes, _stream(q)))


class _Attention(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, scale, causal, seqlens_k):
        o = torch.empty_like(q)
        lse = torch.empty(q.shape[:-1], dtype=torch.float32, device=q.device)
        fa2_fwd(q, k, v, o, scale, causal=causal, seqlens_k=seqlens_k, lse=lse)
        ctx.save_for_backward(q, k, v, o, lse)
        ctx.scale, ctx.causal, ctx.seqlens_k = scale, causal, seqlens_k
        return o

    @staticmethod
    def backward(ctx, grad):
        q, k, v, o, lse = ctx.saved_tensors
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        fa2_bwd(q, k, v, o, lse, grad.contiguous(), dq, dk, dv, ctx.scale, ctx.causal, ctx.seqlens_k)
        return dq, dk, dv, None, None, None


def attention(q, k, v, scale: Optional[float] = None, causal: bool = False,
              seqlens_k: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Differentiable attention, dense [B, H, N, D] fp16 or bf16 (D in 32, 64, 96, 128): returns
    o = softmax(q k^T * scale (masked)) v from :func:`fa2_fwd`, and its backward is :func:`fa2_bwd`, which gives the
    gradients of q, k and v (``seqlens_k``, int32 [B]: valid keys per batch, is not differentiable)."""
    return _Attention.apply(q, k, v, scale, causal, seqlens_k)


def fa2_bwd_varlen_workspace_bytes(total_q: int, H: int) -> int:
    """Workspace bytes :func:`fa2_bwd_varlen` needs for these shapes."""
    n = ctypes.c_size_t(0)
    L.check(_lib.b200k_fa2_bwd_varlen_workspace_bytes(total_q, H, ctypes.byref(n)))
    return n.value


def fa2_bwd_varlen(q, k, v, o, lse, do, dq, dk, dv, cu_seqlens_q: torch.Tensor, cu_seqlens_k: torch.Tensor,
                   max_seqlen_q: int, max_seqlen_k: int, scale: Optional[float] = None, causal: bool = False) -> None:
    """Gradients of :func:`fa2_fwd_varlen` (packed sequences, grouped K/V heads) into dq [total_q, H, D] and dk, dv
    [total_k, H_kv, D]: o and ``lse`` (fp32 [total_q, H]) are what the forward wrote with ``lse=``, ``do`` the gradient
    of o.  ``scale``, ``causal`` and the ``cu_seqlens`` must be the forward's; ``max_seqlen_q`` / ``max_seqlen_k``
    (Python ints, >= every length) size the grids.  dk / dv of a K/V head sum over its query heads; rows of tokens
    outside every sequence are 0.  Deterministic and graph-capturable; the workspace is allocated per call on the
    current stream."""
    dt = q.dtype if q.dtype == torch.bfloat16 else torch.float16
    for t in (q, k, v, o, do, dq, dk, dv):
        _check_dtype(t, dt)
    if q.dim() != 3 or k.dim() != 3:
        raise RuntimeError("Tensor size mismatch!")
    total_q, H, D = q.shape
    total_k, H_kv = k.size(0), k.size(1)
    if (tuple(k.shape) != (total_k, H_kv, D) or any(tuple(t.shape) != tuple(k.shape) for t in (v, dk, dv))
            or any(tuple(t.shape) != tuple(q.shape) for t in (o, do, dq))):
        raise RuntimeError("Tensor size mismatch!")
    if H_kv < 1 or H % H_kv:
        raise RuntimeError("Tensor size mismatch!")
    if D not in FA2_HEADDIMS:
        raise RuntimeError("headdim not support!")
    _check_dtype(cu_seqlens_q, torch.int32)
    _check_dtype(cu_seqlens_k, torch.int32)
    B = cu_seqlens_q.numel() - 1
    if B < 1 or cu_seqlens_k.numel() != B + 1:
        raise RuntimeError("Tensor size mismatch!")
    _check_lse(lse, o)
    _check_cuda_contig(q, k, v, o, lse, do, dq, dk, dv, cu_seqlens_q, cu_seqlens_k)
    with _DeviceGuard(q):
        nbytes = fa2_bwd_varlen_workspace_bytes(total_q, H)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=q.device)
        L.check(_lib.b200k_fa2_bwd_varlen(
            q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(), do.data_ptr(), dq.data_ptr(),
            dk.data_ptr(), dv.data_ptr(), cu_seqlens_q.data_ptr(), cu_seqlens_k.data_ptr(), B, int(max_seqlen_q),
            int(max_seqlen_k), total_q, total_k, H, H_kv, D, float(scale) if scale else 0.0, _DTYPE_ENUM[dt],
            1 if causal else 0, ws.data_ptr(), nbytes, _stream(q)))


class _AttentionVarlen(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, scale, causal):
        o = torch.empty_like(q)
        lse = torch.empty(q.shape[:-1], dtype=torch.float32, device=q.device)
        fa2_fwd_varlen(q, k, v, o, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, scale, causal=causal, lse=lse)
        ctx.save_for_backward(q, k, v, o, lse, cu_seqlens_q, cu_seqlens_k)
        ctx.max_seqlen_q, ctx.max_seqlen_k, ctx.scale, ctx.causal = max_seqlen_q, max_seqlen_k, scale, causal
        return o

    @staticmethod
    def backward(ctx, grad):
        q, k, v, o, lse, cu_q, cu_k = ctx.saved_tensors
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        fa2_bwd_varlen(q, k, v, o, lse, grad.contiguous(), dq, dk, dv, cu_q, cu_k, ctx.max_seqlen_q, ctx.max_seqlen_k,
                       ctx.scale, ctx.causal)
        return dq, dk, dv, None, None, None, None, None, None


def attention_varlen(q, k, v, cu_seqlens_q: torch.Tensor, cu_seqlens_k: torch.Tensor, max_seqlen_q: int,
                     max_seqlen_k: int, scale: Optional[float] = None, causal: bool = False) -> torch.Tensor:
    """Differentiable packed variable-length attention in ``flash_attn_varlen_func``'s argument order: q [total_q, H, D],
    k, v [total_k, H_kv, D] (fp16 or bf16, D in 32, 64, 96, 128, H % H_kv == 0), int32 ``cu_seqlens`` [B + 1] on the
    device.  Returns o from :func:`fa2_fwd_varlen`; its backward is :func:`fa2_bwd_varlen`, which gives the gradients of
    q, k and v."""
    return _AttentionVarlen.apply(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, scale, causal)


def ffpa_fwd(q, k, v, o, scale: Optional[float] = None, variant: int = 0) -> None:
    B, H, N, D = _check_qkvo(q, k, v, o)
    with _DeviceGuard(q):
        rc = _lib.b200k_ffpa_fwd_f16(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), B, H, N, D,
                                     float(scale) if scale else 0.0, variant, _stream(q))
    if rc == L.EHEADDIM:
        raise RuntimeError("headdim not support!")
    L.check(rc)


# ------------------------------------------------------------------------------------------------ support kernels
_ws_cache: dict = {}


def _workspace(dev: torch.device) -> torch.Tensor:
    """Reduction workspace (partials + ticket), one per (device, stream): two streams running reductions concurrently
    on one device must not share partials.  The library zeroes the ticket itself on every call."""
    key = (dev.type, dev.index, torch.cuda.current_stream(dev).cuda_stream)
    ws = _ws_cache.get(key)
    if ws is None:
        ws = torch.empty(int(_lib.b200k_reduce_workspace_bytes()), dtype=torch.uint8, device=dev)
        _ws_cache[key] = ws
    return ws


def elementwise_add(a, b, c) -> None:
    if a.dtype not in (torch.float32, torch.float16, torch.bfloat16):
        raise RuntimeError("values must be torch::kFloat32 or torch::kHalf")
    _check_dtype(b, a.dtype)
    _check_dtype(c, a.dtype)
    if a.numel() != b.numel() or a.numel() != c.numel():
        raise RuntimeError("Tensor size mismatch!")
    _check_cuda_contig(a, b, c)
    with _DeviceGuard(a):
        L.check(_lib.b200k_elementwise_add(a.data_ptr(), b.data_ptr(), c.data_ptr(), a.numel(), _DTYPE_ENUM[a.dtype],
                                           _stream(a)))


def block_all_reduce_sum(x: torch.Tensor, acc_f16: bool = False) -> torch.Tensor:
    """Returns a new 1-element tensor (f32, or i32 for int8 input) like the reference bindings
    (kernels/reduce/block_all_reduce.cu:L734-760)."""
    if x.dtype not in _DTYPE_ENUM or x.dtype == torch.int32:
        raise RuntimeError("values must be a float/half/bfloat16/fp8/int8 tensor")
    _check_cuda_contig(x)
    out = torch.empty(1, dtype=torch.int32 if x.dtype == torch.int8 else torch.float32, device=x.device)
    with _DeviceGuard(x):
        L.check(_lib.b200k_block_all_reduce_sum(x.data_ptr(), out.data_ptr(), x.numel(), _DTYPE_ENUM[x.dtype],
                                                1 if acc_f16 else 0, _workspace(x.device).data_ptr(), _stream(x)))
    return out


SOFTMAX_ALL, SOFTMAX_PER_TOKEN, SOFTMAX_SAFE, SOFTMAX_ONLINE = 0, 1, 2, 3


def softmax(x, y, mode: int) -> None:
    if x.dtype not in (torch.float32, torch.float16):
        raise RuntimeError("values must be torch::kFloat32")
    _check_dtype(y, x.dtype)
    if x.shape != y.shape:
        raise RuntimeError("Tensor size mismatch!")
    _check_cuda_contig(x, y)
    if mode == SOFTMAX_ALL:
        # The total is global in this mode, so the row shape is free: the reference calls softmax_f32 with a flat
        # tensor (softmax.py:L63); fold it into rows of the largest power of two <= 4096 dividing numel so that the
        # normalisation pass runs on the whole grid instead of one CTA.
        n = x.numel()
        if x.dim() >= 2 and x.size(-1) <= 16384:
            S, H = n // x.size(-1), x.size(-1)
        else:
            H = 4096
            while H > 1 and n % H:
                H //= 2
            S, H = (n // H, H) if H >= 32 else (1, n)
    else:
        S, H = x.numel() // x.size(-1), x.size(-1)
    with _DeviceGuard(x):
        L.check(_lib.b200k_softmax(x.data_ptr(), y.data_ptr(), S, H, _DTYPE_ENUM[x.dtype], mode,
                                   _workspace(x.device).data_ptr(), _stream(x)))


def rms_norm(x, y, g: float, eps: float = 1e-5, acc_f16: bool = False, eps_inside_k: bool = False) -> None:
    if x.dtype not in (torch.float32, torch.float16):
        raise RuntimeError("values must be torch::kFloat32")
    _check_dtype(y, x.dtype)
    if x.shape != y.shape or x.dim() != 2:
        raise RuntimeError("Tensor size mismatch!")
    _check_cuda_contig(x, y)
    with _DeviceGuard(x):
        L.check(_lib.b200k_rms_norm(x.data_ptr(), y.data_ptr(), x.size(0), x.size(1), float(g), float(eps),
                                    _DTYPE_ENUM[x.dtype], 1 if acc_f16 else 0, 1 if eps_inside_k else 0, _stream(x)))


def rope_f32(x, out, ref_quirk: bool = True) -> None:
    _check_dtype(x, torch.float32)
    _check_dtype(out, torch.float32)
    if x.shape != out.shape or x.dim() != 2:
        raise RuntimeError("Tensor size mismatch!")
    _check_cuda_contig(x, out)
    with _DeviceGuard(x):
        L.check(_lib.b200k_rope_f32(x.data_ptr(), out.data_ptr(), x.size(0), x.size(1), 1 if ref_quirk else 0,
                                    _stream(x)))


def histogram_i32(a: torch.Tensor, nbins: Optional[int] = None) -> torch.Tensor:
    """Returns int32 counts of length max(a)+1, like the reference (kernels/histogram/histogram.cu:L50-68), which
    also reads max(a) back to the host to size its output."""
    _check_dtype(a, torch.int32)
    _check_cuda_contig(a)
    with _DeviceGuard(a):
        if nbins is None:
            mx = torch.empty(1, dtype=torch.int32, device=a.device)
            L.check(_lib.b200k_max_i32(a.data_ptr(), a.numel(), mx.data_ptr(), _stream(a)))
            nbins = int(mx.item()) + 1
        y = torch.empty(max(nbins, 1), dtype=torch.int32, device=a.device)
        L.check(_lib.b200k_histogram_i32(a.data_ptr(), a.numel(), y.data_ptr(), y.numel(), _stream(a)))
    return y


def embedding(idx, weight, out) -> None:
    _check_dtype(idx, torch.int32)
    if weight.dtype not in (torch.float32, torch.float16, torch.bfloat16):
        raise RuntimeError("values must be torch::kFloat32 or torch::kHalf")
    _check_dtype(out, weight.dtype)
    if weight.dim() != 2 or out.numel() != idx.numel() * weight.size(1):
        raise RuntimeError("Tensor size mismatch!")
    _check_cuda_contig(idx, weight, out)
    with _DeviceGuard(idx):
        L.check(_lib.b200k_embedding(idx.data_ptr(), weight.data_ptr(), out.data_ptr(), idx.numel(), weight.size(0),
                                     weight.size(1), _DTYPE_ENUM[weight.dtype], _stream(idx)))


# ------------------------------------------------------------------------------------------------ support kernels, set 2
ACT_OPS = {"relu": L.ACT_RELU, "sigmoid": L.ACT_SIGMOID, "gelu": L.ACT_GELU, "swish": L.ACT_SWISH, "elu": L.ACT_ELU,
           "hardswish": L.ACT_HARDSWISH, "hardshrink": L.ACT_HARDSHRINK}


def activation(x, y, op: str, ref_clamp: bool = True) -> None:
    """y = op(x) elementwise; f32 or f16.  ``ref_clamp`` keeps the reference's input clamp for sigmoid / gelu
    (kernels/sigmoid/sigmoid.cu:L19-22, kernels/gelu/gelu.cu:L19-22)."""
    if x.dtype not in (torch.float32, torch.float16):
        raise RuntimeError("values must be torch::kFloat32 or torch::kHalf")
    _check_dtype(y, x.dtype)
    if x.numel() != y.numel():
        raise RuntimeError("Tensor size mismatch!")
    _check_cuda_contig(x, y)
    with _DeviceGuard(x):
        L.check(_lib.b200k_activation(x.data_ptr(), y.data_ptr(), x.numel(), _DTYPE_ENUM[x.dtype], ACT_OPS[op],
                                      1 if ref_clamp else 0, _stream(x)))


def layer_norm(x, y, g: float, b: float, eps: float = 1e-5, eps_inside_k: bool = True) -> None:
    """Row-wise layer norm with scalar scale / bias, x[N,K] f32 or f16.  ``eps_inside_k`` = the reference's
    rsqrt(sum/(K + eps)) (kernels/layer-norm/layer_norm.cu:L69)."""
    if x.dtype not in (torch.float32, torch.float16):
        raise RuntimeError("values must be torch::kFloat32 or torch::kHalf")
    _check_dtype(y, x.dtype)
    if x.shape != y.shape or x.dim() != 2:
        raise RuntimeError("Tensor size mismatch!")
    _check_cuda_contig(x, y)
    with _DeviceGuard(x):
        L.check(_lib.b200k_layer_norm(x.data_ptr(), y.data_ptr(), x.size(0), x.size(1), float(g), float(b), float(eps),
                                      _DTYPE_ENUM[x.dtype], 1 if eps_inside_k else 0, _stream(x)))


def dot_prod(a, b) -> torch.Tensor:
    """Returns a new 1-element f32 tensor like the reference bindings (kernels/dot-product/dot_product.cu:L233-283)."""
    if a.dtype not in (torch.float32, torch.float16):
        raise RuntimeError("values must be torch::kFloat32 or torch::kHalf")
    _check_dtype(b, a.dtype)
    if a.numel() != b.numel():
        raise RuntimeError("Tensor size mismatch!")
    _check_cuda_contig(a, b)
    out = torch.empty(1, dtype=torch.float32, device=a.device)
    with _DeviceGuard(a):
        L.check(_lib.b200k_dot_prod(a.data_ptr(), b.data_ptr(), out.data_ptr(), a.numel(), _DTYPE_ENUM[a.dtype],
                                    _workspace(a.device).data_ptr(), _stream(a)))
    return out


def mat_transpose(x, y) -> None:
    """y[N,M] = x[M,N]^T, f32 (kernels/mat-transpose/mat_transpose.cu:L296-339)."""
    _check_dtype(x, torch.float32)
    _check_dtype(y, torch.float32)
    if x.dim() != 2 or y.numel() != x.numel():
        raise RuntimeError("Tensor size mismatch!")
    _check_cuda_contig(x, y)
    with _DeviceGuard(x):
        L.check(_lib.b200k_mat_transpose_f32(x.data_ptr(), y.data_ptr(), x.size(0), x.size(1), _stream(x)))


def transpose_16bit_batched(x: torch.Tensor, y: torch.Tensor) -> None:
    """y[..., N, M] = x[..., M, N]^T for f16 / bf16 tensors (leading dims are the batch); exact."""
    if x.dtype not in (torch.float16, torch.bfloat16):
        raise RuntimeError("values must be torch::kHalf or torch::kBFloat16")
    _check_dtype(y, x.dtype)
    if x.dim() < 2 or y.numel() != x.numel():
        raise RuntimeError("Tensor size mismatch!")
    _check_cuda_contig(x, y)
    M, N = x.size(-2), x.size(-1)
    with _DeviceGuard(x):
        L.check(_lib.b200k_transpose_u16_batched(x.data_ptr(), y.data_ptr(), x.numel() // (M * N), M, N, _stream(x)))


def gemv(a, x, y) -> None:
    """y[M,1] = a[M,K] @ x[K,1], f32 or f16 with f32 accumulation (kernels/sgemv/sgemv.cu:L126-195, hgemv.cu:L130-199)."""
    if a.dtype not in (torch.float32, torch.float16):
        raise RuntimeError("values must be torch::kFloat32 or torch::kHalf")
    _check_dtype(x, a.dtype)
    _check_dtype(y, a.dtype)
    if a.dim() != 2 or x.numel() != a.size(1) or y.numel() != a.size(0):
        raise RuntimeError("Tensor size mismatch!")
    _check_cuda_contig(a, x, y)
    with _DeviceGuard(a):
        L.check(_lib.b200k_gemv(a.data_ptr(), x.data_ptr(), y.data_ptr(), a.size(0), a.size(1), _DTYPE_ENUM[a.dtype],
                                _stream(a)))


def default_scale(D: int) -> float:
    return 1.0 / math.sqrt(D)
