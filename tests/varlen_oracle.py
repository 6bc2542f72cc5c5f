"""CPU reference for packed variable-length attention with grouped-query K/V heads (b200k_fa2_fwd_varlen), used by
test_attention_varlen_cpu.py and test_gpu_attention_varlen.py.  The reference project has no such interface; this is the
textbook definition of flash-attn's flash_attn_varlen_func forward, checked against oracle.attention and per-sequence
scaled_dot_product_attention in test_attention_varlen_cpu.py."""
from __future__ import annotations

import math

import torch


def attention_varlen(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, cu_seqlens_q, cu_seqlens_k,
                     scale: float | None = None, causal: bool = False) -> torch.Tensor:
    """Packed attention in fp32 on the CPU, rounded once to the input dtype.  q [total_q, H, D], k / v [total_k, H_kv, D];
    sequence b is query tokens [cu_q[b], cu_q[b+1]) and key tokens [cu_k[b], cu_k[b+1]).  K/V heads are expanded with
    repeat_interleave (query head h reads K/V head h // (H // H_kv)); `causal` is aligned bottom-right (row r sees keys
    j <= r + Lk - Lq, flash-attn >= 2.1); rows that see no key are 0, and so are tokens outside every sequence."""
    q32, k32, v32 = q.float().cpu(), k.float().cpu(), v.float().cpu()
    H, H_kv, D = q.shape[1], k.shape[1], q.shape[2]
    if scale is None:
        scale = 1.0 / math.sqrt(D)
    cq = torch.as_tensor(cu_seqlens_q).cpu().tolist()
    ck = torch.as_tensor(cu_seqlens_k).cpu().tolist()
    out = torch.zeros(q32.shape)
    for b in range(len(cq) - 1):
        Lq, Lk = cq[b + 1] - cq[b], ck[b + 1] - ck[b]
        qs = q32[cq[b]:cq[b + 1]].transpose(0, 1)                                          # [H, Lq, D]
        ks = k32[ck[b]:ck[b + 1]].transpose(0, 1).repeat_interleave(H // H_kv, dim=0)     # [H, Lk, D]
        vs = v32[ck[b]:ck[b + 1]].transpose(0, 1).repeat_interleave(H // H_kv, dim=0)
        keep = torch.ones(Lq, Lk, dtype=torch.bool)
        if causal:
            keep = torch.arange(Lk).view(1, Lk) <= torch.arange(Lq).view(Lq, 1) + (Lk - Lq)
        s = (qs @ ks.transpose(-1, -2) * scale).masked_fill(~keep, float("-inf"))
        p = torch.softmax(s, dim=-1).masked_fill(~keep.any(dim=-1, keepdim=True), 0.0)   # no visible key: 0, not NaN
        out[cq[b]:cq[b + 1]] = (p @ vs).transpose(0, 1)
    return out.to(q.dtype if q.dtype in (torch.float16, torch.bfloat16) else torch.float16)
