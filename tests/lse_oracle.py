"""fp64 reference for the softmax log-sum-exp of the attention calls (the ``lse=`` outputs of ops.fa2_fwd,
fa2_fwd_varlen and fa2_fwd_kvcache) and for merging partial attentions by it (ops.attn_merge).  Used by
test_attention_lse_cpu.py, which checks it against torch.logsumexp, and test_gpu_attention_lse.py.

lse[row] = ln sum_j exp(scale * q_row . k_j) over exactly the keys the row sees, -inf for a row that sees none.  The
layouts are O's without its last dim: dense [B, H, N], packed [total_q, H], decode [B, Lq, H]."""
from __future__ import annotations

import math

import numpy as np
import torch

import graded_attention
import kvcache_oracle


def lse_varlen(q, k, cu_seqlens_q, cu_seqlens_k, scale=None, causal=False) -> torch.Tensor:
    """fp64 [total_q, H] on the CPU for packed sequences (the rules of varlen_oracle.attention_varlen).  Tokens outside
    every sequence are NaN: no lse is defined, and none is written there."""
    q64, k64 = q.double().cpu(), k.double().cpu()
    H, H_kv, D = q.shape[1], k.shape[1], q.shape[2]
    scale = 1.0 / math.sqrt(D) if scale is None else scale
    cq = torch.as_tensor(cu_seqlens_q).cpu().tolist()
    ck = torch.as_tensor(cu_seqlens_k).cpu().tolist()
    out = torch.full(q.shape[:2], float("nan"), dtype=torch.float64)
    for b in range(len(cq) - 1):
        Lq, Lk = cq[b + 1] - cq[b], ck[b + 1] - ck[b]
        qs = q64[cq[b]:cq[b + 1]].transpose(0, 1)                                          # [H, Lq, D]
        ks = k64[ck[b]:ck[b + 1]].transpose(0, 1).repeat_interleave(H // H_kv, dim=0)     # [H, Lk, D]
        keep = torch.ones(Lq, Lk, dtype=torch.bool)
        if causal:
            keep = torch.arange(Lk).view(1, Lk) <= torch.arange(Lq).view(Lq, 1) + (Lk - Lq)
        s = (qs @ ks.transpose(-1, -2) * scale).masked_fill(~keep, float("-inf"))
        out[cq[b]:cq[b + 1]] = torch.logsumexp(s, dim=-1).transpose(0, 1) if Lk else float("-inf")
    return out


def lse_dense(q, k, scale=None, causal=False, seqlens_k=None) -> torch.Tensor:
    """fp64 [B, H, N] for [B, H, N, D] inputs: row r of batch b sees keys j < seqlens_k[b] (all N without) and, causal,
    j <= r."""
    B, H, N, D = q.shape
    scale = 1.0 / math.sqrt(D) if scale is None else scale
    s = (q.double().cpu() @ k.double().cpu().transpose(-1, -2)) * scale                  # [B, H, N, N]
    j = torch.arange(N)
    keep = torch.ones(B, 1, N, N, dtype=torch.bool)
    if seqlens_k is not None:
        keep = keep & (j.view(1, 1, 1, N) < torch.as_tensor(seqlens_k).cpu().view(B, 1, 1, 1))
    if causal:
        keep = keep & (j.view(1, 1, 1, N) <= j.view(1, 1, N, 1))
    return torch.logsumexp(s.masked_fill(~keep, float("-inf")), dim=-1)


def lse_kvcache(q, k_cache, v_cache, cache_seqlens, block_table=None, scale=None, causal=False) -> torch.Tensor:
    """fp64 [B, Lq, H] for KV-cache decode (the rules of kvcache_oracle.attention_kvcache)."""
    B, Lq, H, D = q.shape
    k, _, cu_k = kvcache_oracle.gather(k_cache, v_cache, cache_seqlens, block_table)
    cu_q = torch.arange(B + 1, dtype=torch.int32) * Lq
    return lse_varlen(q.cpu().reshape(B * Lq, H, D), k, cu_q, cu_k, scale=scale, causal=causal).view(B, Lq, H)


def merge(o_parts, lse_parts):
    """(O, lse) in fp64 from S partial attentions over disjoint key sets: o_parts [S, ..., D], lse_parts [S, ...] natural
    log.  Parts with lse = -inf weigh nothing, whatever their O holds; a row with no part left is 0 / -inf."""
    o64, l64 = o_parts.double().cpu(), lse_parts.double().cpu()
    lse = torch.logsumexp(l64, dim=0)
    w = torch.exp(l64 - torch.where(torch.isinf(lse), torch.zeros_like(lse), lse))          # [S, ...]
    live = torch.isfinite(l64).unsqueeze(-1)
    o = torch.where(live, w.unsqueeze(-1) * o64, torch.zeros_like(o64)).sum(0)
    return o, lse


def emulate_lse(s, n, scale_log2, dtype, bn, splits=1):
    """The lse the kernel forms, through the fp32 loop of graded_attention.emulate(): s [R, L] raw scores, row r sees
    keys [0, n[r]), tiles of bn keys, `splits` contiguous tile ranges.  Per split the running max m (base 2) and the row
    sum l of P rounded to dtype give (m + log2 l) * fp32(ln 2); several splits are merged as attn_combine_kernel merges
    them, (mx + log2 den) * fp32(ln 2) with den = sum of ex2(lse_s - mx) flushed below 2^-126.  -inf for a row that sees
    no key.  Returns fp32 [R]."""
    f = np.float32
    ln2 = f(graded_attention.LN2_F32)
    s, sl, n = np.asarray(s, f), f(scale_log2), np.asarray(n)
    R, L = s.shape
    nt = -(-L // bn)
    parts = []
    with np.errstate(all="ignore"):
        for sp in range(splits):
            m, l = np.full(R, -np.inf, f), np.zeros(R, f)
            for t in range(sp * nt // splits, (sp + 1) * nt // splits):
                j = np.arange(t * bn, min(L, (t + 1) * bn))
                x = np.where(j[None] < n[:, None], s[:, j], f(-np.inf))
                m_new = np.maximum(m, x.max(1) * sl)
                mu = np.where(m_new == -np.inf, f(0), m_new)
                alpha = np.where(m == -np.inf, f(0), np.exp2(m - mu))
                m, l = m_new, l * alpha
                p = np.exp2((x.astype(np.float64) * np.float64(sl) - mu[:, None]).astype(f))
                p[p < f(2.0 ** -126)] = 0                             # ex2.approx.ftz
                l = l + graded_attention.round_to(p, dtype).sum(1, dtype=f)
            parts.append(np.where(l > 0, m + np.log2(l), f(-np.inf)).astype(f))
        if splits == 1:
            return (parts[0] * ln2).astype(f)
        mx = np.stack(parts).max(0)
        den = np.zeros(R, f)
        for ls in parts:
            w = np.where(mx == -np.inf, f(0), np.exp2(ls - mx)).astype(f)
            w[w < f(2.0 ** -126)] = 0
            den = den + w
        return np.where(den > 0, (mx + np.log2(den)) * ln2, f(-np.inf)).astype(f)
