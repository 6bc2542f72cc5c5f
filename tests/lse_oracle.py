"""Merging partial attentions by their log-sum-exp (ops.attn_merge) in fp64, and the lse the kernel forms in its fp32
loop.  Used by test_attention_lse_cpu.py and test_gpu_attention_lse.py; the fp64 lse of each layout is attention_ref's.

lse[row] = ln sum_j exp(scale * q_row . k_j) over exactly the keys the row sees, -inf for a row that sees none.  The
layouts are O's without its last dim: dense [B, H, N], packed [total_q, H], decode [B, Lq, H]."""
from __future__ import annotations

import numpy as np
import torch

import graded_attention


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
