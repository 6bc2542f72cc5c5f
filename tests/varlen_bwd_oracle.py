"""fp64 reference of the packed (variable-length, grouped-query) attention backward, b200k_fa2_bwd_varlen, computed one
sequence at a time: sequence b is tokens [cu_q[b], cu_q[b+1]) of q / o / do ([total_q, H, D]) and [cu_k[b], cu_k[b+1])
of k / v ([total_k, H_kv, D]); query head h reads K/V head h // (H // H_kv); causal is bottom-right (row r sees key j iff
j <= r + Lk - Lq).  K/V heads are expanded with repeat_interleave, and dk / dv summed back over each group.  A row that
sees no key has lse = -inf, o = 0 and gradient 0; tokens outside every sequence have gradient 0.
grads_given takes o and lse as inputs, as the kernels do; grads forms them.  Used by test_attention_varlen_bwd_cpu.py
(against torch autograd and the dense reference) and test_gpu_attention_varlen_bwd.py (against the kernels)."""
from __future__ import annotations

import math
from typing import Optional

import torch


def seqs(cu_q, cu_k):
    """[(q0, q1, k0, k1)] per sequence."""
    cq, ck = [int(x) for x in cu_q], [int(x) for x in cu_k]
    return [(cq[b], cq[b + 1], ck[b], ck[b + 1]) for b in range(len(cq) - 1)]


def visible(Lq: int, Lk: int, causal: bool, device="cpu") -> torch.Tensor:
    """[Lq, Lk] bool: row r sees key j."""
    vis = torch.ones(Lq, Lk, dtype=torch.bool, device=device)
    if causal:
        vis &= torch.arange(Lk, device=device).view(1, Lk) <= torch.arange(Lq, device=device).view(Lq, 1) + Lk - Lq
    return vis


def _scores(q, k, scale, causal):
    """[H, Lq, Lk] masked scores of one sequence, q [Lq, H, D], k [Lk, H, D] (heads already expanded)."""
    s = torch.einsum("qhd,khd->hqk", q, k) * scale
    return s.masked_fill(~visible(q.size(0), k.size(0), causal, q.device), float("-inf"))


def forward(q, k, v, cu_q, cu_k, scale: Optional[float] = None, causal: bool = False):
    """(o [total_q, H, D], lse [total_q, H]) in q's dtype's promotion: differentiable, for torch.autograd and gradcheck.
    Rows that see no key get o = 0 and lse = -inf; tokens outside every sequence get 0 and -inf."""
    total_q, H, D = q.shape
    G = H // k.size(1)
    scale = scale if scale else 1.0 / math.sqrt(D)
    o = torch.zeros_like(q)
    lse = torch.full((total_q, H), float("-inf"), dtype=q.dtype, device=q.device)
    for q0, q1, k0, k1 in seqs(cu_q, cu_k):
        if q1 == q0:
            continue
        kk, vv = (t[k0:k1].repeat_interleave(G, dim=1) for t in (k, v))
        s = _scores(q[q0:q1], kk, scale, causal)                           # [H, Lq, Lk]
        seen = torch.isfinite(s).any(-1, keepdim=True)                     # rows that see a key
        p = torch.softmax(torch.where(seen, s, torch.zeros_like(s)), -1) * seen
        o = o.index_put((torch.arange(q0, q1, device=q.device),), torch.einsum("hqk,khd->qhd", p, vv))
        l = torch.logsumexp(torch.where(seen, s, torch.zeros_like(s)), -1).masked_fill(~seen.squeeze(-1), float("-inf"))
        lse = lse.index_put((torch.arange(q0, q1, device=q.device),), l.transpose(0, 1))
    return o, lse


def grads_given(q, k, v, o, lse, do, cu_q, cu_k, scale: Optional[float] = None, causal: bool = False):
    """(dq, dk, dv) in fp64 from the explicit formulas, with o and lse taken as inputs: P = exp(s - lse) (0 where lse is
    -inf), Delta = rowsum(do o), dS = P (dP - Delta), dq = scale dS k, dk = scale dS^T q, dv = P^T do, dk / dv summed
    over each K/V head's query heads."""
    q, k, v, o, lse, do = (t.double() for t in (q, k, v, o, lse, do))
    total_q, H, D = q.shape
    H_kv = k.size(1)
    G = H // H_kv
    scale = scale if scale else 1.0 / math.sqrt(D)
    dq, dk, dv = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
    for q0, q1, k0, k1 in seqs(cu_q, cu_k):
        Lq, Lk = q1 - q0, k1 - k0
        if Lq == 0 or Lk == 0:
            continue
        kk, vv = (t[k0:k1].repeat_interleave(G, dim=1) for t in (k, v))
        s = _scores(q[q0:q1], kk, scale, causal)
        l = lse[q0:q1].transpose(0, 1).unsqueeze(-1)                       # [H, Lq, 1]
        p = torch.where(torch.isinf(l) & (l < 0), torch.zeros_like(s), torch.exp(s - l))
        delta = (do[q0:q1] * o[q0:q1]).sum(-1).transpose(0, 1).unsqueeze(-1)
        ds = p * (torch.einsum("qhd,khd->hqk", do[q0:q1], vv) - delta)
        dq[q0:q1] = scale * torch.einsum("hqk,khd->qhd", ds, kk)
        dk[k0:k1] = (scale * torch.einsum("hqk,qhd->khd", ds, q[q0:q1])).view(Lk, H_kv, G, D).sum(2)
        dv[k0:k1] = torch.einsum("hqk,qhd->khd", p, do[q0:q1]).view(Lk, H_kv, G, D).sum(2)
    return dq, dk, dv


def grads(q, k, v, do, cu_q, cu_k, scale: Optional[float] = None, causal: bool = False):
    """(dq, dk, dv, o, lse) in fp64, o and lse from forward()."""
    q, k, v, do = (t.double() for t in (q, k, v, do))
    o, lse = forward(q, k, v, cu_q, cu_k, scale, causal)
    return grads_given(q, k, v, o, lse, do, cu_q, cu_k, scale, causal) + (o, lse)
