"""fp64 reference of the dense attention backward (b200k_fa2_bwd), from the explicit formulas the kernels follow:
    s = q k^T * scale, masked (keys >= seqlens_k[b] clamped to [1, N]; causal: key > row), lse = log sum_j exp(s),
    P = exp(s - lse), Delta_i = sum_d dO_id O_id, dP = dO v^T, dS = P (dP - Delta),
    dV = P^T dO, dQ = scale dS k, dK = scale dS^T q.
grads_given takes O and lse as inputs instead of forming them.  Used by test_attention_bwd_cpu.py (against torch.autograd) and test_gpu_attention_bwd.py (against the kernels)."""
from __future__ import annotations

import math
from typing import Optional

import torch


def visible(B: int, N: int, causal: bool, seqlens_k: Optional[torch.Tensor], device="cpu") -> torch.Tensor:
    """[B, 1, N, N] bool: row r of batch b sees key j.  seqlens_k is clamped to [1, N] as the forward does."""
    j = torch.arange(N, device=device)
    if seqlens_k is None:
        n = torch.full((B,), N, device=device)
    else:
        n = seqlens_k.to(device).long().clamp(1, N)
    vis = (j.view(1, 1, 1, N) < n.view(B, 1, 1, 1)).expand(B, 1, N, N)
    if causal:
        vis = vis & (j.view(1, 1, 1, N) <= j.view(1, 1, N, 1))
    return vis


def forward(q, k, v, scale: Optional[float] = None, causal: bool = False, seqlens_k=None):
    """(o, lse) in q's dtype's promotion with fp64: differentiable, for torch.autograd and gradcheck."""
    B, H, N, D = q.shape
    scale = scale if scale else 1.0 / math.sqrt(D)
    s = (q @ k.transpose(-1, -2)) * scale
    s = s.masked_fill(~visible(B, N, causal, seqlens_k, q.device), float("-inf"))
    lse = torch.logsumexp(s, -1)
    return torch.softmax(s, -1) @ v, lse


def grads_given(q, k, v, o, lse, do, scale: Optional[float] = None, causal: bool = False, seqlens_k=None):
    """(dq, dk, dv) in fp64 from the explicit formulas with O and lse taken as inputs, as the kernels take them (they
    need not be the forward of q, k, v): P = exp(s - lse), Delta = rowsum(dO O)."""
    q, k, v, o, lse, do = (t.double() for t in (q, k, v, o, lse, do))
    B, H, N, D = q.shape
    scale = scale if scale else 1.0 / math.sqrt(D)
    vis = visible(B, N, causal, seqlens_k, q.device)
    s = ((q @ k.transpose(-1, -2)) * scale).masked_fill(~vis, float("-inf"))
    p = torch.exp(s - lse.unsqueeze(-1))
    delta = (do * o).sum(-1, keepdim=True)
    ds = p * (do @ v.transpose(-1, -2) - delta)
    return scale * (ds @ k), scale * (ds.transpose(-1, -2) @ q), p.transpose(-1, -2) @ do


def grads(q, k, v, do, scale: Optional[float] = None, causal: bool = False, seqlens_k=None):
    """(dq, dk, dv, o, lse) in fp64 from the explicit formulas."""
    q, k, v, do = (t.double() for t in (q, k, v, do))
    B, H, N, D = q.shape
    scale = scale if scale else 1.0 / math.sqrt(D)
    vis = visible(B, N, causal, seqlens_k, q.device)
    s = ((q @ k.transpose(-1, -2)) * scale).masked_fill(~vis, float("-inf"))
    lse = torch.logsumexp(s, -1)
    o = torch.exp(s - lse.unsqueeze(-1)) @ v
    return grads_given(q, k, v, o, lse, do, scale, causal, seqlens_k) + (o, lse)
