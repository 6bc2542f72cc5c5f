"""The reference for every attention call of the library, forward and backward, in fp64 by default.

One function, `sequence`, computes attention of one sequence under one visibility rule: q [Lq, H, D] against
k, v [Lk, H_kv, D], query head h reading K/V head h // (H // H_kv), row r seeing key j iff diag is None or
j <= r + diag.  A row that sees no key has o = 0 and lse = -inf.  `sequence_grads_given` states the backward's formulas
with o and lse as inputs, as the kernels take them.

Each layout only decides which keys a sequence owns and where its diagonal lies:
  dense [B, H, N, D]: keys [0, clamp(seqlens_k[b], 1, N)) of batch b; causal is top-left (diag = 0);
  packed [total, H, D]: sequence b is query tokens [cu_q[b], cu_q[b+1]) and key tokens [cu_k[b], cu_k[b+1]); causal is
      bottom-right (diag = Lk - Lq); tokens outside every sequence have o = 0, lse = -inf and gradient 0;
  kvcache and paged: the keys gathered from the cache through the block table, then packed.
Every layout slices each sequence's owned keys out before it computes, so NaN or Inf in an element a call does not own
never reaches its result.  Used by every attention test, and checked against torch in test_attention_ref_cpu.py."""
from __future__ import annotations

import math

import torch

import kvcache_oracle
import varlen_paged_oracle

# the GPU attention tests' tolerance against this reference, per output dtype
TOL = {torch.float16: dict(rtol=1e-2, atol=1e-3), torch.bfloat16: dict(rtol=2e-2, atol=4e-3)}


def cu(lens, device="cpu") -> torch.Tensor:
    """int32 cu_seqlens [len(lens) + 1] of the sequence lengths `lens`."""
    return torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=device)


def seqs(cu_q, cu_k) -> list:
    """[(q0, q1, k0, k1)] per sequence."""
    cq, ck = torch.as_tensor(cu_q).tolist(), torch.as_tensor(cu_k).tolist()
    return [(cq[b], cq[b + 1], ck[b], ck[b + 1]) for b in range(len(cq) - 1)]


def kv_lens(seqlens_k, B: int, N: int) -> list:
    """The dense key count of each batch: seqlens_k clamped to [1, N], N without seqlens_k."""
    if seqlens_k is None:
        return [N] * B
    return [min(max(int(x), 1), N) for x in torch.as_tensor(seqlens_k).cpu().tolist()]


def visible(Lq: int, Lk: int, diag=None, device="cpu") -> torch.Tensor:
    """[Lq, Lk] bool: row r sees key j."""
    vis = torch.ones(Lq, Lk, dtype=torch.bool, device=device)
    if diag is not None:
        vis &= torch.arange(Lk, device=device).view(1, Lk) <= torch.arange(Lq, device=device).view(Lq, 1) + diag
    return vis


def _scores(q, k, scale, diag):
    """[H, Lq, Lk] scores of one sequence, -inf where a row does not see a key (k's heads already expanded)."""
    s = torch.einsum("qhd,khd->hqk", q, k) * scale
    return s.masked_fill(~visible(q.size(0), k.size(0), diag, q.device), float("-inf"))


def _scale(scale, D):
    return scale if scale else 1.0 / math.sqrt(D)


# ------------------------------------------------------------------------------------------------ one sequence
def sequence(q, k, v, scale, diag=None, dtype=torch.float64):
    """(o [Lq, H, D], lse [Lq, H]) computed in `dtype` on the inputs' device; differentiable (out-of-place only), for
    torch.autograd and gradcheck."""
    q, k, v = (t.to(dtype) for t in (q, k, v))
    Lq, Lk, G = q.size(0), k.size(0), q.size(1) // k.size(1)
    kk, vv = (t.repeat_interleave(G, dim=1) for t in (k, v))
    s = _scores(q, kk, scale, diag)
    seen = visible(Lq, Lk, diag, q.device).any(-1).view(1, Lq, 1)
    s = torch.where(seen, s, torch.zeros_like(s))                          # no NaN from a row that sees no key
    o = torch.einsum("hqk,khd->qhd", torch.softmax(s, -1) * seen, vv)
    lse = torch.logsumexp(s, -1).masked_fill(~seen.view(1, Lq), float("-inf"))
    return o, lse.transpose(0, 1)


def sequence_grads_given(q, k, v, o, lse, do, scale, diag=None):
    """(dq, dk, dv) of one sequence in fp64 from the explicit formulas, with o and lse taken as inputs (they need not be
    the forward of q, k, v): P = exp(s - lse) (0 where lse = -inf), Delta = rowsum(dO O), dP = dO V^T,
    dS = P (dP - Delta), dq = scale dS K, dk = scale dS^T Q, dv = P^T dO; dk and dv summed over each K/V head's group."""
    q, k, v, o, lse, do = (t.double() for t in (q, k, v, o, lse, do))
    Lq, H, D = q.shape
    Lk, H_kv = k.size(0), k.size(1)
    G = H // H_kv
    kk, vv = (t.repeat_interleave(G, dim=1) for t in (k, v))
    s = _scores(q, kk, scale, diag)
    lse = lse.transpose(0, 1).unsqueeze(-1)                                 # [H, Lq, 1]
    p = torch.where(torch.isinf(lse) & (lse < 0), torch.zeros_like(s), torch.exp(s - lse))
    delta = (do * o).sum(-1).transpose(0, 1).unsqueeze(-1)
    ds = p * (torch.einsum("qhd,khd->hqk", do, vv) - delta)
    dq = scale * torch.einsum("hqk,khd->qhd", ds, kk)
    dk = (scale * torch.einsum("hqk,qhd->khd", ds, q)).view(Lk, H_kv, G, D).sum(2)
    dv = torch.einsum("hqk,qhd->khd", p, do).view(Lk, H_kv, G, D).sum(2)
    return dq, dk, dv


# ------------------------------------------------------------------------------------------------ dense [B, H, N, D]
def dense(q, k, v, scale=None, causal=False, seqlens_k=None, dtype=torch.float64):
    """(o [B, H, N, D], lse [B, H, N]) in `dtype`, differentiable."""
    B, H, N, D = q.shape
    t = [sequence(q[b].transpose(0, 1), k[b, :, :n].transpose(0, 1), v[b, :, :n].transpose(0, 1), _scale(scale, D),
                  0 if causal else None, dtype) for b, n in enumerate(kv_lens(seqlens_k, B, N))]
    return torch.stack([o.transpose(0, 1) for o, _ in t]), torch.stack([lse.transpose(0, 1) for _, lse in t])


def dense_grads_given(q, k, v, o, lse, do, scale=None, causal=False, seqlens_k=None):
    """(dq, dk, dv) in fp64 with o and lse as inputs; dk and dv of the keys past the length are 0."""
    B, H, N, D = q.shape
    dq, dk, dv = (torch.zeros(t.shape, dtype=torch.float64, device=t.device) for t in (q, k, v))
    for b, n in enumerate(kv_lens(seqlens_k, B, N)):
        g = sequence_grads_given(*(t.transpose(0, 1) for t in (q[b], k[b, :, :n], v[b, :, :n], o[b], lse[b], do[b])),
                                 _scale(scale, D), 0 if causal else None)
        dq[b], dk[b, :, :n], dv[b, :, :n] = (x.transpose(0, 1) for x in g)
    return dq, dk, dv


def dense_grads(q, k, v, do, scale=None, causal=False, seqlens_k=None):
    """(dq, dk, dv, o, lse) in fp64, o and lse from dense()."""
    o, lse = dense(q, k, v, scale, causal, seqlens_k)
    return dense_grads_given(q, k, v, o, lse, do, scale, causal, seqlens_k) + (o, lse)


# ------------------------------------------------------------------------------------------------ packed [total, H, D]
def packed(q, k, v, cu_q, cu_k, scale=None, causal=False, dtype=torch.float64):
    """(o [total_q, H, D], lse [total_q, H]) in `dtype`, differentiable."""
    total_q, H, D = q.shape
    o = torch.zeros(q.shape, dtype=dtype, device=q.device)
    lse = torch.full((total_q, H), float("-inf"), dtype=dtype, device=q.device)
    for q0, q1, k0, k1 in seqs(cu_q, cu_k):
        if q1 > q0:
            os_, ls = sequence(q[q0:q1], k[k0:k1], v[k0:k1], _scale(scale, D), k1 - k0 - (q1 - q0) if causal else None,
                               dtype)
            rows = (torch.arange(q0, q1, device=q.device),)
            o, lse = o.index_put(rows, os_), lse.index_put(rows, ls)
    return o, lse


def packed_grads_given(q, k, v, o, lse, do, cu_q, cu_k, scale=None, causal=False):
    """(dq, dk, dv) in fp64 with o and lse as inputs; tokens outside every sequence get 0."""
    dq, dk, dv = (torch.zeros(t.shape, dtype=torch.float64, device=t.device) for t in (q, k, v))
    for q0, q1, k0, k1 in seqs(cu_q, cu_k):
        if q1 > q0 and k1 > k0:
            dq[q0:q1], dk[k0:k1], dv[k0:k1] = sequence_grads_given(
                q[q0:q1], k[k0:k1], v[k0:k1], o[q0:q1], lse[q0:q1], do[q0:q1], _scale(scale, q.size(2)),
                k1 - k0 - (q1 - q0) if causal else None)
    return dq, dk, dv


def packed_grads(q, k, v, do, cu_q, cu_k, scale=None, causal=False):
    """(dq, dk, dv, o, lse) in fp64, o and lse from packed()."""
    o, lse = packed(q, k, v, cu_q, cu_k, scale, causal)
    return packed_grads_given(q, k, v, o, lse, do, cu_q, cu_k, scale, causal) + (o, lse)


# ------------------------------------------------------------------------------------------------ caches
def kvcache(q, k_cache, v_cache, cache_seqlens, block_table=None, scale=None, causal=False, dtype=torch.float64):
    """(o [B, Lq, H, D], lse [B, Lq, H]) on the CPU: Q [B, Lq, H, D] as B packed sequences of Lq tokens over the keys
    kvcache_oracle.gather reads from the cache."""
    B, Lq, H, D = q.shape
    k, v, cu_k = kvcache_oracle.gather(k_cache, v_cache, cache_seqlens, block_table)
    o, lse = packed(q.cpu().reshape(B * Lq, H, D), k, v, torch.arange(B + 1) * Lq, cu_k, scale, causal, dtype)
    return o.view(B, Lq, H, D), lse.view(B, Lq, H)


def paged(q, k_cache, v_cache, cu_q, cu_k, block_table, scale=None, causal=False, dtype=torch.float64):
    """(o [total_q, H, D], lse [total_q, H]) on the CPU over the keys varlen_paged_oracle.gather reads through the table
    (each length clamped to the table's capacity)."""
    k, v, cu_kg = varlen_paged_oracle.gather(k_cache, v_cache, cu_k, block_table)
    return packed(q.cpu(), k, v, cu_q, cu_kg, scale, causal, dtype)
