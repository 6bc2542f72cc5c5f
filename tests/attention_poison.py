"""The elements an attention call does not own, and fp64 references that never read them, used by
test_attention_poison_cpu.py and test_gpu_attention_poison.py.

An element is not owned by a call when:
  dense (fa2_fwd / fa2_bwd / ops.attention) with seqlens_k: K and V rows j >= clamp(seqlens_k[b], 1, N) of every head
      of batch b (V stored [D, N]: those columns);
  packed (fa2_fwd_varlen / fa2_bwd_varlen / ops.attention_varlen): Q, O, dO and lse tokens >= cu_seqlens_q[B], K and V
      tokens >= cu_seqlens_k[B]; and, for the outputs of sequence b, every token of every other sequence.
Filling them with NaN, +Inf or -Inf must leave every output bit-identical to the same call with zeros there.

oracle.attention and attn_bwd_oracle mask scores with -inf and then multiply by the whole of V (or K, Q, dO), so a NaN
or an Inf they should ignore makes them NaN too: 0 * NaN = NaN in fp64 as in the tensor core.  The dense references
here slice each batch to its owned keys instead.  The packed ones are varlen_bwd_oracle's, which already slice each
sequence out of the pack (test_attention_poison_cpu.py proves both kinds unchanged under poison)."""
from __future__ import annotations

import math
from typing import Optional

import torch

import varlen_bwd_oracle as vo

VALUES = (float("nan"), float("inf"), float("-inf"))
VALUE_IDS = ("nan", "+inf", "-inf")


def kv_lens(seqlens_k, B: int, N: int) -> list:
    """The dense key count of each batch: seqlens_k clamped to [1, N], N without seqlens_k."""
    if seqlens_k is None:
        return [N] * B
    return [min(max(int(x), 1), N) for x in torch.as_tensor(seqlens_k).cpu().tolist()]


def dense_kv_mask(shape, seqlens_k, v_dn: bool = False) -> torch.Tensor:
    """bool of a dense K or V [B, H, N, D] (v_dn: V [B, H, D, N]): the rows (columns) no row of the batch may read."""
    B = shape[0]
    N = shape[3] if v_dn else shape[2]
    n = torch.tensor(kv_lens(seqlens_k, B, N))
    past = torch.arange(N).view(1, N) >= n.view(B, 1)                                     # [B, N]
    return (past.view(B, 1, 1, N) if v_dn else past.view(B, 1, N, 1)).expand(shape).clone()


def packed_masks(cu_q, cu_k, q_shape, k_shape):
    """(mask of a [total_q, ...] tensor, mask of a [total_k, ...] tensor): the tokens past cu_q[B] / cu_k[B]."""
    return _tokens(int(cu_q[-1]), q_shape), _tokens(int(cu_k[-1]), k_shape)


def sequence_masks(cu_q, cu_k, b: int, q_shape, k_shape):
    """(q-side mask, k-side mask) of every token that is not sequence b's: what b's outputs must never read."""
    cq, ck = [int(x) for x in cu_q], [int(x) for x in cu_k]
    return _outside(cq[b], cq[b + 1], q_shape), _outside(ck[b], ck[b + 1], k_shape)


def _tokens(lo: int, shape) -> torch.Tensor:
    m = torch.zeros(shape, dtype=torch.bool)
    m[lo:] = True
    return m


def _outside(lo: int, hi: int, shape) -> torch.Tensor:
    m = torch.ones(shape, dtype=torch.bool)
    m[lo:hi] = False
    return m


def poison(t: torch.Tensor, mask: torch.Tensor, value: float) -> torch.Tensor:
    """A copy of t with `value` wherever mask is set (mask on the CPU or on t's device)."""
    return t.masked_fill(mask.to(t.device), value)


# ------------------------------------------------------------------------------------------------ dense references
def _dense_scores(q, k, n: int, scale: float, causal: bool):
    """[H, N, n] scores of one batch against its n owned keys; causal: row r sees keys <= r (key 0 always)."""
    s = (q @ k[:, :n].transpose(-1, -2)) * scale
    if causal:
        N = q.size(1)
        s = s.masked_fill(torch.arange(n).view(1, n) > torch.arange(N).view(N, 1), float("-inf"))
    return s


def dense_forward(q, k, v, scale: Optional[float] = None, causal: bool = False, seqlens_k=None):
    """(o [B, H, N, D], lse [B, H, N]) in fp64 from q, k, v [B, H, N, D], reading only each batch's owned keys."""
    q, k, v = (t.double().cpu() for t in (q, k, v))
    B, H, N, D = q.shape
    scale = scale if scale else 1.0 / math.sqrt(D)
    o, lse = torch.zeros_like(q), torch.zeros(B, H, N, dtype=torch.float64)
    for b, n in enumerate(kv_lens(seqlens_k, B, N)):
        s = _dense_scores(q[b], k[b], n, scale, causal)
        lse[b] = torch.logsumexp(s, -1)
        o[b] = torch.exp(s - lse[b].unsqueeze(-1)) @ v[b, :, :n]
    return o, lse


def dense_grads_given(q, k, v, o, lse, do, scale: Optional[float] = None, causal: bool = False, seqlens_k=None):
    """(dq, dk, dv) in fp64 with o and lse as inputs (attn_bwd_oracle.grads_given's formulas), reading only owned keys;
    dk and dv of the keys past the length are 0."""
    q, k, v, o, lse, do = (t.double().cpu() for t in (q, k, v, o, lse, do))
    B, H, N, D = q.shape
    scale = scale if scale else 1.0 / math.sqrt(D)
    dq, dk, dv = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
    for b, n in enumerate(kv_lens(seqlens_k, B, N)):
        p = torch.exp(_dense_scores(q[b], k[b], n, scale, causal) - lse[b].unsqueeze(-1))
        delta = (do[b] * o[b]).sum(-1, keepdim=True)
        ds = p * (do[b] @ v[b, :, :n].transpose(-1, -2) - delta)
        dq[b] = scale * (ds @ k[b, :, :n])
        dk[b, :, :n] = scale * (ds.transpose(-1, -2) @ q[b])
        dv[b, :, :n] = p.transpose(-1, -2) @ do[b]
    return dq, dk, dv


def dense_grads(q, k, v, do, scale: Optional[float] = None, causal: bool = False, seqlens_k=None):
    """(dq, dk, dv, o, lse) in fp64, o and lse from dense_forward."""
    o, lse = dense_forward(q, k, v, scale, causal, seqlens_k)
    return dense_grads_given(q, k, v, o, lse, do, scale, causal, seqlens_k) + (o, lse)


# ------------------------------------------------------------------------------------------------ packed references
def packed_forward(q, k, v, cu_q, cu_k, scale: Optional[float] = None, causal: bool = False):
    """(o, lse) in fp64 of packed sequences, one sequence sliced out at a time; tokens outside every sequence get 0 and
    -inf."""
    q, k, v = (t.double().cpu() for t in (q, k, v))
    return vo.forward(q, k, v, torch.as_tensor(cu_q).cpu(), torch.as_tensor(cu_k).cpu(), scale, causal)


def packed_grads(q, k, v, do, cu_q, cu_k, scale: Optional[float] = None, causal: bool = False):
    """(dq, dk, dv, o, lse) in fp64, one sequence sliced out at a time; tokens outside every sequence get 0."""
    q, k, v, do = (t.double().cpu() for t in (q, k, v, do))
    return vo.grads(q, k, v, do, torch.as_tensor(cu_q).cpu(), torch.as_tensor(cu_k).cpu(), scale, causal)
