"""The elements an attention call does not own, used by test_attention_poison_cpu.py and test_gpu_attention_poison.py.

An element is not owned by a call when:
  dense (fa2_fwd / fa2_bwd / ops.attention) with seqlens_k: K and V rows j >= clamp(seqlens_k[b], 1, N) of every head
      of batch b (V stored [D, N]: those columns);
  packed (fa2_fwd_varlen / fa2_bwd_varlen / ops.attention_varlen): Q, O, dO and lse tokens >= cu_seqlens_q[B], K and V
      tokens >= cu_seqlens_k[B]; and, for the outputs of sequence b, every token of every other sequence.
Filling them with NaN, +Inf or -Inf must leave every output bit-identical to the same call with zeros there.

oracle.attention masks scores with -inf and then multiplies by the whole of V, so a NaN or an Inf it should ignore makes
it NaN too: 0 * NaN = NaN in fp64 as in the tensor core.  attention_ref slices each sequence to its owned keys instead
(test_attention_poison_cpu.py proves it unchanged under poison)."""
from __future__ import annotations

import torch

from attention_ref import kv_lens

VALUES = (float("nan"), float("inf"), float("-inf"))
VALUE_IDS = ("nan", "+inf", "-inf")


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
