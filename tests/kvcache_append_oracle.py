"""CPU reference for KV-cache decode with append and rotary (b200k_fa2_fwd_kvcache_append), used by
test_attention_kvcache_append_cpu.py and test_gpu_attention_kvcache_append.py.  The new rows are rotated in fp64 and
rounded once to the dtype, written into a copy of the cache through the table, and attention_ref.kvcache runs on the
rotated Q with the lengths plus L_new."""
from __future__ import annotations

import torch

import attention_ref


def rotate(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, pos: torch.Tensor, interleaved: bool) -> torch.Tensor:
    """x [B, L, heads, D] with token (b, i) rotated at position pos[b, i] (clamped to the table), in fp64, rounded once
    to x's dtype.  cos / sin [rotary_seqlen, rotary_dim / 2]; pair j is (2j, 2j + 1) when interleaved, else
    (j, j + rotary_dim / 2); pair j at position p becomes (x0 c - x1 s, x0 s + x1 c)."""
    half = cos.size(1)
    rd = 2 * half
    p = pos.cpu().long().clamp(0, cos.size(0) - 1)
    c = cos.cpu().double()[p].unsqueeze(2)   # [B, L, 1, half]
    s = sin.cpu().double()[p].unsqueeze(2)
    xd = x.cpu().double()
    r = xd[..., :rd]
    if interleaved:
        x0, x1 = r[..., 0::2], r[..., 1::2]
    else:
        x0, x1 = r[..., :half], r[..., half:]
    y0, y1 = x0 * c - x1 * s, x0 * s + x1 * c
    out = xd.clone()
    if interleaved:
        out[..., 0:rd:2], out[..., 1:rd:2] = y0, y1
    else:
        out[..., :half], out[..., half:rd] = y0, y1
    out = out.to(x.dtype)
    out[..., rd:] = x.cpu()[..., rd:]   # copied, not rounded through fp64 (the same bits either way for f16 / bf16)
    return out


def bases(cache_seqlens) -> torch.Tensor:
    return torch.as_tensor(cache_seqlens).cpu().long().clamp(min=0)


def write(cache: torch.Tensor, new: torch.Tensor, cache_seqlens, block_table=None) -> torch.Tensor:
    """A copy of `cache` (on the CPU) with new token i of sequence b at position base_b + i, for positions below the
    capacity only.  Without a table the cache is [B, S, H_kv, D]; with one, slot p % page_size of page
    block_table[b, p // page_size]."""
    out = cache.cpu().clone()
    newc = new.cpu()
    base = bases(cache_seqlens)
    ps = out.size(1)
    table = None if block_table is None else torch.as_tensor(block_table).cpu().long()
    cap = ps * (1 if table is None else table.size(1))
    for b in range(newc.size(0)):
        for i in range(newc.size(1)):
            p = int(base[b]) + i
            if p >= cap:
                continue
            if table is None:
                out[b, p] = newc[b, i]
            else:
                out[table[b, p // ps], p % ps] = newc[b, i]
    return out


def attention_append(q, k_cache, v_cache, cache_seqlens, k_new, v_new, block_table=None, rotary_cos=None,
                     rotary_sin=None, rotary_interleaved=True, scale=None, causal=False):
    """(O, K cache, V cache) on the CPU after the call: O [B, Lq, H, D] in q's dtype."""
    B, Lq = q.shape[:2]
    L_new = k_new.size(1)
    base = bases(cache_seqlens)
    if rotary_cos is not None:
        kpos = base.view(B, 1) + torch.arange(L_new).view(1, L_new)
        qpos = base.view(B, 1) + (torch.arange(Lq).view(1, Lq) if causal else torch.zeros(1, Lq, dtype=torch.long))
        k_new = rotate(k_new, rotary_cos, rotary_sin, kpos, rotary_interleaved)
        q = rotate(q, rotary_cos, rotary_sin, qpos, rotary_interleaved)
    kc = write(k_cache, k_new, cache_seqlens, block_table)
    vc = write(v_cache, v_new, cache_seqlens, block_table)
    cap = kc.size(1) * (1 if block_table is None else block_table.size(1))
    lens = (base + L_new).clamp(max=cap).to(torch.int32)
    o = attention_ref.kvcache(q.cpu(), kc, vc, lens, block_table, scale=scale, causal=causal)[0].to(q.dtype)
    return o, kc, vc
