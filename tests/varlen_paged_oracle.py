"""Paged caches for packed attention (ops.fa2_fwd_varlen with block_table), used by test_attention_varlen_paged_cpu.py and
test_gpu_attention_varlen_paged.py: packed K/V scattered into the pages of a shuffled block table, the gather back through
the table, and a per-sequence fp64 reference that reads keys straight from the pages."""
from __future__ import annotations

import math

import torch

import kvcache_oracle


def lengths(cu_seqlens_k, capacity: int) -> list[int]:
    """Key count of each sequence as the paged call takes it: cu_k[b + 1] - cu_k[b], clamped to [0, capacity]."""
    c = torch.as_tensor(cu_seqlens_k).cpu().tolist()
    return [min(max(c[b + 1] - c[b], 0), capacity) for b in range(len(c) - 1)]


def to_pages(k: torch.Tensor, v: torch.Tensor, cu_seqlens_k, page_size: int, pages_per_seq: int | None = None,
             spare_pages: int = 3, seed: int = 0, fill=None, share: int = 0):
    """(k_cache, v_cache, block_table) on k's device holding packed k / v [total_k, H_kv, D] (sequence b at tokens
    [cu_k[b], cu_k[b + 1])).  Every sequence owns pages_per_seq table entries (default: just enough for the longest) on
    distinct pages in shuffled order, and `spare_pages` pages are listed nowhere.  Slots at or past a sequence's length,
    its unused entries' pages and the spare pages hold `fill` (a scalar) or zeros.  share > 0: sequence 1's first
    `share` entries are sequence 0's pages, so both must start with the same share * page_size keys."""
    lens = torch.as_tensor(cu_seqlens_k).diff().tolist()
    c = torch.as_tensor(cu_seqlens_k).cpu().tolist()
    B, H_kv, D = len(lens), k.size(1), k.size(2)
    pps = pages_per_seq or max(1, max(-(-n // page_size) for n in lens))
    num_pages = B * pps + spare_pages
    g = torch.Generator().manual_seed(seed)
    table = torch.randperm(num_pages, generator=g)[:B * pps].view(B, pps)
    if share:
        table[1, :share] = table[0, :share]
    value = 0.0 if fill is None else fill
    kc = torch.full((num_pages, page_size, H_kv, D), value, dtype=k.dtype, device=k.device)
    vc = torch.full_like(kc, value)
    for b in range(B):
        j = torch.arange(min(lens[b], pps * page_size))
        page, slot = table[b, j // page_size].to(k.device), (j % page_size).to(k.device)
        kc[page, slot] = k[c[b] + j.to(k.device)]
        vc[page, slot] = v[c[b] + j.to(k.device)]
    return kc, vc, table.to(torch.int32).to(k.device)


def gather(k_cache, v_cache, cu_seqlens_k, block_table):
    """Packed K, V (on the CPU) and int32 cu_seqlens_k of the keys the paged call reads: the clamped lengths."""
    cap = block_table.size(1) * k_cache.size(1)
    return kvcache_oracle.gather(k_cache, v_cache, lengths(cu_seqlens_k, cap), block_table)


def attention_pages(q, k_cache, v_cache, cu_seqlens_q, cu_seqlens_k, block_table, scale=None, causal=False):
    """(O [total_q, H, D] fp64, lse [total_q, H] fp64) on the CPU, one sequence at a time, each key read from its page.
    Rows that see no key are 0 with lse -inf; tokens outside every sequence are 0 and -inf."""
    total_q, H, D = q.shape
    ps, H_kv = k_cache.size(1), k_cache.size(2)
    scale = 1.0 / math.sqrt(D) if scale is None else scale
    cq = torch.as_tensor(cu_seqlens_q).cpu().tolist()
    table = torch.as_tensor(block_table).cpu().long()
    lens = lengths(cu_seqlens_k, table.size(1) * ps)
    kc, vc, qd = k_cache.cpu().double(), v_cache.cpu().double(), q.cpu().double()
    out = torch.zeros(total_q, H, D, dtype=torch.float64)
    lse = torch.full((total_q, H), float("-inf"), dtype=torch.float64)
    for b, Lk in enumerate(lens):
        Lq = cq[b + 1] - cq[b]
        for h in range(H):
            hk = h // (H // H_kv)
            keys = torch.stack([kc[table[b, j // ps], j % ps, hk] for j in range(Lk)]) if Lk else torch.zeros(0, D)
            vals = torch.stack([vc[table[b, j // ps], j % ps, hk] for j in range(Lk)]) if Lk else torch.zeros(0, D)
            for r in range(Lq):
                n = min(Lk, r + Lk - Lq + 1) if causal else Lk
                if n <= 0:
                    continue
                s = (keys[:n] @ qd[cq[b] + r, h]) * scale
                lse[cq[b] + r, h] = torch.logsumexp(s, 0)
                out[cq[b] + r, h] = torch.softmax(s, 0) @ vals[:n]
    return out, lse
