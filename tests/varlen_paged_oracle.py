"""Paged caches for packed attention (ops.fa2_fwd_varlen with block_table), used by test_attention_varlen_paged_cpu.py and
test_gpu_attention_varlen_paged.py: packed K/V scattered into the pages of a shuffled block table, and the gather back
through the table that attention_ref.paged attends over."""
from __future__ import annotations

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
