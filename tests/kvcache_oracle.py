"""KV caches for decode attention (b200k_fa2_fwd_kvcache): each sequence's keys gathered from the cache through its block
table into packed K/V with cu_seqlens (attention_ref.kvcache attends over them), and a contiguous cache copied into the
pages of a shuffled table."""
from __future__ import annotations

import torch


def gather(k_cache: torch.Tensor, v_cache: torch.Tensor, cache_seqlens, block_table=None):
    """Packed K, V [sum Lk_b, H_kv, D] (on the CPU) and int32 cu_seqlens_k [B + 1].  Without a table the caches are
    [B, S, H_kv, D]; with one they are [num_pages, page_size, H_kv, D] and key j of sequence b is slot j % page_size of
    page block_table[b, j // page_size]."""
    lens = torch.as_tensor(cache_seqlens).cpu().tolist()
    kc, vc = k_cache.cpu(), v_cache.cpu()
    table = None if block_table is None else torch.as_tensor(block_table).cpu().long()
    ks, vs = [], []
    for b, n in enumerate(lens):
        if table is None:
            ks.append(kc[b, :n])
            vs.append(vc[b, :n])
        else:
            j = torch.arange(n)
            page, slot = table[b, j // kc.size(1)], j % kc.size(1)
            ks.append(kc[page, slot])
            vs.append(vc[page, slot])
    cu = torch.tensor([0] + torch.tensor(lens, dtype=torch.int64).cumsum(0).tolist(), dtype=torch.int32)
    return torch.cat(ks), torch.cat(vs), cu


def paged_copy(k_cache: torch.Tensor, v_cache: torch.Tensor, page_size: int, spare_pages: int = 3, seed: int = 0,
               fill=None):
    """The contiguous caches [B, S, H_kv, D] (S a multiple of page_size) as [num_pages, page_size, H_kv, D] caches under
    a shuffled, non-monotonic block table [B, S / page_size], with `spare_pages` pages no table lists.  Unlisted pages
    hold `fill` (a callable giving a tensor of the page shape) or zeros."""
    B, S, H_kv, D = k_cache.shape
    assert S % page_size == 0
    pps = S // page_size
    num_pages = B * pps + spare_pages
    g = torch.Generator().manual_seed(seed)
    perm = torch.randperm(num_pages, generator=g)
    table = perm[:B * pps].view(B, pps).to(torch.int32)
    spare = perm[B * pps:]
    out = []
    for c in (k_cache, v_cache):
        p = torch.zeros(num_pages, page_size, H_kv, D, dtype=c.dtype, device=c.device)
        p[table.view(-1).long().to(c.device)] = c.reshape(B * pps, page_size, H_kv, D)
        if fill is not None:
            for s in spare.tolist():
                p[s] = fill(p[s].shape).to(c.dtype)
        out.append(p)
    return out[0], out[1], table.to(k_cache.device), spare
