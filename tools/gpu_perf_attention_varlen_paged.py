"""Packed attention over paged caches (ops.fa2_fwd_varlen with block_table) against the calls a serving engine makes
without it, one JSON line per case.  fp16, H = 32, H_kv = 8, D = 128, causal.  CUDA-event time per call after warm-up;
the calls of a case alternate within this process, `iters` calls per turn, and each is reported as the median and
min - max over the rounds.  Every line carries the GPU's name and power limit, read in the same run.

  1. mixed prompts: 64 sequences, seeded lengths uniform in [128, 8192], Lq = Lk, in caches of page_size 16, 64, 256
  2. chunked prefill: B = 8 sequences of Lq = 1024 new queries against Lk = 8K or 32K keys each, the queries aligned
     bottom-right (query t sees keys <= t + Lk - 1024), so every chunk reads its whole cached context
Comparators: `contiguous`, ops.fa2_fwd_varlen on K / V already packed contiguously (the floor); `gather`, a torch
gather of every sequence's keys through the table followed by that call (today's path); in case 2 also `kvcache`,
ops.fa2_fwd_kvcache with Lq = 1024 on the same pages.  `paged` is the call measured.  TFLOP/s count only useful
work, 4 * H * D per visible (query row, key) pair, as gpu_perf_attention_varlen.py does.

    python tools/gpu_perf_attention_varlen_paged.py [--iters 5] [--rounds 7]
"""
import argparse
import json

import numpy as np
import torch
from gpu_timing import gpu_info, stats, time_rounds, visible_pairs
from b200k import ops

H, H_KV, D = 32, 8, 128
PAGE_SIZES = (16, 64, 256)


def paged_cache(k, v, lens, page_size, seed):
    """Caches [num_pages, page_size, H_kv, D] holding packed k / v under a shuffled table [B, pages_per_seq], 8 spare
    pages, the slots past each length NaN."""
    B = len(lens)
    pps = int(max(-(-n // page_size) for n in lens))
    num_pages = B * pps + 8
    table = torch.randperm(num_pages, generator=torch.Generator().manual_seed(seed))[:B * pps].view(B, pps)
    table = table.to(torch.int32).cuda()
    rows = cache_rows(table, lens, page_size)
    kc = torch.full((num_pages * page_size, H_KV, D), float("nan"), dtype=k.dtype, device="cuda")
    vc = torch.full_like(kc, float("nan"))
    kc[rows], vc[rows] = k, v
    return kc.view(num_pages, page_size, H_KV, D), vc.view(num_pages, page_size, H_KV, D), table


def cache_rows(table, lens, page_size):
    """Cache row of every key, in packed order: the index a torch gather through the table uses."""
    out = []
    for b, n in enumerate(lens):
        j = torch.arange(int(n), device="cuda")
        out.append(table[b, j // page_size].long() * page_size + j % page_size)
    return torch.cat(out)


def line(info, case, t, useful, **kw):
    out = dict(case=case, **kw)
    for name, (med, lo, hi) in t.items():
        out[name + "_ms"] = round(med * 1e3, 3)
        out[name + "_ms_min_max"] = [round(lo * 1e3, 3), round(hi * 1e3, 3)]
        out[name + "_useful_tflops"] = round(useful / med * 1e-12, 1)
    for name in t:
        if name != "paged":
            out["paged_speed_vs_" + name] = round(t[name][0] / t["paged"][0], 3)
    print(json.dumps(dict(out, **info)), flush=True)


def run_case(info, args, case, lq, lk, seed, with_kvcache=False):
    torch.manual_seed(seed)
    cq = torch.tensor(np.concatenate([[0], np.cumsum(lq)]), dtype=torch.int32, device="cuda")
    ck = torch.tensor(np.concatenate([[0], np.cumsum(lk)]), dtype=torch.int32, device="cuda")
    q = torch.randn(int(sum(lq)), H, D, dtype=torch.half, device="cuda")
    k, v = [torch.randn(int(sum(lk)), H_KV, D, dtype=torch.half, device="cuda") for _ in range(2)]
    o, o_ref = torch.empty_like(q), torch.empty_like(q)
    max_q = int(max(lq))
    useful = 4 * H * D * sum(visible_pairs(a, b, True) for a, b in zip(lq, lk))
    for ps in PAGE_SIZES:
        kc, vc, table = paged_cache(k, v, lk, ps, seed)
        rows = cache_rows(table, lk, ps)
        flat_k, flat_v = kc.view(-1, H_KV, D), vc.view(-1, H_KV, D)

        def gather():
            ops.fa2_fwd_varlen(q, flat_k.index_select(0, rows), flat_v.index_select(0, rows), o_ref, cq, ck, max_q,
                               causal=True)

        fns = {
            "contiguous": lambda: ops.fa2_fwd_varlen(q, k, v, o_ref, cq, ck, max_q, causal=True),
            "gather": gather,
            "paged": lambda: ops.fa2_fwd_varlen(q, kc, vc, o, cq, ck, max_q, causal=True, block_table=table),
        }
        if with_kvcache:
            B, Lq = len(lq), int(lq[0])
            q4, o4 = q.view(B, Lq, H, D), torch.empty(B, Lq, H, D, dtype=torch.half, device="cuda")
            lens = torch.tensor(lk, dtype=torch.int32, device="cuda")
            fns["kvcache"] = lambda: ops.fa2_fwd_kvcache(q4, kc, vc, o4, lens, table, causal=True)
        t = {name: stats(ts) for name, ts in time_rounds(fns, args.iters, args.rounds).items()}
        ops.fa2_fwd_varlen(q, k, v, o_ref, cq, ck, max_q, causal=True)
        ops.fa2_fwd_varlen(q, kc, vc, o, cq, ck, max_q, causal=True, block_table=table)
        line(info, case, t, useful, page_size=ps, B=len(lq), total_q=int(sum(lq)), total_k=int(sum(lk)), H=H,
             H_kv=H_KV, D=D, causal=True, same_bits_as_contiguous=bool(torch.equal(o, o_ref)))
        del kc, vc, table, rows, flat_k, flat_v, fns
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    info = gpu_info(torch)
    lens = np.random.RandomState(2024).randint(128, 8192 + 1, size=64)
    run_case(info, args, "1_mixed_prompts", lens, lens, seed=1)
    for cached in (8192, 32768):
        run_case(info, args, "2_chunked_prefill_%dk" % (cached // 1024), [1024] * 8, [cached] * 8, seed=2,
                 with_kvcache=True)


if __name__ == "__main__":
    main()
