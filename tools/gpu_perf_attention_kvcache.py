"""KV-cache decode attention (ops.fa2_fwd_kvcache) against the calls a caller makes without it, one JSON line per case.
D = 128, fp16.  Each call is captured `--iters` times into one CUDA graph, so the time is GPU time without the Python
launch cost of a call that takes microseconds; the graphs of a case alternate within this process for `--rounds` rounds,
and each call reports the median and the min - max of its per-call time over the rounds.  Every line carries the GPU's
name and power limit, read in the same run.

Comparators: ops.fa2_fwd_varlen on the same tokens, packed beforehand (what a caller runs today: one query row per
sequence and head; the packing is not timed), and F.scaled_dot_product_attention(enable_gqa=True) with fused backends
only, where every length equals the capacity and the call is not causal (SDPA's is_causal aligns top-left).

Metric: the bytes the problem must move, sum_b Lk_b * H_kv * D * 2 (K and V) * 2 bytes plus Q and O, over the call's
time, as GB/s and as a fraction of the H100 SXM data-sheet 3.35 TB/s.  It is a whole-call figure (both kernels of a
split call), not a kernel's share of peak.

    python tools/gpu_perf_attention_kvcache.py [--iters 20] [--rounds 7]
"""
import argparse
import json

import numpy as np
import torch
import torch.nn.functional as F
from gpu_timing import gpu_info, stats, time_rounds
from b200k import ops

PEAK_BYTES_PER_S = 3.35e12
D = 128


def splits_of(B, Lq, H, H_kv, cap):
    ws = ops.fa2_fwd_kvcache_workspace_bytes(B, Lq, H, H_kv, D, cap)
    return 1 if ws == 0 else ws // (B * Lq * H * (D + 1) * 4)


def run_case(info, args, name, B, Lq, H, H_kv, lens, cap, causal=False, page_sizes=(), seed=0):
    torch.manual_seed(seed)
    q = torch.randn(B, Lq, H, D, dtype=torch.half, device="cuda")
    kc, vc = [torch.randn(B, cap, H_kv, D, dtype=torch.half, device="cuda") for _ in range(2)]
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    o = torch.empty_like(q)
    fns = {"kvcache": lambda: ops.fa2_fwd_kvcache(q, kc, vc, o, sl, causal=causal)}
    paged = {}
    for ps in page_sizes:
        pps = cap // ps
        perm = torch.randperm(B * pps, device="cuda")
        table = perm.to(torch.int32).view(B, pps)
        kp, vp = [torch.empty(B * pps, ps, H_kv, D, dtype=torch.half, device="cuda") for _ in range(2)]
        kp[perm] = kc.view(B * pps, ps, H_kv, D)
        vp[perm] = vc.view(B * pps, ps, H_kv, D)
        op = torch.empty_like(q)
        paged[ps] = (kp, vp, table, op)
        fns["paged%d" % ps] = (lambda kp=kp, vp=vp, table=table, op=op:
                               ops.fa2_fwd_kvcache(q, kp, vp, op, sl, table, causal=causal))
    # what callers run today: the same tokens packed for fa2_fwd_varlen (packing not timed)
    pk = torch.cat([kc[b, :n] for b, n in enumerate(lens)])
    pv = torch.cat([vc[b, :n] for b, n in enumerate(lens)])
    cu_k = torch.tensor([0] + np.cumsum(lens).tolist(), dtype=torch.int32, device="cuda")
    cu_q = torch.arange(B + 1, dtype=torch.int32, device="cuda") * Lq
    pq, ov = q.view(B * Lq, H, D), torch.empty(B * Lq, H, D, dtype=torch.half, device="cuda")
    fns["varlen"] = lambda: ops.fa2_fwd_varlen(pq, pk, pv, ov, cu_q, cu_k, Lq, causal=causal)
    sdpa_note = None
    if all(n == cap for n in lens) and not causal:
        from torch.nn.attention import SDPBackend, sdpa_kernel

        q4, k4, v4 = q.transpose(1, 2), kc.transpose(1, 2), vc.transpose(1, 2)
        fused = [SDPBackend.FLASH_ATTENTION, SDPBackend.EFFICIENT_ATTENTION, SDPBackend.CUDNN_ATTENTION]

        def sdpa():
            with sdpa_kernel(fused):
                return F.scaled_dot_product_attention(q4, k4, v4, enable_gqa=True)

        try:
            sdpa()
            fns["sdpa_enable_gqa"] = sdpa
        except Exception as e:  # no fused backend takes this call: reported, never replaced by the math backend
            sdpa_note = str(e).splitlines()[0][:200]
    else:
        sdpa_note = "not run: lengths differ from the capacity" if not causal else "not run: causal (SDPA aligns top-left)"
    try:
        t = time_rounds(fns, args.iters, args.rounds, graph=True)
    except Exception as e:   # e.g. a comparator that cannot be captured: reported, the case still runs without it
        sdpa_note = "dropped: " + str(e).splitlines()[0][:200]
        fns.pop("sdpa_enable_gqa", None)
        t = time_rounds(fns, args.iters, args.rounds, graph=True)
    nbytes = sum(lens) * H_kv * D * 2 * 2 + 2 * B * Lq * H * D * 2
    line = dict(case=name, B=B, Lq=Lq, H=H, H_kv=H_kv, D=D, causal=causal, capacity=cap,
                lens=lens if len(set(lens)) > 1 and len(lens) <= 16 else None,
                total_keys=int(sum(lens)), splits=int(splits_of(B, Lq, H, H_kv, cap)), bytes=int(nbytes))
    med = {}
    for k, ts in t.items():
        med[k], lo, hi = stats(ts)
        line[k + "_us"] = round(med[k] * 1e6, 2)
        line[k + "_us_min_max"] = [round(lo * 1e6, 2), round(hi * 1e6, 2)]
        line[k + "_GBps"] = round(nbytes / med[k] * 1e-9, 1)
        line[k + "_frac_3350GBps"] = round(nbytes / med[k] / PEAK_BYTES_PER_S, 3)
    line["speed_vs_varlen"] = round(med["varlen"] / med["kvcache"], 3)
    if "sdpa_enable_gqa" in t:
        line["speed_vs_sdpa"] = round(med["sdpa_enable_gqa"] / med["kvcache"], 3)
    if sdpa_note:
        line["sdpa_note"] = sdpa_note
    # the compared calls compute the same rows (paged: the same bits as contiguous)
    ops.fa2_fwd_kvcache(q, kc, vc, o, sl, causal=causal)
    ops.fa2_fwd_varlen(pq, pk, pv, ov, cu_q, cu_k, Lq, causal=causal)
    line["max_abs_diff_vs_varlen"] = float((o.view(B * Lq, H, D).float() - ov.float()).abs().max())
    for ps, (kp, vp, table, op) in paged.items():
        ops.fa2_fwd_kvcache(q, kp, vp, op, sl, table, causal=causal)
        line["paged%d_same_bits" % ps] = bool(torch.equal(op, o))
    print(json.dumps(dict(line, **info)), flush=True)
    del q, kc, vc, pk, pv, paged, fns
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    info = gpu_info(torch)
    for B in (1, 8, 64):
        for L in (1024, 8192, 32768):
            run_case(info, args, "1_decode_gqa4", B, 1, 32, 8, [L] * B, L, seed=B + L)
    run_case(info, args, "1_decode_gqa8", 8, 1, 64, 8, [32768] * 8, 32768, seed=1)
    run_case(info, args, "2_speculative_lq4_causal", 8, 4, 32, 8, [8192] * 8, 8192, causal=True, seed=2)
    run_case(info, args, "2_mha", 8, 1, 32, 32, [8192] * 8, 8192, seed=3)
    mixed = np.random.RandomState(2024).randint(1, 32768 + 1, size=16).tolist()
    run_case(info, args, "3_mixed_lengths", 16, 1, 32, 8, mixed, 32768, seed=4)
    run_case(info, args, "4_paged", 8, 1, 32, 8, [8192] * 8, 8192, page_sizes=(16, 256), seed=5)
    run_case(info, args, "4_paged", 1, 1, 32, 8, [32768], 32768, page_sizes=(16, 256), seed=6)
    run_case(info, args, "4_paged_mixed", 16, 1, 32, 8, mixed, 32768, page_sizes=(16, 256), seed=7)


if __name__ == "__main__":
    main()
