"""Packed variable-length attention (ops.fa2_fwd_varlen) against the calls a caller makes without it, one JSON line per
case.  CUDA-event time per call after warm-up; the calls compared in a case alternate within this process (median of
the rounds).  Every line carries the GPU's name and power limit, read in the same run.

  1. equal lengths, MHA: varlen on the packed [B*N, H, D] copy vs dense ops.fa2_fwd on [B,H,N,D], same data
  2. GQA (H = 64, H_kv = 8, D = 128, 4 x 8192 tokens): vs varlen with K/V repeated to H heads, and vs
     F.scaled_dot_product_attention(enable_gqa=True) on the [B,H,N,D] view (fused backends only)
  3. mixed lengths (64 sequences, seeded lengths uniform in [128, 8192], H = 32, D = 128): vs the padded dense call
     (ops.fa2_fwd with seqlens_k); TFLOP/s count only useful work, 4 * H * D per visible (query row, key) pair

    python tools/gpu_perf_attention_varlen.py [--iters 10] [--rounds 3]
"""
import argparse
import json

import numpy as np
import torch
import torch.nn.functional as F
from gpu_timing import gpu_info, stats, time_rounds, visible_pairs
from b200k import ops


def emit(info, **kw):
    print(json.dumps(dict(kw, **info)), flush=True)


def case_equal_lengths(info, args):
    for (B, H, N, D) in ((4, 48, 8192, 64), (4, 64, 8192, 128)):
        torch.manual_seed(0)
        q, k, v = [torch.randn(B, H, N, D, dtype=torch.half, device="cuda") for _ in range(3)]
        pq, pk, pv = [t.transpose(1, 2).contiguous().view(B * N, H, D) for t in (q, k, v)]
        o, po = torch.empty_like(q), torch.empty_like(pq)
        cu = torch.arange(0, (B + 1) * N, N, dtype=torch.int32, device="cuda")
        for causal in (False, True):
            t = {name: stats(ts)[0] for name, ts in time_rounds({
                "dense": lambda: ops.fa2_fwd(q, k, v, o, causal=causal),
                "varlen": lambda: ops.fa2_fwd_varlen(pq, pk, pv, po, cu, cu, N, causal=causal),
            }, args.iters, args.rounds).items()}
            flop = 4 * H * D * B * visible_pairs(N, N, causal)
            same = torch.equal(po.view(B, N, H, D).transpose(1, 2), o)
            emit(info, case="1_equal_lengths_mha", shape=[B, H, N, D], causal=causal, dense_ms=round(t["dense"] * 1e3, 3),
                 varlen_ms=round(t["varlen"] * 1e3, 3), varlen_speed_vs_dense=round(t["dense"] / t["varlen"], 3),
                 varlen_tflops=round(flop / t["varlen"] * 1e-12, 1), same_bits_as_dense=bool(same))
        del q, k, v, pq, pk, pv, o, po
        torch.cuda.empty_cache()


def case_gqa(info, args):
    B, N, H, H_kv, D = 4, 8192, 64, 8, 128
    torch.manual_seed(1)
    q = torch.randn(B * N, H, D, dtype=torch.half, device="cuda")
    k, v = [torch.randn(B * N, H_kv, D, dtype=torch.half, device="cuda") for _ in range(2)]
    kr, vr = [t.repeat_interleave(H // H_kv, dim=1).contiguous() for t in (k, v)]
    o, o_rep = torch.empty_like(q), torch.empty_like(q)
    cu = torch.arange(0, (B + 1) * N, N, dtype=torch.int32, device="cuda")
    q4, k4, v4 = [t.view(B, N, t.size(1), D).transpose(1, 2) for t in (q, k, v)]
    from torch.nn.attention import SDPBackend, sdpa_kernel

    fused = [SDPBackend.FLASH_ATTENTION, SDPBackend.EFFICIENT_ATTENTION, SDPBackend.CUDNN_ATTENTION]
    for causal in (False, True):
        fns = {
            "varlen_gqa": lambda: ops.fa2_fwd_varlen(q, k, v, o, cu, cu, N, causal=causal),
            "varlen_mha_repeated_kv": lambda: ops.fa2_fwd_varlen(q, kr, vr, o_rep, cu, cu, N, causal=causal),
        }
        sdpa_error = None

        def sdpa():
            with sdpa_kernel(fused):
                return F.scaled_dot_product_attention(q4, k4, v4, is_causal=causal, enable_gqa=True)

        try:
            sdpa()
            fns["sdpa_enable_gqa"] = sdpa
        except Exception as e:  # no fused backend takes this call: reported, never replaced by the math backend
            sdpa_error = str(e).splitlines()[0][:200]
        t = {name: stats(ts)[0] for name, ts in time_rounds(fns, args.iters, args.rounds).items()}
        flop = 4 * H * D * B * visible_pairs(N, N, causal)
        line = dict(case="2_gqa", B=B, N=N, H=H, H_kv=H_kv, D=D, causal=causal,
                    same_bits_as_repeated_kv=bool(torch.equal(o, o_rep)))
        for name, s in t.items():
            line[name + "_ms"] = round(s * 1e3, 3)
            line[name + "_tflops"] = round(flop / s * 1e-12, 1)
        if "sdpa_enable_gqa" in t:
            line["varlen_speed_vs_sdpa"] = round(t["sdpa_enable_gqa"] / t["varlen_gqa"], 3)
        else:
            line["sdpa_error"] = sdpa_error
        line["varlen_speed_vs_repeated_kv"] = round(t["varlen_mha_repeated_kv"] / t["varlen_gqa"], 3)
        emit(info, **line)
    del q, k, v, kr, vr, o, o_rep
    torch.cuda.empty_cache()


def case_mixed_lengths(info, args):
    nseq, H, D = 64, 32, 128
    lens = np.random.RandomState(2024).randint(128, 8192 + 1, size=nseq)
    N = int(lens.max())
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device="cuda")
    total = int(lens.sum())
    torch.manual_seed(2)
    q, k, v = [torch.randn(total, H, D, dtype=torch.half, device="cuda") for _ in range(3)]
    o = torch.empty_like(q)
    # the padded layout a caller builds today: [B, H, N_max, D] with the tail of each sequence zero
    pad = []
    for t in (q, k, v):
        p = torch.zeros(nseq, H, N, D, dtype=torch.half, device="cuda")
        for b in range(nseq):
            p[b, :, :lens[b]] = t[int(cu[b]):int(cu[b + 1])].transpose(0, 1)
        pad.append(p)
    op = torch.empty_like(pad[0])
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    for causal in (False, True):
        t = {name: stats(ts)[0] for name, ts in time_rounds({
            "padded_dense": lambda: ops.fa2_fwd(pad[0], pad[1], pad[2], op, causal=causal, seqlens_k=sl),
            "varlen": lambda: ops.fa2_fwd_varlen(q, k, v, o, cu, cu, N, causal=causal),
        }, args.iters, args.rounds).items()}
        useful = 4 * H * D * sum(visible_pairs(L, L, causal) for L in lens)
        emit(info, case="3_mixed_lengths", nseq=nseq, H=H, D=D, total_tokens=total, max_len=N, causal=causal,
             padded_dense_ms=round(t["padded_dense"] * 1e3, 3), varlen_ms=round(t["varlen"] * 1e3, 3),
             varlen_speedup_vs_padded=round(t["padded_dense"] / t["varlen"], 3),
             padded_dense_useful_tflops=round(useful / t["padded_dense"] * 1e-12, 1),
             varlen_useful_tflops=round(useful / t["varlen"] * 1e-12, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    info = gpu_info(torch)
    case_equal_lengths(info, args)
    case_gqa(info, args)
    case_mixed_lengths(info, args)


if __name__ == "__main__":
    main()
