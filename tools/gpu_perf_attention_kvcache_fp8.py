"""KV-cache attention over fp8 caches against the same call over 16-bit caches, one JSON line per case.  D = 128, fp16
queries.  As in gpu_perf_attention_kvcache.py, each call is captured `--iters` times into one CUDA graph; the fp8 and
16-bit graphs of a case alternate within this process for `--rounds` rounds, and each reports the median and the
min - max of its per-call time.  Every line carries the GPU's name and power limit, read in the same run.

Cases:
  decode       H = 32, H_kv = 8, Lq = 1, B in {1, 8, 64} x {1K, 8K, 32K} keys, contiguous caches, and pages of 16 and
               256 keys at B = 8 and 64 with 8K keys; a mixed-length batch; one append + rotary row
  prefill      chunked prefill through a block table (gpu_perf_attention_varlen_paged.py's rows): 8 sequences of 1024
               new queries against 8K or 32K cached keys, pages of 256

Metric: GB/s counted with the bytes each call must move: K and V at 1 byte (fp8) or 2 bytes (16-bit) per element, plus
Q and O.  `speedup` is the 16-bit median over the fp8 median; the bound from halving K/V bytes is below 2x.

    python tools/gpu_perf_attention_kvcache_fp8.py [--iters 20] [--rounds 7] [--fmt e4m3|e5m2] [--only NAME,...]
"""
import argparse
import json

import numpy as np
import torch
from gpu_timing import gpu_info, stats, time_rounds
from b200k import ops

D, H, H_KV = 128, 32, 8
FMTS = {"e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}


def report(info, args, name, t, bytes16, bytes8, extra):
    line = dict(case=name, fmt=args.fmt, **extra)
    med = {}
    for k, nb in (("fp8", bytes8), ("f16", bytes16)):
        med[k], lo, hi = stats(t[k])
        line[k + "_us"] = round(med[k] * 1e6, 2)
        line[k + "_us_min_max"] = [round(lo * 1e6, 2), round(hi * 1e6, 2)]
        line[k + "_GBps"] = round(nb / med[k] * 1e-9, 1)
    line["speedup"] = round(med["f16"] / med["fp8"], 3)
    line.update(info)
    print(json.dumps(line), flush=True)


def paged(kc, vc, ps, perm):
    """[B, S, H_kv, D] caches as pages of ps keys under the table `perm` (through bytes, so fp8 works too)."""
    B, S = kc.shape[:2]
    pps = S // ps
    out = []
    for c in (kc, vc):
        u = c.view(torch.uint8) if c.element_size() == 1 else c.view(torch.int16)
        p = torch.empty((B * pps, ps) + tuple(u.shape[2:]), dtype=u.dtype, device="cuda")
        p[perm] = u.reshape((B * pps, ps) + tuple(u.shape[2:]))
        out.append(p.view(c.dtype))
    return out[0], out[1], perm.to(torch.int32).view(B, pps)


def decode_case(info, args, name, B, lens, cap, page_size=None, append=False):
    if args.only and name not in args.only.split(","):
        return
    torch.manual_seed(0)
    fmt = FMTS[args.fmt]
    q = torch.randn(B, 1, H, D, dtype=torch.half, device="cuda")
    k16, v16 = [torch.randn(B, cap, H_KV, D, dtype=torch.half, device="cuda") for _ in range(2)]
    ks, vs = torch.full((H_KV,), 0.5, device="cuda"), torch.full((H_KV,), 0.25, device="cuda")
    k8, v8 = (k16.float() / 0.5).to(fmt), (v16.float() / 0.25).to(fmt)
    table = None
    if page_size:
        perm = torch.randperm(B * (cap // page_size), device="cuda")
        k16, v16, table = paged(k16, v16, page_size, perm)
        k8, v8, _ = paged(k8, v8, page_size, perm)
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    o8, o16 = torch.empty_like(q), torch.empty_like(q)
    kw = {}
    if append:
        kn, vn = [torch.randn(B, 1, H_KV, D, dtype=torch.half, device="cuda") for _ in range(2)]
        ang = torch.rand(cap, D // 2, device="cuda") * 6.28
        kw = dict(k=kn, v=vn, rotary_cos=ang.cos().half(), rotary_sin=ang.sin().half())
        sl = sl - 1  # the appended key brings each sequence to its length
    fns = {"fp8": lambda: ops.fa2_fwd_kvcache(q, k8, v8, o8, sl, table if page_size else None, k_scale=ks, v_scale=vs,
                                              **kw),
           "f16": lambda: ops.fa2_fwd_kvcache(q, k16, v16, o16, sl, table if page_size else None, **kw)}
    t = time_rounds(fns, args.iters, args.rounds, graph=True)
    keys = int(sum(lens))
    qo = 2 * B * H * D * 2
    report(info, args, name, t, keys * H_KV * D * 2 * 2 + qo, keys * H_KV * D * 2 + qo,
           dict(B=B, H=H, H_kv=H_KV, D=D, capacity=cap, page_size=page_size, total_keys=keys, append_rotary=append))


def prefill_case(info, args, name, Lq, Lk, ps=256):
    if args.only and name not in args.only.split(","):
        return
    torch.manual_seed(2)
    fmt = FMTS[args.fmt]
    B = len(Lq)
    cap = max(Lk)
    q = torch.randn(sum(Lq), H, D, dtype=torch.half, device="cuda")
    k16, v16 = [torch.randn(B, cap, H_KV, D, dtype=torch.half, device="cuda") for _ in range(2)]
    k8, v8 = k16.to(fmt), v16.to(fmt)
    perm = torch.randperm(B * (cap // ps), device="cuda")
    k16, v16, table = paged(k16, v16, ps, perm)
    k8, v8, _ = paged(k8, v8, ps, perm)
    cu_q = torch.tensor([0] + np.cumsum(Lq).tolist(), dtype=torch.int32, device="cuda")
    cu_k = torch.tensor([0] + np.cumsum(Lk).tolist(), dtype=torch.int32, device="cuda")
    o8, o16 = torch.empty_like(q), torch.empty_like(q)
    fns = {"fp8": lambda: ops.fa2_fwd_varlen(q, k8, v8, o8, cu_q, cu_k, max(Lq), causal=True, block_table=table),
           "f16": lambda: ops.fa2_fwd_varlen(q, k16, v16, o16, cu_q, cu_k, max(Lq), causal=True, block_table=table)}
    t = time_rounds(fns, args.iters, args.rounds, graph=True)
    keys = int(sum(Lk))
    qo = 2 * sum(Lq) * H * D * 2
    report(info, args, name, t, keys * H_KV * D * 2 * 2 + qo, keys * H_KV * D * 2 + qo,
           dict(B=B, H=H, H_kv=H_KV, D=D, Lq=Lq[0], Lk=Lk[0], page_size=ps))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--fmt", choices=sorted(FMTS), default="e4m3")
    ap.add_argument("--only", default="", help="comma list of case names to run (default: all)")
    args = ap.parse_args()
    info = gpu_info(torch)
    for B in (1, 8, 64):
        for keys in (1024, 8192, 32768):
            decode_case(info, args, "decode_B%d_%dk" % (B, keys // 1024), B, [keys] * B, keys)
    for B in (8, 64):
        for ps in (16, 256):
            decode_case(info, args, "decode_B%d_8k_pages%d" % (B, ps), B, [8192] * B, 8192, page_size=ps)
    mixed = [int(x) for x in np.random.default_rng(0).integers(64, 16384, 32)]
    decode_case(info, args, "decode_mixed_B32", 32, mixed, 16384, page_size=256)
    decode_case(info, args, "decode_append_rotary_B8_8k", 8, [8192] * 8, 8192, page_size=256, append=True)
    for cached in (8192, 32768):
        prefill_case(info, args, "chunked_prefill_%dk" % (cached // 1024), [1024] * 8, [cached] * 8)


if __name__ == "__main__":
    main()
