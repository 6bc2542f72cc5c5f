"""KV-cache decode with append and rotary (ops.fa2_fwd_kvcache with k / v / rotary) against what a caller runs without
it, one JSON line per case.  D = 128, fp16, H = 32, H_kv = 8, L_new = Lq = 1, NeoX rotary over all 128 columns unless
stated.  Three calls, each captured `--iters` times into one CUDA graph (time_rounds of gpu_timing.py), alternate
in this process for `--rounds` rounds:

    append  the new call: rows appended and rotated, then the decode
    floor   fa2_fwd_kvcache alone on a cache that already holds the new tokens
    today   rotary in torch (fp32, then a cast) on q and k, the torch scatter of k / v into the cache, then
            fa2_fwd_kvcache on lengths + L_new, in one graph

Each line reports median and min - max µs per call, append - floor (the append kernel plus one launch), the speed of
append relative to today, whether append and today give O and caches with the same bits without rotary (a separate
check, not timed), and the GPU's name and power limit read in the same run.

    python tools/gpu_perf_attention_kvcache_append.py [--iters 20] [--rounds 7]
"""
import argparse
import json

import torch
from gpu_timing import gpu_info, stats, time_rounds
from b200k import ops

D, H, H_KV = 128, 32, 8


def rope(n, rd):
    inv = 10000.0 ** (-torch.arange(0, rd, 2, device="cuda", dtype=torch.float32) / rd)
    ang = torch.arange(n, device="cuda", dtype=torch.float32).view(n, 1) * inv.view(1, -1)
    return ang.cos().half(), ang.sin().half()


def torch_rotary(x, cos, sin, pos):
    """NeoX rotary over all D columns, x [B, L, heads, D], pos [B, L]: fp32 math, one cast."""
    c, s = cos[pos].float().unsqueeze(2), sin[pos].float().unsqueeze(2)
    x0, x1 = x[..., :D // 2].float(), x[..., D // 2:].float()
    return torch.cat([x0 * c - x1 * s, x0 * s + x1 * c], -1).to(x.dtype)


def make_state(B, cap, ps, seed):
    """Caches [num_pages, page_size, H_kv, D] (contiguous: B pages of cap keys) and the table (None if contiguous)."""
    torch.manual_seed(seed)
    if ps is None:
        kc, vc = [torch.randn(B, cap, H_KV, D, dtype=torch.half, device="cuda") for _ in range(2)]
        return kc, vc, None
    pps = cap // ps
    kc, vc = [torch.randn(B * pps, ps, H_KV, D, dtype=torch.half, device="cuda") for _ in range(2)]
    return kc, vc, torch.randperm(B * pps, device="cuda").to(torch.int32).view(B, pps)


def run_case(info, args, name, B, cap, Lq=1, causal=False, ps=None, seed=0):
    L_new = Lq
    kc, vc, table = make_state(B, cap, ps, seed)
    page = cap if ps is None else ps
    lens = torch.full((B,), cap - 2 * L_new, dtype=torch.int32, device="cuda")   # room for the new tokens
    q = torch.randn(B, Lq, H, D, dtype=torch.half, device="cuda")
    kn, vn = [torch.randn(B, L_new, H_KV, D, dtype=torch.half, device="cuda") for _ in range(2)]
    cos, sin = rope(cap, D)
    o = torch.empty_like(q)
    pos = lens.long().view(B, 1) + torch.arange(L_new, device="cuda").view(1, L_new)
    qpos = lens.long().view(B, 1) + (torch.arange(Lq, device="cuda").view(1, Lq) if causal else 0 * pos[:, :1])
    pg = (table.gather(1, pos // page).long() if table is not None else torch.arange(B, device="cuda").view(B, 1)
          .expand(B, L_new))
    slot = pos % page
    lens_new = lens + L_new
    # caches the timed calls write into (the same slots each call, so the state does not drift)
    ka, va, kt, vt = kc.clone(), vc.clone(), kc.clone(), vc.clone()
    kf, vf = kc.clone(), vc.clone()
    kf[pg, slot] = torch_rotary(kn, cos, sin, pos)
    vf[pg, slot] = vn

    def append():
        ops.fa2_fwd_kvcache(q, ka, va, o, lens, table, causal=causal, k=kn, v=vn, rotary_cos=cos, rotary_sin=sin,
                            rotary_interleaved=False)

    def floor():
        ops.fa2_fwd_kvcache(q, kf, vf, o, lens_new, table, causal=causal)

    def today():
        qr = torch_rotary(q, cos, sin, qpos)
        kt[pg, slot] = torch_rotary(kn, cos, sin, pos)
        vt[pg, slot] = vn
        ops.fa2_fwd_kvcache(qr, kt, vt, o, lens + L_new, table, causal=causal)

    t = time_rounds({"append": append, "floor": floor, "today": today}, args.iters, args.rounds, graph=True)
    line = dict(case=name, B=B, Lq=Lq, L_new=L_new, H=H, H_kv=H_KV, D=D, causal=causal, capacity=cap,
                page_size=ps, rotary="neox 128")
    med = {}
    for k, ts in t.items():
        med[k], lo, hi = stats(ts)
        line[k + "_us"] = round(med[k] * 1e6, 2)
        line[k + "_us_min_max"] = [round(lo * 1e6, 2), round(hi * 1e6, 2)]
    line["append_minus_floor_us"] = round((med["append"] - med["floor"]) * 1e6, 2)
    line["speed_vs_today"] = round(med["today"] / med["append"], 3)
    # without rotary: append and the torch scatter + decode give the same bits
    k1, v1, k2, v2 = kc.clone(), vc.clone(), kc.clone(), vc.clone()
    o1, o2 = torch.empty_like(q), torch.empty_like(q)
    ops.fa2_fwd_kvcache(q, k1, v1, o1, lens, table, causal=causal, k=kn, v=vn)
    k2[pg, slot] = kn
    v2[pg, slot] = vn
    ops.fa2_fwd_kvcache(q, k2, v2, o2, lens + L_new, table, causal=causal)
    line["no_rotary_same_bits"] = bool(torch.equal(o1, o2) and torch.equal(k1, k2) and torch.equal(v1, v2))
    print(json.dumps(dict(line, **info)), flush=True)
    del kc, vc, ka, va, kt, vt, kf, vf, k1, v1, k2, v2
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    info = gpu_info(torch)
    for B in (1, 8, 64):
        for cap in (1024, 8192, 32768):
            run_case(info, args, "decode", B, cap, seed=B + cap)
    for ps in (16, 256):
        run_case(info, args, "paged", 8, 8192, ps=ps, seed=ps)
    run_case(info, args, "speculative_lq4_causal", 8, 8192, Lq=4, causal=True, seed=4)


if __name__ == "__main__":
    main()
