"""Attention backward time on the GPU, in one process: ops.fa2_bwd (backward only) and ops.attention forward + backward,
against scaled_dot_product_attention's flash backend and torch's math path, on the same [B, H, N, D] tensors.

Shapes (4, 48, 8192, 64), (4, 64, 8192, 128) and (8, 16, 2048, 128) in fp16, causal and not.  Backward only: a
prepared forward's O and lse (ours) or autograd graph (SDPA, torch.autograd.grad with retain_graph) and the same dO.
FLOPs are counted as flash-attn counts them: the forward's 4 B H N^2 D, halved when causal; the backward 2.5 times that
(flash-attn's convention, although this backward recomputes S and dP and performs 7 products where an atomic-dQ
backward performs 5).  Each variant runs `iters` calls between two CUDA events; the variants alternate within each round,
and each line gives the median and min - max over rounds.  A variant that runs out of memory (the math path at 8K
keys) is reported as such.  The first line names the GPU, its power limit and its maximum SM clock, read in the same run.
Prints one JSON object per line.

    python tools/gpu_perf_attention_bwd.py [--rounds 7] [--iters 3]
"""
import argparse
import json

from gpu_timing import gpu_info, stats, time_rounds

SHAPES = [(4, 48, 8192, 64), (4, 64, 8192, 128), (8, 16, 2048, 128)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()
    import torch
    from torch.nn.attention import SDPBackend, sdpa_kernel
    from torch.nn.functional import scaled_dot_product_attention as sdpa

    from b200k import ops

    print(json.dumps(gpu_info(torch)), flush=True)
    for B, H, N, D in SHAPES:
        for causal in (False, True):
            g = torch.Generator(device="cuda").manual_seed(0)
            q, k, v, do = (torch.randn(B, H, N, D, generator=g, device="cuda", dtype=torch.half) for _ in range(4))
            o, lse = torch.empty_like(q), torch.empty(B, H, N, device="cuda")
            ops.fa2_fwd(q, k, v, o, causal=causal, lse=lse)
            dq, dk, dv = (torch.empty_like(q) for _ in range(3))
            qa, ka, va = (t.clone().requires_grad_() for t in (q, k, v))

            def ours_bwd():
                ops.fa2_bwd(q, k, v, o, lse, do, dq, dk, dv, causal=causal)

            def ours_fb():
                torch.autograd.grad(ops.attention(qa, ka, va, causal=causal), (qa, ka, va), do)

            def sdpa_bwd_of(backend):
                with sdpa_kernel(backend):
                    out = sdpa(qa, ka, va, is_causal=causal)
                return lambda: torch.autograd.grad(out, (qa, ka, va), do, retain_graph=True)

            def sdpa_fb_of(backend):
                def run():
                    with sdpa_kernel(backend):
                        torch.autograd.grad(sdpa(qa, ka, va, is_causal=causal), (qa, ka, va), do)
                return run

            variants = {"ours_bwd": ours_bwd, "ours_fwd_bwd": ours_fb,
                        "sdpa_flash_bwd": sdpa_bwd_of(SDPBackend.FLASH_ATTENTION),
                        "sdpa_flash_fwd_bwd": sdpa_fb_of(SDPBackend.FLASH_ATTENTION),
                        "math_fwd_bwd": sdpa_fb_of(SDPBackend.MATH)}
            names = list(variants)
            for name in names:  # a variant that does not fit is dropped
                try:
                    variants[name]()
                    torch.cuda.synchronize()
                except torch.OutOfMemoryError:
                    del variants[name]
                    torch.cuda.empty_cache()
            times = time_rounds(variants, args.iters, args.rounds)
            fwd_flops = 4.0 * B * H * N * N * D / (2 if causal else 1)
            row = {"shape": [B, H, N, D], "causal": causal, "dtype": "f16"}
            for name in names:
                if name not in times:
                    row[name] = "out of memory"
                    continue
                med, lo, hi = (s * 1e3 for s in stats(times[name]))
                flops = fwd_flops * (2.5 if name.endswith("_bwd") and "fwd" not in name else 3.5)
                row[name] = {"ms_median": round(med, 3), "ms_min": round(lo, 3), "ms_max": round(hi, 3),
                             "tflops": round(flops / med / 1e9, 1)}
            if "sdpa_flash_bwd" in times:
                row["bwd_ratio_ours_over_flash"] = round(stats(times["ours_bwd"])[0] /
                                                         stats(times["sdpa_flash_bwd"])[0], 2)
            print(json.dumps(row), flush=True)
            del q, k, v, do, o, lse, dq, dk, dv, qa, ka, va, variants
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
