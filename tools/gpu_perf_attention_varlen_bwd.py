"""Packed attention backward time on the GPU, in one process: ops.fa2_bwd_varlen against what a user does without it,
fp16, causal and not.

  1. equal lengths, MHA, (4, 48, 8192, 64) and (4, 64, 8192, 128): packed against the dense fa2_bwd on the same data,
     whose outputs are checked for the same bits;
  2. GQA, H = 64, H_kv = 8, D = 128, 4 x 8192 tokens: against repeat_interleave of K/V + fa2_bwd + a group sum of dK/dV,
     and against scaled_dot_product_attention(enable_gqa=True)'s backward on the backend torch picks (named);
  3. mixed lengths, 64 sequences uniform in [128, 8192], H = 32, D = 128: against fa2_bwd on the sequences padded to the
     longest with seqlens_k; TFLOP/s counts only the useful (unpadded) work;
  4. MQA, H = 32, H_kv = 1, B = 1, N = 4096, D = 128: the dK/dV grid is 64 CTAs, below the SM count.

FLOPs as flash-attn counts them: the backward is 2.5 times the forward's 4 H Lq Lk D per sequence, halved when causal.
Each variant runs `iters` calls between two CUDA events; the variants alternate within each round, and each line gives
the median and min - max over rounds.  The first line names the GPU, its power limit and its maximum SM clock, read in
the same run.  Prints one JSON object per line.

    python tools/gpu_perf_attention_varlen_bwd.py [--rounds 7] [--iters 3]
"""
import argparse
import json

from gpu_timing import gpu_info, stats, time_rounds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()
    import torch
    import torch.nn.functional as F

    from b200k import ops

    print(json.dumps(gpu_info(torch)), flush=True)
    dev, h = "cuda", torch.half

    def cu_of(lens):
        return torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=dev)

    def packed(lens, H, H_kv, D, causal, seed=0):
        g = torch.Generator(device=dev).manual_seed(seed)
        T = sum(lens)
        q, do = (torch.randn(T, H, D, generator=g, device=dev, dtype=h) for _ in range(2))
        k, v = (torch.randn(T, H_kv, D, generator=g, device=dev, dtype=h) for _ in range(2))
        cu = cu_of(lens)
        o, lse = torch.empty_like(q), torch.empty(T, H, device=dev)
        ops.fa2_fwd_varlen(q, k, v, o, cu, cu, max(lens), causal=causal, lse=lse)
        outs = [torch.empty_like(t) for t in (q, k, v)]
        fn = lambda: ops.fa2_bwd_varlen(q, k, v, o, lse, do, *outs, cu, cu, max(lens), max(lens), causal=causal)  # noqa
        return (q, k, v, o, lse, do, cu), outs, fn

    def flops(lens, H, D, causal):
        return 2.5 * sum(4.0 * H * n * n * D / (2 if causal else 1) for n in lens)

    def report(case, lens, H, D, causal, times, extra=None):
        row = {"case": case, "causal": causal, "dtype": "f16"}
        useful = flops(lens, H, D, causal)
        for n, t in times.items():
            med, lo, hi = (s * 1e3 for s in stats(t))
            row[n] = {"ms_median": round(med, 3), "ms_min": round(lo, 3), "ms_max": round(hi, 3),
                      "useful_tflops": round(useful / med / 1e9, 1)}
        row.update(extra or {})
        print(json.dumps(row), flush=True)

    for causal in (False, True):
        # 1. equal lengths, MHA: packed vs dense, same bits
        for B, H, N, D in ((4, 48, 8192, 64), (4, 64, 8192, 128)):
            (q, k, v, o, lse, do, cu), outs, ours = packed([N] * B, H, H, D, causal)
            dn = lambda t: t.view(B, N, t.size(1), D).transpose(1, 2).contiguous()  # noqa: E731
            qd, kd, vd, od, dod = (dn(t) for t in (q, k, v, o, do))
            lsed = lse.view(B, N, H).transpose(1, 2).contiguous()
            dd = [torch.empty_like(qd) for _ in range(3)]
            dense = lambda: ops.fa2_bwd(qd, kd, vd, od, lsed, dod, *dd, causal=causal)  # noqa: E731
            times = time_rounds({"packed": ours, "dense": dense}, args.iters, args.rounds)
            same = all(torch.equal(a.view(torch.int16), dn(b).view(torch.int16)) for a, b in zip(dd, outs))
            report("mha %dx%dx%dx%d" % (B, H, N, D), [N] * B, H, D, causal, times, {"same_bits_as_dense": same})
            del q, k, v, o, lse, do, outs, qd, kd, vd, od, dod, lsed, dd
            torch.cuda.empty_cache()
        # 2. GQA 64 / 8
        B, N, H, H_kv, D = 4, 8192, 64, 8, 128
        (q, k, v, o, lse, do, cu), outs, ours = packed([N] * B, H, H_kv, D, causal)
        dn = lambda t: t.view(B, N, t.size(1), D).transpose(1, 2).contiguous()  # noqa: E731
        qd, od, dod = (dn(t) for t in (q, o, do))
        lsed = lse.view(B, N, H).transpose(1, 2).contiguous()
        dd = [torch.empty_like(qd) for _ in range(3)]

        def expand():
            kd, vd = (dn(t).repeat_interleave(H // H_kv, dim=1) for t in (k, v))
            ops.fa2_bwd(qd, kd, vd, od, lsed, dod, *dd, causal=causal)
            return dd[1].view(B, H_kv, H // H_kv, N, D).sum(2), dd[2].view(B, H_kv, H // H_kv, N, D).sum(2)

        qa, ka, va = (dn(t).requires_grad_() for t in (q, k, v))
        out = F.scaled_dot_product_attention(qa, ka, va, is_causal=causal, enable_gqa=True)
        backend = out.grad_fn.name()
        sd = lambda: torch.autograd.grad(out, (qa, ka, va), dod, retain_graph=True)  # noqa: E731
        times = time_rounds({"packed": ours, "repeat_interleave_fa2_bwd_sum": expand, "sdpa_gqa": sd},
                            args.iters, args.rounds)
        report("gqa %dx%dx%d H_kv=%d" % (B, H, N, H_kv), [N] * B, H, D, causal, times, {"sdpa_backend": backend})
        del q, k, v, o, lse, do, outs, qd, od, dod, lsed, dd, qa, ka, va, out
        torch.cuda.empty_cache()
        # 3. mixed lengths vs padded
        g = torch.Generator().manual_seed(1)
        lens = torch.randint(128, 8193, (64,), generator=g).tolist()
        H, D, Nmax = 32, 128, max(lens)
        (q, k, v, o, lse, do, cu), outs, ours = packed(lens, H, H, D, causal)
        pad = lambda t: torch.stack([F.pad(t[s:s + n], (0, 0, 0, 0, 0, Nmax - n)) for s, n in  # noqa: E731
                                     zip(cu[:-1].tolist(), lens)]).transpose(1, 2).contiguous()
        qp, kp, vp, dop = (pad(t) for t in (q, k, v, do))
        sl = torch.tensor(lens, dtype=torch.int32, device=dev)
        op, lsep = torch.empty_like(qp), torch.empty(64, H, Nmax, device=dev)
        ops.fa2_fwd(qp, kp, vp, op, causal=causal, seqlens_k=sl, lse=lsep)
        dp = [torch.empty_like(qp) for _ in range(3)]
        padded = lambda: ops.fa2_bwd(qp, kp, vp, op, lsep, dop, *dp, causal=causal, seqlens_k=sl)  # noqa: E731
        times = time_rounds({"packed": ours, "padded_fa2_bwd": padded}, args.iters, args.rounds)
        report("mixed 64 seqs [128, 8192] H=32 D=128", lens, H, D, causal, times, {"tokens": sum(lens), "padded_to": Nmax})
        del q, k, v, o, lse, do, outs, qp, kp, vp, dop, op, lsep, dp
        torch.cuda.empty_cache()
        # 4. MQA, low parallelism
        (q, k, v, o, lse, do, cu), outs, ours = packed([4096], 32, 1, 128, causal)
        times = time_rounds({"packed": ours}, args.iters, args.rounds)
        report("mqa 1x32x4096 H_kv=1", [4096], 32, 128, causal, times, {"dkdv_ctas": 4096 // 64})
        del q, k, v, o, lse, do, outs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
