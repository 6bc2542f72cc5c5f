"""What the attention log-sum-exp costs, and what merging by it costs, on the GPU, in one process.

  (a) LSE overhead: each call with ``lse=`` against the same call without, alternating, at bench.py's attention shapes
      (dense (4, 48, 8192, 64) and (4, 64, 8192, 128)), packed GQA (4 x 8192 tokens, H 64, H_kv 8, D 128, causal) and
      decode against an 8K cache at B = 1 (split) and B = 64.
  (b) Merge bandwidth: ops.attn_merge at S = 2 and 4, D = 128, from decode sizes (B * H rows) to prefill (16K tokens x
      32 heads), in GB/s over (S + 1) * rows * D * 2 + (S + 1) * rows * 4 bytes, against the torch composition (fp32
      weights, weighted sum, cast) and against the 3.35 TB/s of the H100 SXM data sheet.
  (c) Cascade decode: a shared 8K prefix, B = 64 sequences with 1K suffixes, D 128, H 32, H_kv 8: prefix (fa2_fwd_varlen,
      all query rows against one copy) + suffix (fa2_fwd_kvcache) + merge, against fa2_fwd_kvcache over B full copies.

Each measurement is one CUDA graph of `iters` calls, timed with CUDA events; the compared variants alternate within each
round, and each line gives the median and min - max over rounds.  The first line names the GPU, its power limit and its
maximum SM clock, read in the same run.  Prints one JSON object per line.

    python tools/gpu_perf_attention_lse.py [--rounds 9] [--iters 20]
"""
import argparse
import json

from gpu_timing import gpu_info, stats, time_rounds


def us(samples):
    med, lo, hi = stats(samples)
    return {"median_us": round(med * 1e6, 2), "min_us": round(lo * 1e6, 2), "max_us": round(hi * 1e6, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    import torch

    from b200k import ops

    print(json.dumps(gpu_info(torch)), flush=True)
    dev = "cuda"
    torch.manual_seed(0)

    def rn(*shape):
        return torch.randn(*shape, device=dev).half()

    def report(section, name, times, **extra):
        line = {"section": section, "case": name}
        line.update({k: us(v) for k, v in times.items()})
        line.update(extra)
        print(json.dumps(line), flush=True)

    # (a) overhead of writing lse
    for B, H, N, D in ((4, 48, 8192, 64), (4, 64, 8192, 128)):
        q, k, v = [rn(B, H, N, D) for _ in range(3)]
        o, lse = torch.empty_like(q), torch.empty(B, H, N, device=dev)
        t = time_rounds({"without": lambda: ops.fa2_fwd(q, k, v, o), "with": lambda: ops.fa2_fwd(q, k, v, o, lse=lse)},
                        max(1, args.iters // 4), args.rounds, graph=True)
        report("a", "dense B%d H%d N%d D%d" % (B, H, N, D), t)
        del q, k, v, o, lse
    T, H, H_kv, D = 4 * 8192, 64, 8, 128
    cu = torch.arange(5, dtype=torch.int32, device=dev) * 8192
    q, k, v = rn(T, H, D), rn(T, H_kv, D), rn(T, H_kv, D)
    o, lse = torch.empty_like(q), torch.empty(T, H, device=dev)
    t = time_rounds({"without": lambda: ops.fa2_fwd_varlen(q, k, v, o, cu, cu, 8192, causal=True),
                     "with": lambda: ops.fa2_fwd_varlen(q, k, v, o, cu, cu, 8192, causal=True, lse=lse)},
                    max(1, args.iters // 4), args.rounds, graph=True)
    report("a", "packed GQA 4x8192 H64 Hkv8 D128 causal", t)
    del q, k, v, o, lse
    for B in (1, 64):
        H, H_kv, D, S = 32, 8, 128, 8192
        q = rn(B, 1, H, D)
        kc, vc = rn(B, S, H_kv, D), rn(B, S, H_kv, D)
        lens = torch.full((B,), S, dtype=torch.int32, device=dev)
        o, lse = torch.empty_like(q), torch.empty(B, 1, H, device=dev)
        t = time_rounds({"without": lambda: ops.fa2_fwd_kvcache(q, kc, vc, o, lens),
                         "with": lambda: ops.fa2_fwd_kvcache(q, kc, vc, o, lens, lse=lse)}, args.iters, args.rounds,
                        graph=True)
        report("a", "decode B%d 8K cache H32 Hkv8 D128 (%s)" % (B, "split" if ops.fa2_fwd_kvcache_workspace_bytes(
            B, 1, H, H_kv, D, S) else "unsplit"), t)
        del q, kc, vc, o, lse

    # (b) merge bandwidth
    D = 128
    for S in (2, 4):
        for rows in (64 * 32, 16384 * 32):
            parts = rn(S, rows, D)
            lps = torch.randn(S, rows, device=dev)
            o, lse = torch.empty(rows, D, dtype=torch.half, device=dev), torch.empty(rows, device=dev)

            def composed():
                m = lps.max(0).values
                w = torch.exp(lps - m)
                x = (w.unsqueeze(-1) * parts.float()).sum(0) / w.sum(0).unsqueeze(-1)
                o.copy_(x.half())
                lse.copy_(m + torch.log(w.sum(0)))

            t = time_rounds({"attn_merge": lambda: ops.attn_merge(parts, lps, o, lse), "torch": composed},
                            args.iters, args.rounds, graph=True)
            nbytes = (S + 1) * rows * D * 2 + (S + 1) * rows * 4
            gbs = {name: round(nbytes / (us(v)["median_us"] * 1e3), 1) for name, v in t.items()}
            report("b", "merge S%d rows%d D%d" % (S, rows, D), t, bytes=nbytes, gb_per_s=gbs,
                   share_of_3350_gbs=round(gbs["attn_merge"] / 3350.0, 3))
            del parts, lps, o, lse

    # (c) cascade decode
    B, H, H_kv, D, P, Ls = 64, 32, 8, 128, 8192, 1024
    q = rn(B, 1, H, D)
    kp, vp = rn(P, H_kv, D), rn(P, H_kv, D)
    ks, vs = rn(B, Ls, H_kv, D), rn(B, Ls, H_kv, D)
    lens = torch.full((B,), Ls, dtype=torch.int32, device=dev)
    cu_q = torch.tensor([0, B], dtype=torch.int32, device=dev)
    cu_k = torch.tensor([0, P], dtype=torch.int32, device=dev)
    parts, lps = torch.empty(2, B, 1, H, D, dtype=torch.half, device=dev), torch.empty(2, B, 1, H, device=dev)
    om = torch.empty_like(q)

    def cascade():
        ops.fa2_fwd_varlen(q.view(B, H, D), kp, vp, parts[0].view(B, H, D), cu_q, cu_k, B, lse=lps[0].view(B, H))
        ops.fa2_fwd_kvcache(q, ks, vs, parts[1], lens, lse=lps[1])
        ops.attn_merge(parts, lps, om)

    fk = torch.cat([kp.expand(B, P, H_kv, D), ks], 1).contiguous()
    fv = torch.cat([vp.expand(B, P, H_kv, D), vs], 1).contiguous()
    flens = lens + P
    of = torch.empty_like(q)
    t = time_rounds({"cascade": cascade, "full_copies": lambda: ops.fa2_fwd_kvcache(q, fk, fv, of, flens)},
                    args.iters, args.rounds, graph=True)
    cascade()
    ops.fa2_fwd_kvcache(q, fk, fv, of, flens)
    torch.cuda.synchronize()
    report("c", "cascade B64 prefix 8K suffix 1K H32 Hkv8 D128", t,
           max_abs_diff_vs_full=float((om.float() - of.float()).abs().max()))


if __name__ == "__main__":
    main()
