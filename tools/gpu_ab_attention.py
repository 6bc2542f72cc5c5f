"""A/B of the attention entry points against an earlier build of the library, in one process: same bits, then time.

A second copy of libb200k.so, built from another git revision, is loaded through ctypes next to the one in the tree, with
the signatures of b200k._loader.  Every call goes through b200k.ops, pointed at one library or the other, so both builds
see the same arguments.

  1. Seeded random inputs through both builds; every output (and, for append, both caches) must have the same bits:
     dense f16 / bf16 at D 32 - 128 (causal, key padding, ragged N), V stored [B,H,D,N], FFPA at D 160 - 1024, packed
     GQA / MQA with empty sequences, decode on contiguous caches and pages of 16 / 64 / 256 at one split and at many
     (G = 72 among them: two 64-row head tiles), and append with and without rotary; decode and rotary append with
     lse over 16-bit and fp8 (e4m3 / e5m2, with and without scales) caches, at one split and at many; packed prefill
     over 16-bit and fp8 pages of 16 and 256; the backward's dQ, dK and dV, dense f16 / bf16 at D 64 and 128 (causal,
     key padding, ragged N) and packed GQA with empty sequences and Lq != Lk.
  2. Time per call of each build, alternating, one CUDA graph of `iters` calls per build per round: bench.py's
     attention shapes (dense (4, 48, 8192, 64) and (4, 64, 8192, 128), FFPA (1, 32, 4096, 512)), packed GQA (4 x 8192
     tokens, H 64, H_kv 8, D 128, causal) and decode against an 8K cache at B 1 and 64; the backward at the dense
     shapes and the packed GQA one, causal and not.  Then decode and append at B 1 against an 8K cache, call by call
     without a graph, so the host's share of each call counts.  Each line gives the median and min - max of both
     builds and whether the new median lies inside the base's min - max.

The first line names the GPU, its power limit and its maximum SM clock, read in the same run.

    python tools/gpu_ab_attention.py --build-base REV        # CPU is enough: git archive REV -> build_ab/base, make
    python tools/gpu_ab_attention.py [--base-lib PATH] [--rounds 9]
"""
import argparse
import json
import os
import sys

from gpu_timing import BASE_LIB, ROOT, build_base, compare_and_time, gpu_info, load_lib


def equal_cases(torch, ops):
    """(name, run) pairs; run() makes fresh outputs (and caches) from the case's seeded inputs and returns them."""
    dev = "cuda"
    cases = []

    def rn(*shape, dt=torch.float16):
        return torch.randn(*shape, device=dev).to(dt)

    def i32(x):
        return torch.as_tensor(x, dtype=torch.int32, device=dev)

    for dt in (torch.float16, torch.bfloat16):
        for D in (32, 64, 96, 128):
            for causal in (False, True):
                for pad in (False, True):
                    torch.manual_seed(D + 2 * causal + 4 * pad)
                    B, H, N = 3, 4, 1000
                    q, k, v = [rn(B, H, N, D, dt=dt) for _ in range(3)]
                    sl = i32([1, 129, 700]) if pad else None

                    def run(q=q, k=k, v=v, sl=sl, causal=causal):
                        o = torch.full_like(q, float("nan"))
                        ops.fa2_fwd(q, k, v, o, causal=causal, seqlens_k=sl)
                        return [o]
                    cases.append(("dense %s D=%d causal=%d pad=%d" % (str(dt)[6:], D, causal, pad), run))
    for D in (64, 128):
        for causal in (False, True):
            torch.manual_seed(10 + D + causal)
            q, k = rn(2, 3, 1000, D), rn(2, 3, 1000, D)
            vt = rn(2, 3, D, 1000)
            sl = i32([1000, 129])

            def run(q=q, k=k, vt=vt, sl=sl, causal=causal):
                o = torch.full_like(q, float("nan"))
                ops.fa2_fwd(q, k, vt, o, v_is_dn=True, causal=causal, seqlens_k=sl)
                return [o]
            cases.append(("dense V [D,N] D=%d causal=%d" % (D, causal), run))
    for D in (160, 192, 256, 288, 512, 544, 1024):
        torch.manual_seed(D)
        q, k, v = [rn(1, 3, 777, D) for _ in range(3)]

        def run(q=q, k=k, v=v):
            o = torch.full_like(q, float("nan"))
            ops.ffpa_fwd(q, k, v, o)
            return [o]
        cases.append(("ffpa D=%d" % D, run))
    lq, lk = [77, 0, 1, 129, 300, 0, 200, 64, 5], [300, 5, 0, 128, 129, 0, 200, 63, 700]
    cq, ck = [i32([0] + torch.tensor(x).cumsum(0).tolist()) for x in (lq, lk)]
    for dt in (torch.float16, torch.bfloat16):
        for D in (64, 128):
            for H_kv in (4, 1):
                for causal in (False, True):
                    torch.manual_seed(D + H_kv + causal)
                    q, k, v = rn(sum(lq), 16, D, dt=dt), rn(sum(lk), H_kv, D, dt=dt), rn(sum(lk), H_kv, D, dt=dt)

                    def run(q=q, k=k, v=v, causal=causal):
                        o = torch.full_like(q, float("nan"))
                        ops.fa2_fwd_varlen(q, k, v, o, cq, ck, max(lq), causal=causal)
                        return [o]
                    cases.append(("packed %s D=%d H=16 H_kv=%d causal=%d" % (str(dt)[6:], D, H_kv, causal), run))

    def paged(kc, vc, ps, seed):
        """[B, S, H_kv, D] caches as [pages, ps, H_kv, D] under a shuffled table, two pages no table lists."""
        B, S = kc.shape[:2]
        pps = S // ps
        g = torch.Generator().manual_seed(seed)
        perm = torch.randperm(B * pps + 2, generator=g).to(dev)
        table = perm[:B * pps].view(B, pps)
        out = []
        for c in (kc, vc):
            p = torch.randn(B * pps + 2, ps, *c.shape[2:], device=dev).to(c.dtype)
            p[table.reshape(-1)] = c.reshape(B * pps, ps, *c.shape[2:])
            out.append(p)
        return out[0], out[1], table.to(torch.int32)

    # decode: (B, Lq, G, H_kv) with one split (B * H_kv CTAs fill the SMs) and with many
    for dt in (torch.float16, torch.bfloat16):
        for D in (64, 128):
            for kind in ("contig", 16, 64, 256):
                for B, Lq, G, H_kv in ((16, 1, 4, 8), (1, 3, 8, 1), (64, 1, 72, 2), (2, 2, 72, 2)):
                    for causal in (False, True):
                        S = 2048
                        seed = D + B + G + causal + (0 if kind == "contig" else kind)
                        torch.manual_seed(seed)
                        q = rn(B, Lq, G * H_kv, D, dt=dt)
                        kc, vc = rn(B, S, H_kv, D, dt=dt), rn(B, S, H_kv, D, dt=dt)
                        table = None
                        if kind != "contig":
                            kc, vc, table = paged(kc, vc, kind, seed)
                        lens = i32(torch.randint(0, S + 1, (B,)).tolist())
                        splits = ops.fa2_fwd_kvcache_workspace_bytes(B, Lq, G * H_kv, H_kv, D, S) > 0

                        def run(q=q, kc=kc, vc=vc, lens=lens, table=table, causal=causal):
                            o = torch.full_like(q, float("nan"))
                            ops.fa2_fwd_kvcache(q, kc, vc, o, lens, table, causal=causal)
                            return [o]
                        cases.append(("decode %s D=%d %s B=%d Lq=%d G=%d H_kv=%d causal=%d %s" % (
                            str(dt)[6:], D, kind, B, Lq, G, H_kv, causal, "split" if splits else "one split"), run))
    for kind in ("contig", 64):
        for rotary in (None, "neox", "interleaved"):
            for B, H_kv in ((16, 8), (1, 1)):
                torch.manual_seed(B + H_kv + (rotary is None))
                Lq, G, D, S, L_new = 2, 4, 128, 1024, 2
                q = rn(B, Lq, G * H_kv, D)
                kc0, vc0 = rn(B, S, H_kv, D), rn(B, S, H_kv, D)
                table = None
                if kind != "contig":
                    kc0, vc0, table = paged(kc0, vc0, kind, B)
                kn, vn = rn(B, L_new, H_kv, D), rn(B, L_new, H_kv, D)
                lens = i32(torch.randint(0, S - L_new + 1, (B,)).tolist())
                rot = {}
                if rotary:
                    theta = torch.rand(S, 32, device=dev) * 6.283
                    rot = dict(rotary_cos=theta.cos().half(), rotary_sin=theta.sin().half(),
                               rotary_interleaved=rotary == "interleaved")

                def run(q=q, kc0=kc0, vc0=vc0, kn=kn, vn=vn, lens=lens, table=table, rot=rot):
                    kc, vc = kc0.clone(), vc0.clone()
                    o = torch.full_like(q, float("nan"))
                    ops.fa2_fwd_kvcache(q, kc, vc, o, lens, table, causal=True, k=kn, v=vn, **rot)
                    return [o, kc, vc]
                cases.append(("append %s rotary=%s B=%d H_kv=%d" % (kind, rotary, B, H_kv), run))

    # decode and append with lse, 16-bit or fp8 caches (e4m3 / e5m2, with and without per-head scales), at one split
    # (B 16, H_kv 8) and at many (B 1, H_kv 1); appends with NeoX or interleaved rotary
    for kvdt in (None, torch.float8_e4m3fn, torch.float8_e5m2):
        for scaled in ((False,) if kvdt is None else (False, True)):
            for B, H_kv in ((16, 8), (1, 1)):
                for rotary in (None, "neox", "interleaved"):
                    torch.manual_seed(40 + B + scaled + (rotary is None))
                    Lq, G, D, S, L_new, ps = 2, 4, 128, 1024, 2, 64
                    q, kn, vn = rn(B, Lq, G * H_kv, D), rn(B, L_new, H_kv, D), rn(B, L_new, H_kv, D)
                    kc0, vc0, table = paged(rn(B, S, H_kv, D), rn(B, S, H_kv, D), ps, B)
                    if kvdt is not None:
                        kc0, vc0 = kc0.to(kvdt), vc0.to(kvdt)
                    lens = i32(torch.randint(0, S - L_new + 1, (B,)).tolist())
                    kw = dict(k_scale=torch.rand(H_kv, device=dev) + 0.5, v_scale=torch.rand(H_kv, device=dev) + 0.5) \
                        if scaled else {}
                    if rotary:
                        theta = torch.rand(S, 32, device=dev) * 6.283
                        kw.update(k=kn, v=vn, rotary_cos=theta.cos().half(), rotary_sin=theta.sin().half(),
                                  rotary_interleaved=rotary == "interleaved")

                    def run(q=q, kc0=kc0, vc0=vc0, lens=lens, table=table, kw=kw):
                        kc, vc = kc0.clone(), vc0.clone()
                        o, lse = torch.full_like(q, float("nan")), torch.full(q.shape[:-1], float("nan"), device=dev)
                        ops.fa2_fwd_kvcache(q, kc, vc, o, lens, table, causal=True, lse=lse, **kw)
                        return [o, lse, kc, vc]
                    cases.append(("kvcache lse %s scaled=%d B=%d H_kv=%d %s" % (
                        str(kvdt)[6:] or "f16", scaled, B, H_kv, "rotary=%s" % rotary if rotary else "decode"), run))

    # packed prefill over paged caches, 16-bit or fp8, with and without lse
    for kvdt in (None, torch.float8_e4m3fn, torch.float8_e5m2):
        for ps in (16, 256):
            for causal in (False, True):
                torch.manual_seed(50 + ps + causal)
                H_kv, D, S = 4, 128, 768
                q = rn(sum(lq), 16, D)
                kc, vc, table = paged(rn(len(lk), S, H_kv, D), rn(len(lk), S, H_kv, D), ps, ps + causal)
                kw = {}
                if kvdt is not None:
                    kc, vc = kc.to(kvdt), vc.to(kvdt)
                    kw = dict(k_scale=torch.rand(H_kv, device=dev) + 0.5, v_scale=torch.rand(H_kv, device=dev) + 0.5)

                def run(q=q, kc=kc, vc=vc, table=table, causal=causal, kw=kw):
                    o = torch.full_like(q, float("nan"))
                    lse = torch.full(q.shape[:-1], float("nan"), device=dev) if causal else None
                    ops.fa2_fwd_varlen(q, kc, vc, o, cq, ck, max(lq), causal=causal, lse=lse, block_table=table, **kw)
                    return [o] + ([lse] if causal else [])
                cases.append(("paged prefill %s page=%d causal=%d" % (str(kvdt)[6:] or "f16", ps, causal), run))

    # backward: o and lse from the in-tree forward, so both builds take the same inputs
    for dt in (torch.float16, torch.bfloat16):
        for D in (64, 128):
            for causal in (False, True):
                for pad in (False, True):
                    torch.manual_seed(20 + D + 2 * causal + 4 * pad)
                    B, H, N = 3, 4, 1000
                    q, k, v, do = [rn(B, H, N, D, dt=dt) for _ in range(4)]
                    sl = i32([1, 129, 700]) if pad else None
                    o, lse = torch.empty_like(q), torch.empty(B, H, N, device=dev)
                    ops.fa2_fwd(q, k, v, o, causal=causal, seqlens_k=sl, lse=lse)

                    def run(q=q, k=k, v=v, o=o, lse=lse, do=do, sl=sl, causal=causal):
                        g = [torch.full_like(t, float("nan")) for t in (q, k, v)]
                        ops.fa2_bwd(q, k, v, o, lse, do, *g, causal=causal, seqlens_k=sl)
                        return g
                    cases.append(("bwd dense %s D=%d causal=%d pad=%d" % (str(dt)[6:], D, causal, pad), run))
            for H_kv in (4, 1):
                for causal in (False, True):
                    torch.manual_seed(30 + D + H_kv + causal)
                    q, do = rn(sum(lq), 16, D, dt=dt), rn(sum(lq), 16, D, dt=dt)
                    k, v = rn(sum(lk), H_kv, D, dt=dt), rn(sum(lk), H_kv, D, dt=dt)
                    o, lse = torch.empty_like(q), torch.empty(sum(lq), 16, device=dev)
                    ops.fa2_fwd_varlen(q, k, v, o, cq, ck, max(lq), causal=causal, lse=lse)

                    def run(q=q, k=k, v=v, o=o, lse=lse, do=do, causal=causal):
                        g = [torch.full_like(t, float("nan")) for t in (q, k, v)]
                        ops.fa2_bwd_varlen(q, k, v, o, lse, do, *g, cq, ck, max(lq), max(lk), causal=causal)
                        return g
                    cases.append(("bwd packed %s D=%d H=16 H_kv=%d causal=%d" % (str(dt)[6:], D, H_kv, causal), run))
    return cases


def timed_cases(torch, ops):
    """(name, flop, run) for the timed shapes; run() is one call on preallocated tensors."""
    dev = "cuda"
    cases = []
    for B, H, N, D in ((4, 48, 8192, 64), (4, 64, 8192, 128)):
        q, k, v = [torch.randn(B, H, N, D, dtype=torch.half, device=dev) for _ in range(3)]
        o = torch.empty_like(q)
        cases.append(("dense (%d, %d, %d, %d)" % (B, H, N, D), 4.0 * B * H * N * N * D,
                      lambda q=q, k=k, v=v, o=o: ops.fa2_fwd(q, k, v, o)))
    B, H, N, D = 1, 32, 4096, 512
    q, k, v = [torch.randn(B, H, N, D, dtype=torch.half, device=dev) for _ in range(3)]
    o = torch.empty_like(q)
    cases.append(("ffpa (1, 32, 4096, 512)", 4.0 * B * H * N * N * D, lambda q=q, k=k, v=v, o=o: ops.ffpa_fwd(q, k, v, o)))
    B, N, H, H_kv, D = 4, 8192, 64, 8, 128
    q = torch.randn(B * N, H, D, dtype=torch.half, device=dev)
    k, v = [torch.randn(B * N, H_kv, D, dtype=torch.half, device=dev) for _ in range(2)]
    o = torch.empty_like(q)
    cu = torch.arange(0, (B + 1) * N, N, dtype=torch.int32, device=dev)
    cases.append(("packed GQA 4 x 8192 H 64 H_kv 8 D 128 causal", 2.0 * B * H * N * N * D,
                  lambda q=q, k=k, v=v, o=o: ops.fa2_fwd_varlen(q, k, v, o, cu, cu, N, causal=True)))
    for B in (1, 64):
        S, Lq, H, H_kv, D = 8192, 1, 32, 8, 128
        q = torch.randn(B, Lq, H, D, dtype=torch.half, device=dev)
        kc, vc = [torch.randn(B, S, H_kv, D, dtype=torch.half, device=dev) for _ in range(2)]
        o = torch.empty_like(q)
        lens = torch.full((B,), S, dtype=torch.int32, device=dev)
        cases.append(("decode B %d Lq 1 H 32 H_kv 8 D 128, 8K cache" % B, 4.0 * B * Lq * H * S * D,
                      lambda q=q, kc=kc, vc=vc, o=o, lens=lens: ops.fa2_fwd_kvcache(q, kc, vc, o, lens)))
    # the backward's work counted as flash-attn does: 2.5 times the forward's (5 products), half of it when causal
    for causal in (False, True):
        for B, H, N, D in ((4, 48, 8192, 64), (4, 64, 8192, 128)):
            q, k, v, do = [torch.randn(B, H, N, D, dtype=torch.half, device=dev) for _ in range(4)]
            o, lse = torch.empty_like(q), torch.empty(B, H, N, device=dev)
            ops.fa2_fwd(q, k, v, o, causal=causal, lse=lse)
            g = [torch.empty_like(q) for _ in range(3)]
            cases.append(("bwd dense (%d, %d, %d, %d)%s" % (B, H, N, D, " causal" if causal else ""),
                          10.0 * B * H * N * N * D / (2 if causal else 1),
                          lambda q=q, k=k, v=v, o=o, lse=lse, do=do, g=g, causal=causal:
                          ops.fa2_bwd(q, k, v, o, lse, do, *g, causal=causal)))
        B, N, H, H_kv, D = 4, 8192, 64, 8, 128
        q, do = [torch.randn(B * N, H, D, dtype=torch.half, device=dev) for _ in range(2)]
        k, v = [torch.randn(B * N, H_kv, D, dtype=torch.half, device=dev) for _ in range(2)]
        o, lse = torch.empty_like(q), torch.empty(B * N, H, device=dev)
        cu = torch.arange(0, (B + 1) * N, N, dtype=torch.int32, device=dev)
        ops.fa2_fwd_varlen(q, k, v, o, cu, cu, N, causal=causal, lse=lse)
        g = [torch.empty_like(t) for t in (q, k, v)]
        cases.append(("bwd packed GQA 4 x 8192 H 64 H_kv 8 D 128%s" % (" causal" if causal else ""),
                      10.0 * B * H * N * N * D / (2 if causal else 1),
                      lambda q=q, k=k, v=v, o=o, lse=lse, do=do, g=g, cu=cu, causal=causal:
                      ops.fa2_bwd_varlen(q, k, v, o, lse, do, *g, cu, cu, N, N, causal=causal)))
    return cases


def eager_cases(torch, ops):
    """(name, flop, run) timed call by call without a graph, so the host's share of a call of about 10 us shows:
    decode and append (one new token, no rotary) at B 1 against an 8K cache."""
    dev = "cuda"
    S, H, H_kv, D = 8192, 32, 8, 128
    q = torch.randn(1, 1, H, D, dtype=torch.half, device=dev)
    kc, vc = [torch.randn(1, S, H_kv, D, dtype=torch.half, device=dev) for _ in range(2)]
    kn, vn = [torch.randn(1, 1, H_kv, D, dtype=torch.half, device=dev) for _ in range(2)]
    o = torch.empty_like(q)
    lens = torch.full((1,), S - 1, dtype=torch.int32, device=dev)
    return [("eager decode B 1 Lq 1 H 32 H_kv 8 D 128, 8K cache", 4.0 * H * S * D,
             lambda: ops.fa2_fwd_kvcache(q, kc, vc, o, lens)),
            ("eager append B 1 L_new 1 H 32 H_kv 8 D 128, 8K cache", 4.0 * H * S * D,
             lambda: ops.fa2_fwd_kvcache(q, kc, vc, o, lens, k=kn, v=vn))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build-base", metavar="REV", help="build REV's library into build_ab/base and exit")
    ap.add_argument("--base-lib", default=BASE_LIB, help="the library to compare against (default: build_ab/base's)")
    ap.add_argument("--rounds", type=int, default=9)
    args = ap.parse_args()
    if args.build_base:
        build_base(args.build_base)
        return

    import torch

    info = gpu_info(torch)
    from b200k import _loader, ops

    libs = {"base": load_lib(args.base_lib), "new": _loader.lib}
    print(json.dumps(dict(info, base_lib=os.path.relpath(os.path.abspath(args.base_lib), ROOT), rounds=args.rounds)),
          flush=True)

    bad, slow = compare_and_time(torch, libs, equal_cases(torch, ops), timed_cases(torch, ops), args.rounds)
    _, slow_eager = compare_and_time(torch, libs, [], eager_cases(torch, ops), args.rounds, graph=False)
    print(json.dumps({"differing_cases": bad, "new_median_above_base_max": slow + slow_eager}), flush=True)
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
