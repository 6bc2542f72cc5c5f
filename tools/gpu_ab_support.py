"""A/B of the bandwidth kernels against an earlier build of the library, in one process: same bits, then time.

Built like tools/gpu_ab_attention.py, on the loader and the compare-and-time loop of tools/gpu_timing.py: the base
build's libb200k.so is loaded through ctypes next to the one in the tree, and every call goes through b200k.ops, pointed
at one library or the other.

  1. Seeded inputs through both builds; the raw bits of every output must be equal (NaN and -0 count):
     softmax modes 0-3, RMS norm in every acc_f16 / eps_inside_k combination and layer norm with both eps forms, f32
     and f16, at H = 1024, 1024 + VN, 4096, 4096 + VN, 8192, 8192 + VN and 1024 + VN - 1 (both sides of every R, cached /
     re-read and vector / scalar switch), aligned and one element off; block_all_reduce_sum for all six dtypes with and
     without half accumulation, aligned and off; dot_prod f32 / f16, aligned and off; the fp32 transpose (16-byte,
     ragged, off) and the batched 16-bit one (f16, bf16, ragged); the seven activations in both dtypes with both
     ref_clamp settings; and the fp32 NN GEMM, which transposes B through the 16-byte fp32 transpose.
  2. Time per call of each build, alternating, one CUDA graph per build per round: the support rows of bench.py and
     the workloads on the other side of each path switch (see timed_cases), on inputs larger than the 50 MB L2, and
     the fp32 NN GEMM at 8192.  Each line gives the median and min - max of both builds.

The first line names the GPU, its power limit and its maximum SM clock, read in the same run.

    python tools/gpu_ab_support.py --build-base REV        # CPU is enough: git archive REV -> build_ab/base, make
    python tools/gpu_ab_support.py [--base-lib PATH] [--rounds 9]
"""
import argparse
import json
import os
import sys

from gpu_timing import BASE_LIB, ROOT, build_base, compare_and_time, gpu_info, load_lib


def equal_cases(torch, ops):
    """(name, run) pairs; run() makes fresh NaN-filled outputs from the case's seeded inputs and returns them."""
    dev = "cuda"
    cases = []

    def inp(shape, dt, off, scale=1.0, shift=0.0):
        """Seeded values in a view `off` elements into its buffer (off = 1: not 16-byte aligned)."""
        n = 1
        for d in shape:
            n *= d
        if dt == torch.int8:
            buf = torch.randint(-128, 128, (n + off,), dtype=dt, device=dev)
        else:
            buf = (torch.randn(n + off, device=dev) * scale + shift).to(dt)
        return buf[off:].view(shape)

    def out(shape, dt, off=0):
        n = 1
        for d in shape:
            n *= d
        return torch.full((n + off,), float("nan"), device=dev).to(dt)[off:].view(shape)

    S = 333  # not a multiple of the 8 or 2 rows a CTA holds at R = 32, 128
    for dt, vn in ((torch.float32, 4), (torch.float16, 8)):
        dn = str(dt)[6:]
        for H in (1024, 1024 + vn, 4096, 4096 + vn, 8192, 8192 + vn, 1024 + vn - 1):
            for off in (0, 1):
                torch.manual_seed(H + off)
                x = inp((S, H), dt, off, scale=4.0)
                xl = inp((S, H), dt, off, shift=0.5)
                tag = "%s H=%d off=%d" % (dn, H, off)
                for mode in ((0, 1, 2, 3) if dt == torch.float32 else (1, 2, 3)):
                    def run(x=x, mode=mode, off=off):
                        y = out(x.shape, x.dtype, off)
                        ops.softmax(x, y, mode)
                        return [y]
                    cases.append(("softmax mode %d %s" % (mode, tag), run))
                for acc in (False, True):
                    for inside in (False, True):
                        def run(x=x, acc=acc, inside=inside, off=off):
                            y = out(x.shape, x.dtype, off)
                            ops.rms_norm(x, y, 1.25, 1e-5, acc_f16=acc, eps_inside_k=inside)
                            return [y]
                        cases.append(("rms_norm acc_f16=%d eps_inside_k=%d %s" % (acc, inside, tag), run))
                for inside in (False, True):
                    def run(x=xl, inside=inside, off=off):
                        y = out(x.shape, x.dtype, off)
                        ops.layer_norm(x, y, 1.25, 0.375, 1e-5, eps_inside_k=inside)
                        return [y]
                    cases.append(("layer_norm eps_inside_k=%d %s" % (inside, tag), run))

    n = 10_000_019
    fp8 = [torch.float8_e4m3fn, torch.float8_e5m2] if hasattr(torch, "float8_e4m3fn") else []
    for dt in [torch.float32, torch.float16, torch.bfloat16, torch.int8] + fp8:
        for acc in (False, True):
            for off in (0, 1):
                torch.manual_seed(7 + off)
                x = inp((n,), dt, off)

                def run(x=x, acc=acc):
                    return [ops.block_all_reduce_sum(x, acc_f16=acc)]
                cases.append(("block_all_reduce_sum %s acc_f16=%d off=%d" % (str(dt)[6:], acc, off), run))
    for dt in (torch.float32, torch.float16):
        for off in (0, 1):
            torch.manual_seed(11 + off)
            a, b = inp((n,), dt, off), inp((n,), dt, off)
            cases.append(("dot_prod %s off=%d" % (str(dt)[6:], off), lambda a=a, b=b: [ops.dot_prod(a, b)]))

    for (M, N, off) in ((1024, 2048, 0), (1001, 777, 0), (1024, 2048, 1)):
        torch.manual_seed(M + N + off)
        x = inp((M, N), torch.float32, off)

        def run(x=x, off=off):
            y = out((x.shape[1], x.shape[0]), torch.float32, off)
            ops.mat_transpose(x, y)
            return [y]
        cases.append(("mat_transpose f32 %dx%d off=%d" % (M, N, off), run))
    for dt, shape in ((torch.float16, (4, 256, 512)), (torch.bfloat16, (3, 1001, 333)), (torch.float16, (2, 77, 1001))):
        torch.manual_seed(shape[1])
        x = inp(shape, dt, 0)

        def run(x=x):
            y = out(x.shape[:-2] + (x.shape[-1], x.shape[-2]), x.dtype)
            ops.transpose_16bit_batched(x, y)
            return [y]
        cases.append(("transpose_16bit_batched %s %s" % (str(dt)[6:], shape), run))

    for dt in (torch.float32, torch.float16):
        torch.manual_seed(13)
        x = inp((1_000_003,), dt, 0, scale=30.0)
        for op in ops.ACT_OPS:
            for clamp in (False, True):
                def run(x=x, op=op, clamp=clamp):
                    y = out(x.shape, x.dtype)
                    ops.activation(x, y, op, ref_clamp=clamp)
                    return [y]
                cases.append(("activation %s %s ref_clamp=%d" % (op, str(dt)[6:], clamp), run))

    for M, K, N in ((512, 1024, 768), (333, 1004, 780)):  # the fp32 GEMM takes K, N multiples of 4
        torch.manual_seed(K)
        a, b = inp((M, K), torch.float32, 0), inp((K, N), torch.float32, 0)

        def run(a=a, b=b):
            c = out((a.shape[0], b.shape[1]), torch.float32)
            ops.gemm(a, b, c)
            return [c]
        cases.append(("gemm f32 NN %dx%dx%d" % (M, K, N), run))
    return cases


def timed_cases(torch, ops):
    """(name, bytes, fn) for the bandwidth workloads: algorithmic bytes moved per call, fn one call on preallocated
    tensors, every input larger than L2."""
    dev = "cuda"
    torch.manual_seed(0)
    ne = 64 * 1024 * 1024  # bench.py's support shapes
    xa, xb, xc = torch.randn(ne, device=dev), torch.randn(ne, device=dev), torch.empty(ne, device=dev)
    xr = torch.randn(16384, 8192, dtype=torch.half, device=dev)
    yr = torch.empty_like(xr)
    xs = torch.randn(262144, 1024, dtype=torch.half, device=dev)
    ys = torch.empty_like(xs)
    x32 = torch.randn(32768, 4096, device=dev)
    y32 = torch.empty_like(x32)
    xlong = torch.randn(8192, 16384, dtype=torch.half, device=dev)  # past the 8192 values R = 256 threads cache
    ylong = torch.empty_like(xlong)
    x4097 = torch.randn(16384, 4097, device=dev)
    y4097 = torch.empty_like(x4097)
    r16 = torch.randn(128 * 1024 * 1024, device=dev).half()
    r8 = torch.randint(-128, 128, (256 * 1024 * 1024,), dtype=torch.int8, device=dev)
    ha, hb = xa.half(), xb.half()
    xt = torch.randn(32767, 4095, device=dev)
    yt = torch.empty_like(xt)
    xq = torch.randn(128, 256, 8192, dtype=torch.half, device=dev)
    yq = torch.empty(128, 8192, 256, dtype=torch.half, device=dev)
    cases = [
        ("elementwise_add_f32", 3 * ne * 4, lambda: ops.elementwise_add(xa, xb, xc)),
        ("block_all_reduce_sum_f32", ne * 4, lambda: ops.block_all_reduce_sum(xa)),
        ("safe_softmax_f16_h8192", 2 * xr.numel() * 2, lambda: ops.softmax(xr, yr, ops.SOFTMAX_SAFE)),
        ("rms_norm_f16_k8192", 2 * xr.numel() * 2, lambda: ops.rms_norm(xr, yr, 1.0)),
        ("layer_norm_f16_k8192", 2 * xr.numel() * 2, lambda: ops.layer_norm(xr, yr, 1.0, 0.0)),
        ("gelu_f32", 2 * ne * 4, lambda: ops.activation(xa, xc, "gelu")),
        ("dot_prod_f32", 2 * ne * 4, lambda: ops.dot_prod(xa, xb)),
        ("safe_softmax_f16_h1024", 2 * xs.numel() * 2, lambda: ops.softmax(xs, ys, ops.SOFTMAX_SAFE)),
        ("safe_softmax_f32_h4096", 2 * x32.numel() * 4, lambda: ops.softmax(x32, y32, ops.SOFTMAX_SAFE)),
        ("online_softmax_f32_h4096", 2 * x32.numel() * 4, lambda: ops.softmax(x32, y32, ops.SOFTMAX_ONLINE)),
        ("softmax_all_f32", 3 * x32.numel() * 4, lambda: ops.softmax(x32, y32, ops.SOFTMAX_ALL)),
        ("rms_norm_f16_k8192_acc_f16", 2 * xr.numel() * 2, lambda: ops.rms_norm(xr, yr, 1.0, acc_f16=True)),
        ("layer_norm_f16_k1024", 2 * xs.numel() * 2, lambda: ops.layer_norm(xs, ys, 1.0, 0.0)),
        ("layer_norm_f32_k4096", 2 * x32.numel() * 4, lambda: ops.layer_norm(x32, y32, 1.0, 0.0)),
        ("safe_softmax_f16_h16384_reread", 2 * xlong.numel() * 2, lambda: ops.softmax(xlong, ylong, ops.SOFTMAX_SAFE)),
        ("layer_norm_f16_k16384_reread", 2 * xlong.numel() * 2, lambda: ops.layer_norm(xlong, ylong, 1.0, 0.0)),
        ("layer_norm_f32_k4097_scalar", 2 * x4097.numel() * 4, lambda: ops.layer_norm(x4097, y4097, 1.0, 0.0)),
        ("block_all_reduce_sum_f16", r16.numel() * 2, lambda: ops.block_all_reduce_sum(r16)),
        ("block_all_reduce_sum_i8", r8.numel(), lambda: ops.block_all_reduce_sum(r8)),
    ]
    if hasattr(torch, "float8_e4m3fn"):
        r8e = r8.view(torch.float8_e4m3fn)
        cases.append(("block_all_reduce_sum_e4m3", r8e.numel(), lambda: ops.block_all_reduce_sum(r8e)))
    cases += [
        ("dot_prod_f16", 2 * ha.numel() * 2, lambda: ops.dot_prod(ha, hb)),
        ("mat_transpose_f32_32768x4096", 2 * x32.numel() * 4, lambda: ops.mat_transpose(x32, y32.view(4096, 32768))),
        ("mat_transpose_f32_32767x4095", 2 * xt.numel() * 4, lambda: ops.mat_transpose(xt, yt.view(4095, 32767))),
        ("transpose_16bit_batched_128x256x8192", 2 * xq.numel() * 2, lambda: ops.transpose_16bit_batched(xq, yq)),
    ]
    return cases


def gemm_case(torch, ops):
    """The fp32 NN GEMM at 8192 (TF32 tensor cores, B transposed through scratch by the fp32 transpose)."""
    n = 8192
    torch.manual_seed(1)
    a, b = torch.randn(n, n, device="cuda"), torch.randn(n, n, device="cuda")
    c = torch.empty_like(a)
    return [("gemm_f32_nn_8192", 2.0 * n ** 3, lambda: ops.gemm(a, b, c))]


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
    bad, slow = compare_and_time(torch, libs, equal_cases(torch, ops), timed_cases(torch, ops), args.rounds,
                                 unit=("gbps", 1e-9))
    torch.cuda.empty_cache()
    _, slow_gemm = compare_and_time(torch, libs, [], gemm_case(torch, ops), args.rounds)
    print(json.dumps({"differing_cases": bad, "new_median_above_base_max": slow + slow_gemm}), flush=True)
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
