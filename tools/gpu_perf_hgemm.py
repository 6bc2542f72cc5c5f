"""A/B timing of the GEMM against an earlier build of the library and against cuBLAS, in one process.

A second copy of libb200k.so, built from another git revision, is loaded through ctypes next to the one in the tree.
Each case alternates the base build, the tree's build and torch.matmul (cuBLAS) on the same tensors, one batch of
calls per arm per round, timed with CUDA events.  Every case checks that the two builds give the same bits.  The first
line names the GPU, its power limit and its maximum SM clock, read in the same run.

    python tools/gpu_perf_hgemm.py --build-base REV        # CPU is enough: git archive REV -> build_ab/base, make
    python tools/gpu_perf_hgemm.py [--base-lib PATH] [--rounds 15]

Cases: fp16 NN at 2048, 4096, 8192 and 16384; fp16 TN (B stored [N,K]), bf16 NN and TF32 NN (fp32 storage) at 8192.
"""
import argparse
import json
import os
import time

from gpu_timing import BASE_LIB, ROOT, build_base, gpu_info, load_lib, stats, time_rounds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build-base", metavar="REV", help="build REV's library into build_ab/base and exit")
    ap.add_argument("--base-lib", default=BASE_LIB, help="the library to compare against (default: build_ab/base's)")
    ap.add_argument("--rounds", type=int, default=15)
    args = ap.parse_args()
    if args.build_base:
        build_base(args.build_base)
        return

    import torch

    info = gpu_info(torch)
    from b200k import _loader

    libs = {"base": load_lib(args.base_lib), "new": _loader.lib}
    print(json.dumps(dict(info, base_lib=os.path.relpath(os.path.abspath(args.base_lib), ROOT), rounds=args.rounds)),
          flush=True)

    F32, F16, BF16 = _loader.F32, _loader.F16, _loader.BF16
    cases = [("f16_nn", torch.float16, F16, False, n) for n in (2048, 4096, 8192, 16384)]
    cases += [("f16_tn", torch.float16, F16, True, 8192), ("bf16_nn", torch.bfloat16, BF16, False, 8192),
              ("tf32_nn", torch.float32, F32, False, 8192)]
    torch.backends.cuda.matmul.allow_tf32 = True  # cuBLAS on the same TF32 tensor-core path
    for name, dt, enum, tn, n in cases:
        torch.manual_seed(1)
        a = torch.randn(n, n, device="cuda").to(dt)
        b = torch.randn(n, n, device="cuda").to(dt)  # tn: this is B^T, stored [N,K]
        outs = {k: torch.zeros(n, n, dtype=dt, device="cuda") for k in ("base", "new", "cublas")}
        stream = torch.cuda.current_stream().cuda_stream

        def ours(key):
            lib, c = libs[key], outs[key]

            def run():
                rc = lib.b200k_gemm(a.data_ptr(), b.data_ptr(), c.data_ptr(), n, n, n, int(tn), enum, 0, stream)
                if rc != 0:
                    raise RuntimeError("%s: %s" % (key, lib.b200k_last_error().decode()))
            return run

        bmat = b.t() if tn else b
        arms = {"base": ours("base"), "new": ours("new"), "cublas": lambda: torch.matmul(a, bmat, out=outs["cublas"])}
        flop = 2.0 * n ** 3
        # about 200 ms of work per arm per round: at a 400 W limit the clock swings on a scale of tens of milliseconds
        iters = max(3, int(200e-3 / (flop / 400e12)))
        # the GPU out of its idle state, as bench.py does: untimed launches of every arm, then a pause
        for _ in range(max(1, 40 // iters)):
            for fn in arms.values():
                for _ in range(iters):
                    fn()
        torch.cuda.synchronize()
        time.sleep(1.0)
        tflops = {k: [flop / s * 1e-12 for s in v] for k, v in time_rounds(arms, iters, args.rounds).items()}
        med = {k: stats(v)[0] for k, v in tflops.items()}
        line = {"case": name, "mnk": n, "iters_per_round": iters, "bit_equal_new_base": bool(torch.equal(outs["new"], outs["base"]))}
        for k, v in tflops.items():
            line[k + "_tflops"] = round(med[k], 1)
            line[k + "_min_max"] = [round(min(v), 1), round(max(v), 1)]
        line["new_over_base"] = round(med["new"] / med["base"], 4)
        line["new_over_cublas"] = round(med["new"] / med["cublas"], 4)
        line["new_min_above_base_max"] = min(tflops["new"]) > max(tflops["base"])
        print(json.dumps(line), flush=True)
        del a, b, outs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
