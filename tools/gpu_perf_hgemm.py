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
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "cuda-learn-notes_b200", "b200k", "libb200k.so")
BASE_DIR = os.path.join(ROOT, "build_ab", "base")
BASE_LIB = os.path.join(BASE_DIR, "cuda-learn-notes_b200", "b200k", "libb200k.so")

# dtype enums of include/b200k.h
F32, F16, BF16 = 0, 1, 2


def build_base(rev):
    """The whole tree at `rev` into build_ab/base (git-ignored), then its library with its own Makefile."""
    if os.path.isdir(BASE_DIR):
        subprocess.run(["rm", "-rf", BASE_DIR], check=True)
    os.makedirs(BASE_DIR)
    archive = subprocess.run(["git", "-C", ROOT, "archive", rev], capture_output=True, check=True).stdout
    subprocess.run(["tar", "-x", "-C", BASE_DIR], input=archive, check=True)
    subprocess.run(["make", "-C", os.path.join(BASE_DIR, "cuda-learn-notes_b200", "csrc"), "-j", str(os.cpu_count() or 4)],
                   check=True, stdout=subprocess.DEVNULL)
    print("built %s at %s" % (BASE_LIB, subprocess.run(["git", "-C", ROOT, "rev-parse", rev], capture_output=True,
                                                      text=True, check=True).stdout.strip()))


def load(path):
    lib = ctypes.CDLL(os.path.abspath(path))
    c_void_p, c_int, c_int64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
    lib.b200k_gemm.argtypes = [c_void_p] * 3 + [c_int64] * 3 + [c_int, c_int, c_int, c_void_p]
    lib.b200k_gemm.restype = c_int
    lib.b200k_last_error.restype = ctypes.c_char_p
    return lib


def gpu_info(torch):
    """Name, power limit and maximum SM clock of the current GPU (read-only nvidia-smi query)."""
    info = {"gpu": torch.cuda.get_device_name(), "power_limit_w": None, "max_sm_mhz": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, power, mhz = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        info.update(gpu=name, power_limit_w=float(power), max_sm_mhz=float(mhz))
    except Exception as e:  # the name from torch stays; the missing fields are reported as such
        info["nvidia_smi_error"] = str(e)[:200]
    return info


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

    if not torch.cuda.is_available():
        sys.exit("gpu_perf_hgemm.py needs a CUDA device")
    libs = {"base": load(args.base_lib), "new": load(LIB)}
    info = gpu_info(torch)
    print(json.dumps(dict(info, base_lib=os.path.relpath(os.path.abspath(args.base_lib), ROOT), rounds=args.rounds)),
          flush=True)

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
        times = {k: [] for k in arms}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(args.rounds):
            for k, fn in arms.items():
                e0.record()
                for _ in range(iters):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                times[k].append(flop * iters / (e0.elapsed_time(e1) * 1e-3) * 1e-12)
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        line = {"case": name, "mnk": n, "iters_per_round": iters, "bit_equal_new_base": bool(torch.equal(outs["new"], outs["base"]))}
        for k, v in times.items():
            line[k + "_tflops"] = round(med[k], 1)
            line[k + "_min_max"] = [round(min(v), 1), round(max(v), 1)]
        line["new_over_base"] = round(med["new"] / med["base"], 4)
        line["new_over_cublas"] = round(med["new"] / med["cublas"], 4)
        line["new_min_above_base_max"] = min(times["new"]) > max(times["base"])
        print(json.dumps(line), flush=True)
        del a, b, outs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
