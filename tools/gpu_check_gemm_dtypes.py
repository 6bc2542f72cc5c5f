"""bf16 / TF32 builds of the GEMM kernel: quick correctness probe and throughput next to torch.matmul (cuBLAS)."""
import json, sys
import torch
from gpu_timing import ROOT, gpu_info, time_rounds
from b200k import ops
sys.path.insert(0, ROOT)
from oracle import oracle


def main():
    print(json.dumps(gpu_info(torch)), flush=True)
    torch.backends.cuda.matmul.allow_tf32 = True
    for dt in (torch.bfloat16, torch.float32):
        for tn in (False, True):
            torch.manual_seed(1)
            M, N, K = 512, 384, 256
            a = torch.randn(M, K, device="cuda").to(dt); b = torch.randn(K, N, device="cuda").to(dt)
            c = torch.full((M, N), float("nan"), device="cuda").to(dt)
            bb = b.t().contiguous().t() if tn else b
            try:
                ops.gemm(a, bb, c, tn=tn)
                torch.cuda.synchronize()
                exact, bound = oracle.gemm_tf32_bound(a, b)
                err = (c.double().cpu() - exact).abs()
                print(json.dumps({"dtype": str(dt), "tn": tn, "max_err_over_bound": float((err / bound).max()),
                                  "mean_rel": float(err.mean() / exact.abs().mean()), "finite": bool(torch.isfinite(c).all())}), flush=True)
            except Exception as e:  # noqa
                print(json.dumps({"dtype": str(dt), "tn": tn, "error": str(e)[:200]}), flush=True)
    for dt in (torch.float16, torch.bfloat16, torch.float32):
        for n in (4096, 8192):
            a = torch.randn(n, n, device="cuda").to(dt); b = torch.randn(n, n, device="cuda").to(dt); c = torch.empty(n, n, device="cuda").to(dt)
            # two rounds of 20 calls each, ours then cuBLAS; the second round is reported
            times = time_rounds({"ours": lambda: ops.gemm(a, b, c), "cublas": lambda: torch.matmul(a, b, out=c)}, 20, 2)
            t, tc = times["ours"][-1], times["cublas"][-1]
            print(json.dumps({"dtype": str(dt), "mnk": n, "tflops": round(2.0 * n ** 3 / t * 1e-12, 1), "cublas_tflops": round(2.0 * n ** 3 / tc * 1e-12, 1)}), flush=True)


if __name__ == "__main__":
    main()
