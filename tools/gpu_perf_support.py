"""Achieved HBM bandwidth of the support kernels (algorithmic bytes / CUDA-event time), one JSON line per kernel after
a first line that names the GPU, its power limit and its maximum SM clock, read in the same run.  Inputs are larger
than the 50 MB L2 or rotated over several buffers, so every launch streams from HBM.

    python tools/gpu_perf_support.py [--iters 20]
"""
import argparse
import json
import os

import torch
from gpu_timing import ROOT, gpu_info, time_rounds
from b200k import ops


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    print(json.dumps(gpu_info(torch)), flush=True)
    peak = None
    try:
        peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))).get("hbm_gbs")
    except Exception:
        pass
    torch.manual_seed(0)
    dev = "cuda"
    n = 128 * 1024 * 1024
    a = torch.randn(n, device=dev)
    b = torch.randn(n, device=dev)
    c = torch.empty_like(a)
    ah, bh, ch = a.half(), b.half(), torch.empty(n, dtype=torch.half, device=dev)
    x16 = torch.randn(32768, 8192, dtype=torch.half, device=dev)
    y16 = torch.empty_like(x16)
    x32 = torch.randn(32768, 4096, device=dev)
    y32 = torch.empty_like(x32)
    xs = torch.randn(262144, 1024, dtype=torch.half, device=dev)
    ys = torch.empty_like(xs)
    w = torch.randn(131072, 1024, dtype=torch.half, device=dev)
    idx = torch.randint(0, 131072, (262144,), dtype=torch.int32, device=dev)
    eo = torch.empty(262144, 1024, dtype=torch.half, device=dev)
    hin = torch.randint(0, 256, (n,), dtype=torch.int32, device=dev)
    gx32, gy32 = torch.randn(4096, 1, device=dev), torch.empty(32768, 1, device=dev)
    gx16, gy16 = torch.randn(8192, 1, dtype=torch.half, device=dev), torch.empty(32768, 1, dtype=torch.half, device=dev)
    cases = [
        ("elementwise_add_f32", lambda: ops.elementwise_add(a, b, c), 3 * n * 4),
        ("elementwise_add_f16", lambda: ops.elementwise_add(ah, bh, ch), 3 * n * 2),
        ("block_all_reduce_sum_f32", lambda: ops.block_all_reduce_sum(a), n * 4),
        ("block_all_reduce_sum_f16", lambda: ops.block_all_reduce_sum(ah), n * 2),
        ("safe_softmax_f16_h8192", lambda: ops.softmax(x16, y16, ops.SOFTMAX_SAFE), 2 * x16.numel() * 2),
        ("safe_softmax_f16_h1024", lambda: ops.softmax(xs, ys, ops.SOFTMAX_SAFE), 2 * xs.numel() * 2),
        ("safe_softmax_f32_h4096", lambda: ops.softmax(x32, y32, ops.SOFTMAX_SAFE), 2 * x32.numel() * 4),
        ("online_softmax_f32_h4096", lambda: ops.softmax(x32, y32, ops.SOFTMAX_ONLINE), 2 * x32.numel() * 4),
        ("softmax_all_f32", lambda: ops.softmax(x32, y32, ops.SOFTMAX_ALL), 3 * x32.numel() * 4),
        ("rms_norm_f16_k8192", lambda: ops.rms_norm(x16, y16, 1.0), 2 * x16.numel() * 2),
        ("rms_norm_f32_k4096", lambda: ops.rms_norm(x32, y32, 1.0), 2 * x32.numel() * 4),
        ("rope_f32_ref_quirk", lambda: ops.rope_f32(x32, y32, True), 2 * x32.numel() * 4),
        ("rope_f32_textbook", lambda: ops.rope_f32(x32, y32, False), 2 * x32.numel() * 4),
        ("embedding_f16_e1024", lambda: ops.embedding(idx, w, eo), 2 * eo.numel() * 2 + idx.numel() * 4),
        ("histogram_i32_256bins", lambda: ops.histogram_i32(hin, nbins=256), n * 4),
        # second set (SURVEY.md section 8f-3)
        ("relu_f32", lambda: ops.activation(a, c, "relu"), 2 * n * 4),
        ("gelu_f32", lambda: ops.activation(a, c, "gelu"), 2 * n * 4),
        ("sigmoid_f16", lambda: ops.activation(ah, ch, "sigmoid"), 2 * n * 2),
        ("gelu_f16", lambda: ops.activation(ah, ch, "gelu"), 2 * n * 2),
        ("swish_f16", lambda: ops.activation(ah, ch, "swish"), 2 * n * 2),
        ("elu_f16", lambda: ops.activation(ah, ch, "elu"), 2 * n * 2),
        ("hardswish_f16", lambda: ops.activation(ah, ch, "hardswish"), 2 * n * 2),
        ("layer_norm_f16_k8192", lambda: ops.layer_norm(x16, y16, 1.0, 0.0), 2 * x16.numel() * 2),
        ("layer_norm_f16_k1024", lambda: ops.layer_norm(xs, ys, 1.0, 0.0), 2 * xs.numel() * 2),
        ("layer_norm_f32_k4096", lambda: ops.layer_norm(x32, y32, 1.0, 0.0), 2 * x32.numel() * 4),
        ("dot_prod_f32", lambda: ops.dot_prod(a, b), 2 * n * 4),
        ("dot_prod_f16", lambda: ops.dot_prod(ah, bh), 2 * n * 2),
        ("mat_transpose_f32_32768x4096", lambda: ops.mat_transpose(x32, y32.view(4096, 32768)), 2 * x32.numel() * 4),
        ("sgemv_32768x4096", lambda: ops.gemv(x32, gx32, gy32), x32.numel() * 4),
        ("hgemv_32768x8192", lambda: ops.gemv(x16, gx16, gy16), x16.numel() * 2),
    ]
    for name, fn, nbytes in cases:
        t = time_rounds({name: fn}, args.iters, 1)[name][0]
        out = {"kernel": name, "us": round(t * 1e6, 1), "algorithmic_bytes": nbytes, "gbps": round(nbytes / t * 1e-9, 1)}
        if peak:
            out["frac_of_measured_hbm_peak"] = round(out["gbps"] / peak, 3)
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
