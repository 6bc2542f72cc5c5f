"""CPU reference for KV-cache attention over fp8 caches (b200k_fa2_kvcache_fp8, b200k_fa2_varlen_paged_fp8), used by
test_attention_kvcache_fp8_cpu.py and test_gpu_attention_kvcache_fp8.py.  The attention itself is the 16-bit one on
dequantized caches; what is new is the two conversions:
  quantize    x -> fp8: torch's float8 cast of float(x) / scale[h] after a clamp to the format's largest finite value,
              which is cvt.rn.satfinite (round to nearest even, saturate, NaN stays NaN)
  dequantize  fp8 -> dtype(fp8) * scale[h]: exact for every code (both formats fit f16 and bf16) and, with power-of-two
              scales, for every product that stays a normal dtype value
Scales are per K/V head, the third dim of a [pages, page_size, H_kv, D] or [B, S, H_kv, D] cache."""
from __future__ import annotations

import torch

FORMATS = (torch.float8_e4m3fn, torch.float8_e5m2)
FMAX = {torch.float8_e4m3fn: 448.0, torch.float8_e5m2: 57344.0}


def _per_head(scale, H_kv: int) -> torch.Tensor:
    if scale is None:
        return torch.ones(H_kv, dtype=torch.float32)
    return torch.as_tensor(scale, dtype=torch.float32).cpu().reshape(H_kv)


def quantize(x: torch.Tensor, fmt: torch.dtype, scale=None) -> torch.Tensor:
    """The fp8 cache (on the CPU) for 16-bit values x [..., H_kv, D]: satfinite(float(x) / scale[h])."""
    H_kv = x.size(-2)
    s = _per_head(scale, H_kv).view(H_kv, 1)
    y = x.cpu().float() / s
    return y.clamp(-FMAX[fmt], FMAX[fmt]).to(fmt)


def dequantize(x8: torch.Tensor, dtype: torch.dtype, scale=None) -> torch.Tensor:
    """fp8 [..., H_kv, D] -> dtype(x8) * scale[h] on the CPU, rounded once to dtype (torch.float32: not rounded)."""
    H_kv = x8.size(-2)
    s = _per_head(scale, H_kv).view(H_kv, 1)
    return (x8.cpu().float() * s).to(dtype)


def every_code(fmt: torch.dtype) -> torch.Tensor:
    """All 256 codes of the format, as fp8 values in code order."""
    return torch.arange(256, dtype=torch.int32).to(torch.uint8).view(fmt)
