"""CPU: the fp8 quantise / dequantise reference (kvcache_fp8_oracle.py) and every argument check of the fp8 KV-cache
entry points, b200k_fa2_kvcache_fp8 (decode, with or without append) and b200k_fa2_varlen_paged_fp8, each made before
any CUDA call with the argument named.  No device is touched: the pointers are never dereferenced."""
import ctypes
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kvcache_fp8_oracle as fo  # noqa: E402

from b200k import _loader as L  # noqa: E402
from b200k import ops  # noqa: E402

P = 1 << 20  # a 16-byte aligned fake device address


# ------------------------------------------------------------------------------------------------ the reference
@pytest.mark.parametrize("fmt", fo.FORMATS)
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_every_code_converts_exactly(fmt, dtype):
    codes = fo.every_code(fmt)
    exact = codes.to(torch.float64)
    got = fo.dequantize(codes.view(1, 256, 1), dtype).view(256).to(torch.float64)
    fin = torch.isfinite(exact)
    assert torch.equal(got[fin], exact[fin])
    assert torch.isnan(got[torch.isnan(exact)]).all() and torch.isnan(exact).sum() > 0
    inf = torch.isinf(exact)
    assert torch.equal(got[inf], exact[inf])
    assert (inf.sum() == 2) == (fmt == torch.float8_e5m2)


@pytest.mark.parametrize("fmt", fo.FORMATS)
def test_quantise_round_trips_every_finite_code_and_saturates(fmt):
    codes = fo.every_code(fmt)
    vals = codes.float()
    fin = torch.isfinite(vals)
    for scale in (1.0, 0.25, 8.0):
        x = (vals[fin] * scale).view(1, 1, -1)  # one head; exact in fp32
        back = fo.quantize(x, fmt, torch.tensor([scale]))
        assert torch.equal(back.view(-1).view(torch.uint8), codes[fin].view(torch.uint8)) or \
            torch.equal(back.view(-1).float(), vals[fin])  # +0 / -0 both round-trip as values
    big = torch.tensor([1e30, -1e30, math.inf, -math.inf]).view(1, 1, 4)
    assert fo.quantize(big, fmt).view(-1).float().tolist() == [fo.FMAX[fmt], -fo.FMAX[fmt]] * 2
    assert torch.isnan(fo.quantize(torch.tensor([math.nan]).view(1, 1, 1), fmt).float()).all()


def test_quantise_rounds_to_nearest_even_per_head():
    # e4m3 spacing between 1 and 2 is 1/8: 1 + 1/16 ties to 1, 1 + 3/16 ties to 1 + 1/4
    x = torch.tensor([[[1 + 1 / 16, 1 + 3 / 16], [2 + 2 / 16, 2 + 6 / 16]]])  # [1, H_kv = 2, D = 2]
    q = fo.quantize(x, torch.float8_e4m3fn, torch.tensor([1.0, 2.0]))
    assert q.float()[0].tolist() == [[1.0, 1.25], [1.0, 1.25]]


# ------------------------------------------------------------------------------------------------ argument checks
def _decode_args(**kw):
    a = dict(Q=P, K=P, V=P, O=P, lse=None, seqlens=P, table=None, k_scale=None, v_scale=None, kv=L.FP8_E4M3,
             K_new=None, V_new=None, L_new=0, cos=None, sin=None, rs=0, rd=0, inter=0, B=2, Lq=1, H=8, H_kv=2, D=64,
             num_pages=2, page_size=256, pps=1, scale=0.0, dtype=L.F16, causal=0, ws=P, ws_bytes=1 << 30, stream=None)
    a.update(kw)
    return list(a.values())


def _decode(**kw):
    return L.lib.b200k_fa2_kvcache_fp8(*_decode_args(**kw))


def _paged(**kw):
    a = dict(Q=P, K=P, V=P, O=P, lse=None, cu_q=P, cu_k=P, table=P, k_scale=None, v_scale=None, kv=L.FP8_E4M3, B=2,
             max_q=8, total_q=16, H=8, H_kv=2, D=64, num_pages=8, page_size=64, pps=4, scale=0.0, dtype=L.F16,
             causal=0, stream=None)
    a.update(kw)
    return L.lib.b200k_fa2_varlen_paged_fp8(*a.values())


def _err():
    return L.last_error()


CASES_DECODE = [
    (dict(Q=None), L.EARG, "null pointer"),
    (dict(seqlens=None), L.EARG, "null pointer"),
    (dict(dtype=L.F32), L.EDTYPE, "dtype"),
    (dict(dtype=L.FP8_E4M3), L.EDTYPE, "dtype"),
    (dict(kv=L.F16), L.EDTYPE, "kv_dtype"),
    (dict(kv=L.BF16), L.EDTYPE, "kv_dtype"),
    (dict(kv=L.I8), L.EDTYPE, "kv_dtype"),
    (dict(D=80), L.EHEADDIM, "headdim"),
    (dict(H=6, H_kv=4), L.ESHAPE, "H % H_kv"),
    (dict(num_pages=3), L.ESHAPE, "contiguous cache"),
    (dict(table=P, num_pages=8, page_size=48, pps=4), L.ESHAPE, "page_size"),
    (dict(K=P + 8), L.EALIGN, "K_cache"),
    (dict(V=P + 8), L.EALIGN, "V_cache"),
    (dict(Q=P + 8), L.EALIGN, "Q"),
    (dict(O=P + 2), L.EALIGN, "O"),
    (dict(k_scale=P + 2), L.EALIGN, "k_scale"),
    (dict(v_scale=P + 1), L.EALIGN, "v_scale"),
    (dict(lse=P + 2), L.EALIGN, "lse"),
    (dict(ws=P + 8), L.EALIGN, "workspace"),
    (dict(cos=P, sin=P, rs=256, rd=64), L.EARG, "need K_new / V_new"),
    (dict(K_new=P), L.EARG, "K_new / V_new"),
    (dict(V_new=P), L.EARG, "K_new / V_new"),
    (dict(K_new=P, V_new=P, L_new=0), L.ESHAPE, "L_new"),
    (dict(K_new=P, V_new=P, L_new=1, cos=P), L.EARG, "rotary_cos and rotary_sin"),
    (dict(K_new=P, V_new=P, L_new=1, cos=P, sin=P, rs=256, rd=24), L.ESHAPE, "rotary_dim"),
    (dict(K_new=P, V_new=P, L_new=1, cos=P, sin=P, rs=100, rd=64), L.ESHAPE, "rotary_seqlen"),
    (dict(K_new=P + 8, V_new=P, L_new=1), L.EALIGN, "K_new"),
    (dict(K_new=P, V_new=P + 8, L_new=1), L.EALIGN, "V_new"),
    (dict(K_new=P, V_new=P, L_new=1, cos=P + 8, sin=P, rs=256, rd=64), L.EALIGN, "rotary_cos"),
    (dict(K_new=P, V_new=P, L_new=1, ws=P + 8), L.EALIGN, "workspace"),
]


@pytest.mark.parametrize("kw,code,msg", CASES_DECODE, ids=[str(c[0]) for c in CASES_DECODE])
def test_decode_refusals_before_cuda(kw, code, msg):
    assert _decode(**kw) == code
    err = _err()
    assert "b200k_fa2_kvcache_fp8:" in err and msg in err, err


CASES_PAGED = [
    (dict(table=None), L.EARG, "null pointer"),
    (dict(cu_k=None), L.EARG, "null pointer"),
    (dict(dtype=L.FP8_E5M2), L.EDTYPE, "dtype"),
    (dict(kv=L.F16), L.EDTYPE, "kv_dtype"),
    (dict(kv=7), L.EDTYPE, "kv_dtype"),
    (dict(D=40), L.EHEADDIM, "headdim"),
    (dict(page_size=24), L.ESHAPE, "page_size"),
    (dict(max_q=17), L.ESHAPE, "max_seqlen_q"),
    (dict(K=P + 4), L.EALIGN, "K_cache"),
    (dict(V=P + 4), L.EALIGN, "V_cache"),
    (dict(k_scale=P + 2), L.EALIGN, "k_scale"),
    (dict(v_scale=P + 3), L.EALIGN, "v_scale"),
    (dict(lse=P + 2), L.EALIGN, "lse"),
    (dict(table=P + 2), L.EALIGN, "block_table"),
]


@pytest.mark.parametrize("kw,code,msg", CASES_PAGED, ids=[str(c[0]) for c in CASES_PAGED])
def test_paged_refusals_before_cuda(kw, code, msg):
    assert _paged(**kw) == code
    err = _err()
    assert "b200k_fa2_varlen_paged_fp8:" in err and msg in err, err


def test_workspace_query_checks_before_the_device():
    n = ctypes.c_size_t(0)
    assert L.lib.b200k_fa2_kvcache_fp8_workspace_bytes(1, 1, 8, 2, 64, 128, 0, 0, None) == L.EARG
    assert L.lib.b200k_fa2_kvcache_fp8_workspace_bytes(1, 1, 8, 2, 48, 128, 0, 0, ctypes.byref(n)) == L.EHEADDIM
    assert L.lib.b200k_fa2_kvcache_fp8_workspace_bytes(1, 1, 8, 3, 64, 128, 1, 0, ctypes.byref(n)) == L.ESHAPE


# ------------------------------------------------------------------------------------------------ the Python wrapper
def _cpu(shape, dtype):
    return torch.zeros(shape, dtype=dtype)


@pytest.mark.parametrize("fmt", fo.FORMATS)
def test_wrapper_refuses_mixed_caches_and_scales_on_16_bit_caches(fmt):
    q, o = _cpu((2, 1, 8, 64), torch.float16), _cpu((2, 1, 8, 64), torch.float16)
    k8, v16 = _cpu((2, 128, 2, 64), fmt), _cpu((2, 128, 2, 64), torch.float16)
    lens, s = torch.zeros(2, dtype=torch.int32), torch.ones(2)
    with pytest.raises(RuntimeError, match="same fp8 dtype"):
        ops.fa2_fwd_kvcache(q, k8, v16, o, lens)
    with pytest.raises(RuntimeError, match="dequantize fp8 caches"):
        ops.fa2_fwd_kvcache(q, v16, v16, o, lens, k_scale=s)
    with pytest.raises(RuntimeError, match="dequantize fp8 caches"):
        ops.fa2_fwd_varlen(q[:, 0], v16, v16, o[:, 0], lens, lens, 1, v_scale=s)
    with pytest.raises(RuntimeError, match="block_table"):
        ops.fa2_fwd_varlen(q[:, 0], k8, k8, o[:, 0], lens, lens, 1)
    with pytest.raises(RuntimeError, match="CUDA device"):  # every check passes up to the device
        ops.fa2_fwd_kvcache(q, k8, k8, o, lens, k_scale=s, v_scale=s)
