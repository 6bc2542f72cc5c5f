"""CPU: argument validation of the packed variable-length attention entry point (before any CUDA call), the Python
wrapper's checks, and the packed layout of the CPU reference (attention_ref.py) against the dense oracle and against
per-sequence SDPA."""
import ctypes
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))  # attention_ref.py sits next to this file
import attention_ref as ar  # noqa: E402

from b200k import _loader as L
from oracle import oracle

ONE = ctypes.c_void_p(16)  # never dereferenced: validation fails first


def _call(ptrs=(ONE,) * 6, B=2, max_q=64, total_q=100, total_k=100, H=8, H_kv=2, D=64, dtype=L.F16, causal=0):
    return L.lib.b200k_fa2_fwd_varlen(*ptrs, B, max_q, total_q, total_k, H, H_kv, D, 0.0, dtype, causal, None)


@pytest.mark.parametrize("null_at", range(6))
def test_null_pointers_are_refused(null_at):
    ptrs = [ONE] * 6
    ptrs[null_at] = None
    assert _call(ptrs=ptrs) == L.EARG


@pytest.mark.parametrize("dtype", [L.F32, L.I8, L.FP8_E4M3, 99])
def test_unsupported_dtypes_are_refused(dtype):
    assert _call(dtype=dtype) == L.EDTYPE


@pytest.mark.parametrize("D", [0, 16, 48, 80, 160, 256])
def test_unsupported_head_dims_are_refused(D):
    assert _call(D=D) == L.EHEADDIM
    assert b"headdim not support!" in L.lib.b200k_last_error()


@pytest.mark.parametrize("kw", [
    dict(B=0), dict(B=-1),
    dict(H=0), dict(H_kv=0), dict(H=8, H_kv=3), dict(H=2, H_kv=4),
    dict(max_q=0), dict(max_q=101),                            # max_seqlen_q outside [1, total_q]
    dict(total_q=0, max_q=1), dict(total_k=0), dict(total_k=-5),
    dict(total_q=2 ** 31, max_q=1), dict(total_k=2 ** 31),
    dict(B=65536, H=1, H_kv=1), dict(B=2, H=32768, H_kv=1),    # B * H CTAs per query tile exceed the grid
])
def test_bad_shapes_are_refused(kw):
    assert _call(**kw) == L.ESHAPE


def test_valid_arguments_reach_the_device():
    """Validation passes; without a GPU the call then fails loudly at the device query instead of doing anything else."""
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    for kw in (dict(), dict(total_q=2 ** 31 - 1, max_q=2 ** 31 - 1), dict(B=65535, H=1, H_kv=1), dict(H=8, H_kv=8),
               dict(dtype=L.BF16, D=128, causal=1)):
        assert _call(**kw) in (L.ECUDA, L.EARCH), kw


def test_python_wrapper_checks():
    from b200k import ops

    q = torch.zeros(10, 4, 64, dtype=torch.half)
    k = torch.zeros(12, 2, 64, dtype=torch.half)
    cu = torch.tensor([0, 4, 10], dtype=torch.int32)
    cuk = torch.tensor([0, 5, 12], dtype=torch.int32)
    with pytest.raises(RuntimeError, match="values must be torch::kHalf"):
        ops.fa2_fwd_varlen(q, k.float(), k, q, cu, cuk, 6)
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        ops.fa2_fwd_varlen(q, k, k[:, :1].contiguous(), q, cu, cuk, 6)            # V heads differ from K heads
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        ops.fa2_fwd_varlen(q, torch.zeros(12, 3, 64, dtype=torch.half), torch.zeros(12, 3, 64, dtype=torch.half), q, cu,
                           cuk, 6)                                                   # H % H_kv != 0
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        ops.fa2_fwd_varlen(q[None], k, k, q, cu, cuk, 6)
    with pytest.raises(RuntimeError, match="headdim not support!"):
        q2, k2 = torch.zeros(10, 4, 48, dtype=torch.half), torch.zeros(12, 2, 48, dtype=torch.half)
        ops.fa2_fwd_varlen(q2, k2, k2, q2, cu, cuk, 6)
    with pytest.raises(RuntimeError, match="values must be torch::kInt32"):
        ops.fa2_fwd_varlen(q, k, k, q, cu.long(), cuk, 6)
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        ops.fa2_fwd_varlen(q, k, k, q, cu, cuk[:2], 6)                              # B + 1 entries each
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        ops.fa2_fwd_varlen(q, k, k, q, cu[:1], cuk[:1], 6)                          # B >= 1
    with pytest.raises(RuntimeError, match="CUDA device"):
        ops.fa2_fwd_varlen(q, k, k, q, cu, cuk, 6)                                  # there is no CPU path


def _pack(lens, H, D, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0).tolist()), dtype=torch.int32)
    return torch.randn(int(cu[-1]), H, D, generator=g).to(dtype), cu


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("causal", [False, True])
def test_oracle_equal_lengths_matches_dense_oracle(dtype, causal):
    B, H, N, D = 3, 4, 37, 32
    g = torch.Generator().manual_seed(3)
    q, k, v = [torch.randn(B, H, N, D, generator=g).to(dtype) for _ in range(3)]
    want = oracle.attention(q, k, v, causal=causal)                                  # [B, H, N, D]
    packed = [t.transpose(1, 2).reshape(B * N, H, D) for t in (q, k, v)]
    cu = torch.arange(0, (B + 1) * N, N, dtype=torch.int32)
    got = ar.packed(*packed, cu, cu, causal=causal)[0].to(dtype)
    assert got.dtype == dtype
    assert torch.allclose(got.float(), want.transpose(1, 2).reshape(B * N, H, D).float(), rtol=1e-2, atol=1e-3)


def _sdpa_per_sequence(q, k, v, cq, ck, causal):
    """F.scaled_dot_product_attention(enable_gqa=True) per sequence, fp32, explicit bottom-right boolean mask."""
    out = torch.zeros(q.shape)
    for b in range(len(cq) - 1):
        Lq, Lk = cq[b + 1] - cq[b], ck[b + 1] - ck[b]
        if Lq == 0 or Lk == 0:
            continue
        qs, ks, vs = (t.float().transpose(0, 1)[None] for t in (q[cq[b]:cq[b + 1]], k[ck[b]:ck[b + 1]], v[ck[b]:ck[b + 1]]))
        mask = None
        if causal:
            mask = torch.arange(Lk).view(1, Lk) <= torch.arange(Lq).view(Lq, 1) + (Lk - Lq)
        o = F.scaled_dot_product_attention(qs, ks, vs, attn_mask=mask, enable_gqa=True)[0].transpose(0, 1)
        if causal:
            o = o.masked_fill(~mask.any(-1).view(Lq, 1, 1), 0.0)                   # SDPA gives NaN for rows with no key
        out[cq[b]:cq[b + 1]] = o
    return out


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("H,H_kv", [(4, 4), (4, 2), (8, 1)])
@pytest.mark.parametrize("lq,lk", [([5, 0, 33, 1, 70], [5, 9, 40, 1, 70]),       # Lq <= Lk, an empty query sequence
                                   ([30, 12, 1, 64], [7, 12, 3, 0]),              # Lq > Lk, an empty key sequence
                                   ([128, 129, 77], [129, 128, 200])])
def test_oracle_matches_sdpa_gqa_with_bottom_right_mask(lq, lk, H, H_kv, causal):
    D = 32
    q, cq = _pack(lq, H, D, torch.float16, seed=sum(lq) + H)
    k, ck = _pack(lk, H_kv, D, torch.float16, seed=sum(lk) + H_kv)
    v, _ = _pack(lk, H_kv, D, torch.float16, seed=sum(lk) + 7)
    got = ar.packed(q, k, v, cq, ck, causal=causal)[0].half()
    want = _sdpa_per_sequence(q, k, v, cq.tolist(), ck.tolist(), causal).half()
    assert torch.allclose(got.float(), want.float(), rtol=1e-3, atol=1e-3)


def test_oracle_rows_that_see_no_key_are_zero():
    H, D = 2, 32
    lq, lk = [6, 4, 3], [2, 0, 3]
    q, cq = _pack(lq, H, D, torch.float16, seed=1)
    k, ck = _pack(lk, H, D, torch.float16, seed=2)
    v, _ = _pack(lk, H, D, torch.float16, seed=3)
    o = ar.packed(q, k, v, cq, ck, causal=True)[0].half()
    assert torch.isfinite(o.float()).all()
    assert (o[0:4] == 0).all()                 # sequence 0: Lq - Lk = 4 rows before the first key
    assert (o[4:6] != 0).any()
    assert (o[6:10] == 0).all()                # sequence 1: no keys at all
    assert (o[10:13] != 0).any()
    o = ar.packed(q, k, v, cq, ck, causal=False)[0].half()
    assert (o[6:10] == 0).all() and (o[0:6] != 0).any()
    # a row that sees exactly one key returns that key's V row
    assert torch.equal(ar.packed(q, k, v, cq, ck, causal=True)[0][4].half(), v[0])
