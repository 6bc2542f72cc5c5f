"""CPU: argument validation of the KV-cache decode entry points (before any CUDA call), the Python wrapper's checks, and
the gather step of the CPU reference (kvcache_oracle.py): a contiguous cache and the same data paged under a shuffled
table give the same packed K/V."""
import ctypes
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))  # kvcache_oracle.py sits next to this file
import attention_ref as ar  # noqa: E402
import kvcache_oracle  # noqa: E402

from b200k import _loader as L

ONE = ctypes.c_void_p(16)  # never dereferenced: validation fails first


def _call(ptrs=(ONE,) * 6, B=2, Lq=1, H=8, H_kv=2, D=64, num_pages=10, page_size=64, pages_per_seq=4, dtype=L.F16,
          causal=0, ws=None, ws_bytes=0):
    return L.lib.b200k_fa2_fwd_kvcache(*ptrs, B, Lq, H, H_kv, D, num_pages, page_size, pages_per_seq, 0.0, dtype, causal,
                                       ws, ws_bytes, None)


@pytest.mark.parametrize("null_at", range(5))   # Q, K_cache, V_cache, O, cache_seqlens (a NULL block_table is valid)
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
    n = ctypes.c_size_t(7)
    assert L.lib.b200k_fa2_fwd_kvcache_workspace_bytes(1, 1, 8, 2, D, 1024, ctypes.byref(n)) == L.EHEADDIM


@pytest.mark.parametrize("kw", [
    dict(B=0), dict(Lq=0), dict(H=0), dict(H_kv=0), dict(H=8, H_kv=3), dict(H=2, H_kv=4),
    dict(num_pages=0), dict(page_size=0), dict(pages_per_seq=0), dict(page_size=-64),
    dict(page_size=8), dict(page_size=48), dict(page_size=96), dict(page_size=200),
    dict(num_pages=2 ** 26, page_size=64), dict(pages_per_seq=2 ** 25, page_size=64),   # > INT32_MAX cache rows
    dict(B=2 ** 16, Lq=2 ** 15, H=1, H_kv=1),                                            # B * Lq > INT32_MAX
    dict(B=65536, H=1, H_kv=1), dict(B=2, H=65536, H_kv=65536),                         # B * H_kv > 65535
    dict(B=1, Lq=65536 * 64 + 1, H=1, H_kv=1),                                           # token tiles > 65535
    dict(B=1, H=65536 * 64 + 64, H_kv=1),                                                # head tiles > 65535
])
def test_bad_shapes_are_refused(kw):
    assert _call(**kw) == L.ESHAPE


@pytest.mark.parametrize("kw", [dict(num_pages=3, pages_per_seq=1), dict(num_pages=2, pages_per_seq=2)])
def test_contiguous_cache_must_be_one_page_per_sequence(kw):
    ptrs = [ONE] * 5 + [None]
    assert _call(ptrs=ptrs, **kw) == L.ESHAPE


def test_workspace_query_checks():
    n = ctypes.c_size_t(0)
    assert L.lib.b200k_fa2_fwd_kvcache_workspace_bytes(1, 1, 8, 2, 64, 1024, None) == L.EARG
    for args in ((0, 1, 8, 2, 64, 1024), (1, 1, 8, 3, 64, 1024), (1, 1, 8, 2, 64, 0), (1, 1, 8, 2, 64, 2 ** 31)):
        assert L.lib.b200k_fa2_fwd_kvcache_workspace_bytes(*args, ctypes.byref(n)) == L.ESHAPE, args


def test_valid_arguments_reach_the_device():
    """Validation passes; without a GPU the call then fails loudly at the device query instead of doing anything else."""
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    n = ctypes.c_size_t(0)
    for kw in (dict(), dict(page_size=16), dict(page_size=256, num_pages=4, pages_per_seq=2), dict(H=71 * 2, H_kv=2),
               dict(dtype=L.BF16, D=128, causal=1, Lq=16), dict(B=65535, H=1, H_kv=1)):
        assert _call(**kw) in (L.ECUDA, L.EARCH), kw
    assert _call(ptrs=[ONE] * 5 + [None], num_pages=2, pages_per_seq=1, page_size=100) in (L.ECUDA, L.EARCH)
    assert L.lib.b200k_fa2_fwd_kvcache_workspace_bytes(1, 1, 32, 8, 128, 32768, ctypes.byref(n)) in (L.ECUDA, L.EARCH)


def test_python_wrapper_checks():
    from b200k import ops

    q = torch.zeros(2, 1, 8, 64, dtype=torch.half)
    kc = torch.zeros(2, 100, 2, 64, dtype=torch.half)
    pc = torch.zeros(6, 16, 2, 64, dtype=torch.half)
    lens = torch.tensor([5, 9], dtype=torch.int32)
    table = torch.zeros(2, 3, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="values must be torch::kHalf"):
        ops.fa2_fwd_kvcache(q, kc.float(), kc, q, lens)
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        ops.fa2_fwd_kvcache(q, kc, kc[:, :, :1].contiguous(), q, lens)                  # V heads differ from K heads
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        k3 = torch.zeros(2, 100, 3, 64, dtype=torch.half)
        ops.fa2_fwd_kvcache(q, k3, k3, q, lens)                                           # H % H_kv != 0
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        ops.fa2_fwd_kvcache(q[0], kc, kc, q[0], lens)                                     # q must be [B, Lq, H, D]
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        ops.fa2_fwd_kvcache(q, kc[:1], kc[:1], q, lens)                                   # contiguous: one page per sequence
    with pytest.raises(RuntimeError, match="headdim not support!"):
        q2, k2 = torch.zeros(2, 1, 8, 48, dtype=torch.half), torch.zeros(2, 100, 2, 48, dtype=torch.half)
        ops.fa2_fwd_kvcache(q2, k2, k2, q2, lens)
    with pytest.raises(RuntimeError, match="values must be torch::kInt32"):
        ops.fa2_fwd_kvcache(q, kc, kc, q, lens.long())
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        ops.fa2_fwd_kvcache(q, kc, kc, q, lens[:1])                                       # B lengths
    with pytest.raises(RuntimeError, match="values must be torch::kInt32"):
        ops.fa2_fwd_kvcache(q, pc, pc, q, lens, table.long())
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        ops.fa2_fwd_kvcache(q, pc, pc, q, lens, table[:1])                                # one table row per sequence
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        ops.fa2_fwd_kvcache(q, pc, pc, q, lens, table.view(-1))
    with pytest.raises(RuntimeError, match="CUDA device"):
        ops.fa2_fwd_kvcache(q, kc, kc, q, lens)                                           # there is no CPU path
    with pytest.raises(RuntimeError, match="CUDA device"):
        ops.fa2_fwd_kvcache(q, pc, pc, q, lens, table)


@pytest.mark.parametrize("page_size", [16, 64, 256])
def test_gather_paged_equals_contiguous(page_size):
    B, S, H_kv, D = 3, 512, 2, 32
    g = torch.Generator().manual_seed(page_size)
    kc, vc = [torch.randn(B, S, H_kv, D, generator=g).half() for _ in range(2)]
    lens = torch.tensor([0, 300, 512], dtype=torch.int32)
    kp, vp, table, spare = kvcache_oracle.paged_copy(kc, vc, page_size, seed=page_size,
                                                     fill=lambda shape: torch.full(shape, float("nan")))
    assert len(set(table.view(-1).tolist())) == table.numel() and not set(spare.tolist()) & set(table.view(-1).tolist())
    assert table.view(-1).tolist() != sorted(table.view(-1).tolist())                    # shuffled
    k1, v1, cu1 = kvcache_oracle.gather(kc, vc, lens)
    k2, v2, cu2 = kvcache_oracle.gather(kp, vp, lens, table)
    assert torch.equal(cu1, cu2) and cu1.tolist() == [0, 0, 300, 812]
    assert torch.equal(k1, k2) and torch.equal(v1, v2)
    assert torch.equal(k1[300:], kc[2]) and torch.equal(k1[:300], kc[1, :300])


def test_reference_is_varlen_with_lq_tokens_per_sequence():
    B, Lq, H, H_kv, D = 2, 3, 4, 2, 32
    g = torch.Generator().manual_seed(1)
    q = torch.randn(B, Lq, H, D, generator=g).half()
    kc, vc = [torch.randn(B, 40, H_kv, D, generator=g).half() for _ in range(2)]
    lens = torch.tensor([2, 40], dtype=torch.int32)
    o = ar.kvcache(q, kc, vc, lens, causal=True)[0].half()
    assert o.shape == q.shape
    assert (o[0, 0] == 0).all()                                 # token 0 of sequence 0 sees keys <= 0 + 2 - 3 < 0
    assert torch.equal(o[0, 1], vc[0, 0].repeat_interleave(2, dim=0))   # token 1 sees exactly key 0
    assert torch.isfinite(o.float()).all()
