"""CPU: argument validation of the KV-cache append entry points (before any CUDA call), the Python wrapper's checks for
k / v / rotary, and self-checks of the append reference (kvcache_append_oracle.py): the rotation's identity, pairing
and inverse, and where the new rows land under a shuffled table."""
import ctypes
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))  # the oracles sit next to this file
import attention_ref as ar  # noqa: E402
import kvcache_append_oracle as ko  # noqa: E402
import kvcache_oracle  # noqa: E402

from b200k import _loader as L

ONE = ctypes.c_void_p(16)      # never dereferenced: validation fails first
ODD = ctypes.c_void_p(16 + 8)  # 8-byte aligned only


def _call(ptrs=(ONE,) * 6, k_new=ONE, v_new=ONE, L_new=1, cos=ONE, sin=ONE, rotary_seqlen=256, rotary_dim=64,
          interleaved=1, B=2, Lq=1, H=8, H_kv=2, D=64, num_pages=10, page_size=64, pages_per_seq=4, dtype=L.F16,
          causal=0, ws=ONE, ws_bytes=1 << 20):
    return L.lib.b200k_fa2_fwd_kvcache_append(*ptrs, k_new, v_new, L_new, cos, sin, rotary_seqlen, rotary_dim,
                                              interleaved, B, Lq, H, H_kv, D, num_pages, page_size, pages_per_seq, 0.0,
                                              dtype, causal, ws, ws_bytes, None)


@pytest.mark.parametrize("null_at", range(5))   # Q, K_cache, V_cache, O, cache_seqlens (a NULL block_table is valid)
def test_null_pointers_of_the_decode_call_are_refused(null_at):
    ptrs = [ONE] * 6
    ptrs[null_at] = None
    assert _call(ptrs=ptrs) == L.EARG


@pytest.mark.parametrize("kw", [dict(k_new=None), dict(v_new=None), dict(k_new=None, v_new=None)])
def test_null_new_rows_are_refused(kw):
    assert _call(**kw) == L.EARG


@pytest.mark.parametrize("kw", [dict(cos=None), dict(sin=None)])
def test_cos_without_sin_is_refused(kw):
    assert _call(**kw) == L.EARG
    assert b"rotary_cos and rotary_sin" in L.lib.b200k_last_error()


@pytest.mark.parametrize("dtype", [L.F32, L.I8, L.FP8_E4M3, 99])
def test_unsupported_dtypes_are_refused(dtype):
    assert _call(dtype=dtype) == L.EDTYPE


@pytest.mark.parametrize("D", [0, 16, 48, 80, 160, 256])
def test_unsupported_head_dims_are_refused(D):
    assert _call(D=D, rotary_dim=16) == L.EHEADDIM
    assert b"headdim not support!" in L.lib.b200k_last_error()
    n = ctypes.c_size_t(7)
    assert L.lib.b200k_fa2_fwd_kvcache_append_workspace_bytes(1, 1, 8, 2, D, 1024, 1, ctypes.byref(n)) == L.EHEADDIM


@pytest.mark.parametrize("L_new", [0, -1, 2 ** 31])
def test_bad_new_token_counts_are_refused(L_new):
    assert _call(L_new=L_new) == L.ESHAPE


@pytest.mark.parametrize("rotary_dim", [0, 8, 24, 64 + 16])
def test_bad_rotary_dims_are_refused(rotary_dim):
    assert _call(rotary_dim=rotary_dim) == L.ESHAPE
    assert b"rotary_dim" in L.lib.b200k_last_error()


def test_rotary_table_shorter_than_the_capacity_is_refused():
    assert _call(rotary_seqlen=4 * 64 - 1) == L.ESHAPE
    assert b"capacity" in L.lib.b200k_last_error()


def test_rotary_arguments_are_ignored_without_cos_and_sin():
    """No rotary: rotary_dim and rotary_seqlen are not checked; validation passes and the call reaches the device."""
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    assert _call(cos=None, sin=None, rotary_dim=0, rotary_seqlen=0) in (L.ECUDA, L.EARCH)


@pytest.mark.parametrize("kw", [dict(k_new=ODD), dict(v_new=ODD), dict(cos=ODD), dict(sin=ODD),
                                dict(ptrs=[ODD] + [ONE] * 5), dict(ptrs=[ONE, ODD] + [ONE] * 4), dict(ws=ODD)])
def test_unaligned_pointers_are_refused(kw):
    assert _call(**kw) == L.EALIGN


@pytest.mark.parametrize("kw", [dict(page_size=48), dict(H=8, H_kv=3), dict(B=65536, H=1, H_kv=1),
                                dict(ptrs=[ONE] * 5 + [None], num_pages=3, pages_per_seq=1)])
def test_decode_shape_rules_are_shared(kw):
    """The rules of b200k_fa2_fwd_kvcache apply with the same codes and messages (named after the entry point)."""
    assert _call(**kw) == L.ESHAPE
    msg = L.lib.b200k_last_error().replace(b"b200k_fa2_fwd_kvcache_append", b"b200k_fa2_fwd_kvcache")
    a = dict(ptrs=[ONE] * 6, B=2, H=8, H_kv=2, num_pages=10, page_size=64, pages_per_seq=4)
    a.update(kw)
    assert L.lib.b200k_fa2_fwd_kvcache(*a["ptrs"], a["B"], 1, a["H"], a["H_kv"], 64, a["num_pages"], a["page_size"],
                                       a["pages_per_seq"], 0.0, L.F16, 0, None, 0, None) == L.ESHAPE
    assert L.lib.b200k_last_error() == msg


def test_workspace_query_checks():
    n = ctypes.c_size_t(0)
    assert L.lib.b200k_fa2_fwd_kvcache_append_workspace_bytes(1, 1, 8, 2, 64, 1024, 1, None) == L.EARG
    for args in ((0, 1, 8, 2, 64, 1024), (1, 1, 8, 3, 64, 1024), (1, 1, 8, 2, 64, 0), (1, 1, 8, 2, 64, 2 ** 31)):
        assert L.lib.b200k_fa2_fwd_kvcache_append_workspace_bytes(*args, 0, ctypes.byref(n)) == L.ESHAPE, args


def test_valid_arguments_reach_the_device():
    """Validation passes; without a GPU the call then fails loudly at the device query instead of doing anything else."""
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    n = ctypes.c_size_t(0)
    for kw in (dict(), dict(page_size=16, rotary_dim=16), dict(interleaved=0, rotary_dim=48, L_new=7, Lq=3),
               dict(dtype=L.BF16, D=128, rotary_dim=128, causal=1), dict(ws=None, ws_bytes=0)):
        assert _call(**kw) in (L.ECUDA, L.EARCH), kw
    assert _call(ptrs=[ONE] * 5 + [None], num_pages=2, pages_per_seq=1, page_size=100, rotary_seqlen=100) in (L.ECUDA, L.EARCH)
    assert L.lib.b200k_fa2_fwd_kvcache_append_workspace_bytes(1, 1, 32, 8, 128, 32768, 1, ctypes.byref(n)) in (L.ECUDA, L.EARCH)


def test_python_wrapper_checks():
    from b200k import ops

    q = torch.zeros(2, 1, 8, 64, dtype=torch.half)
    kc = torch.zeros(2, 100, 2, 64, dtype=torch.half)
    lens = torch.tensor([5, 9], dtype=torch.int32)
    k = torch.zeros(2, 3, 2, 64, dtype=torch.half)
    cos = torch.zeros(100, 16, dtype=torch.half)
    with pytest.raises(RuntimeError, match="both k and v"):
        ops.fa2_fwd_kvcache(q, kc, kc, q, lens, k=k)                                       # k without v
    with pytest.raises(RuntimeError, match="both k and v"):
        ops.fa2_fwd_kvcache(q, kc, kc, q, lens, v=k)                                       # v without k
    with pytest.raises(RuntimeError, match="both k and v"):
        ops.fa2_fwd_kvcache(q, kc, kc, q, lens, rotary_cos=cos, rotary_sin=cos)            # rotary without k / v
    with pytest.raises(RuntimeError, match="rotary_cos and rotary_sin"):
        ops.fa2_fwd_kvcache(q, kc, kc, q, lens, k=k, v=k, rotary_cos=cos)                  # cos without sin
    with pytest.raises(RuntimeError, match="values must be torch::kHalf"):
        ops.fa2_fwd_kvcache(q, kc, kc, q, lens, k=k.float(), v=k)
    with pytest.raises(RuntimeError, match="values must be torch::kHalf"):
        ops.fa2_fwd_kvcache(q, kc, kc, q, lens, k=k, v=k, rotary_cos=cos, rotary_sin=cos.bfloat16())
    for bad in (k[:1], k[:, :, :1], k[..., :32], k[0]):                                   # B, H_kv, D, rank
        with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
            ops.fa2_fwd_kvcache(q, kc, kc, q, lens, k=bad.contiguous(), v=bad.contiguous())
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        ops.fa2_fwd_kvcache(q, kc, kc, q, lens, k=k, v=k[:, :2].contiguous())              # v differs from k
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        ops.fa2_fwd_kvcache(q, kc, kc, q, lens, k=k, v=k, rotary_cos=cos, rotary_sin=cos[:, :8].contiguous())
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        ops.fa2_fwd_kvcache(q, kc, kc, q, lens, k=k, v=k, rotary_cos=cos.view(-1), rotary_sin=cos.view(-1))
    with pytest.raises(RuntimeError, match="CUDA device"):
        ops.fa2_fwd_kvcache(q, kc, kc, q, lens, k=k, v=k, rotary_cos=cos, rotary_sin=cos)  # there is no CPU path


def _angles(n, half, seed=0, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    theta = torch.rand(n, half, generator=g, dtype=torch.float64) * 2 * math.pi
    return theta.cos().to(dtype), theta.sin().to(dtype), theta


@pytest.mark.parametrize("interleaved", [False, True])
def test_rotation_by_zero_is_the_identity(interleaved):
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 3, 4, 64, generator=g).half()
    cos, sin = torch.ones(50, 24).half(), torch.zeros(50, 24).half()
    pos = torch.randint(0, 50, (2, 3), generator=g)
    assert torch.equal(ko.rotate(x, cos, sin, pos, interleaved), x)


def test_interleaved_and_neox_differ_by_a_column_permutation():
    """Interleaved pairs (2j, 2j + 1), NeoX pairs (j, j + rd/2): permuting the rotated columns maps one onto the other."""
    rd, D = 32, 64
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 5, 3, D, generator=g, dtype=torch.float64)
    cos, sin, _ = _angles(40, rd // 2, seed=3)
    pos = torch.randint(0, 40, (2, 5), generator=g)
    perm = torch.cat([torch.arange(0, rd, 2), torch.arange(1, rd, 2), torch.arange(rd, D)])   # interleaved -> NeoX
    neox = ko.rotate(x[..., perm], cos, sin, pos, interleaved=False)
    inter = ko.rotate(x, cos, sin, pos, interleaved=True)
    assert torch.equal(neox, inter[..., perm])


@pytest.mark.parametrize("interleaved", [False, True])
def test_rotating_back_gives_the_input(interleaved):
    g = torch.Generator().manual_seed(4)
    x = torch.randn(3, 4, 2, 128, generator=g, dtype=torch.float64)
    cos, sin, _ = _angles(30, 32, seed=5)
    pos = torch.randint(0, 30, (3, 4), generator=g)
    back = ko.rotate(ko.rotate(x, cos, sin, pos, interleaved), cos, -sin, pos, interleaved)
    assert torch.allclose(back, x, rtol=0, atol=1e-12)
    assert torch.equal(back[..., 64:], x[..., 64:])


def test_rotation_matches_the_textbook_formula():
    """One row by hand: pair j at position p is (x0 cos - x1 sin, x0 sin + x1 cos)."""
    x = torch.arange(1, 17, dtype=torch.float64).view(1, 1, 1, 16)
    cos, sin, theta = _angles(4, 8, seed=6)
    got = ko.rotate(x, cos, sin, torch.tensor([[2]]), interleaved=False)[0, 0, 0]
    c, s = cos[2], sin[2]
    assert torch.allclose(got[:8], x[0, 0, 0, :8] * c - x[0, 0, 0, 8:] * s)
    assert torch.allclose(got[8:], x[0, 0, 0, :8] * s + x[0, 0, 0, 8:] * c)


@pytest.mark.parametrize("page_size", [16, 64])
def test_rows_land_in_their_page_slots_under_a_shuffled_table(page_size):
    B, S, H_kv, D, L_new = 3, 256, 2, 32, 5
    g = torch.Generator().manual_seed(page_size)
    kc = torch.randn(B, S, H_kv, D, generator=g).half()
    kp, _, table, spare = kvcache_oracle.paged_copy(kc, kc, page_size, seed=page_size)
    assert table.view(-1).tolist() != sorted(table.view(-1).tolist())
    new = torch.randn(B, L_new, H_kv, D, generator=g).half()
    lens = torch.tensor([0, page_size - 2, S - 3], dtype=torch.int32)   # the second crosses a page, the third overflows
    out = ko.write(kp, new, lens, table)
    want = kc.clone()
    for b, n in enumerate(lens.tolist()):
        m = min(L_new, S - n)
        want[b, n:n + m] = new[b, :m]
    k, _, _ = kvcache_oracle.gather(out, out, torch.full((B,), S, dtype=torch.int32), table)
    assert torch.equal(k, want.reshape(B * S, H_kv, D))
    assert torch.equal(out[spare], kp[spare])                      # unlisted pages untouched
    contiguous = ko.write(kc, new, lens)                           # the same rows without a table
    assert torch.equal(contiguous, want)


def test_reference_attends_over_old_and_new_keys():
    """Lengths are taken as base + L_new, with negative lengths as 0, and the result equals attention_ref.kvcache on a cache
    that already holds the new rows."""
    B, Lq, H, H_kv, D, S = 2, 2, 4, 2, 32, 64
    g = torch.Generator().manual_seed(7)
    q = torch.randn(B, Lq, H, D, generator=g).half()
    kc, vc = [torch.randn(B, S, H_kv, D, generator=g).half() for _ in range(2)]
    kn, vn = [torch.randn(B, 3, H_kv, D, generator=g).half() for _ in range(2)]
    lens = torch.tensor([-4, 10], dtype=torch.int32)
    o, k2, v2 = ko.attention_append(q, kc, vc, lens, kn, vn, causal=True)
    assert torch.equal(k2[0, :3], kn[0]) and torch.equal(k2[1, 10:13], kn[1]) and torch.equal(k2[1, :10], kc[1, :10])
    want = ar.kvcache(q, k2, v2, torch.tensor([3, 13], dtype=torch.int32), causal=True)[0].half()
    assert torch.equal(o, want)
