"""CPU: the attention backward.  The fp64 reference (attention_ref.py, dense layout) against torch.autograd on its own
forward and gradcheck; every argument check of b200k_fa2_bwd before any CUDA call (fake pointers, never dereferenced); the workspace
size; the checks of the fa2_bwd wrapper."""
import ctypes
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attention_ref as ar  # noqa: E402

from b200k import _loader as L  # noqa: E402

SL = torch.tensor([3, 5])


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("seqlens", [None, SL, torch.tensor([0, 9])], ids=["full", "seqlens", "clamped"])
def test_reference_gradients_are_torch_autograd_of_the_reference_forward(causal, seqlens):
    g = torch.Generator().manual_seed(1)
    B, H, N, D = 2, 3, 7, 8
    q, k, v, do = [torch.randn(B, H, N, D, generator=g, dtype=torch.float64) for _ in range(4)]
    qa, ka, va = [t.clone().requires_grad_() for t in (q, k, v)]
    o, lse = ar.dense(qa, ka, va, 0.3, causal, seqlens)
    o.backward(do)
    dq, dk, dv, o64, lse64 = ar.dense_grads(q, k, v, do, 0.3, causal, seqlens)
    for got, want in ((dq, qa.grad), (dk, ka.grad), (dv, va.grad), (o64, o), (lse64, lse)):
        assert torch.allclose(got, want.detach(), rtol=1e-12, atol=1e-12)
    # keys no row sees have zero dK and dV
    if seqlens is SL:
        assert (dk[0, :, 3:] == 0).all() and (dv[0, :, 3:] == 0).all()
        assert (dk[1, :, 5:] == 0).all() and (dv[1, :, 5:] == 0).all()


@pytest.mark.parametrize("causal", [False, True])
def test_reference_forward_passes_gradcheck(causal):
    g = torch.Generator().manual_seed(2)
    q, k, v = [torch.randn(2, 1, 5, 4, generator=g, dtype=torch.float64, requires_grad=True) for _ in range(3)]
    assert torch.autograd.gradcheck(lambda a, b, c: ar.dense(a, b, c, None, causal, SL)[0], (q, k, v))


# ------------------------------------------------------------------------------------------------ the C entry points
P = 1 << 20  # fake device pointers, 16-byte aligned, never dereferenced: validation fails first


def _bwd(**kw):
    a = dict(Q=P, K=P, V=P, O=P, lse=P, dO=P, dQ=P, dK=P, dV=P, B=1, H=2, N=8, D=64, scale=0.0, dtype=L.F16, causal=0,
             seqlens=None, ws=P, ws_bytes=1 << 20)
    a.update(kw)
    ptr = lambda x: None if x is None else ctypes.c_void_p(x)  # noqa: E731
    return L.lib.b200k_fa2_bwd(*(ptr(a[n]) for n in ("Q", "K", "V", "O", "lse", "dO", "dQ", "dK", "dV")), a["B"], a["H"],
                               a["N"], a["D"], a["scale"], a["dtype"], a["causal"], ptr(a["seqlens"]), ptr(a["ws"]),
                               a["ws_bytes"], None)


@pytest.mark.parametrize("name", ["Q", "K", "V", "O", "lse", "dO", "dQ", "dK", "dV", "ws"])
def test_null_pointer(name):
    assert _bwd(**{name: None}) == L.EARG
    assert b"null pointer" in L.lib.b200k_last_error()


def test_codes_and_their_order():
    for dt in (L.F32, L.I8, 99):
        assert _bwd(dtype=dt) == L.EDTYPE
    for D in (16, 48, 256):
        assert _bwd(D=D) == L.EHEADDIM
        assert b"headdim not support" in L.lib.b200k_last_error()
    for kw in (dict(B=0), dict(H=0), dict(N=0), dict(N=1 << 31), dict(B=256, H=256)):
        assert _bwd(**kw) == L.ESHAPE, kw
    # the order: null pointer, dtype, head dim, shape, alignment, workspace size
    assert _bwd(Q=None, dtype=L.F32) == L.EARG
    assert _bwd(dtype=L.F32, D=48) == L.EDTYPE
    assert _bwd(D=48, N=0) == L.EHEADDIM
    assert _bwd(N=0, Q=P + 8) == L.ESHAPE
    assert _bwd(Q=P + 8, ws_bytes=0) == L.EALIGN


@pytest.mark.parametrize("name,rule", [("Q", 16), ("K", 16), ("V", 16), ("O", 16), ("dO", 16), ("ws", 16), ("dQ", 4),
                                       ("dK", 4), ("dV", 4), ("lse", 4), ("seqlens", 4)])
def test_alignment_is_checked_and_named(name, rule):
    assert _bwd(**{name: P + rule // 2}) == L.EALIGN
    label = {"ws": "workspace", "seqlens": "seqlens_k"}.get(name, name)
    assert ("%s must be %d-byte aligned" % (label, rule)).encode() in L.lib.b200k_last_error()


def test_short_workspace_is_refused_before_cuda():
    need = ops_ws(2, 3, 100)
    assert _bwd(B=2, H=3, N=100, ws_bytes=need - 1) == L.EARG
    assert b"workspace bytes needed" in L.lib.b200k_last_error()


def ops_ws(B, H, N):
    n = ctypes.c_size_t(0)
    L.check(L.lib.b200k_fa2_bwd_workspace_bytes(B, H, N, ctypes.byref(n)))
    return n.value


@pytest.mark.parametrize("B,H,N", [(1, 1, 1), (1, 1, 64), (1, 1, 65), (2, 3, 100), (4, 48, 8192), (65535, 1, 7)])
def test_workspace_is_two_fp32_rows_sections_on_256_byte_boundaries(B, H, N):
    section = (B * H * N * 4 + 255) // 256 * 256
    assert ops_ws(B, H, N) == 2 * section


def test_workspace_function_checks():
    assert L.lib.b200k_fa2_bwd_workspace_bytes(1, 1, 1, None) == L.EARG
    n = ctypes.c_size_t(0)
    for shape in ((0, 1, 1), (1, 0, 1), (1, 1, 0), (300, 300, 1), (1, 1, 1 << 31)):
        assert L.lib.b200k_fa2_bwd_workspace_bytes(*shape, ctypes.byref(n)) == L.ESHAPE, shape


def test_wrapper_checks():
    from b200k import ops

    q = torch.zeros(1, 2, 8, 64, dtype=torch.half)
    lse = torch.zeros(1, 2, 8)

    def call(**kw):
        a = dict(q=q, k=q, v=q, o=q, lse=lse, do=q, dq=q.clone(), dk=q.clone(), dv=q.clone())
        a.update(kw)
        ops.fa2_bwd(**a)

    for kw, msg in ((dict(do=q.bfloat16()), "values must be torch::kHalf"), (dict(dv=q[:, :, :4]), "Tensor size mismatch!"),
                    (dict(lse=lse.half()), "values must be torch::kFloat32"), (dict(lse=lse[:, :1]), "Tensor size mismatch!"),
                    (dict(q=q[..., :48], k=q[..., :48], v=q[..., :48], o=q[..., :48], do=q[..., :48], dq=q[..., :48],
                          dk=q[..., :48], dv=q[..., :48]), "headdim not support!"),
                    (dict(seqlens_k=torch.zeros(2, dtype=torch.int32)), "Tensor size mismatch!"),
                    (dict(seqlens_k=torch.zeros(1, dtype=torch.int64)), "values must be torch::kInt32"),
                    ({}, "CUDA device")):
        with pytest.raises(RuntimeError, match=msg):
            call(**kw)
    with pytest.raises(RuntimeError, match="CUDA device"):
        ops.attention(q, q, q)
