"""CPU: the fp64 reference of the packed attention backward (attention_ref.py, packed layout) against torch autograd and
gradcheck; b200k_fa2_bwd_varlen's argument checks, all made before any CUDA call (fake pointers, never
dereferenced); and ops.fa2_bwd_varlen's checks."""
import ctypes
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attention_ref as ar  # noqa: E402

from b200k import _loader as L  # noqa: E402


def _inputs(lq, lk, H, H_kv, D, seed):
    g = torch.Generator().manual_seed(seed)
    q, do = (torch.randn(sum(lq), H, D, generator=g, dtype=torch.float64) for _ in range(2))
    k, v = (torch.randn(sum(lk), H_kv, D, generator=g, dtype=torch.float64) for _ in range(2))
    return q, k, v, do


@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("lq,lk,H,H_kv", [((5, 3), (5, 3), 4, 2), ((2, 7, 4), (6, 3, 4), 4, 1), ((3, 4), (5, 2), 2, 2)])
def test_reference_gradients_are_torch_autograd_of_the_reference_forward(causal, lq, lk, H, H_kv):
    q, k, v, do = _inputs(lq, lk, H, H_kv, 8, sum(lq) + H)
    qa, ka, va = (t.clone().requires_grad_() for t in (q, k, v))
    ar.packed(qa, ka, va, ar.cu(lq), ar.cu(lk), None, causal)[0].backward(do)
    got = ar.packed_grads(q, k, v, do, ar.cu(lq), ar.cu(lk), None, causal)[:3]
    for a, r in zip(got, (qa.grad, ka.grad, va.grad)):
        assert torch.allclose(a, r, rtol=1e-10, atol=1e-12)


def test_reference_forward_passes_gradcheck():
    q, k, v, _ = _inputs((3, 2), (2, 4), 4, 2, 4, 1)
    for t in (q, k, v):
        t.requires_grad_()
    for causal in (False, True):
        assert torch.autograd.gradcheck(lambda a, b, c: ar.packed(a, b, c, ar.cu((3, 2)), ar.cu((2, 4)), None, causal)[0],
                                        (q, k, v))


def test_explicit_edges_are_zero_not_nan():
    """Lq > Lk and Lq < Lk, Lq = 0, Lk = 0, causal rows that see no key, and two tokens past cu_seqlens[B]."""
    lq, lk = (6, 0, 4, 2), (3, 5, 0, 7)
    q, k, v, do = _inputs(lq, lk, 4, 2, 8, 9)
    q, do = (torch.cat([t, torch.randn(2, 4, 8, dtype=torch.float64)]) for t in (q, do))
    for causal in (False, True):
        dq, dk, dv, o, lse = ar.packed_grads(q, k, v, do, ar.cu(lq), ar.cu(lk), None, causal)
        for t in (dq, dk, dv, o):
            assert not torch.isnan(t).any()
        assert (dk[3:8] == 0).all() and (dv[3:8] == 0).all()        # Lq = 0
        assert (dq[6:10] == 0).all() and (o[6:10] == 0).all()       # Lk = 0
        assert (dq[-2:] == 0).all() and torch.isinf(lse[-2:]).all()  # outside every sequence
        assert (dq[:3] == 0).all() == causal                        # rows r < Lq - Lk = 3 see no key when causal
        assert torch.isinf(lse[:3]).all() == causal


# ------------------------------------------------------------------------------------------------ the C entry points
P = 1 << 20  # fake device pointers, 16-byte aligned


def _bwd(**kw):
    a = dict(Q=P, K=P, V=P, O=P, lse=P, dO=P, dQ=P, dK=P, dV=P, cu_q=P, cu_k=P, B=2, mq=8, mk=8, tq=16, tk=16, H=4,
             H_kv=2, D=64, scale=0.0, dtype=L.F16, causal=0, ws=P, ws_bytes=1 << 20)
    a.update(kw)
    ptr = lambda x: None if x is None else ctypes.c_void_p(x)  # noqa: E731
    return L.lib.b200k_fa2_bwd_varlen(*(ptr(a[n]) for n in ("Q", "K", "V", "O", "lse", "dO", "dQ", "dK", "dV", "cu_q",
                                                            "cu_k")),
                                      a["B"], a["mq"], a["mk"], a["tq"], a["tk"], a["H"], a["H_kv"], a["D"], a["scale"],
                                      a["dtype"], a["causal"], ptr(a["ws"]), a["ws_bytes"], None)


@pytest.mark.parametrize("name", ["Q", "K", "V", "O", "lse", "dO", "dQ", "dK", "dV", "cu_q", "cu_k", "ws"])
def test_null_pointer(name):
    assert _bwd(**{name: None}) == L.EARG
    assert b"null pointer" in L.lib.b200k_last_error()


def test_codes_and_their_order():
    for dt in (L.F32, L.I8, 99):
        assert _bwd(dtype=dt) == L.EDTYPE
    for D in (16, 48, 256):
        assert _bwd(D=D) == L.EHEADDIM
    for kw in (dict(B=0), dict(H=0), dict(H_kv=0), dict(H=4, H_kv=3), dict(mq=0), dict(mq=17), dict(mk=0),
               dict(mk=17), dict(tq=1 << 31, mq=8), dict(tk=1 << 31), dict(B=65536 // 4 + 1), dict(B=2, H=65536, H_kv=1)):
        assert _bwd(**kw) == L.ESHAPE, kw
    assert _bwd(D=16, B=0) == L.EHEADDIM          # head dim before shape
    assert _bwd(B=0, Q=P + 2) == L.ESHAPE         # shape before alignment
    assert _bwd(Q=P + 2, ws_bytes=0) == L.EALIGN  # alignment before the workspace size


RULES = {"Q": 16, "K": 16, "V": 16, "O": 16, "dO": 16, "ws": 16, "dQ": 4, "dK": 4, "dV": 4, "lse": 4, "cu_q": 4, "cu_k": 4}


@pytest.mark.parametrize("name,rule", sorted(RULES.items()))
def test_alignment_is_checked_and_named(name, rule):
    for off in (2, 4, 8, 12):
        # a short workspace stops an accepted pointer at the next check, before any CUDA call
        rc = _bwd(**{name: P + off, "ws_bytes": 0})
        if off % rule:
            assert rc == L.EALIGN, (name, off)
            msg = {"ws": "workspace", "cu_q": "cu_seqlens_q", "cu_k": "cu_seqlens_k"}.get(name, name)
            assert (" %s must be %d-byte aligned" % (msg, rule)).encode() in L.lib.b200k_last_error()
        else:
            assert rc == L.EARG, (name, off)
            assert b"workspace bytes needed" in L.lib.b200k_last_error()


def _ws(total_q, H):
    n = ctypes.c_size_t(0)
    rc = L.lib.b200k_fa2_bwd_varlen_workspace_bytes(total_q, H, ctypes.byref(n))
    return rc, n.value


def test_short_workspace_is_refused_before_cuda():
    _, need = _ws(16, 4)
    assert _bwd(ws_bytes=need - 1) == L.EARG
    assert b"workspace bytes needed" in L.lib.b200k_last_error()


@pytest.mark.parametrize("total_q,H", [(1, 1), (16, 4), (1000, 7), (65, 64)])
def test_workspace_is_two_fp32_sections_on_256_byte_boundaries(total_q, H):
    assert _ws(total_q, H) == (L.OK, 2 * ((total_q * H * 4 + 255) // 256 * 256))


def test_workspace_function_checks():
    assert L.lib.b200k_fa2_bwd_varlen_workspace_bytes(1, 1, None) == L.EARG
    for tq, H in ((0, 1), (1, 0), (1 << 31, 1), (1, 65536)):
        assert _ws(tq, H)[0] == L.ESHAPE


def test_wrapper_checks():
    from b200k import ops

    def t(*s, dt=torch.float16):
        return torch.zeros(*s, dtype=dt)

    q, k = t(16, 4, 64), t(16, 2, 64)
    cu = torch.tensor([0, 8, 16], dtype=torch.int32)
    lse = torch.zeros(16, 4)

    def call(**kw):
        a = dict(q=q, k=k, v=k, o=q, lse=lse, do=q, dq=q, dk=k, dv=k, cu_seqlens_q=cu, cu_seqlens_k=cu, max_seqlen_q=8,
                 max_seqlen_k=8)
        a.update(kw)
        ops.fa2_bwd_varlen(**a)

    for kw, msg in ((dict(dq=t(16, 4, 64, dt=torch.bfloat16)), "values must be"), (dict(dk=t(16, 4, 64)), "size mismatch"),
                    (dict(k=t(16, 3, 64), v=t(16, 3, 64), dk=t(16, 3, 64), dv=t(16, 3, 64)), "size mismatch"),
                    (dict(q=t(16, 4, 48), o=t(16, 4, 48), do=t(16, 4, 48), dq=t(16, 4, 48), k=t(16, 2, 48),
                          v=t(16, 2, 48), dk=t(16, 2, 48), dv=t(16, 2, 48)), "headdim"),
                    (dict(lse=torch.zeros(16, 2)), "size mismatch"), (dict(lse=torch.zeros(16, 4, dtype=torch.float64)),
                                                                     "values must be"),
                    (dict(cu_seqlens_q=cu.long()), "values must be"), (dict(cu_seqlens_k=cu[:2]), "size mismatch"),
                    ({}, "CUDA device")):
        with pytest.raises(RuntimeError, match=msg):
            call(**kw)
