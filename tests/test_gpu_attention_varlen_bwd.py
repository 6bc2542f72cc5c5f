"""GPU: the packed attention backward (ops.fa2_bwd_varlen, b200k_fa2_bwd_varlen) and ops.attention_varlen.

  - exact needle answers per sequence and query head, GQA groups of 1, 2 and 8 and MQA: dQ = dK = 0 and dV of K/V head
    k, key j = the sum over the group of the dO rows whose needle is j, bit for bit;
  - H_kv = H and equal lengths: the bits of the dense fa2_bwd;
  - each sequence of a packed call has the bits of that sequence passed alone;
  - random inputs against the fp64 reference (attention_ref.py) by flash-attn's rule;
  - rows that see no key, keys no query sees and tokens outside every sequence are +0, nothing is NaN;
  - every element is written once, guards and inputs are untouched, two calls and a graph replay give the same bits,
    a call from a fresh thread works;
  - ops.attention_varlen's gradients are the bits of fa2_fwd_varlen(lse=) + fa2_bwd_varlen, and within the fp64 rule of
    scaled_dot_product_attention(enable_gqa=True) per sequence."""
import math
import os
import sys
import threading

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attention_ref as ar  # noqa: E402
import exact_attention as ea  # noqa: E402

from b200k import ops  # noqa: E402

pytestmark = pytest.mark.gpu
GUARD = 30
DTYPES = [torch.float16, torch.bfloat16]


def _out(shape, dtype):
    n = math.prod(shape)
    buf = torch.full((n + 2 * GUARD,), float("nan"), dtype=dtype, device="cuda")
    return buf[GUARD:GUARD + n].view(shape), buf


def _fwd(q, k, v, cu_q, cu_k, mq, scale=None, causal=False):
    o = torch.zeros_like(q)
    lse = torch.full(q.shape[:-1], float("-inf"), device="cuda")
    ops.fa2_fwd_varlen(q, k, v, o, cu_q, cu_k, mq, scale, causal=causal, lse=lse)
    return o, lse


def _bwd(q, k, v, o, lse, do, cu_q, cu_k, mq, mk, scale=None, causal=False):
    outs = [_out(q.shape, q.dtype), _out(k.shape, k.dtype), _out(v.shape, v.dtype)]
    ops.fa2_bwd_varlen(q, k, v, o, lse, do, *(t for t, _ in outs), cu_q, cu_k, mq, mk, scale=scale, causal=causal)
    return [t for t, _ in outs], [b for _, b in outs]


def _bits(t):
    return t.view(torch.int16)


def _pos_zero(t):
    return bool((_bits(t) == 0).all())


# ------------------------------------------------------------------------------------------------ exact answers
def _needles(lq, lk, H, H_kv, D, dtype, causal, g):
    """Packed q, k and each row's needle token (-1: the row sees no key), per sequence and query head as the dense test
    builds them: column c of K/V head kh holds its needle at key nk[c] (nk[0] = 0), and row r of query head h takes a
    column whose needle it sees."""
    G = H // H_kv
    q = torch.zeros(sum(lq), H, D, dtype=dtype)
    k = torch.zeros(sum(lk), H_kv, D, dtype=dtype)
    needle = torch.full((sum(lq), H), -1, dtype=torch.long)
    q0 = k0 = 0
    for Lq, Lk in zip(lq, lk):
        if Lk > 0:
            for kh in range(H_kv):
                nk = torch.randint(0, Lk, (D,), generator=g)
                nk[0] = 0
                k[k0 + nk, kh, torch.arange(D)] = ea.A
                for h in range(kh * G, (kh + 1) * G):
                    rows = torch.arange(Lq)
                    ok = (nk.view(1, D) <= rows.view(Lq, 1) + Lk - Lq) if causal else torch.ones(Lq, D, dtype=torch.bool)
                    col = torch.where(ok, torch.rand(Lq, D, generator=g), torch.full((Lq, D), -1.0)).argmax(1)
                    sees = ok.any(1)
                    q[q0 + rows[sees], h, col[sees]] = ea.A
                    needle[q0 + rows[sees], h] = k0 + nk[col[sees]]
        q0 += Lq
        k0 += Lk
    return q, k, needle


NEEDLES = [((1, 63, 64), (1, 63, 64), 2, 2), ((65, 127, 128), (65, 127, 128), 4, 2), ((129, 1000), (129, 1000), 8, 1),
           ((100, 0, 64), (37, 64, 0), 8, 8), ((40, 129), (200, 65), 16, 2)]


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("D", [32, 128])
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("lq,lk,H,H_kv", NEEDLES, ids=["G1", "G2", "MQA", "G1-empty", "G8"])
def test_exact_needles(dtype, D, causal, lq, lk, H, H_kv):
    g = torch.Generator().manual_seed(sum(lq) + D + 7 * causal + H)
    q, k, needle = _needles(lq, lk, H, H_kv, D, dtype, causal, g)
    v = torch.randint(-8, 9, k.shape, generator=g).to(dtype)
    do = torch.randint(-8, 9, q.shape, generator=g).to(dtype)
    q, k, v, do, needle = (t.cuda() for t in (q, k, v, do, needle))
    cu_q, cu_k = ar.cu(lq, "cuda"), ar.cu(lk, "cuda")
    o, lse = _fwd(q, k, v, cu_q, cu_k, max(lq), None, causal)
    (dq, dk, dv), bufs = _bwd(q, k, v, o, lse, do, cu_q, cu_k, max(lq), max(max(lk), 1), None, causal)
    assert _pos_zero(dq) and _pos_zero(dk)
    G = H // H_kv
    want = torch.zeros(k.shape, dtype=torch.float64, device="cuda")
    seen = needle >= 0
    tok = needle[seen]
    kvh = (torch.arange(H, device="cuda") // G).view(1, H).expand_as(needle)[seen]
    want.index_put_((tok, kvh), do[seen].double(), accumulate=True)
    assert torch.equal(dv, want.to(dtype))
    for buf in bufs:
        assert torch.isnan(buf[:GUARD].float()).all() and torch.isnan(buf[-GUARD:].float()).all()


# ------------------------------------------------------------------------------------------------ same bits as dense
@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("D", [32, 64, 96, 128])
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
def test_equal_lengths_are_the_dense_bits(dtype, D, causal):
    g = torch.Generator(device="cuda").manual_seed(D + causal)
    B, H, N = 3, 4, 333
    q, k, v, do = (torch.randn(B, H, N, D, generator=g, device="cuda").to(dtype) for _ in range(4))
    o = torch.empty_like(q)
    lse = torch.empty(B, H, N, device="cuda")
    ops.fa2_fwd(q, k, v, o, causal=causal, lse=lse)
    dense = [torch.empty_like(q) for _ in range(3)]
    ops.fa2_bwd(q, k, v, o, lse, do, *dense, causal=causal)
    pk = lambda t: t.transpose(1, 2).reshape(B * N, H, D).contiguous()  # noqa: E731
    cu = ar.cu([N] * B, "cuda")
    got, _ = _bwd(pk(q), pk(k), pk(v), pk(o), lse.transpose(1, 2).reshape(B * N, H).contiguous(), pk(do), cu, cu, N, N,
                  None, causal)
    for a, d in zip(got, dense):
        assert torch.equal(_bits(a), _bits(pk(d)))


# ------------------------------------------------------------------------------------------------ isolation, fp64
CASES = [((300, 64, 1, 500), (200, 64, 77, 500), 8, 2, None), ((129, 1000, 65), (1000, 129, 65), 4, 1, 0.2),
         ((128, 1, 700), (128, 900, 700), 16, 16, None)]


def _random(lq, lk, H, H_kv, D, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q, do = (torch.randn(sum(lq), H, D, generator=g, device="cuda").to(dtype) for _ in range(2))
    k, v = (torch.randn(sum(lk), H_kv, D, generator=g, device="cuda").to(dtype) for _ in range(2))
    return q, k, v, do


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("lq,lk,H,H_kv,scale", CASES, ids=["G4", "MQA-scale", "MHA"])
def test_random_against_fp64_and_isolation(dtype, causal, lq, lk, H, H_kv, scale):
    D = 128 if H_kv == 1 else 64
    q, k, v, do = _random(lq, lk, H, H_kv, D, dtype, sum(lq) + H)
    cu_q, cu_k = ar.cu(lq, "cuda"), ar.cu(lk, "cuda")
    o, lse = _fwd(q, k, v, cu_q, cu_k, max(lq), scale, causal)
    got, _ = _bwd(q, k, v, o, lse, do, cu_q, cu_k, max(lq), max(lk), scale, causal)
    assert all(bool(torch.isfinite(t).all()) for t in got)
    g64 = ar.packed_grads(q.cpu(), k.cpu(), v.cpu(), do.cpu(), cu_q.cpu(), cu_k.cpu(), scale, causal)[:3]
    qa, ka, va = (t.clone().requires_grad_() for t in (q, k, v))  # the same math in the dtype through torch autograd
    ar.packed(qa, ka, va, cu_q, cu_k, scale, causal, q.dtype)[0].backward(do)
    for name, a, r, w in zip(("dq", "dk", "dv"), got, (qa.grad, ka.grad, va.grad), g64):
        w = w.cuda()
        err, err_ref = (a.double() - w).abs().max().item(), (r.double() - w).abs().max().item()
        eps = ea.ulp(w.abs().max().view(1), a.dtype).item()
        assert err <= 2 * err_ref + eps, (name, err, err_ref, eps)
    # each sequence alone: the same bits
    for q0, q1, k0, k1 in ar.seqs(cu_q.cpu(), cu_k.cpu()):
        if q1 == q0 or k1 == k0:
            continue
        c1, c2 = ar.cu([q1 - q0], "cuda"), ar.cu([k1 - k0], "cuda")
        sl = [t[q0:q1].contiguous() for t in (q, o, do)] + [t[k0:k1].contiguous() for t in (k, v)]
        alone, _ = _bwd(sl[0], sl[3], sl[4], sl[1], lse[q0:q1].contiguous(), sl[2], c1, c2, q1 - q0, k1 - k0, scale, causal)
        assert torch.equal(_bits(alone[0]), _bits(got[0][q0:q1]))
        assert torch.equal(_bits(alone[1]), _bits(got[1][k0:k1]))
        assert torch.equal(_bits(alone[2]), _bits(got[2][k0:k1]))


# ------------------------------------------------------------------------------------------------ edges, bounds
@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_edge_rows_bounds_determinism_graph_and_thread(dtype):
    """Causal with Lq > Lk (rows that see no key), Lq < Lk (keys no query sees), an empty query and an empty key
    sequence, and 50 query / 30 key tokens past cu_seqlens[B]."""
    lq, lk, H, H_kv, D = (200, 0, 70, 5), (90, 40, 0, 300), 8, 2, 96
    q, k, v, do = _random(lq, lk, H, H_kv, D, dtype, 5)
    q, do = (torch.cat([t, torch.randn(50, H, D, device="cuda").to(dtype)]) for t in (q, do))
    k, v = (torch.cat([t, torch.randn(30, H_kv, D, device="cuda").to(dtype)]) for t in (k, v))
    cu_q, cu_k = ar.cu(lq, "cuda"), ar.cu(lk, "cuda")
    o, lse = _fwd(q, k, v, cu_q, cu_k, max(lq), None, True)
    inputs = [t.clone() for t in (q, k, v, o, lse, do, cu_q, cu_k)]
    first, bufs = _bwd(q, k, v, o, lse, do, cu_q, cu_k, max(lq), max(lk), None, True)
    second, _ = _bwd(q, k, v, o, lse, do, cu_q, cu_k, max(lq), max(lk), None, True)
    dq, dk, dv = first
    for a, b, buf in zip(first, second, bufs):
        assert torch.equal(_bits(a), _bits(b))
        assert not torch.isnan(a.float()).any()
        assert torch.isnan(buf[:GUARD].float()).all() and torch.isnan(buf[-GUARD:].float()).all()
    for a, b in zip(inputs, (q, k, v, o, lse, do, cu_q, cu_k)):
        assert torch.equal(a, b)
    assert _pos_zero(dq[:110]) and not _pos_zero(dq[110:200])  # rows r < Lq - Lk = 110 see no key
    assert _pos_zero(dq[200:270]) and _pos_zero(dk[90:130]) and _pos_zero(dv[90:130])  # Lk = 0, Lq = 0
    assert _pos_zero(dq[-50:]) and _pos_zero(dk[-30:]) and _pos_zero(dv[-30:])  # outside every sequence
    g64 = ar.packed_grads(q.cpu(), k.cpu(), v.cpu(), do.cpu(), cu_q.cpu(), cu_k.cpu(), None, True)[:3]
    for a, w in zip(first, g64):
        assert (a.double().cpu() - w).abs().max().item() < 0.1
    # graph replay
    outs = [torch.full_like(t, float("nan")) for t in (q, k, v)]
    args = (q, k, v, o, lse, do, *outs, cu_q, cu_k, max(lq), max(lk))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.fa2_bwd_varlen(*args, causal=True)
    torch.cuda.current_stream().wait_stream(s)
    for t in outs:
        t.fill_(float("nan"))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.fa2_bwd_varlen(*args, causal=True)
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(first, outs):
        assert torch.equal(_bits(a), _bits(b))
    # a fresh thread
    res = []
    th = threading.Thread(target=lambda: res.append(_bwd(q, k, v, o, lse, do, cu_q, cu_k, max(lq), max(lk), None, True)[0]))
    th.start()
    th.join()
    torch.cuda.synchronize()
    for a, b in zip(first, res[0]):
        assert torch.equal(_bits(a), _bits(b))


# ------------------------------------------------------------------------------------------------ autograd
@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
def test_attention_varlen_autograd(dtype, causal):
    lq, lk, H, H_kv, D = (300, 77, 513), (300, 150, 513), 8, 2, 64
    q, k, v, do = _random(lq, lk, H, H_kv, D, dtype, 3 + causal)
    cu_q, cu_k = ar.cu(lq, "cuda"), ar.cu(lk, "cuda")
    qa, ka, va = (t.clone().requires_grad_() for t in (q, k, v))
    out = ops.attention_varlen(qa, ka, va, cu_q, cu_k, max(lq), max(lk), causal=causal)
    out.backward(do.transpose(0, 1).contiguous().transpose(0, 1))  # a non-contiguous upstream gradient
    o, lse = _fwd(q, k, v, cu_q, cu_k, max(lq), None, causal)
    want, _ = _bwd(q, k, v, o, lse, do, cu_q, cu_k, max(lq), max(lk), None, causal)
    for a, b in zip((qa.grad, ka.grad, va.grad), want):
        assert torch.equal(_bits(a), _bits(b))
    g64 = ar.packed_grads(q.cpu(), k.cpu(), v.cpu(), do.cpu(), cu_q.cpu(), cu_k.cpu(), None, causal)[:3]
    ref = [torch.zeros_like(t) for t in (q, k, v)]
    for q0, q1, k0, k1 in ar.seqs(cu_q.cpu(), cu_k.cpu()):
        qs, ks, vs = (t[a:b].transpose(0, 1).unsqueeze(0).clone().requires_grad_() for t, a, b in
                      ((q, q0, q1), (k, k0, k1), (v, k0, k1)))
        mask = ar.visible(q1 - q0, k1 - k0, k1 - k0 - (q1 - q0) if causal else None, "cuda")
        torch.nn.functional.scaled_dot_product_attention(qs, ks, vs, attn_mask=mask, enable_gqa=True).backward(
            do[q0:q1].transpose(0, 1).unsqueeze(0))
        for r, t, a, b in zip(ref, (qs, ks, vs), (q0, k0, k0), (q1, k1, k1)):
            r[a:b] = t.grad[0].transpose(0, 1)
    for a, r, w in zip((qa.grad, ka.grad, va.grad), ref, g64):
        w = w.cuda()
        err, err_ref = (a.double() - w).abs().max().item(), (r.double() - w).abs().max().item()
        assert err <= 2 * err_ref + ea.ulp(w.abs().max().view(1), a.dtype).item(), (err, err_ref)
