"""GPU: the attention backward (ops.fa2_bwd, b200k_fa2_bwd) and the differentiable ops.attention.

  - exact answers on the needle inputs of exact_attention.py with every row's needle visible: dQ = dK = 0 and dV_j = the
    sum of the dO rows whose needle is j, bit for bit;
  - random inputs against the fp64 reference (attention_ref.py) by flash-attn's rule: the error is at most twice
    that of the same math in the input dtype through torch autograd, plus one ulp of the dtype;
  - two calls and a CUDA-graph replay give the same bits; outputs go into NaN-filled buffers with guards, exactly the
    documented elements change and the inputs do not;
  - ops.attention's gradients are the bits of fa2_fwd(lse=) + fa2_bwd, and match scaled_dot_product_attention's."""
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
GUARD = 30  # 60 bytes: the outputs sit 4- but not 16-byte aligned, as the header allows
DTYPES = [torch.float16, torch.bfloat16]


def _out(shape, dtype):
    """(view of `shape` in a NaN-filled buffer, the buffer with GUARD elements on each side)."""
    n = math.prod(shape)
    buf = torch.full((n + 2 * GUARD,), float("nan"), dtype=dtype, device="cuda")
    return buf[GUARD:GUARD + n].view(shape), buf


def _fwd(q, k, v, scale=None, causal=False, sl=None):
    o = torch.empty_like(q)
    lse = torch.empty(q.shape[:-1], device="cuda")
    ops.fa2_fwd(q, k, v, o, scale, causal=causal, seqlens_k=sl, lse=lse)
    return o, lse


def _bwd(q, k, v, o, lse, do, scale=None, causal=False, sl=None):
    """(dq, dk, dv, the three guarded buffers)."""
    outs = [_out(q.shape, q.dtype) for _ in range(3)]
    ops.fa2_bwd(q, k, v, o, lse, do, *(t for t, _ in outs), scale=scale, causal=causal, seqlens_k=sl)
    return [t for t, _ in outs], [b for _, b in outs]


def _bits(t):
    return t.view(torch.int16)


# ------------------------------------------------------------------------------------------------ exact answers
def _needle_inputs(B, H, N, D, dtype, causal, kv_len, g):
    """Q, K as exact_attention.py builds them, per (b, h): column c of K holds its needle at key nk[c] < kv_len[b]
    (nk[0] = 0), and row r takes a column whose needle it sees (nk[c] <= r when causal).  Returns q, k, the needle key of
    every row [B, H, N]."""
    q = torch.zeros(B, H, N, D, dtype=dtype)
    k = torch.zeros(B, H, N, D, dtype=dtype)
    needle = torch.zeros(B, H, N, dtype=torch.long)
    rows = torch.arange(N)
    for b in range(B):
        for h in range(H):
            nk = torch.randint(0, kv_len[b], (D,), generator=g)
            nk[0] = 0
            k[b, h, nk, torch.arange(D)] = ea.A
            ok = (nk.view(1, D) <= rows.view(N, 1)) if causal else torch.ones(N, D, dtype=torch.bool)
            col = torch.where(ok, torch.rand(N, D, generator=g), torch.full((N, D), -1.0)).argmax(1)
            q[b, h, rows, col] = ea.A
            needle[b, h] = nk[col]
    return q, k, needle


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("D", [32, 64, 96, 128])
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("N,lens", [(1, None), (77, None), (77, (77, 30)), (130, None), (130, (1, 129)),
                                    (1000, None), (1000, (640, 999))])
def test_exact_needles(dtype, D, causal, N, lens):
    """P is 1 at the needle and 0 elsewhere (M = A^2 scale log2 e = 1044 at D = 32 down to 522 at D = 128, so every
    other key's 2^-M underflows), and dP - Delta = 0 exactly at the needle (O = V[needle], and both are exact integer
    sums in fp32).  So dS = 0 everywhere: dQ = dK = 0, and dV_j sums the integer dO rows whose needle is j, exactly, then
    rounds once.  That needs the needle's P to round to 1.0 in the dtype: the exponent s scale log2 e - lse log2 e is
    off by the fp32 roundings of m (the forward's max), of lse and of lse log2 e, each at most half an fp32 ulp of a
    value below 2048 (2^-14), so P is within 3 * 2^-14 * ln 2 = 1.3e-4 of 1, inside fp16's half-spacing below 1
    (2^-12 = 2.4e-4)."""
    g = torch.Generator().manual_seed(N * 1000 + D + 7 * causal)
    B, H = 2, 2
    kv_len = lens if lens is not None else (N, N)
    q, k, needle = _needle_inputs(B, H, N, D, dtype, causal, kv_len, g)
    v = torch.randint(-8, 9, (B, H, N, D), generator=g).to(dtype)
    do = torch.randint(-8, 9, (B, H, N, D), generator=g).to(dtype)
    q, k, v, do = (t.cuda() for t in (q, k, v, do))
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda") if lens is not None else None
    o, lse = _fwd(q, k, v, None, causal, sl)
    idx = needle.cuda().unsqueeze(-1).expand(B, H, N, D)
    assert torch.equal(o, torch.gather(v, 2, idx))  # the forward's exact answer
    (dq, dk, dv), bufs = _bwd(q, k, v, o, lse, do, None, causal, sl)
    zero = torch.zeros_like(dq)
    assert torch.equal(dq, zero) and torch.equal(dk, zero)
    want = torch.zeros(B, H, N, D, dtype=torch.float64, device="cuda").scatter_add_(2, idx, do.double())
    assert torch.equal(dv, want.to(dtype))
    for b in range(B):  # keys no row sees: past the length, and (by construction) keys that are nobody's needle
        assert (dv[b, :, kv_len[b]:] == 0).all() and (dk[b, :, kv_len[b]:] == 0).all()
    for buf in bufs:
        assert torch.isnan(buf[:GUARD].float()).all() and torch.isnan(buf[-GUARD:].float()).all()


# ------------------------------------------------------------------------------------------------ random inputs
def _check_against_fp64(got, ref, g64, what):
    """max|g - g64| <= 2 max|g_ref - g64| + one ulp of the dtype at max|g64|: both round each output once, which alone
    can leave them an ulp apart at the largest element where the reference happens to round exactly."""
    for name, a, r, w in zip(("dq", "dk", "dv"), got, ref, g64):
        err, err_ref = (a.double() - w).abs().max().item(), (r.double() - w).abs().max().item()
        eps = ea.ulp(w.abs().max().view(1), a.dtype).item()
        assert err <= 2 * err_ref + eps, (what, name, err, err_ref, eps)


def _torch_grads(q, k, v, do, scale, causal, sl):
    """The same math in q's dtype through torch autograd (the reference forward)."""
    qa, ka, va = (t.clone().requires_grad_() for t in (q, k, v))
    ar.dense(qa, ka, va, scale, causal, sl, q.dtype)[0].backward(do)
    return qa.grad, ka.grad, va.grad


RANDOM = [(1, 2, 64, 32, None), (2, 3, 77, 64, (50, 77)), (1, 4, 200, 96, None), (2, 2, 333, 128, (333, 100)),
          (1, 8, 1024, 64, None), (2, 4, 1500, 32, (1500, 999)), (2, 16, 4096, 128, None)]


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("B,H,N,D,lens", RANDOM, ids=["x".join(map(str, s[:4])) + ("-sl" if s[4] else "") for s in RANDOM])
def test_random_against_fp64(dtype, causal, B, H, N, D, lens):
    g = torch.Generator(device="cuda").manual_seed(B * 7 + N + D)
    q, k, v, do = (torch.randn(B, H, N, D, generator=g, device="cuda").to(dtype) for _ in range(4))
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda") if lens is not None else None
    scale = 0.3 if N == 200 else None  # one explicit scale
    o, lse = _fwd(q, k, v, scale, causal, sl)
    got, _ = _bwd(q, k, v, o, lse, do, scale, causal, sl)
    assert all(bool(torch.isfinite(t).all()) for t in got)
    g64 = ar.dense_grads(q, k, v, do, scale, causal, sl)[:3]
    _check_against_fp64(got, _torch_grads(q, k, v, do, scale, causal, sl), g64, (B, H, N, D, lens))


# ------------------------------------------------------------------------------------------------ determinism, bounds
@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_deterministic_graph_replay_and_write_bounds(dtype):
    g = torch.Generator(device="cuda").manual_seed(11)
    B, H, N, D = 2, 3, 700, 96
    q, k, v, do = (torch.randn(B, H, N, D, generator=g, device="cuda").to(dtype) for _ in range(4))
    sl = torch.tensor([700, 333], dtype=torch.int32, device="cuda")
    o, lse = _fwd(q, k, v, None, True, sl)
    inputs = [t.clone() for t in (q, k, v, o, lse, do, sl)]
    first, bufs = _bwd(q, k, v, o, lse, do, None, True, sl)
    second, _ = _bwd(q, k, v, o, lse, do, None, True, sl)
    for a, b, buf in zip(first, second, bufs):
        assert torch.equal(_bits(a), _bits(b))
        assert not torch.isnan(a.float()).any()  # every element written
        assert torch.isnan(buf[:GUARD].float()).all() and torch.isnan(buf[-GUARD:].float()).all()  # nothing else
    for a, b in zip(inputs, (q, k, v, o, lse, do, sl)):
        assert torch.equal(a, b)
    # the same call captured in a CUDA graph (workspace allocated inside the capture, from the graph's pool)
    outs = [torch.full_like(q, float("nan")) for _ in range(3)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.fa2_bwd(q, k, v, o, lse, do, *outs, causal=True, seqlens_k=sl)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    for t in outs:
        t.fill_(float("nan"))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.fa2_bwd(q, k, v, o, lse, do, *outs, causal=True, seqlens_k=sl)
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(first, outs):
        assert torch.equal(_bits(a), _bits(b))


# ------------------------------------------------------------------------------------------------ autograd
@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("D", [64, 128])
def test_attention_autograd(dtype, causal, D):
    g = torch.Generator(device="cuda").manual_seed(D + causal)
    B, H, N = 2, 4, 513
    q, k, v, do = (torch.randn(B, H, N, D, generator=g, device="cuda").to(dtype) for _ in range(4))
    qa, ka, va = (t.clone().requires_grad_() for t in (q, k, v))
    out = ops.attention(qa, ka, va, causal=causal)
    out.backward(do)
    o, lse = _fwd(q, k, v, None, causal)
    assert torch.equal(_bits(out.detach()), _bits(o))
    want, _ = _bwd(q, k, v, o, lse, do, None, causal)
    for a, b in zip((qa.grad, ka.grad, va.grad), want):
        assert torch.equal(_bits(a), _bits(b))
    qs, ks, vs = (t.clone().requires_grad_() for t in (q, k, v))
    torch.nn.functional.scaled_dot_product_attention(qs, ks, vs, is_causal=causal).backward(do)
    g64 = ar.dense_grads(q, k, v, do, None, causal, None)[:3]
    _check_against_fp64((qa.grad, ka.grad, va.grad), (qs.grad, ks.grad, vs.grad), g64, ("sdpa", D))
    # a non-contiguous upstream gradient is made contiguous
    qa.grad = ka.grad = va.grad = None
    ops.attention(qa, ka, va, causal=causal).backward(do.transpose(1, 2).contiguous().transpose(1, 2))
    for a, b in zip((qa.grad, ka.grad, va.grad), want):
        assert torch.equal(_bits(a), _bits(b))


def test_backward_from_a_fresh_thread():
    """torch runs a backward on an autograd thread of its own; a thread on which no CUDA call has run yet must work."""
    g = torch.Generator(device="cuda").manual_seed(5)
    q, k, v, do = (torch.randn(1, 2, 200, 64, generator=g, device="cuda", dtype=torch.half) for _ in range(4))
    o, lse = _fwd(q, k, v)
    want, _ = _bwd(q, k, v, o, lse, do)
    got = [torch.empty_like(q) for _ in range(3)]
    err = []

    def run():
        try:
            ops.fa2_bwd(q, k, v, o, lse, do, *got)
        except Exception as e:  # reported in the main thread
            err.append(e)

    t = threading.Thread(target=run)
    t.start()
    t.join()
    torch.cuda.synchronize()
    assert not err, err
    for a, b in zip(got, want):
        assert torch.equal(_bits(a), _bits(b))
