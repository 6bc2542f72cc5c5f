"""GPU: NaN, +Inf and -Inf in every element an attention call does not own (attention_poison.py) leave every output
bit-identical to the same call with zeros there, in the dense forward and backward with seqlens_k (V stored [N, D] and
[D, N]), the packed forward and backward, and the autograd wrappers ops.attention and ops.attention_varlen.

Each case checks the clean call against the fp64 slicing reference (the forward within the suite's TOL, the backward by
flash-attn's rule: at most twice the error of the same math in the dtype through torch autograd, plus one ulp), then runs
the call once per poison value and compares O, lse, dQ, dK and dV bit for bit, the sign of zero included.  Outputs go
into NaN-filled buffers with guards, which must keep their NaNs; packed O and lse rows outside every sequence must keep
whatever they held.  Exact-answer cases (needles forward and backward, graded integers backward) tie the bits under
poison to a closed form.

Lengths sit on both sides of the forward's 128-key tiles and the backward's 64-key tiles (1, 63, 64, 65, 127, 128, 129,
N - 1) and include the clamped seqlens_k 0 and -5; packed query lengths have Lq % 64 in {0, 1, 63}, Lq > Lk and Lq < Lk
under causal masking, an empty sequence between two others, GQA groups 1, 2, 8 and MQA, and padding tokens past
cu_seqlens[B] that a sequence's last tiles read."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attention_poison as ap  # noqa: E402
import attention_ref as ar  # noqa: E402
import exact_attention as ea  # noqa: E402
import graded_attention_bwd as gb  # noqa: E402
import test_gpu_attention_bwd as tb  # noqa: E402
import test_gpu_attention_varlen_bwd as tvb  # noqa: E402

from b200k import ops  # noqa: E402

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]
N = 200
LENS = [1, 63, 64, 65, 127, 128, 129, N - 1, 0, -5]
H = 2
PAD = 70                                    # tokens past cu_seqlens[B]: more than a query or key tile's overhang


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _same_bits(got, want, what):
    for name, a, b in zip(("o/dq", "lse/dk", "dv"), got, want):
        bad = _bits(a) != _bits(b)
        assert not bool(bad.any()), "%s %s: %d elements differ, first at %s" % (
            what, name, int(bad.sum()), bad.nonzero()[0].tolist())


def _guards_kept(bufs):
    for buf in bufs:
        assert torch.isnan(buf[:tb.GUARD].float()).all() and torch.isnan(buf[-tb.GUARD:].float()).all()


def _grad_rule(got, ref, g64, what):
    """max|g - g64| <= 2 max|g_ref - g64| + one ulp of the dtype at max|g64| (test_gpu_attention_bwd's rule)."""
    for name, a, r, w in zip(("dq", "dk", "dv"), got, ref, g64):
        w = w.to(a.device)
        err, err_ref = (a.double() - w).abs().max().item(), (r.double() - w).abs().max().item()
        eps = ea.ulp(w.abs().max().view(1), a.dtype).item()
        assert err <= 2 * err_ref + eps, (what, name, err, err_ref, eps)


# ------------------------------------------------------------------------------------------------ dense
def _dense_inputs(dtype, D, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q, k, v, do = (torch.randn(len(LENS), H, N, D, generator=g, device="cuda").to(dtype) for _ in range(4))
    sl = torch.tensor(LENS, dtype=torch.int32, device="cuda")
    m = ap.dense_kv_mask(k.shape, sl)
    k, v = ap.poison(k, m, 0.0), ap.poison(v, m, 0.0)   # the clean call: zeros where the poison goes
    return q, k, v, do, sl, m


def _dense_fwd(q, k, v, sl, causal, v_dn=False):
    """(o, lse, guarded buffers); v is [B, H, D, N] when v_dn."""
    (o, ob), (lse, lb) = tb._out(q.shape, q.dtype), tb._out(q.shape[:-1], torch.float32)
    ops.fa2_fwd(q, k, v, o, causal=causal, seqlens_k=sl, lse=lse, v_is_dn=v_dn)
    return (o, lse), (ob, lb)


DENSE_FWD = [(dt, D, False) for dt in DTYPES for D in (32, 64, 96, 128)] + [(torch.float16, D, True) for D in (64, 128)]


@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("dtype,D,v_dn", DENSE_FWD,
                         ids=["%s-D%d%s" % ("f16" if c[0] == torch.float16 else "bf16", c[1], "-vdn" if c[2] else "")
                              for c in DENSE_FWD])
def test_dense_forward_poisoned_keys(dtype, D, v_dn, causal):
    q, k, v, _, sl, m = _dense_inputs(dtype, D, seed=D + 2 * causal + v_dn)
    vt = (lambda t: t.transpose(-1, -2).contiguous()) if v_dn else (lambda t: t)  # noqa: E731
    clean, bufs = _dense_fwd(q, k, vt(v), sl, causal, v_dn)
    o64, lse64 = ar.dense(q.cpu(), k.cpu(), v.cpu(), None, causal, sl)
    assert torch.allclose(clean[0].float().cpu(), o64.to(dtype).float(), **ar.TOL[dtype])
    assert torch.allclose(clean[1].double().cpu(), lse64, rtol=0, atol=1e-2)
    _guards_kept(bufs)
    mv = m.transpose(-1, -2) if v_dn else m
    for value in ap.VALUES:
        got, bufs = _dense_fwd(q, ap.poison(k, m, value), ap.poison(vt(v), mv, value), sl, causal, v_dn)
        _same_bits(got, clean, "poison %s" % value)
        _guards_kept(bufs)


@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("D", [32, 64, 96, 128])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_dense_backward_poisoned_keys(dtype, D, causal):
    q, k, v, do, sl, m = _dense_inputs(dtype, D, seed=3 * D + causal)
    o, lse = (t.clone() for t in _dense_fwd(q, k, v, sl, causal)[0])  # O 16-byte aligned, as the backward needs
    clean, bufs = tb._bwd(q, k, v, o, lse, do, None, causal, sl)
    _guards_kept(bufs)
    g64 = ar.dense_grads(q.cpu(), k.cpu(), v.cpu(), do.cpu(), None, causal, sl)[:3]
    _grad_rule(clean, tb._torch_grads(q, k, v, do, None, causal, sl), g64, "clean")
    for value in ap.VALUES:
        got, bufs = tb._bwd(q, ap.poison(k, m, value), ap.poison(v, m, value), o, lse, do, None, causal, sl)
        _same_bits(got, clean, "poison %s" % value)
        _guards_kept(bufs)


@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_dense_exact_needles_poisoned_keys(dtype, causal):
    """test_gpu_attention_bwd's needles with poisoned padding: O = V[needle], dQ = dK = +0 and dV the sum of the dO rows
    whose needle is each key, bit for bit."""
    lens = (1, 63, 64, 65, 127, 128, 129, N - 1)
    B, D = len(lens), 64
    g = torch.Generator().manual_seed(17 + causal)
    q, k, needle = tb._needle_inputs(B, H, N, D, dtype, causal, lens, g)
    v, do = (torch.randint(-8, 9, (B, H, N, D), generator=g).to(dtype) for _ in range(2))
    q, k, v, do, needle = (t.cuda() for t in (q, k, v, do, needle))
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    m = ap.dense_kv_mask(k.shape, sl)
    idx = needle.unsqueeze(-1).expand(B, H, N, D)
    want_dv = torch.zeros(B, H, N, D, dtype=torch.float64, device="cuda").scatter_add_(2, idx, do.double()).to(dtype)
    zero = torch.zeros_like(q)
    for value in ap.VALUES:
        kp, vp = ap.poison(k, m, value), ap.poison(v, m, value)
        o, lse = (t.clone() for t in _dense_fwd(q, kp, vp, sl, causal)[0])
        assert torch.equal(_bits(o), _bits(torch.gather(v, 2, idx))), value
        (dq, dk, dv), bufs = tb._bwd(q, kp, vp, o, lse, do, None, causal, sl)
        _same_bits((dq, dk, dv), (zero, zero, want_dv), "poison %s" % value)
        _guards_kept(bufs)


@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_dense_graded_backward_poisoned_keys(dtype, D, causal):
    """graded_attention_bwd's closed form (nonzero dS, rounded dS and P) with the keys past seqlens_k poisoned."""
    case = gb.make_case(dtype, 4, 2, 130, D, causal, lens=(1, 64, 65, 0), seed=D + causal, k=1)
    case = {n: (t.cuda() if isinstance(t, torch.Tensor) else t) for n, t in case.items()}
    q, k, v, o, lse, do, sl, scale = (case[n] for n in ("q", "k", "v", "o", "lse", "do", "seqlens", "scale"))
    want, info = gb.closed_form(q, k, v, o, lse, do, scale, causal, sl)
    assert info["ds_nonzero"] > 0
    m = ap.dense_kv_mask(k.shape, sl)
    for value in ap.VALUES:
        got, bufs = tb._bwd(q, ap.poison(k, m, value), ap.poison(v, m, value), o, lse, do, scale, causal, sl)
        _same_bits(got, want, "poison %s" % value)
        _guards_kept(bufs)


@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_attention_autograd_poisoned_keys(dtype, causal):
    q, k, v, do, sl, m = _dense_inputs(dtype, 64, seed=5 + causal)

    def run(k, v):
        qa, ka, va = (t.clone().requires_grad_() for t in (q, k, v))
        out = ops.attention(qa, ka, va, causal=causal, seqlens_k=sl)
        out.backward(do)
        return out.detach(), qa.grad, ka.grad, va.grad

    clean = run(k, v)
    for value in ap.VALUES:
        got = run(ap.poison(k, m, value), ap.poison(v, m, value))
        _same_bits(got[:1], clean[:1], "o, poison %s" % value)
        _same_bits(got[1:], clean[1:], "grads, poison %s" % value)


# ------------------------------------------------------------------------------------------------ packed
def _packed_inputs(lq, lk, Hq, H_kv, D, dtype, seed):
    """q, k, v, do with PAD zero tokens past cu_seqlens[B], the cu_seqlens and the masks of the padding."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    z = lambda h: torch.zeros(PAD, h, D, device="cuda", dtype=dtype)  # noqa: E731
    q, do = (torch.cat([torch.randn(sum(lq), Hq, D, generator=g, device="cuda").to(dtype), z(Hq)]) for _ in range(2))
    k, v = (torch.cat([torch.randn(sum(lk), H_kv, D, generator=g, device="cuda").to(dtype), z(H_kv)]) for _ in range(2))
    cu_q, cu_k = ar.cu(lq, "cuda"), ar.cu(lk, "cuda")
    mq, mk = ap.packed_masks(cu_q.cpu(), cu_k.cpu(), q.shape, k.shape)
    return q, k, v, do, cu_q, cu_k, mq, mk


def _packed_fwd(q, k, v, cu_q, cu_k, mq_value, causal, mq=None):
    """(o, lse): o and lse start as zeros (or `mq_value` on the tokens of mq) in guarded NaN buffers."""
    (o, ob), (lse, lb) = tb._out(q.shape, q.dtype), tb._out(q.shape[:-1], torch.float32)
    o.zero_()
    lse.zero_()
    if mq is not None:
        o.copy_(ap.poison(o, mq, mq_value))
        lse.copy_(ap.poison(lse, mq[..., 0], mq_value))
    mlq = int((cu_q[1:] - cu_q[:-1]).max())
    ops.fa2_fwd_varlen(q, k, v, o, cu_q, cu_k, max(mlq, 1), causal=causal, lse=lse)
    return (o, lse), (ob, lb)


def _packed_bwd(q, k, v, o, lse, do, cu_q, cu_k, causal):
    mlq, mlk = (max(int((c[1:] - c[:-1]).max()), 1) for c in (cu_q, cu_k))
    return tvb._bwd(q, k, v, o, lse, do, cu_q, cu_k, mlq, mlk, None, causal)


# (lq, lk): Lq % 64 in {0, 1, 63}, lengths around the 128-key tile, Lq > Lk and Lq < Lk; an empty sequence between two
PACKS = {"tails": ((64, 1, 63, 127, 128, 129), (129, 127, 63, 65, 128, 1)),
         "empty": ((65, 0, 70, 1), (100, 0, 30, 64))}
# (pack, H, H_kv): GQA groups 1, 2, 8 and MQA
PACKED = [("tails", 4, 4), ("tails", 16, 2), ("empty", 4, 2), ("empty", 8, 1)]
PACKED_IDS = ["%s-G%d" % (p, h // hk) if hk > 1 else "%s-MQA" % p for p, h, hk in PACKED]


@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("D", [32, 64, 96, 128])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("pack,Hq,H_kv", PACKED, ids=PACKED_IDS)
def test_packed_forward_poisoned_padding(pack, Hq, H_kv, dtype, D, causal):
    lq, lk = PACKS[pack]
    q, k, v, _, cu_q, cu_k, mq, mk = _packed_inputs(lq, lk, Hq, H_kv, D, dtype, seed=D + Hq + causal)
    clean, bufs = _packed_fwd(q, k, v, cu_q, cu_k, 0.0, causal)
    _guards_kept(bufs)
    o64, lse64 = ar.packed(q.cpu(), k.cpu(), v.cpu(), cu_q, cu_k, None, causal)
    assert torch.allclose(clean[0].float().cpu(), o64.to(dtype).float(), **ar.TOL[dtype])
    assert torch.allclose(clean[1].double().cpu(), lse64.masked_fill(mq[..., 0], 0.0), rtol=0, atol=1e-2)
    for value in ap.VALUES:
        got, bufs = _packed_fwd(ap.poison(q, mq, value), ap.poison(k, mk, value), ap.poison(v, mk, value), cu_q, cu_k,
                                value, causal, mq)
        want = (ap.poison(clean[0], mq, value), ap.poison(clean[1], mq[..., 0], value))  # padding rows: not written
        _same_bits(got, want, "poison %s" % value)
        _guards_kept(bufs)


@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("D", [32, 64, 96, 128])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("pack,Hq,H_kv", PACKED, ids=PACKED_IDS)
def test_packed_backward_poisoned_padding(pack, Hq, H_kv, dtype, D, causal):
    lq, lk = PACKS[pack]
    q, k, v, do, cu_q, cu_k, mq, mk = _packed_inputs(lq, lk, Hq, H_kv, D, dtype, seed=3 * D + Hq + causal)
    o, lse = (t.clone() for t in _packed_fwd(q, k, v, cu_q, cu_k, 0.0, causal)[0])
    clean, bufs = _packed_bwd(q, k, v, o, lse, do, cu_q, cu_k, causal)
    _guards_kept(bufs)
    g64 = ar.packed_grads(q.cpu(), k.cpu(), v.cpu(), do.cpu(), cu_q, cu_k, None, causal)[:3]
    qa, ka, va = (t.clone().requires_grad_() for t in (q, k, v))  # the same math in the dtype through torch autograd
    ar.packed(qa, ka, va, cu_q, cu_k, None, causal, dtype)[0].backward(do)
    _grad_rule(clean, (qa.grad, ka.grad, va.grad), g64, "clean")
    mlse = mq[..., 0]
    for value in ap.VALUES:
        qs = [ap.poison(t, mq, value) for t in (q, o, do)]
        got, bufs = _packed_bwd(qs[0], ap.poison(k, mk, value), ap.poison(v, mk, value), qs[1],
                                ap.poison(lse, mlse, value), qs[2], cu_q, cu_k, causal)
        _same_bits(got, clean, "poison %s" % value)
        _guards_kept(bufs)


@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("H_kv", [4, 1], ids=["G2", "MQA"])
def test_packed_exact_needles_poisoned_padding(H_kv, dtype, causal):
    """test_gpu_attention_varlen_bwd's needles with poisoned padding: O = V[needle] (0 for a row that sees no key),
    dQ = dK = +0 and dV of each key the sum over the group of the dO rows whose needle it is, bit for bit."""
    lq, lk, Hq, D = (65, 127, 0, 64), (129, 63, 0, 1), 8, 64
    g = torch.Generator().manual_seed(23 + H_kv + causal)
    q, k, needle = tvb._needles(lq, lk, Hq, H_kv, D, dtype, causal, g)
    v = torch.randint(-8, 9, k.shape, generator=g).to(dtype)
    do = torch.randint(-8, 9, q.shape, generator=g).to(dtype)
    pad = lambda t: torch.cat([t, torch.zeros(PAD, *t.shape[1:], dtype=t.dtype)]).cuda()  # noqa: E731
    q, k, v, do = (pad(t) for t in (q, k, v, do))
    needle = torch.cat([needle, torch.full((PAD, Hq), -1, dtype=torch.long)]).cuda()
    cu_q, cu_k = ar.cu(lq, "cuda"), ar.cu(lk, "cuda")
    mq, mk = ap.packed_masks(cu_q.cpu(), cu_k.cpu(), q.shape, k.shape)
    seen = needle >= 0
    kvh = (torch.arange(Hq, device="cuda") // (Hq // H_kv)).view(1, Hq).expand_as(needle)
    want_o = torch.where(seen.unsqueeze(-1), v[needle.clamp(min=0), kvh], torch.zeros_like(q))
    want_dv = torch.zeros(k.shape, dtype=torch.float64, device="cuda")
    want_dv.index_put_((needle[seen], kvh[seen]), do[seen].double(), accumulate=True)
    for value in ap.VALUES:
        qp, kp, vp, dop = (ap.poison(t, m, value) for t, m in ((q, mq), (k, mk), (v, mk), (do, mq)))
        o, lse = (t.clone() for t in _packed_fwd(qp, kp, vp, cu_q, cu_k, value, causal, mq)[0])
        _same_bits((o,), (ap.poison(want_o, mq, value),), "o, poison %s" % value)
        got, bufs = _packed_bwd(qp, kp, vp, o, lse, dop, cu_q, cu_k, causal)
        _same_bits(got, (torch.zeros_like(q), torch.zeros_like(k), want_dv.to(dtype)), "grads, poison %s" % value)
        _guards_kept(bufs)


@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_packed_isolation(dtype, D, causal):
    """Sequences 1 and 3, right after ones of 65 and 129 tokens, poisoned whole (Q, K, V, O, dO and lse): every other
    sequence keeps the bits of its O, lse, dQ, dK and dV."""
    lq, lk, Hq, H_kv = (65, 50, 129, 40, 30), (65, 70, 129, 100, 20), 8, 2
    q, k, v, do, cu_q, cu_k, _, _ = _packed_inputs(lq, lk, Hq, H_kv, D, dtype, seed=D + causal)
    o, lse = (t.clone() for t in _packed_fwd(q, k, v, cu_q, cu_k, 0.0, causal)[0])
    clean = _packed_bwd(q, k, v, o, lse, do, cu_q, cu_k, causal)[0]
    seqs = ar.seqs(cu_q.cpu(), cu_k.cpu())
    mq = torch.zeros(q.shape, dtype=torch.bool)
    mk = torch.zeros(k.shape, dtype=torch.bool)
    for b in (1, 3):
        mq[seqs[b][0]:seqs[b][1]] = True
        mk[seqs[b][2]:seqs[b][3]] = True
    for value in ap.VALUES:
        qp, kp, vp, op, dop = (ap.poison(t, m, value) for t, m in ((q, mq), (k, mk), (v, mk), (o, mq), (do, mq)))
        (o2, lse2), _ = _packed_fwd(qp, kp, vp, cu_q, cu_k, 0.0, causal)
        got = _packed_bwd(qp, kp, vp, op, ap.poison(lse, mq[..., 0], value), dop, cu_q, cu_k, causal)[0]
        for b in (0, 2, 4):
            q0, q1, k0, k1 = seqs[b]
            what = "sequence %d, poison %s" % (b, value)
            _same_bits((o2[q0:q1], lse2[q0:q1]), (o[q0:q1], lse[q0:q1]), what)
            _same_bits((got[0][q0:q1], got[1][k0:k1], got[2][k0:k1]),
                       (clean[0][q0:q1], clean[1][k0:k1], clean[2][k0:k1]), what)


@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_attention_varlen_autograd_poisoned_padding(dtype, causal):
    lq, lk = PACKS["tails"]
    q, k, v, do, cu_q, cu_k, mq, mk = _packed_inputs(lq, lk, 8, 2, 64, dtype, seed=9 + causal)

    def run(q, k, v, do):
        qa, ka, va = (t.clone().requires_grad_() for t in (q, k, v))
        out = ops.attention_varlen(qa, ka, va, cu_q, cu_k, max(lq), max(lk), causal=causal)
        out.backward(do)
        return out.detach()[:int(cu_q[-1])], qa.grad, ka.grad, va.grad

    clean = run(q, k, v, do)
    for value in ap.VALUES:
        got = run(*(ap.poison(t, m, value) for t, m in ((q, mq), (k, mk), (v, mk), (do, mq))))
        _same_bits(got[:1], clean[:1], "o, poison %s" % value)
        _same_bits(got[1:], clean[1:], "grads, poison %s" % value)
