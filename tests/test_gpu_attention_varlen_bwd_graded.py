"""GPU: the packed attention backward (ops.fa2_bwd_varlen, b200k_fa2_bwd_varlen) bit for bit against the closed form of
graded_attention_varlen_bwd.py, whose every case test_attention_varlen_bwd_graded_cpu.py proves on the CPU:
  - fp16 and bf16, D = 32, 64, 96, 128, full and causal, G = 1, 2, 8 and MQA with nonzero dS summed over the group,
    lengths 0 .. 1000 on both sides of the 64-row and 64-key tiles, bottom-right causal shifts of 0, +-1, +-63, +-64,
    +-65 and beyond, empty query and key sequences first, middle and last, tokens before cu[0] and after cu[B], and one
    2048-key sequence per dtype within a factor of two of the fp32 window in dK;
  - keys of an empty query sequence, rows that see no key (lse = -inf) and tokens outside every sequence are +0, no
    output is a negative zero, and the guards around every output keep their NaNs;
  - B * H = 65535, the largest dQ grid;
  - the forward's own O and lse on a consistent GQA case (lse = fp32(t * 0.6931472f) exactly), and ops.attention_varlen
    giving the same O and the same gradient bits;
  - a call past 2^31 elements of Q and dQ, whose graded sequences straddle element 2^31 and end the call.
Outputs go into NaN-filled buffers with guards (test_gpu_attention_varlen_bwd.py's helpers)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import graded_attention_bwd as gb  # noqa: E402
import graded_attention_varlen_bwd as gv  # noqa: E402
import test_gpu_attention_varlen_bwd as tv  # noqa: E402

from b200k import ops  # noqa: E402

pytestmark = pytest.mark.gpu
NAMES = ("dq", "dk", "dv")


def _cuda(x):
    return {n: (t.cuda() if isinstance(t, torch.Tensor) and n not in ("col", "t", "kind") else t) for n, t in x.items()}


def _zero(t):
    return int(torch.count_nonzero(tv._bits(t))) == 0


def _bwd(x):
    return tv._bwd(x["q"], x["k"], x["v"], x["o"], x["lse"], x["do"], x["cu_q"], x["cu_k"], x["max_q"], x["max_k"],
                   x["scale"], x["causal"])


def _check(x, got, want, bufs):
    """got == want bit for bit (so every zero is +0), then by name: keys of empty query sequences, rows that see no
    key, tokens outside every sequence, and the guards."""
    for name, a, w in zip(NAMES, got, want):
        assert torch.equal(tv._bits(a), tv._bits(w)), gv.describe(x, name, w, a)
    dq, dk, dv = got
    cq, ck = x["cu_q"].tolist(), x["cu_k"].tolist()
    for b in range(len(cq) - 1):
        if cq[b + 1] == cq[b]:
            assert _zero(dk[ck[b]:ck[b + 1]]) and _zero(dv[ck[b]:ck[b + 1]]), "keys of empty query sequence %d" % b
    assert _zero(dq[(x["lse"] == float("-inf"))]), "a row that sees no key"
    assert _zero(dq[:cq[0]]) and _zero(dq[cq[-1]:]), "query tokens outside every sequence"
    assert all(_zero(t[:ck[0]]) and _zero(t[ck[-1]:]) for t in (dk, dv)), "key tokens outside every sequence"
    for buf in bufs:
        assert torch.isnan(buf[:tv.GUARD].float()).all() and torch.isnan(buf[-tv.GUARD:].float()).all()


def _run(c):
    x = _cuda(gv.make_case(**c))
    want, info = gv.closed_form(x)
    got, bufs = _bwd(x)
    _check(x, got, want, bufs)
    return info


@pytest.mark.parametrize("c", gv.all_cases(), ids=gv.case_id)
def test_graded_packed_backward_bit_for_bit(c):
    _run(c)


def test_grid_limit_65535_heads():
    info = _run(gv.grid_case())
    assert info["ds_rounded"] > 0 and info["ds_group"] > 0


@pytest.mark.parametrize("c", gv.forward_cases(), ids=lambda c: "fwd-D%d-H%d-%d" % (c["D"], c["H"], c["H_kv"]))
def test_forward_then_backward_and_autograd(c):
    """O and lse from fa2_fwd_varlen: lse is exact and O the exact P V rounded once, the gradients are the closed form of
    those O and lse, and ops.attention_varlen returns the same O and the same gradient bits."""
    x = _cuda(gv.make_forward_case(**c))
    q, k, v, do, cu_q, cu_k = (x[n] for n in ("q", "k", "v", "do", "cu_q", "cu_k"))
    o, lse = tv._fwd(q, k, v, cu_q, cu_k, x["max_q"], x["scale"], False)
    assert torch.equal(lse, gb.forward_lse(x["t"]).cuda()), "forward lse is not fp32(t * 0.6931472f)"
    o_cpu, _ = gv.forward_outputs({n: (t.cpu() if isinstance(t, torch.Tensor) else t) for n, t in x.items()})
    assert torch.equal(tv._bits(o), tv._bits(o_cpu.cuda())), "forward O is not the exact P V rounded once"
    x["o"], x["lse"] = o, lse
    want, _ = gv.closed_form(x)
    got, bufs = _bwd(x)
    _check(x, got, want, bufs)
    qa, ka, va = (t.clone().requires_grad_() for t in (q, k, v))
    out = ops.attention_varlen(qa, ka, va, cu_q, cu_k, x["max_q"], x["max_k"], scale=x["scale"], causal=False)
    out.backward(do)
    assert torch.equal(tv._bits(out.detach()), tv._bits(o))
    for name, a, w in zip(NAMES, (qa.grad, ka.grad, va.grad), got):
        assert torch.equal(tv._bits(a), tv._bits(w)), name


def test_past_2_31_elements():
    """H = 16, H_kv = 2, D = 128 and 2052 sequences, 1,050,729 query tokens: 2^31 + 4.4 M elements of Q, O, dO and dQ
    (about 18 GiB in all).  The graded sequences of big_core straddle element 2^31 (token 2^20) and end the call; every
    other token is zero with lse = 0, so its gradients are +0, and any element a wrapped offset wrote elsewhere, or left
    NaN, shows."""
    c = gv.big_core()
    small = gv.make_case(**c)
    H, H_kv, D, dt = c["H"], c["H_kv"], c["D"], c["dtype"]
    (lq0, lk0), (lq1, lk1) = c["lens"]
    ZQ, ZK, before, after = 512, 64, 2047, 3
    lens = [(ZQ, ZK)] * before + [(lq0, lk0)] + [(ZQ, ZK)] * after + [(lq1, lk1)]
    cu_q = torch.tensor([0] + [a for a, _ in lens], dtype=torch.int64).cumsum(0)
    cu_k = torch.tensor([0] + [b for _, b in lens], dtype=torch.int64).cumsum(0)
    Tq, Tk = int(cu_q[-1]), int(cu_k[-1])
    s0, s1 = int(cu_q[before]), int(cu_q[-2])                 # the graded sequences' first query tokens
    t0, t1 = int(cu_k[before]), int(cu_k[-2])
    assert s0 < 2 ** 20 < s0 + lq0 and Tq * H * D > 2 ** 31
    q, o, do = (torch.zeros(Tq, H, D, dtype=dt, device="cuda") for _ in range(3))
    k, v = (torch.zeros(Tk, H_kv, D, dtype=dt, device="cuda") for _ in range(2))
    lse = torch.zeros(Tq, H, device="cuda")
    for big, name in ((q, "q"), (o, "o"), (do, "do"), (lse, "lse")):
        big[s0:s0 + lq0] = small[name][:lq0].cuda()
        big[s1:s1 + lq1] = small[name][lq0:lq0 + lq1].cuda()
    for big, name in ((k, "k"), (v, "v")):
        big[t0:t0 + lk0] = small[name][:lk0].cuda()
        big[t1:t1 + lk1] = small[name][lk0:lk0 + lk1].cuda()
    x = _cuda(small)
    want, _ = gv.closed_form(x)
    got, bufs = tv._bwd(q, k, v, o, lse, do, cu_q.int().cuda(), cu_k.int().cuda(), max(a for a, _ in lens),
                        max(b for _, b in lens), x["scale"], True)
    for name, a, w in zip(NAMES, got, want):
        (a0, n0), (a1, n1) = ((s0, lq0), (s1, lq1)) if name == "dq" else ((t0, lk0), (t1, lk1))
        graded = torch.cat([a[a0:a0 + n0], a[a1:a1 + n1]])   # big_core's own layout
        assert torch.equal(tv._bits(graded), tv._bits(w)), gv.describe(x, name, w, graded)
        a[a0:a0 + n0], a[a1:a1 + n1] = 0, 0
        assert _zero(a), "%s: %d nonzero elements outside the graded sequences" % (name, int(torch.count_nonzero(
            tv._bits(a))))
    for buf in bufs:
        assert torch.isnan(buf[:tv.GUARD].float()).all() and torch.isnan(buf[-tv.GUARD:].float()).all()
