"""GPU: the attention backward (ops.fa2_bwd, b200k_fa2_bwd) bit for bit against the closed form of graded_attention_bwd.py,
with nonzero dS, dS rounded to nearest (ties to even), fractional P rounded, every mask edge and decoys a wrong mask would
let through:
  - fp16 and bf16, D = 32, 64, 96, 128 (32 and 96 on their padded DP), full and causal, N = 1 .. 1000 on both sides of
    the 64-key tiles, seqlens_k of 1, 64, 65, N - 1 and the clamped 0, -5 and N + 5, B * H > 1 with t differing per
    head, and one 2048-key row per dtype within a factor of two of the fp32 window;
  - keys no row sees get dK = dV = 0, and no output is a negative zero: a masked dS is 0 * (0 - Delta), -0 when
    Delta > 0, yet every zero the kernels were found to store is +0, and the bit comparison holds them to it;
  - B * H = 65535, the largest grid the backward launches;
  - the forward's own O and lse on a consistent case (lse = fp32(t * 0.6931472f) exactly), and ops.attention with
    seqlens_k and an explicit scale giving the bits of fa2_fwd(lse=) + fa2_bwd.
Outputs go into NaN-filled buffers with guards (test_gpu_attention_bwd.py's helpers); the guards must keep their NaNs."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import graded_attention_bwd as gb  # noqa: E402
import test_gpu_attention_bwd as tb  # noqa: E402

from b200k import ops  # noqa: E402

pytestmark = pytest.mark.gpu
NAMES = ("dq", "dk", "dv")


def _cuda(case):
    return {n: (case[n].cuda() if isinstance(case[n], torch.Tensor) else case[n]) for n in case}


def _check(case, got, want, bufs):
    """got == want bit for bit (zeros included: the kernel's zeros are +0), guards untouched, unseen keys zero."""
    B, H, N, D = want[0].shape
    for name, a, w in zip(NAMES, got, want):
        bad = tb._bits(a) != tb._bits(w)
        assert not bool(bad.any()), gb.describe(case, name, w.cpu(), a.cpu(), count=3)
    kv = gb.kv_lens(None if case["seqlens"] is None else case["seqlens"].cpu(), B, N)
    for b in range(B):  # keys past the length: no row sees them
        for t in got[1:]:
            assert int(tb._bits(t[b, :, int(kv[b]):]).ne(0).sum()) == 0
    for buf in bufs:
        assert torch.isnan(buf[:tb.GUARD].float()).all() and torch.isnan(buf[-tb.GUARD:].float()).all()


def _run(c):
    case = _cuda(gb.make_case(**c))
    want, info = gb.closed_form(case["q"], case["k"], case["v"], case["o"], case["lse"], case["do"], case["scale"],
                                case["causal"], case["seqlens"])
    got, bufs = tb._bwd(case["q"], case["k"], case["v"], case["o"], case["lse"], case["do"], case["scale"], case["causal"],
                        case["seqlens"])
    _check(case, got, want, bufs)
    return info


@pytest.mark.parametrize("c", gb.all_cases(), ids=gb.case_id)
def test_graded_backward_bit_for_bit(c):
    _run(c)


def test_grid_limit_65535_heads():
    info = _run(gb.grid_case())
    assert info["ds_rounded"] > 0   # N = 3: every row is a rounding row


@pytest.mark.parametrize("c", gb.forward_cases(), ids=lambda c: gb.case_id(dict(c, causal=False)))
def test_forward_then_backward_and_autograd(c):
    """O and lse from fa2_fwd: lse is exact, the gradients are the closed form of those O and lse, and ops.attention
    (seqlens_k, explicit scale) returns the same O and the same gradient bits."""
    case = _cuda(gb.make_forward_case(**c))
    q, k, v, do, sl, scale = case["q"], case["k"], case["v"], case["do"], case["seqlens"], case["scale"]
    o, lse = tb._fwd(q, k, v, scale, False, sl)
    assert torch.equal(lse, gb.forward_lse(case["t"])), "forward lse is not fp32(t * 0.6931472f)"
    want, _ = gb.closed_form(q, k, v, o, lse, do, scale, False, sl)
    got, bufs = tb._bwd(q, k, v, o, lse, do, scale, False, sl)
    _check(case, got, want, bufs)
    qa, ka, va = (t.clone().requires_grad_() for t in (q, k, v))
    out = ops.attention(qa, ka, va, scale=scale, causal=False, seqlens_k=sl)
    out.backward(do)
    assert torch.equal(tb._bits(out.detach()), tb._bits(o))
    for name, a, w in zip(NAMES, (qa.grad, ka.grad, va.grad), got):
        assert torch.equal(tb._bits(a), tb._bits(w)), name
