"""CPU: the constructions of graded_attention_bwd.py.  The lse and scale identities hold (and the targets with no exact
lse are the known ones); the closed form is attention_ref.dense_grads_given within fp64; the three kernels' arithmetic,
emulated in fp32, gives the closed form bit for bit on every case the GPU test runs; the rounding paths are exercised;
and each way the backward could be subtly wrong (graded_attention_bwd.MUTATIONS) changes at least one expected bit of
one of those cases:
  ds_trunc      dS~ truncated         the rows whose |dP - Delta| exceeds the dtype's integers
  p_trunc       P~ truncated          the frac rows: dV[:, 0] holds their rounded P
  delta_swap    Delta of row r ^ 8    any row with nonzero P whose partner's Delta differs
  lse2_swap     lse2 of row r ^ 8     rows whose partner has another t (t = beta + W + {0, 1})
  causal_diag   key >= row masked     every causal case: the diagonal's P is lost
  causal_next   key > row + 1 masked  row E - 1 reads the cliff column with DECOY at key E: P = inf
  len_short     one key short         the key at kv_len - 1 is lost
  len_long      one key long          the key at kv_len holds DECOY in every column: P = inf
  scale_dv, dk_unscaled, dq_unscaled  any nonzero output
  ds_sign       dS = P (Delta - dP)   any nonzero dS
  delta_from_v  Delta = dO . V_i      normal and round rows (for frac rows dO . V_i = V_i0 = 1 = dO . O_i)
Mutations no case can see, and why:
  - lse2 = 0 instead of +inf for rows past N: P = 1 there, but TMA zero-fills those rows of Q and dO, so dS = P (0 - 0)
    and P dO add nothing;
  - a P~ truncated where P is an exact power of two: every integer-row P is one, so only the frac rows can tell;
  - the prep kernel's summation order of Delta: every Delta here is an exact fp32 sum."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attention_ref as ar  # noqa: E402
import graded_attention as ga  # noqa: E402
import graded_attention_bwd as gb  # noqa: E402

CASES = gb.all_cases()
_EXPECTED: dict = {}


def _inputs(c):
    x = gb.make_case(**c)
    return x, (x["q"], x["k"], x["v"], x["o"], x["lse"], x["do"], x["scale"], x["causal"], x["seqlens"])


def _expected(c):
    """(inputs, closed form as fp32 arrays, info), cached per case."""
    key = gb.case_id(c)
    if key not in _EXPECTED:
        x, args = _inputs(c)
        want, info = gb.closed_form(*args)
        _EXPECTED[key] = (x, args, [w.float().numpy() for w in want], info)
    return _EXPECTED[key]


def _forward_inputs(c):
    """make_forward_case with O as the forward computes it for these weights (exact softmax, one rounding) and
    lse = fp32(t * 0.6931472f)."""
    x = gb.make_forward_case(**c)
    B, H, N, D = x["q"].shape
    vis = gb.visible(B, H, N, False, x["seqlens"])
    g = (x["q"].double() @ x["k"].double().transpose(-1, -2)) * float(np.float32(x["scale"]) * np.float32(ga.LOG2E_F32))
    p = torch.where(vis, torch.exp2(g - x["t"].unsqueeze(-1)), torch.zeros_like(g))
    assert torch.equal(p.sum(-1), torch.ones(B, H, N, dtype=torch.float64)), "weights do not sum to 1"
    x["o"] = (p @ x["v"].double()).to(x["q"].dtype)
    x["lse"] = gb.forward_lse(x["t"])
    return x, (x["q"], x["k"], x["v"], x["o"], x["lse"], x["do"], x["scale"], False, x["seqlens"])


# ------------------------------------------------------------------------------------------------ identities
def test_scale_and_lse_identities():
    for k in range(4):
        assert np.float32(ga.scale_exact(k)) * np.float32(ga.LOG2E_F32) == np.float32(2.0 ** -k)
    for x in [0, 1, -1, 7, 12, 244, -5.625, 2.5, 5.125]:
        lse = gb.lse_exact(x)
        assert lse is not None and gb.lse2_of(lse) == np.float32(x)
    assert gb.no_exact_lse(-31, 31) == [-31, -30, -27, -26, -15, -13, 13, 15, 26, 27, 30, 31]
    assert [t for t in range(244, 256) if t in gb.no_exact_lse(240, 260)] == [248, 249, 250, 251]
    assert gb.lse_exact(3.375) is None and gb.lse_exact(1.875) is None      # eighths miss too
    # the forward's lse of a row whose max is m and whose weights sum to 2^u, t = m + u, survives lse * log2 e for
    # |t| <= 12 (and not at 13)
    t = torch.arange(-12, 13)
    assert torch.equal(torch.from_numpy(gb.lse2_of(gb.forward_lse(t).numpy())), t.float())
    assert gb.lse2_of(gb.forward_lse(torch.tensor([13])).numpy())[0] != 13
    e, lse = gb.exact_lse_of(torch.tensor([8 * 13, 8 * 15 + 3, 0]))
    assert e.tolist() == [8 * 14, 8 * 15 + 3, 0] and bool((torch.from_numpy(gb.lse2_of(lse.numpy())) == e / 8).all())


def test_window_is_enforced():
    A = torch.full((1, 1, 1, 600), 0.5, dtype=torch.float64)
    B = torch.full((1, 1, 600, 1), 2.0 ** 5, dtype=torch.float64)
    assert gb._window_mm(A, B, "ok") < 1                  # 600 terms of 2^4, G = -4: 600 * 2^4 * 2^-4 < 2^24
    A[..., 0] = 1 + 2.0 ** -20                           # one term of 21 bits: G = 15 and the sum is about 2^13
    with pytest.raises(AssertionError, match="window"):
        gb._window_mm(A, B, "too wide")


# ------------------------------------------------------------------------------------------------ closed form vs fp64
SMALL = [c for c in CASES if c["N"] in (63, 129) and c["D"] in (32, 96)][:6]


@pytest.mark.parametrize("c", SMALL, ids=gb.case_id)
def test_closed_form_is_grads_given(c):
    x, args = _inputs(c)
    _check_grads_given(x, args)


@pytest.mark.parametrize("c", gb.forward_cases()[:2], ids=lambda c: "fwd-%d" % c["N"])
def test_forward_case_closed_form_is_grads_given(c):
    x, args = _forward_inputs(c)
    _check_grads_given(x, args)


def _check_grads_given(x, args):
    """closed_form without the dtype roundings is the fp64 formula with O and lse as given, at the exponent's exact
    scale: scale_log2 ln 2, lse = lse2 ln 2."""
    q, k, v, o, lse, do, scale, causal, sl = args
    got, _ = gb.closed_form(*args, rounded=False)
    sl2 = float(np.float32(scale) * np.float32(ga.LOG2E_F32))
    lse_n = torch.from_numpy(gb.lse2_of(lse.numpy())).double() * math.log(2)
    want = ar.dense_grads_given(q, k, v, o, lse_n, do, sl2 * math.log(2), causal, sl)
    for a, w in zip(got, want):
        assert torch.allclose(a, w, rtol=1e-12, atol=1e-12 * float(w.abs().max() + 1))


# ------------------------------------------------------------------------------------------------ the kernels' arithmetic
@pytest.mark.parametrize("c", CASES, ids=gb.case_id)
def test_emulation_is_the_closed_form(c):
    x, args, want, info = _expected(c)
    got = gb.emulate_bwd(*args)
    for name, a, w in zip(("dq", "dk", "dv"), got, want):
        assert gb.same_bits(a, w), name


@pytest.mark.parametrize("c", gb.forward_cases(), ids=lambda c: "fwd-%d-%d" % (c["N"], c["D"]))
def test_forward_case_emulation_is_the_closed_form(c):
    x, args = _forward_inputs(c)
    want, _ = gb.closed_form(*args)
    got = gb.emulate_bwd(*args)
    for name, a, w in zip(("dq", "dk", "dv"), got, want):
        assert gb.same_bits(a, w.float().numpy()), name


def test_grid_case_builds():
    """The 65535-head case: its closed form holds (windows, exactness) and it has rounding rows."""
    _, args = _inputs(gb.grid_case())
    _, info = gb.closed_form(*args)
    assert info["ds_rounded"] > 0


def test_rounding_paths_are_exercised():
    """Over the GPU cases: dS rounded (some away from zero, where truncation differs, some ties), fractional P rounded,
    and the long case near the window."""
    tot = {}
    for c in CASES:
        info = _expected(c)[3]
        for key in ("ds_rounded", "ds_away", "ds_ties", "p_rounded", "ds_nonzero"):
            tot[key] = tot.get(key, 0) + info[key]
    print("graded backward cases:", len(CASES), tot)
    assert tot["ds_rounded"] > 1000 and tot["ds_away"] > 100 and tot["ds_ties"] > 100 and tot["p_rounded"] > 1000
    assert max(_expected(c)[3]["win_dq"] for c in gb.long_cases()) > 0.25


def test_every_mutation_changes_a_bit():
    """Each mutation of the emulated kernels changes at least one expected bit of some GPU case (smallest cases tried
    first)."""
    order = sorted(CASES, key=lambda c: c["B"] * c["H"] * c["N"] * c["N"] * c["D"])
    found = {}
    for mut in gb.MUTATIONS:
        for c in order:
            x, args, want, info = _expected(c)
            got = gb.emulate_bwd(*args, mut=mut)
            if not all(gb.same_bits(a, w) for a, w in zip(got, want)):
                found[mut] = gb.case_id(c)
                break
    print("mutations rejected by:", found)
    assert sorted(found) == sorted(gb.MUTATIONS), set(gb.MUTATIONS) - set(found)
