"""CPU: the constructions of graded_attention_varlen_bwd.py.  The closed form is attention_ref.packed_grads_given within fp64;
the three kernels' arithmetic, emulated in fp32 at tile granularity, gives the closed form bit for bit on every case the
GPU test runs; the rounding paths and the group sums are exercised; and each way the packed backward could be subtly
wrong (graded_attention_varlen_bwd.MUTATIONS) changes at least one expected bit of one of those cases.  Besides the
dense file's mutations (test_attention_bwd_graded_cpu.py), the packed ones and what rejects them:
  group_first_only   any G > 1 case: the other heads' dS~ and P~ are lost from dK / dV
  group_interleaved  G > 1 with H_kv > 1: head h reads another K/V head's grades and V
  top_left           causal Lq != Lk: the diagonal moves by the shift, cliff rows see DECOY
  first_tile_late    causal shifts that are not multiples of 64: the rows of the partial first tile are lost from dK / dV
  q_tail_stats       the last sequence's last query tile runs into the junk past cu_q[B], whose lse = -100 gives
                     P = 2^144 = inf against zeroed Q and dO: NaN in dK / dV
  lse_head_major     any H > 1: rows take another row's lse2 / Delta
  no_key_lse         causal Lq > Lk with Lq - Lk not a multiple of 64: a row that sees no key sits in a visited tile,
                     where 2^(-inf + inf) = NaN
  kv_tail_len        the next sequence's Lk is longer (the dQ rows see its keys, DECOY in the boundary columns) or
                     shorter (keys are lost)
Mutations no case can see, and why:
  - the order of the group sum (heads, then tiles): every partial sum of dK and dV stays inside the fp32 window, so any
    order gives the same bits (and two calls giving the same bits is tested on the GPU);
  - a prep that leaves Delta or lse2 unwritten for tokens outside every sequence: no correct kernel reads them;
  - the dense file's three (lse2 = 0 past N, truncating an exact power of two, Delta's summation order), for the same
    reasons."""
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
import graded_attention_varlen_bwd as gv  # noqa: E402

CASES = gv.all_cases() + [gv.grid_case(), gv.big_core()]
_EXPECTED: dict = {}


def _expected(c):
    """(case, closed form as fp32 arrays, info), cached per case."""
    key = gv.case_id(c)
    if key not in _EXPECTED:
        x = gv.make_case(**c)
        want, info = gv.closed_form(x)
        _EXPECTED[key] = (x, [w.float().numpy() for w in want], info)
    return _EXPECTED[key]


def _forward(c):
    x = gv.make_forward_case(**c)
    x["o"], x["lse"] = gv.forward_outputs(x)
    return x


# ------------------------------------------------------------------------------------------------ closed form vs fp64
SMALL = [dict(dtype=torch.float16, D=32, causal=True, H=16, H_kv=2, lens=[(200, 70), (0, 5), (63, 129), (1, 0)],
              pre=(3, 2), post=(5, 4), seed=1, k=1),
         dict(dtype=torch.bfloat16, D=64, causal=True, H=8, H_kv=1, lens=[(70, 135), (130, 65)], seed=2, k=0),
         dict(dtype=torch.bfloat16, D=96, causal=False, H=4, H_kv=2, lens=[(65, 100), (7, 1)], post=(2, 2), seed=3, k=2)]


@pytest.mark.parametrize("x", [gv.make_case(**c) for c in SMALL] + [_forward(c) for c in gv.forward_cases()[:2]],
                         ids=["G8-causal-long-q", "MQA-causal", "G2-full", "fwd0", "fwd1"])
def test_closed_form_is_grads_given(x):
    """closed_form without the dtype roundings is the fp64 formula with O and lse as given, at the exponent's exact
    scale (scale_log2 ln 2, lse2 ln 2): the same gradients up to fp64 rounding."""
    got, _ = gv.closed_form(x, rounded=False)
    sl2 = float(np.float32(x["scale"]) * np.float32(ga.LOG2E_F32))
    lse_n = torch.from_numpy(gb.lse2_of(x["lse"].numpy())).double() * math.log(2)
    want = ar.packed_grads_given(x["q"], x["k"], x["v"], x["o"], lse_n, x["do"], x["cu_q"], x["cu_k"], sl2 * math.log(2),
                                 x["causal"])
    for a, w in zip(got, want):
        assert torch.allclose(a, w, rtol=1e-12, atol=1e-12 * float(w.abs().max() + 1))
    if x["causal"]:
        assert bool((x["lse"] == float("-inf")).any()), "no row that sees no key"


# ------------------------------------------------------------------------------------------------ the kernels' arithmetic
@pytest.mark.parametrize("c", CASES, ids=gv.case_id)
def test_emulation_is_the_closed_form(c):
    x, want, info = _expected(c)
    got = gv.emulate_bwd(x)
    for name, a, w in zip(("dq", "dk", "dv"), got, want):
        assert gb.same_bits(a, w), gv.describe(x, name, torch.from_numpy(w), torch.from_numpy(a))


@pytest.mark.parametrize("c", gv.forward_cases(), ids=lambda c: "fwd-D%d-H%d-%d" % (c["D"], c["H"], c["H_kv"]))
def test_forward_case_emulation_is_the_closed_form(c):
    x = _forward(c)
    want, _ = gv.closed_form(x)
    got = gv.emulate_bwd(x)
    for name, a, w in zip(("dq", "dk", "dv"), got, want):
        assert gb.same_bits(a, w.float().numpy()), name


def test_rounding_paths_are_exercised():
    """Over the GPU cases: dS rounded (some away from zero, where truncation differs, some ties), fractional P rounded,
    keys whose dK sums nonzero dS~ from two or more heads of the group, and the long cases' dK within a factor of two of
    the fp32 window."""
    tot = {}
    for c in CASES:
        info = _expected(c)[2]
        for key in ("ds_rounded", "ds_away", "ds_ties", "p_rounded", "ds_nonzero", "ds_group"):
            tot[key] = tot.get(key, 0) + info[key]
    print("graded packed backward cases:", len(CASES), tot)
    assert tot["ds_rounded"] > 1000 and tot["ds_away"] > 100 and tot["ds_ties"] > 100 and tot["p_rounded"] > 1000
    assert tot["ds_group"] > 1000
    win = [_expected(c)[2]["win_dk"] for c in gv.long_cases()]
    print("long cases, largest dK sum / fp32 window:", win)
    assert min(win) > 0.5


def test_cases_cover_the_edges():
    """Lengths on both sides of the tile edges, empty sequences first, middle and last, cu[0] > 0, padding after cu[B],
    every shift the cliffs need, and rows that see no key."""
    lq = {a for c in gv.cases() for a, _ in c["lens"]}
    lk = {b for c in gv.cases() for _, b in c["lens"]}
    want = {0, 1, 63, 64, 65, 127, 128, 129, 191, 192, 1000}
    assert want <= lq and want <= lk
    shifts = {b - a for c in gv.cases() for a, b in c["lens"] if a and b}
    assert {0, 1, -1, 63, -63, 64, -64, 65, -65} <= shifts and max(shifts) > 500 and min(shifts) < -500
    for side in (0, 1):
        pos = {i if i == 0 else ("last" if i == len(c["lens"]) - 1 else "middle")
               for c in gv.cases() for i, s in enumerate(c["lens"]) if s[side] == 0}
        assert pos == {0, "middle", "last"}, (side, pos)
    assert any(c["pre"][0] and c["pre"][1] for c in gv.cases()) and any(c["post"][0] and c["post"][1] for c in gv.cases())


def test_every_mutation_changes_a_bit():
    """Each mutation of the emulated kernels changes at least one expected bit of some GPU case (smallest cases tried
    first)."""
    order = sorted(CASES, key=lambda c: sum(a * b for a, b in c["lens"]) * c["H"] * c["D"])
    found = {}
    for mut in gv.MUTATIONS:
        for c in order:
            x, want, _ = _expected(c)
            got = gv.emulate_bwd(x, mut=mut)
            if not all(gb.same_bits(a, w) for a, w in zip(got, want)):
                found[mut] = gv.case_id(c)
                break
    print("mutations rejected by:", found)
    assert sorted(found) == sorted(gv.MUTATIONS), set(gv.MUTATIONS) - set(found)
