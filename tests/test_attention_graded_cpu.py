"""CPU: the constructions of graded_attention.py.  The scale trick is exact; the closed form agrees with attention_ref's packed
and kvcache layouts; the kernel's loop, emulated in fp32 at tile sizes 64, 128 and 192, gives the closed form bit for bit; and
each way the softmax could be subtly wrong (graded_attention.MUTATIONS) is rejected by one of the checks the GPU tests
apply."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))  # the helpers and oracles sit next to this file
import attention_ref as ar  # noqa: E402
import exact_attention as ex  # noqa: E402
import graded_attention as ga  # noqa: E402

DTYPES = [torch.float16, torch.bfloat16]
EDGES = [0, 1, 15, 16, 63, 64, 127, 128, 129, 191, 192, 255, 256, 383, 384, 511, 512]   # as test_gpu_attention_exact.py


def test_scale_times_log2e_is_a_power_of_two_in_fp32():
    for k in range(8):
        s = ga.scale_exact(k)
        assert np.float32(s) * np.float32(1.4426950408889634) == np.float32(2.0 ** -k)
        assert float(np.float32(s)) == s


def test_window_is_enforced():
    assert ga.window(1024) == 10 and ga.window(16384) == 6 and ga.window(64) == 14
    with pytest.raises(AssertionError):
        ga.window(1 << 19)
    g = torch.Generator().manual_seed(0)
    G = torch.full((1, 600, 1), 0, dtype=torch.int16)
    G[0, :300, 0] = 20                                   # spread 20 over 600 keys: sums need more than 24 bits
    G[0, 0, 0] = 0
    V = ex.values(600, 1, torch.float16, g).view(1, 600, 1)
    V[0, 0, 0], V[0, 1, 0] = 1, 8
    with pytest.raises(AssertionError, match="window"):
        ga.expected(G, V, torch.zeros(1), torch.tensor([600]), torch.zeros(1), torch.float16)


def _block(L, R, D, dtype, seed, last=None, k=3):
    """One block of L key slots (valid up to `last`) and R rows with random columns and prefixes that stop on, before and
    after every edge: (G, V, n, cols, raw scores [R, L], 2^-k, W)."""
    g = torch.Generator().manual_seed(seed)
    W = ga.window(L)
    last = L - 1 if last is None else last
    G = ga.grades(1, L, torch.tensor([last]), D, W, EDGES, g)
    V = ex.values(L, D, dtype, g).view(1, L, D)
    cols = ga.columns(R, D, EDGES, g, "cpu")
    stops = torch.tensor([e + d for e in EDGES + [last + 1] for d in (-1, 0, 1)]).clamp(0, last + 1)
    n = torch.cat([stops, torch.randint(0, last + 2, (R,), generator=g)])[:R]
    s = (2.0 ** k) * G[0][:, cols].t().float()
    return G, V, n, cols, s.numpy(), 2.0 ** -k, W


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bn", [64, 128, 192])
def test_the_loop_gives_the_closed_form_at_every_tile_size(bn, dtype):
    for L, last in ((600, None), (300, 200), (1024, 1000)):
        G, V, n, cols, s, sl, W = _block(L, 256, 32, dtype, seed=L + bn, last=last)
        want, info = ga.expected(G, V, torch.zeros(256), n, cols, dtype)
        assert int(info["decoyed"].sum()) > 0 and int((n == 0).sum()) > 0
        for splits in (1, 3):
            got = torch.from_numpy(ga.emulate(s, V[0].float().numpy(), n.numpy(), sl, dtype, bn, splits=splits)).to(dtype)
            if splits == 1:
                assert torch.equal(got, want), ga.describe(G, torch.zeros(256), n, cols, want, got, info, EDGES, W)
            else:
                assert bool(((got.float() - want.float()).abs() <= ga.ulp(want, dtype) + 2.0 ** -14).all())
        assert bool((want[n == 0] == 0).all())


def _pack(X, lk, H_kv):
    B = len(lk)
    X = X.view(B, H_kv, X.size(1), X.size(2))
    return torch.cat([X[b, :, :lk[b]].transpose(0, 1) for b in range(B)])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("causal", [False, True])
def test_closed_form_matches_the_varlen_and_kvcache_oracles(causal, dtype):
    """Packed sequences with grouped heads, and the same blocks as a KV cache with lengths below the capacity (so the
    decoy column's key exists).  The reference's softmax is natural-base: one ulp of the dtype plus 2^-20."""
    g = torch.Generator().manual_seed(5 + causal)
    lq, lk, H, H_kv, D, L, k = [5, 0, 40, 1, 70], [9, 3, 0, 70, 130], 4, 2, 32, 140, 2
    B, W = len(lq), ga.window(L)
    G = ga.grades(B * H_kv, L, torch.tensor(lk).repeat_interleave(H_kv) - 1, D, W, EDGES, g)
    V = ex.values(B * H_kv * L, D, dtype, g).view(B * H_kv, L, D)
    tq = sum(lq)
    cols = ga.columns(tq * H, D, EDGES, g, "cpu")
    q = ex.queries(cols, D, dtype).view(tq, H, D) * (2.0 ** k / ex.A)
    cu_q, cu_k = [torch.tensor([0] + torch.tensor(x).cumsum(0).tolist()) for x in (lq, lk)]
    tok = torch.arange(tq).repeat_interleave(H)
    h = torch.arange(H).repeat(tq)
    b = torch.bucketize(tok, cu_q[1:], right=True)
    Lq, Lk = torch.tensor(lq)[b], torch.tensor(lk)[b]
    n = (tok - cu_q[b] + Lk - Lq + 1).clamp(min=0).minimum(Lk) if causal else Lk
    blk = b * H_kv + h // (H // H_kv)
    want, info = ga.expected(G, V, blk, n, cols, dtype)
    ref = ar.packed(q, _pack(G.to(dtype), lk, H_kv), _pack(V, lk, H_kv), cu_q, cu_k, scale=ga.scale_exact(k),
                    causal=causal)[0].to(dtype)
    tol = ga.ulp(want, dtype) + 2.0 ** -20
    assert bool(((ref.view(-1, D).float() - want.float()).abs() <= tol).all())
    assert int(info["decoyed"].sum()) > 0 and int((n == 0).sum()) > 0
    # the same rows as decode calls: one per sequence, its Lq tokens against cache rows [0, Lk)
    kc, vc = [t.view(B, H_kv, L, D).transpose(1, 2) for t in (G.to(dtype), V)]
    for bb in range(B):
        if lq[bb] == 0:
            continue
        rows = (b == bb)
        qd = q[cu_q[bb]:cu_q[bb + 1]].view(1, lq[bb], H, D)
        ref = ar.kvcache(qd, kc[bb:bb + 1], vc[bb:bb + 1], [lk[bb]], scale=ga.scale_exact(k), causal=causal)[0].to(dtype)
        assert bool(((ref.view(-1, D).float() - want[rows].float()).abs() <= tol[rows]).all())


def test_subnormal_and_vanishing_fp16_weights_by_running_max():
    """fp16, 128-key tiles (the order is pinned: the FFPA path's 64-key tiles would round other keys).  Tile 0: every key
    at grade 0, so its P are 1 and reach the final max 26 through alpha = 2^-26 in fp32, where rounding P against the
    final max would lose them.  Tile 1: the max 26 on a key whose V row is 0, spreads 15 .. 23 (exact subnormal P), 25
    (a tie that rounds to 0) and 26 .. 30 (0)."""
    G, V, n, cols, s = ga.subnormal_case("cpu")
    want, info = ga.expected(G, V, torch.zeros(n.numel()), n, cols, torch.float16, bn=128)
    got = torch.from_numpy(ga.emulate(s, V[0].float().numpy(), n.numpy(), 1.0, torch.float16, 128)).half()
    assert torch.equal(got, want)
    by_final_max, _ = ga.expected(G, V, torch.zeros(n.numel()), n, cols, torch.float16)
    assert not torch.equal(by_final_max, want)
    assert bool((want[n == 256].float().abs().max(1).values > 0).all())


def _fractional(dtype, L=300, R=64, D=32, seed=3):
    g = torch.Generator().manual_seed(seed)
    steps = torch.tensor(ga.fractional_grades(dtype))
    G = -steps[torch.randint(0, steps.numel(), (1, L, D), generator=g)].to(torch.int16)
    G[0, 0] = 0
    V = ex.values(L, D, dtype, g).view(1, L, D)
    cols = torch.randint(0, D, (R,), generator=g)
    n = torch.randint(1, L + 1, (R,), generator=g)
    return G, V, n, cols, (G[0][:, cols].t().float() / 8).numpy()


@pytest.mark.parametrize("dtype", DTYPES)
def test_fractional_weights_tell_rounding_from_truncation(dtype):
    assert len(ga.fractional_grades(dtype)) >= 2
    G, V, n, cols, s = _fractional(dtype)
    want, _ = ga.expected(G, V, torch.zeros(64), n, cols, dtype, unit=0.125)
    for bn in (64, 128, 192):
        run = lambda mut: torch.from_numpy(ga.emulate(s, V[0].float().numpy(), n.numpy(), 1.0, dtype, bn, mut=mut)).to(dtype)  # noqa: E731
        assert torch.equal(run(""), want)
        assert not torch.equal(run("trunc"), want)
        assert not torch.equal(run("rowsum_unrounded"), want)


def _const_v_wrong(dtype, mut, splits, factor, kind):
    rng = np.random.default_rng(7)
    R, L, D = 64, 700, 32
    q, k = [torch.from_numpy(rng.standard_normal((x, D)).astype(np.float32)).to(dtype).float().numpy() for x in (R, L)]
    s = (q * factor) @ k.T
    n = np.minimum(np.arange(R) * 12, L)
    n[1], n[2] = 1, 2
    v, c = ga.const_v((L, D), kind, dtype, "cpu")
    sl = np.float32(1 / np.sqrt(np.float32(D))) * np.float32(ga.LOG2E_F32)
    o = torch.from_numpy(ga.emulate(s, v.float().numpy(), n, sl, dtype, 128, mut=mut, splits=splits)).to(dtype)
    return ga.check_const_v(o, c, torch.from_numpy(n > 0), L, dtype)[0]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", ["ones", "mod17"])
def test_constant_v_comes_back_exactly_and_catches_combine_weights_that_do_not_sum_to_one(kind, dtype):
    """A row sum of unrounded P moves sum(P) / l by less than 2^-12 (fp16) or 2^-9 (bf16), under half an ulp of O, so
    constant V cannot see it; the fractional weights above do.  Here: alpha left off l, and a combine without 1 / den."""
    for factor in (1.0, 4.0):
        for splits in (1, 4):
            assert _const_v_wrong(dtype, "", splits, factor, kind) == 0
        assert _const_v_wrong(dtype, "no_renorm", 4, factor, kind) > 0
        assert _const_v_wrong(dtype, "alpha_skips_l", 1, factor, kind) > 0
    with pytest.raises(AssertionError):
        ga.check_const_v(torch.zeros(1, 1, dtype=dtype), torch.zeros(1, dtype=dtype), torch.ones(1, dtype=torch.bool),
                         ga.CONST_V_MAX_KEYS[dtype] + 1, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mut", ["alpha_skips_l", "alpha_swapped", "decoy_moves_max"])
def test_graded_weights_reject_a_wrong_alpha_and_a_decoy_that_moves_the_max(mut, dtype):
    G, V, n, cols, s, sl, W = _block(600, 256, 32, dtype, seed=9, last=500)
    want, _ = ga.expected(G, V, torch.zeros(256), n, cols, dtype)
    for bn in (64, 128):
        got = torch.from_numpy(ga.emulate(s, V[0].float().numpy(), n.numpy(), sl, dtype, bn, mut=mut)).to(dtype)
        assert int((got != want).any(1).sum()) > 0


def test_every_mutation_has_a_test():
    """rowsum_unrounded and trunc: fractional weights (truncation scales o and l alike and the unrounded row sum is off by
    less than half an ulp of O, so neither constant V nor an error statistic sees them); alpha_*, decoy_moves_max: graded
    weights; alpha_skips_l and no_renorm: constant V."""
    assert sorted(ga.MUTATIONS) == sorted(["rowsum_unrounded", "trunc", "alpha_skips_l", "alpha_swapped",
                                           "decoy_moves_max", "no_renorm"])


@pytest.mark.parametrize("dtype", DTYPES)
def test_fp64_bound_holds_for_the_loop_and_the_model(dtype):
    """The emulated kernel and the 16-bit-P model sit inside the elementwise bound, with comparable rms error."""
    rng = np.random.default_rng(1)
    R, L, D = 64, 500, 64
    q, k, v = [torch.from_numpy(rng.standard_normal((x, D)).astype(np.float32)).to(dtype) for x in (R, L, L)]
    n = torch.arange(R) * 8 + 1
    scale = 1 / np.sqrt(D)
    o64, om, A, T, tiles = ga.reference(q, k, v, n, scale, dtype)
    s = q.float().numpy() @ k.float().numpy().T
    sl = np.float32(scale) * np.float32(ga.LOG2E_F32)
    o = torch.from_numpy(ga.emulate(s, v.float().numpy(), n.numpy(), sl, dtype, 128)).double()
    tol = ga.bound(o64, A, T, tiles, D, dtype)
    assert bool(((o - o64).abs() <= tol).all()) and bool(((om.to(dtype).double() - o64).abs() <= tol).all())
    ratio = float((o - o64).pow(2).mean().sqrt() / (om.to(dtype).double() - o64).pow(2).mean().sqrt())
    assert 0.5 < ratio < 1.5, ratio
