"""CPU: the log-sum-exp outputs of the attention calls and b200k_attn_merge.  Argument checks of every new entry point
(before any CUDA call) and of the ``lse=`` / attn_merge wrappers; the fp64 reference (attention_ref.py) against
torch.logsumexp and a direct sum, merging by it (lse_oracle.merge); and lse_oracle.emulate_lse(), the lse of
graded_attention.emulate()'s fp32 loop, against it."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attention_ref as ar  # noqa: E402
import graded_attention as ga  # noqa: E402
import lse_oracle  # noqa: E402

from b200k import _loader as L  # noqa: E402

ONE = ctypes.c_void_p(256)       # never dereferenced: validation fails first
ODD = ctypes.c_void_p(258)       # 2 bytes past a 16-byte boundary


def _dense(fn, lse=None, **kw):
    a = dict(Q=ONE, K=ONE, V=ONE, O=ONE, B=1, H=1, N=8, D=64, scale=0.0, v_is_dn=0, dtype=L.F16, causal=0,
             seqlens=None, variant=0, stream=None)
    a.update(kw)
    head = [a["Q"], a["K"], a["V"], a["O"]] + ([lse] if fn.endswith("_lse") else [])
    return getattr(L.lib, fn)(*head, a["B"], a["H"], a["N"], a["D"], a["scale"], a["v_is_dn"], a["dtype"], a["causal"],
                              a["seqlens"], a["variant"], a["stream"])


def _varlen(fn, lse=None, **kw):
    a = dict(Q=ONE, cu=ONE, B=1, max_q=8, total_q=8, total_k=8, H=2, H_kv=1, D=64, dtype=L.F16)
    a.update(kw)
    head = [a["Q"], ONE, ONE, ONE] + ([lse] if fn.endswith("_lse") else [])
    return getattr(L.lib, fn)(*head, a["cu"], ONE, a["B"], a["max_q"], a["total_q"], a["total_k"], a["H"], a["H_kv"],
                              a["D"], 0.0, a["dtype"], 0, None)


def _kvcache(fn, lse=None, **kw):
    a = dict(Q=ONE, B=1, Lq=1, H=2, H_kv=1, D=64, pages=1, ps=128, pps=1, dtype=L.F16)
    a.update(kw)
    head = [a["Q"], ONE, ONE, ONE] + ([lse] if fn.endswith("_lse") else [])
    return getattr(L.lib, fn)(*head, ONE, None, a["B"], a["Lq"], a["H"], a["H_kv"], a["D"], a["pages"], a["ps"],
                              a["pps"], 0.0, a["dtype"], 0, None, 0, None)


def _append(fn, lse=None, **kw):
    a = dict(Q=ONE, K_new=ONE, L_new=1, D=64, dtype=L.F16)
    a.update(kw)
    head = [a["Q"], ONE, ONE, ONE] + ([lse] if fn.endswith("_lse") else [])
    return getattr(L.lib, fn)(*head, ONE, None, a["K_new"], ONE, a["L_new"], None, None, 0, 0, 0, 1, 1, 2, 1, a["D"], 1,
                              128, 1, 0.0, a["dtype"], 0, ONE, 1 << 20, None)


CALLS = [(_dense, "b200k_fa2_fwd", [dict(dtype=L.F32), dict(Q=None), dict(N=0), dict(D=48), dict(v_is_dn=1, N=12),
                                    dict(v_is_dn=1, dtype=L.BF16)]),
         (_varlen, "b200k_fa2_fwd_varlen", [dict(Q=None), dict(cu=None), dict(dtype=L.I8), dict(D=80), dict(H_kv=3),
                                            dict(max_q=9), dict(B=70000)]),
         (_kvcache, "b200k_fa2_fwd_kvcache", [dict(Q=None), dict(dtype=L.F32), dict(D=256), dict(B=0), dict(H_kv=3),
                                              dict(ps=0), dict(pages=2)]),
         (_append, "b200k_fa2_fwd_kvcache_append", [dict(Q=None), dict(K_new=None), dict(L_new=0), dict(D=40),
                                                    dict(Q=ODD)])]


@pytest.mark.parametrize("call,name,bad", CALLS, ids=[c[1] for c in CALLS])
def test_lse_entry_points_check_like_the_calls_they_extend(call, name, bad):
    """Every bad argument gives the same code from the call and from its _lse form (with and without an lse), and the
    old call still returns it; then, with good arguments, an lse 2 bytes off a float boundary is B200K_EALIGN before
    the device is touched."""
    for kw in bad:
        rc = call(name, **kw)
        msg = L.lib.b200k_last_error()
        assert rc in (L.EARG, L.EDTYPE, L.ESHAPE, L.EHEADDIM, L.EALIGN), (kw, rc)
        assert call(name + "_lse", None, **kw) == rc, kw
        assert L.lib.b200k_last_error() == msg, kw
        assert call(name + "_lse", ODD, **kw) == rc, kw
    assert call(name + "_lse", ODD) == L.EALIGN
    assert b"lse must be 4-byte aligned" in L.lib.b200k_last_error()


def test_attn_merge_checks_before_cuda():
    m = L.lib.b200k_attn_merge
    good = dict(op=ONE, lp=ONE, o=ctypes.c_void_p(512), lse=ONE, S=2, rows=4, D=64, dtype=L.F16)

    def call(**kw):
        a = dict(good)
        a.update(kw)
        return m(a["op"], a["lp"], a["o"], a["lse"], a["S"], a["rows"], a["D"], a["dtype"], None)

    for kw in (dict(op=None), dict(lp=None), dict(o=None)):
        assert call(**kw) == L.EARG, kw
    for kw in (dict(dtype=L.F32), dict(dtype=L.I8), dict(dtype=99)):
        assert call(**kw) == L.EDTYPE, kw
    for kw in (dict(S=0), dict(rows=0), dict(D=0), dict(D=12), dict(D=4), dict(S=-1)):
        assert call(**kw) == L.ESHAPE, kw
    for kw in (dict(op=ctypes.c_void_p(264)), dict(o=ctypes.c_void_p(520)), dict(lp=ctypes.c_void_p(258)),
               dict(lse=ctypes.c_void_p(258))):
        assert call(**kw) == L.EALIGN, kw


def test_lse_wrapper_checks():
    """dtype and shape of ``lse`` before the device; a CPU lse with CPU tensors is refused for having no CUDA path."""
    from b200k import ops

    q = torch.zeros(1, 2, 8, 64, dtype=torch.half)
    good = torch.zeros(1, 2, 8)
    for bad, msg in ((good.double(), "values must be torch::kFloat32"), (good.half(), "values must be torch::kFloat32"),
                     (torch.zeros(1, 2, 9), "Tensor size mismatch!"), (torch.zeros(2, 8), "Tensor size mismatch!"),
                     (good, "CUDA device")):
        with pytest.raises(RuntimeError, match=msg):
            ops.fa2_fwd(q, q, q, q.clone(), lse=bad)
    qv = torch.zeros(8, 2, 64, dtype=torch.half)
    kv = torch.zeros(8, 1, 64, dtype=torch.half)
    cu = torch.tensor([0, 8], dtype=torch.int32)
    for bad, msg in ((torch.zeros(8, 2, dtype=torch.int32), "values must be torch::kFloat32"),
                     (torch.zeros(2, 8), "Tensor size mismatch!"), (torch.zeros(8, 2), "CUDA device")):
        with pytest.raises(RuntimeError, match=msg):
            ops.fa2_fwd_varlen(qv, kv, kv, qv.clone(), cu, cu, 8, lse=bad)
    qc = torch.zeros(1, 3, 2, 64, dtype=torch.half)
    kc = torch.zeros(1, 128, 1, 64, dtype=torch.half)
    lens = torch.tensor([5], dtype=torch.int32)
    kn = torch.zeros(1, 1, 1, 64, dtype=torch.half)
    for extra in ({}, dict(k=kn, v=kn)):
        for bad, msg in ((torch.zeros(1, 3, 2, dtype=torch.bfloat16), "values must be torch::kFloat32"),
                         (torch.zeros(1, 2, 3), "Tensor size mismatch!"), (torch.zeros(1, 3, 2), "CUDA device")):
            with pytest.raises(RuntimeError, match=msg):
                ops.fa2_fwd_kvcache(qc, kc, kc, qc.clone(), lens, lse=bad, **extra)


def test_attn_merge_wrapper_checks():
    from b200k import ops

    o = torch.zeros(3, 4, 64, dtype=torch.bfloat16)
    parts, lp = torch.zeros(2, 3, 4, 64, dtype=torch.bfloat16), torch.zeros(2, 3, 4)
    cases = [((parts, lp, o.float()), "values must be torch::kHalf or torch::kBFloat16"),
             ((parts.half(), lp, o), "values must be torch::kBFloat16"),
             ((parts, lp.double(), o), "values must be torch::kFloat32"),
             ((parts[:, :2], lp, o), "Tensor size mismatch!"),
             ((parts[0], lp, o), "Tensor size mismatch!"),
             ((parts, lp[:1], o), "Tensor size mismatch!"),
             ((parts, lp, o), "CUDA device")]
    for args, msg in cases:
        with pytest.raises(RuntimeError, match=msg):
            ops.attn_merge(*args)
    for bad, msg in ((torch.zeros(3, 4, dtype=torch.half), "values must be torch::kFloat32"),
                     (torch.zeros(3, 5), "Tensor size mismatch!")):
        with pytest.raises(RuntimeError, match=msg):
            ops.attn_merge(parts, lp, o, bad)


# ------------------------------------------------------------------------------------------------ the fp64 reference
def _packed(seed, lens_q, lens_k, H=4, H_kv=2, D=32, extra_q=3):
    g = torch.Generator().manual_seed(seed)
    cq = torch.tensor([0] + np.cumsum(lens_q).tolist(), dtype=torch.int32)
    ck = torch.tensor([0] + np.cumsum(lens_k).tolist(), dtype=torch.int32)
    q = torch.randn(int(cq[-1]) + extra_q, H, D, generator=g)
    k, v = [torch.randn(max(int(ck[-1]), 1), H_kv, D, generator=g) for _ in range(2)]
    return q, k, v, cq, ck


@pytest.mark.parametrize("causal", [False, True])
def test_reference_lse_is_the_log_of_the_softmax_denominator(causal):
    """The packed lse against a direct fp64 sum per row; -inf for rows that see no key (Lk = 0, causal rows above the
    bottom-right diagonal) and for tokens outside every sequence; the dense lse is the same rule."""
    lens_q, lens_k = [5, 0, 7, 3], [9, 4, 0, 2]
    q, k, v, cq, ck = _packed(1, lens_q, lens_k)
    got = ar.packed(q, k, v, cq, ck, causal=causal)[1]
    H, D = q.shape[1], q.shape[2]
    for b in range(len(lens_q)):
        for r in range(lens_q[b]):
            for h in range(H):
                t = int(cq[b]) + r
                keys = [j for j in range(lens_k[b]) if not causal or j <= r + lens_k[b] - lens_q[b]]
                s = [float(q[t, h].double() @ k[int(ck[b]) + j, h // 2].double()) / math.sqrt(D) for j in keys]
                want = math.log(sum(math.exp(x) for x in s)) if s else float("-inf")
                assert got[t, h].item() == pytest.approx(want, rel=1e-12, abs=1e-12) if s else got[t, h] == want
    assert (got[int(cq[-1]):] == float("-inf")).all()
    assert (got[int(cq[2]):int(cq[3])] == float("-inf")).all()
    # dense: the same rule with a key-padding mask, against torch.logsumexp of the masked scores
    qd, kd = torch.randn(2, 3, 10, 16, dtype=torch.float64), torch.randn(2, 3, 10, 16, dtype=torch.float64)
    sl = torch.tensor([4, 10])
    dense = ar.dense(qd, kd, kd, causal=causal, seqlens_k=sl)[1]
    for b in range(2):
        for r in range(10):
            n = min(int(sl[b]), r + 1) if causal else int(sl[b])
            want = torch.logsumexp(torch.einsum("hd,hjd->hj", qd[b, :, r], kd[b, :, :n]) / 4.0, dim=-1)
            assert torch.allclose(dense[b, :, r], want, rtol=1e-14, atol=1e-14)


def test_reference_merge_of_two_key_ranges_is_the_attention_over_their_union():
    """Attention over keys [0, c) and [c, Lk) of each sequence, merged by lse, is the attention over [0, Lk) in fp64;
    a part with lse = -inf and NaN in O weighs nothing."""
    lens_q, lens_k = [6, 5, 4], [20, 7, 3]
    q, k, v, cq, ck = _packed(2, lens_q, lens_k, extra_q=0)
    cut = [8, 0, 3]
    lo = torch.tensor([0] + np.cumsum(cut).tolist(), dtype=torch.int32)
    hi_len = [n - c for n, c in zip(lens_k, cut)]
    # the two key ranges as packed tensors of their own
    k1 = torch.cat([k[int(ck[b]):int(ck[b]) + cut[b]] for b in range(3)])
    k2 = torch.cat([k[int(ck[b]) + cut[b]:int(ck[b + 1])] for b in range(3)])
    v1 = torch.cat([v[int(ck[b]):int(ck[b]) + cut[b]] for b in range(3)])
    v2 = torch.cat([v[int(ck[b]) + cut[b]:int(ck[b + 1])] for b in range(3)])
    hi = torch.tensor([0] + np.cumsum(hi_len).tolist(), dtype=torch.int32)

    def attn64(kk, vv, cu):
        q64, k64, v64 = q.double(), kk.double(), vv.double()
        out = torch.zeros(q.shape, dtype=torch.float64)
        for b in range(3):
            s = torch.einsum("thd,jhd->htj", q64[int(cq[b]):int(cq[b + 1])],
                             k64[int(cu[b]):int(cu[b + 1])].repeat_interleave(2, dim=1)) / math.sqrt(q.shape[2])
            p = torch.softmax(s, -1) if s.size(-1) else s
            out[int(cq[b]):int(cq[b + 1])] = torch.einsum("htj,jhd->thd", p, v64[int(cu[b]):int(cu[b + 1])]
                                                          .repeat_interleave(2, dim=1))
        return out

    o1, o2, o = attn64(k1, v1, lo), attn64(k2, v2, hi), attn64(k, v, ck)
    l1 = ar.packed(q, k1, v1, cq, lo)[1]
    l2 = ar.packed(q, k2, v2, cq, hi)[1]
    assert (l1[int(cq[1]):int(cq[2])] == float("-inf")).all()       # sequence 1 has no key in its first range
    o1[int(cq[1]):int(cq[2])] = float("nan")
    mo, ml = lse_oracle.merge(torch.stack([o1, o2]), torch.stack([l1, l2]))
    assert torch.allclose(mo, o, rtol=1e-12, atol=1e-12)
    assert torch.allclose(ml, ar.packed(q, k, v, cq, ck)[1], rtol=1e-12, atol=1e-12)
    mo, ml = lse_oracle.merge(torch.full((2, 1, 4), float("nan")), torch.full((2, 1), float("-inf")))
    assert (mo == 0).all() and (ml == float("-inf")).all()


# ------------------------------------------------------------------------------------------------ emulate_lse()
def lse_bound(lse64, T, tiles, D, dtype):
    """|lse - lse64| bound of the kernel's arithmetic: the relative error of the row sum l (P rounded to dtype, ex2.approx
    in P and in each tile's alpha, fp32 sums) and the fp32 score error at the max, both as natural-log offsets, plus 4
    fp32 ulp of the terms of (m + log2f(l)) * ln 2."""
    e = ga.U_P[dtype] + 2 * math.log(2) * 2.0 ** -23 * (D / 16 + 3) * T + 2.0 ** -22 * (1 + tiles) + 2.0 ** -20
    return e + 4 * 2.0 ** -23 * (lse64.abs() + math.log(2) * T + 1)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_emulated_lse_within_its_bound_of_the_reference(dtype):
    rng = np.random.default_rng(3)
    R, L, D = 64, 500, 64
    q, k, v = [torch.from_numpy(rng.standard_normal((x, D)).astype(np.float32)).to(dtype) for x in (R, L, L)]
    n = torch.arange(R) * 8
    scale = 1 / np.sqrt(D)
    _, _, _, T, tiles = ga.reference(q, k, v, n, scale, dtype)
    s = q.float().numpy() @ k.float().numpy().T
    sl = np.float32(scale) * np.float32(ga.LOG2E_F32)
    x =(q.double() @ k.double().t()) * scale
    vis = torch.arange(L).view(1, L) < n.view(R, 1)
    want = torch.logsumexp(torch.where(vis, x, torch.full_like(x, float("-inf"))), dim=1)
    for splits in (1, 3):
        lse = lse_oracle.emulate_lse(s, n.numpy(), sl, dtype, 128, splits=splits)
        got = torch.from_numpy(lse).double()
        assert got.dtype == torch.float64 and lse.dtype == np.float32
        assert got[0] == float("-inf")
        err = (got[1:] - want[1:]).abs()
        assert bool((err <= lse_bound(want[1:], T[1:], tiles[1:].double() + splits, D, dtype)).all()), float(err.max())


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_emulated_lse_exact_on_graded_scores(dtype):
    """Integer scores at scale_log2 = 1 with grades in the window: the running max m is an integer and the row sum l of
    rounded weights an exact fp32 sum whatever the tiling, so emulate_lse is (m + log2 l) * fp32(ln 2) bit for bit."""
    g = torch.Generator().manual_seed(5)
    R, L = 48, 700
    W = ga.window(L)
    G = torch.randint(0, W + 1, (R, L), generator=g).double()
    n = torch.randint(0, L + 1, (R,), generator=g)
    n[:3] = torch.tensor([0, 1, L])
    vis = torch.arange(L).view(1, L) < n.view(R, 1)
    m = torch.where(vis, G, torch.full_like(G, float("-inf"))).max(1).values
    w = torch.where(vis, torch.exp2(G - m.view(R, 1).clamp(min=0)).to(dtype).double(), torch.zeros_like(G))
    l = w.sum(1).numpy().astype(np.float32)
    assert np.array_equal(l.astype(np.float64), w.sum(1).numpy())
    f = np.float32
    with np.errstate(divide="ignore"):
        want = np.where(l > 0, (m.numpy().astype(f) + np.log2(l)) * f(ga.LN2_F32), f(-np.inf)).astype(f)
    for bn in (64, 128):
        got = lse_oracle.emulate_lse(G.numpy().astype(f), n.numpy(), 1.0, dtype, bn)
        assert np.array_equal(got, want), bn
