"""GPU: the log-sum-exp outputs of the attention calls (``lse=``) and ops.attn_merge.

  - the _lse calls give O with the same bits as the calls without, in every mode, and lse within an fp64 bound; lse is
    written into a NaN-filled buffer with guard elements on both sides, and exactly the documented entries change;
  - exact answers from exact_attention.py (needles) and graded_attention.py (lse_oracle.emulate_lse()), unsplit and split decode;
  - the merge: exact cases, real partials over split key ranges, cascade (shared-prefix) decode, and a CUDA graph."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attention_poison as ap  # noqa: E402
import attention_ref as ar  # noqa: E402
import exact_attention as ea  # noqa: E402
import graded_attention as ga  # noqa: E402
import kvcache_oracle  # noqa: E402
import lse_oracle  # noqa: E402

pytestmark = pytest.mark.gpu
LN2_F32 = np.float32(ga.LN2_F32)
GUARD = 37


def _lse_buf(shape):
    """(view of `shape`, the whole NaN-filled buffer with GUARD elements on each side)."""
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * GUARD,), float("nan"), device="cuda")
    return buf[GUARD:GUARD + n].view(shape), buf


def _guards_kept(buf):
    return bool(torch.isnan(buf[:GUARD]).all()) and bool(torch.isnan(buf[-GUARD:]).all())


def _same_bits(a, b):
    """Equal bit patterns (NaN left in place by both calls compares equal)."""
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


def _ulp32(x):
    """One fp32 ulp at |x| (x fp64)."""
    return torch.pow(2.0, torch.floor(torch.log2(x.abs().clamp(min=2.0 ** -126))) - 23)


def _random_bound(want, q, k, scale, dtype):
    """|lse - lse64| for random inputs: the unit roundoff of P in the row sum, the fp32 score error at the max (T is an
    upper bound of sum_d |q_d k_d| * scale * log2 e over the call), ex2.approx and fp32 sums, then 4 fp32 ulp of |lse|
    and of the max m."""
    T = float(q.float().abs().sum(-1).max() * k.float().abs().max()) * scale * ga.LOG2E_F32
    e = ga.U_P[dtype] + 2 * math.log(2) * 2.0 ** -23 * (q.size(-1) / 16 + 3) * T + 2.0 ** -20
    return e + 4 * _ulp32(want) + 4 * 2.0 ** -23 * T


def _check_lse(got, want, bound):
    """got [..] fp32 on the GPU, want fp64 on the CPU: NaN (not written) and -inf where want is, within bound elsewhere."""
    got = got.double().cpu()
    nan, inf = torch.isnan(want), torch.isinf(want)
    assert torch.equal(torch.isnan(got), nan)
    assert (got[inf] == want[inf]).all()
    fin = ~(nan | inf)
    err = (got[fin] - want[fin]).abs()
    b = bound[fin] if torch.is_tensor(bound) else bound
    assert bool((err <= b).all()), float(err.max())


# ------------------------------------------------------------------------------------------------ 1, 4, 5: same O, random
@pytest.mark.parametrize("v_dn", [False, True])
@pytest.mark.parametrize("causal,pad", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("D", [32, 64, 96, 128])
def test_dense_same_o_and_lse(D, dtype, causal, pad, v_dn):
    from b200k import ops

    if v_dn and dtype == torch.bfloat16:
        pytest.skip("V stored [B,H,D,N] is built for fp16 only")
    torch.manual_seed(D + 3 * causal + 7 * pad)
    B, H, N = 3, 4, 1000
    q, k, v = [torch.randn(B, H, N, D, device="cuda").to(dtype) for _ in range(3)]
    vv = v.transpose(-1, -2).contiguous() if v_dn else v
    sl = torch.tensor([1, 129, 700], dtype=torch.int32, device="cuda") if pad else None
    o0, o1 = torch.full_like(q, float("nan")), torch.full_like(q, float("nan"))
    ops.fa2_fwd(q, k, vv, o0, v_is_dn=v_dn, causal=causal, seqlens_k=sl)
    lse, buf = _lse_buf((B, H, N))
    ops.fa2_fwd(q, k, vv, o1, v_is_dn=v_dn, causal=causal, seqlens_k=sl, lse=lse)
    torch.cuda.synchronize()
    assert torch.equal(o0, o1) and _guards_kept(buf)
    want = ar.dense(q.cpu(), k.cpu(), v.cpu(), causal=causal, seqlens_k=sl)[1]
    _check_lse(lse, want, _random_bound(want, q, k, D ** -0.5, dtype))


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("H,H_kv", [(8, 2), (6, 1)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_packed_same_o_and_lse(dtype, H, H_kv, causal):
    """GQA and MQA, empty query and key sequences, ragged lengths, and tokens past the last sequence (left NaN)."""
    from b200k import ops

    torch.manual_seed(H + causal)
    D, lq, lk = 128, [0, 70, 300, 1, 129], [50, 0, 300, 200, 1]
    cq = torch.tensor([0] + np.cumsum(lq).tolist(), dtype=torch.int32, device="cuda")
    ck = torch.tensor([0] + np.cumsum(lk).tolist(), dtype=torch.int32, device="cuda")
    tq = int(cq[-1]) + 5
    q = torch.randn(tq, H, D, device="cuda").to(dtype)
    k, v = [torch.randn(int(ck[-1]), H_kv, D, device="cuda").to(dtype) for _ in range(2)]
    o0, o1 = torch.full_like(q, float("nan")), torch.full_like(q, float("nan"))
    ops.fa2_fwd_varlen(q, k, v, o0, cq, ck, max(lq), causal=causal)
    lse, buf = _lse_buf((tq, H))
    ops.fa2_fwd_varlen(q, k, v, o1, cq, ck, max(lq), causal=causal, lse=lse)
    torch.cuda.synchronize()
    assert _same_bits(o0, o1) and _guards_kept(buf)
    want = ar.packed(q.cpu(), k.cpu(), v.cpu(), cq, ck, causal=causal)[1]
    want = ap.poison(want, ap.packed_masks(cq, ck, want.shape, k.shape)[0], float("nan"))  # past cu[B]: not written
    assert torch.isnan(want[-5:]).all() and (want[cq[1]:cq[2]] == float("-inf")).all()
    _check_lse(lse, want, _random_bound(want, q, k, D ** -0.5, dtype))


def _ws(B, Lq, H, H_kv, D, cap):
    from b200k import ops

    return ops.fa2_fwd_kvcache_workspace_bytes(B, Lq, H, H_kv, D, cap)


LENS = [0, 1, 127, 128, 129, 3000]


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("page_size", [None, 16, 64, 256])
@pytest.mark.parametrize("B_split", ["split", "unsplit"])
def test_decode_same_o_and_lse(B_split, page_size, causal):
    """Six sequences x 2 K/V heads run split; 128 sequences x 8 K/V heads fill the SMs and run unsplit."""
    from b200k import ops

    torch.manual_seed(5 + causal)
    if B_split == "split":
        B, Lq, H, H_kv, D, S, lens_l = 6, 3, 16, 2, 64, 3072, LENS
    else:
        B, Lq, H, H_kv, D, S = 128, 2, 16, 8, 128, 256
        lens_l = [(37 * b) % 257 for b in range(B)]
    assert (_ws(B, Lq, H, H_kv, D, S) > 0) == (B_split == "split")
    dtype = torch.bfloat16 if causal else torch.float16
    q = torch.randn(B, Lq, H, D, device="cuda").to(dtype)
    kc, vc = [torch.randn(B, S, H_kv, D, device="cuda").to(dtype) for _ in range(2)]
    table = None
    if page_size:
        kc, vc, table, _ = kvcache_oracle.paged_copy(kc, vc, page_size, seed=page_size)
    lens = torch.tensor(lens_l, dtype=torch.int32, device="cuda")
    o0, o1 = torch.full_like(q, float("nan")), torch.full_like(q, float("nan"))
    ops.fa2_fwd_kvcache(q, kc, vc, o0, lens, table, causal=causal)
    lse, buf = _lse_buf((B, Lq, H))
    ops.fa2_fwd_kvcache(q, kc, vc, o1, lens, table, causal=causal, lse=lse)
    torch.cuda.synchronize()
    assert torch.equal(o0, o1) and _guards_kept(buf)
    want = ar.kvcache(q, kc, vc, lens, table, causal=causal)[1]
    _check_lse(lse, want, _random_bound(want, q, kc, D ** -0.5, dtype))


@pytest.mark.parametrize("rotary", [None, "neox", "interleaved"])
@pytest.mark.parametrize("B", [6, 128])
def test_append_same_o_and_lse(B, rotary):
    """Append two new tokens (with and without rotary), split (B = 6) and unsplit (B = 128): the caches and O have the
    same bits with and without lse, and lse is the reference over the old keys plus the new ones."""
    from b200k import ops

    torch.manual_seed(B)
    Lq, H, H_kv, D, S = 2, 16, 2 if B == 6 else 8, 64, 1024
    lens_l = [(13 * b * b) % 1000 for b in range(B)]
    q = torch.randn(B, Lq, H, D, device="cuda").half()
    kc, vc = [torch.randn(B, S, H_kv, D, device="cuda").half() for _ in range(2)]
    kn, vn = [torch.randn(B, 2, H_kv, D, device="cuda").half() for _ in range(2)]
    kw = {}
    if rotary:
        ang = torch.arange(S, device="cuda").view(S, 1) * 10000.0 ** (-torch.arange(16, device="cuda").view(1, 16) / 16)
        kw = dict(rotary_cos=ang.cos().half(), rotary_sin=ang.sin().half(), rotary_interleaved=rotary == "interleaved")
    lens = torch.tensor(lens_l, dtype=torch.int32, device="cuda")
    outs = []
    for with_lse in (False, True):
        k2, v2 = kc.clone(), vc.clone()
        o = torch.full_like(q, float("nan"))
        lse, buf = _lse_buf((B, Lq, H))
        ops.fa2_fwd_kvcache(q, k2, v2, o, lens, causal=True, k=kn, v=vn, lse=lse if with_lse else None, **kw)
        outs.append((o, k2, v2, lse, buf))
    torch.cuda.synchronize()
    (o0, k0, v0, _, _), (o1, k1, v1, lse, buf) = outs
    assert torch.equal(o0, o1) and torch.equal(k0, k1) and torch.equal(v0, v1) and _guards_kept(buf)
    if rotary:   # the rotated q is not an output; every row sees the two new keys at least
        assert torch.isfinite(lse).all()
        return
    want = ar.kvcache(q, k1, v1, lens + 2, None, causal=True)[1]
    _check_lse(lse, want, _random_bound(want, q, k1, D ** -0.5, torch.float16))


# ------------------------------------------------------------------------------------------------ 2: needles
def _needle_lse(D, n, visible):
    """Expected lse of a needle row: visible, fp32(fp32(4096 * scale_log2) * fp32(ln 2)) bit for bit (l is exactly 1);
    hidden, every score 0 and l = n, so log n; no key, -inf."""
    sl = np.float32(np.float32(1.0) / np.sqrt(np.float32(D))) * np.float32(ga.LOG2E_F32)
    vis = float(np.float32(np.float32(np.float32(ea.A * ea.A) * sl) * LN2_F32))
    want = torch.where(visible, torch.full(n.shape, vis, dtype=torch.float64), torch.log(n.double().clamp(min=1)))
    return torch.where(n > 0, want, torch.full_like(want, float("-inf")))


def _needle_check(got, want, visible, n, hidden_ulps):
    got = got.double().cpu().reshape(-1)
    want, visible, n = want.reshape(-1), visible.reshape(-1), n.reshape(-1)
    zero = n == 0
    assert (got[zero] == float("-inf")).all()
    vis = visible & ~zero
    assert vis.any() and torch.equal(got[vis], want[vis])
    hid = ~visible & ~zero
    assert hid.any()
    err = (got[hid] - want[hid]).abs()
    assert bool((err <= hidden_ulps * _ulp32(want[hid]) + (0 if hidden_ulps <= 2 else 2.0 ** -21)).all()), float(err.max())


def _needles(nblk, L, D, dtype, g, pos=None):
    """K [nblk, L, D] with the needle of column c of block b at key pos[b, c] (default: a random permutation prefix, so
    one needle per key), V integers."""
    if pos is None:
        pos = torch.stack([torch.randperm(L, generator=g)[:D] for _ in range(nblk)])           # [nblk, D]
    k = torch.zeros(nblk, L, D)
    k[torch.arange(nblk).view(-1, 1), pos, torch.arange(D).view(1, -1)] = ea.A
    v = ea.values(nblk * L, D, dtype, g).view(nblk, L, D)
    return k.to(dtype), v, pos


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("D", [32, 128])
def test_needles_dense_and_packed(D, dtype):
    from b200k import ops

    g = torch.Generator().manual_seed(D)
    # dense: block (b, h); rows of batch b see keys [0, seqlens[b])
    B, H, N = 2, 3, 700
    k, v, pos = _needles(B * H, N, D, dtype, g)
    col = torch.randint(0, D, (B * H, N), generator=g)
    q = ea.queries(col.view(-1), D, dtype).view(B, H, N, D)
    sl = torch.tensor([1, 333], dtype=torch.int32)
    n = sl.repeat_interleave(H).view(B * H, 1).expand(B * H, N)
    visible = pos.gather(1, col) < n
    o = torch.empty(B, H, N, D, dtype=dtype, device="cuda")
    lse = torch.empty(B, H, N, device="cuda")
    ops.fa2_fwd(q.cuda(), k.view(B, H, N, D).cuda(), v.view(B, H, N, D).cuda(), o, seqlens_k=sl.cuda(), lse=lse)
    _needle_check(lse, _needle_lse(D, n, visible), visible, n, 2)
    # packed, one K/V head: sequence b, rows see keys [0, Lk_b); Lk = 0 gives -inf
    lk, lq = [300, 0, 129], [40, 30, 20]
    k, v, pos = _needles(3, 300, D, dtype, g)
    kk = torch.cat([k[b, :lk[b]] for b in range(3)]).view(-1, 1, D)
    vv = torch.cat([v[b, :lk[b]] for b in range(3)]).view(-1, 1, D)
    col = torch.randint(0, D, (sum(lq), 2), generator=g)
    q = ea.queries(col.view(-1), D, dtype).view(-1, 2, D)
    blk = torch.tensor(sum([[b] * lq[b] for b in range(3)], [])).view(-1, 1).expand(-1, 2)
    n = torch.tensor(lk)[blk]
    visible = pos[blk, col] < n
    cq = torch.tensor([0] + np.cumsum(lq).tolist(), dtype=torch.int32, device="cuda")
    ck = torch.tensor([0] + np.cumsum(lk).tolist(), dtype=torch.int32, device="cuda")
    o = torch.empty(sum(lq), 2, D, dtype=dtype, device="cuda")
    lse = torch.empty(sum(lq), 2, device="cuda")
    ops.fa2_fwd_varlen(q.cuda(), kk.cuda(), vv.cuda(), o, cq, ck, max(lq), lse=lse)
    _needle_check(lse, _needle_lse(D, n, visible), visible, n, 2)


@pytest.mark.parametrize("split", [False, True])
def test_needles_decode(split):
    """Unsplit (128 sequences) and split (one sequence of 3000 keys): a visible needle is bit-exact either way, since every
    split without it gets a combine weight that flushes to 0.  A hidden needle is log n within 2 fp32 ulp unsplit; split,
    the combine's ex2.approx weights (relative 2^-22 each) add up to 2^-21 absolute on top of 4 ulp."""
    from b200k import ops

    dtype, D, H = torch.float16, 64, 8
    g = torch.Generator().manual_seed(int(split))
    B, S = (1, 3072) if split else (128, 256)
    lens_l = [3000] if split else [(41 * b) % 257 for b in range(B)]
    pos = None
    if split:   # even columns' needles lie in the first 3000 keys, odd ones' past the length
        c = torch.arange(D)
        pos = torch.where(c % 2 == 0, c * 46, 3000 + c).view(1, D)
    k, v, pos = _needles(B, S, D, dtype, g, pos)
    col = (torch.arange(B * H).view(B, H) * 3) % D
    q = ea.queries(col.view(-1), D, dtype).view(B, 1, H, D)
    n = torch.tensor(lens_l).view(B, 1).expand(B, H)
    visible = pos.gather(1, col) < n
    assert (_ws(B, 1, H, 1, D, S) > 0) == split
    o = torch.empty(B, 1, H, D, dtype=dtype, device="cuda")
    lse = torch.empty(B, 1, H, device="cuda")
    lens = torch.tensor(lens_l, dtype=torch.int32, device="cuda")
    ops.fa2_fwd_kvcache(q.cuda(), k.view(B, S, 1, D).cuda(), v.view(B, S, 1, D).cuda(), o, lens, lse=lse)
    _needle_check(lse, _needle_lse(D, n, visible), visible, n, 4 if split else 2)


# ------------------------------------------------------------------------------------------------ 3: graded, emulate_lse()
def _graded_block(L, D, dtype, seed):
    """Scores that are integers after scale_log2 = 2^-k: Q row = 2^k e_c, K column c integer grades in [0, W]."""
    g = torch.Generator().manual_seed(seed)
    W = ga.window(L)
    kexp = 3
    G = torch.randint(0, W + 1, (L, D), generator=g)
    G[torch.randint(0, L, (D,), generator=g), torch.arange(D)] = W
    v = ea.values(L, D, dtype, g)
    return G.to(dtype), v, kexp, ga.scale_exact(kexp)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_graded_dense_within_2_ulp_of_emulate_lse(dtype):
    from b200k import ops

    B, N, D = 3, 600, 64
    G, v, kexp, scale = _graded_block(N, D, dtype, 1)
    g = torch.Generator().manual_seed(2)
    col = torch.randint(0, D, (B, N), generator=g)
    q = (ea.queries(col.view(-1), D, dtype).float() / ea.A * 2.0 ** kexp).to(dtype).view(B, 1, N, D)
    sl = [1, 300, 600]
    o = torch.empty(B, 1, N, D, dtype=dtype, device="cuda")
    lse = torch.empty(B, 1, N, device="cuda")
    ops.fa2_fwd(q.cuda(), G.view(1, 1, N, D).expand(B, 1, N, D).contiguous().cuda(),
                v.view(1, 1, N, D).expand(B, 1, N, D).contiguous().cuda(), o, scale=scale,
                seqlens_k=torch.tensor(sl, dtype=torch.int32, device="cuda"), lse=lse)
    for b in range(B):
        s = (q[b, 0].float() @ G.float().t()).numpy()
        want = lse_oracle.emulate_lse(s, np.full(N, sl[b]), np.float32(2.0 ** -kexp), dtype, 128)
        want = torch.from_numpy(want).double()
        err = (lse[b, 0].double().cpu() - want).abs()
        assert bool((err <= 2 * _ulp32(want)).all()), float(err.max())


def test_graded_split_decode_against_emulate_lse_splits():
    """One sequence, 3000 keys, split s ways (s from the workspace size): lse against emulate_lse(..., splits=s) within 4 fp32
    ulp + 2^-21 (the combine's ex2.approx and log2f on top of each split's 2 ulp)."""
    from b200k import ops

    dtype, D, H, S, n = torch.float16, 64, 16, 3072, 3000
    G, v, kexp, scale = _graded_block(n, D, dtype, 3)
    ws = _ws(1, 1, H, 1, D, S)
    splits = ws // (H * (D + 1) * 4)
    assert splits > 1 and ws == splits * H * (D + 1) * 4
    kc, vc = torch.zeros(1, S, 1, D, dtype=dtype), torch.zeros(1, S, 1, D, dtype=dtype)
    kc[0, :n, 0], vc[0, :n, 0] = G, v
    col = torch.randint(0, D, (H,), generator=torch.Generator().manual_seed(4))
    q = (ea.queries(col, D, dtype).float() / ea.A * 2.0 ** kexp).to(dtype).view(1, 1, H, D)
    o = torch.empty(1, 1, H, D, dtype=dtype, device="cuda")
    lse = torch.empty(1, 1, H, device="cuda")
    ops.fa2_fwd_kvcache(q.cuda(), kc.cuda(), vc.cuda(), o, torch.tensor([n], dtype=torch.int32, device="cuda"),
                        scale=scale, lse=lse)
    s = (q[0, 0].float() @ G.float().t()).numpy()
    want = lse_oracle.emulate_lse(s, np.full(H, n), np.float32(2.0 ** -kexp), dtype, 128, splits=splits)
    want = torch.from_numpy(want).double()
    err = (lse.view(-1).double().cpu() - want).abs()
    assert bool((err <= 4 * _ulp32(want) + 2.0 ** -21).all()), float(err.max())


# ------------------------------------------------------------------------------------------------ 6: merge, exact
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_merge_exact_answers(dtype):
    from b200k import ops

    torch.manual_seed(0)
    R, D = 1000, 128
    a, b = [torch.randint(-64, 65, (R, D), device="cuda").to(dtype) / 8 for _ in range(2)]
    la = torch.randn(R, device="cuda") * 10

    def merge(parts, lps):
        o = torch.full((R, D), float("nan"), dtype=dtype, device="cuda")
        lse, buf = _lse_buf((R,))
        ops.attn_merge(torch.stack(parts), torch.stack(lps), o, lse)
        torch.cuda.synchronize()
        assert _guards_kept(buf)
        return o, lse

    # one part dominates by more than 126 in base 2: its O bit for bit, its lse
    o, lse = merge([a, b], [la, la - 90.0])
    assert torch.equal(o, a) and torch.equal(lse, ((la * np.float32(1.4426950)) * LN2_F32))
    # equal lse: dtype((a + b) / 2)
    o, lse = merge([a, b], [la, la])
    assert torch.equal(o, ((a.float() + b.float()) * 0.5).to(dtype))
    # S = 1 copies
    o, _ = merge([a], [la])
    assert torch.equal(o, a)
    # all parts -inf: 0 / -inf; a -inf part with NaN O changes nothing
    ninf = torch.full_like(la, float("-inf"))
    o, lse = merge([a, b], [ninf, ninf])
    assert (o == 0).all() and (lse == float("-inf")).all()
    nan = torch.full_like(a, float("nan"))
    o1, l1 = merge([nan, a, b], [ninf, la, la - 1.5])
    o2, l2 = merge([a, b], [la, la - 1.5])
    assert torch.equal(o1, o2) and torch.equal(l1, l2)
    # deterministic; without lse the same O
    o3, l3 = merge([nan, a, b], [ninf, la, la - 1.5])
    assert torch.equal(o1, o3) and torch.equal(l1, l3)
    o4 = torch.empty_like(a)
    ops.attn_merge(torch.stack([nan, a, b]), torch.stack([ninf, la, la - 1.5]), o4)
    assert torch.equal(o4, o1)


# ------------------------------------------------------------------------------------------------ 7: merge of real parts
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_merge_of_split_key_ranges_matches_one_call(dtype):
    """Each sequence's keys split at seeded points into [0, c) and [c, Lk), attended through offset cu_seqlens_k, merged:
    O and lse against one call over all keys, within the fp64 bound (O: the varlen tolerance)."""
    from b200k import ops

    g = torch.Generator().manual_seed(7)
    H, H_kv, D = 8, 2, 128
    lq, lk = [64, 1, 200, 33], [700, 90, 1300, 1]
    cut = [int(torch.randint(0, n + 1, (1,), generator=g)) for n in lk]
    cq = torch.tensor([0] + np.cumsum(lq).tolist(), dtype=torch.int32, device="cuda")
    ck = torch.tensor([0] + np.cumsum(lk).tolist(), dtype=torch.int32, device="cuda")
    q = torch.randn(int(cq[-1]), H, D, device="cuda").to(dtype)
    k, v = [torch.randn(int(ck[-1]), H_kv, D, device="cuda").to(dtype) for _ in range(2)]
    cut_t = torch.tensor(cut, dtype=torch.int32, device="cuda")
    # part 1: keys [ck[b], ck[b] + c) - ends ck[:-1] + c; part 2: [ck[b] + c, ck[b+1])
    parts, lps = [], []
    for lo, hi in ((ck[:-1], ck[:-1] + cut_t), (ck[:-1] + cut_t, ck[1:])):
        # packed as its own K/V: gather the ranges
        idx = torch.cat([torch.arange(int(a), int(b), device="cuda") for a, b in zip(lo, hi)])
        cu = torch.cat([torch.zeros(1, dtype=torch.int32, device="cuda"), (hi - lo).cumsum(0).to(torch.int32)])
        o = torch.empty_like(q)
        lse = torch.empty(q.shape[:2], device="cuda")
        ops.fa2_fwd_varlen(q, k[idx].contiguous(), v[idx].contiguous(), o, cq, cu, max(lq), lse=lse)
        parts.append(o)
        lps.append(lse)
    om, lm = torch.empty_like(q), torch.empty(q.shape[:2], device="cuda")
    ops.attn_merge(torch.stack(parts), torch.stack(lps), om, lm)
    o1, l1 = torch.empty_like(q), torch.empty(q.shape[:2], device="cuda")
    ops.fa2_fwd_varlen(q, k, v, o1, cq, ck, max(lq), lse=l1)
    ref, want = ar.packed(q.cpu(), k.cpu(), v.cpu(), cq, ck)
    bound = _random_bound(want, q, k, D ** -0.5, dtype)
    _check_lse(lm, want, 2 * bound)
    _check_lse(l1, want, bound)
    ref = ref.to(dtype).float()
    tol = dict(rtol=2e-2, atol=8e-3) if dtype == torch.bfloat16 else dict(rtol=1e-2, atol=2e-3)
    assert torch.allclose(om.cpu().float(), ref, **tol)


# ------------------------------------------------------------------------------------------------ 8: cascade decode
def test_cascade_decode_matches_full_cache():
    """A shared prefix (one copy) attended by every sequence's query rows through fa2_fwd_varlen, per-sequence suffixes
    through causal fa2_fwd_kvcache, merged: the result matches fa2_fwd_kvcache over the concatenated caches."""
    from b200k import ops

    torch.manual_seed(8)
    B, Lq, H, H_kv, D, P, Smax = 4, 2, 16, 4, 128, 1000, 512
    suf = [300, 2, 511, 77]
    q = torch.randn(B, Lq, H, D, device="cuda").half()
    kp, vp = [torch.randn(P, H_kv, D, device="cuda").half() for _ in range(2)]
    ks, vs = [torch.randn(B, Smax, H_kv, D, device="cuda").half() for _ in range(2)]
    # prefix: all B * Lq query tokens as one sequence against the prefix keys (the causal rule does not reach them)
    o1, l1 = torch.empty(B * Lq, H, D, dtype=torch.half, device="cuda"), torch.empty(B * Lq, H, device="cuda")
    cu_q = torch.tensor([0, B * Lq], dtype=torch.int32, device="cuda")
    cu_k = torch.tensor([0, P], dtype=torch.int32, device="cuda")
    ops.fa2_fwd_varlen(q.view(B * Lq, H, D), kp, vp, o1, cu_q, cu_k, B * Lq, lse=l1)
    o2, l2 = torch.empty_like(q), torch.empty(B, Lq, H, device="cuda")
    lens = torch.tensor(suf, dtype=torch.int32, device="cuda")
    ops.fa2_fwd_kvcache(q, ks, vs, o2, lens, causal=True, lse=l2)
    om, lm = torch.empty_like(q), torch.empty(B, Lq, H, device="cuda")
    ops.attn_merge(torch.stack([o1.view(B, Lq, H, D), o2]), torch.stack([l1.view(B, Lq, H), l2]), om, lm)
    full_k = torch.cat([kp.expand(B, P, H_kv, D), ks], 1).contiguous()
    full_v = torch.cat([vp.expand(B, P, H_kv, D), vs], 1).contiguous()
    of, lf = torch.empty_like(q), torch.empty(B, Lq, H, device="cuda")
    ops.fa2_fwd_kvcache(q, full_k, full_v, of, lens + P, causal=True, lse=lf)
    ref, want = ar.kvcache(q, full_k, full_v, lens + P, causal=True)
    bound = _random_bound(want, q, full_k, D ** -0.5, torch.float16)
    _check_lse(lm, want, 2 * bound)
    _check_lse(lf, want, bound)
    assert torch.allclose(om.cpu().float(), ref.half().float(), rtol=1e-2, atol=2e-3)
    assert torch.allclose(om.float(), of.float(), rtol=1e-2, atol=2e-3)


# ------------------------------------------------------------------------------------------------ 9: CUDA graph
def test_cuda_graph_append_with_lse_while_the_cache_grows():
    from b200k import ops

    torch.manual_seed(9)
    B, Lq, H, H_kv, D, S = 2, 1, 32, 8, 128, 4096
    q = torch.randn(B, Lq, H, D, device="cuda").half()
    kc, vc = [torch.randn(B, S, H_kv, D, device="cuda").half() for _ in range(2)]
    kn, vn = [torch.randn(B, 1, H_kv, D, device="cuda").half() for _ in range(2)]
    lens = torch.tensor([100, 2000], dtype=torch.int32, device="cuda")
    o, lse = torch.empty_like(q), torch.empty(B, Lq, H, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.fa2_fwd_kvcache(q, kc, vc, o, lens, causal=True, k=kn, v=vn, lse=lse)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.fa2_fwd_kvcache(q, kc, vc, o, lens, causal=True, k=kn, v=vn, lse=lse)
        lens.add_(1)
    for step in range(4):
        kn.copy_(torch.randn_like(kn.float()).half())
        vn.copy_(torch.randn_like(vn.float()).half())
        before = lens.clone()
        o.fill_(float("nan"))
        lse.fill_(float("nan"))
        g.replay()
        o2, l2 = torch.empty_like(q), torch.empty_like(lse)
        ops.fa2_fwd_kvcache(q, kc, vc, o2, before, causal=True, k=kn, v=vn, lse=l2)
        torch.cuda.synchronize()
        assert torch.equal(o, o2) and torch.equal(lse, l2), step
    want = ar.kvcache(q, kc, vc, lens, causal=True)[1]
    _check_lse(lse, want, _random_bound(want, q, kc, D ** -0.5, torch.float16))


def test_lse_wrapper_device_and_contiguity():
    from b200k import ops

    q = torch.zeros(1, 2, 8, 64, dtype=torch.half, device="cuda")
    with pytest.raises(RuntimeError, match="contiguous"):
        ops.fa2_fwd(q, q, q, q.clone(), lse=torch.zeros(1, 8, 2, device="cuda").transpose(1, 2))
    with pytest.raises(RuntimeError, match="CUDA device"):
        ops.fa2_fwd(q, q, q, q.clone(), lse=torch.zeros(1, 2, 8))
    o = torch.zeros(3, 64, dtype=torch.half, device="cuda")
    with pytest.raises(RuntimeError, match="contiguous"):
        ops.attn_merge(torch.zeros(2, 3, 64, dtype=torch.half, device="cuda"), torch.zeros(3, 2, device="cuda").t(), o)
