"""GPU: every attention mode against exact answers (exact_attention.py), the softmax scale in every entry point, V stored
[B,H,D,N] against V stored [B,H,N,D], the largest grid each entry point accepts and 64-bit offsets.

The exact tests put needles where kernels go wrong: key 0, the first and last key of 16 / 64 / 128-key boxes and tiles,
page and split boundaries, the last valid key and the one after it (a decoy that must not be seen), the last key a causal
row sees and the one after it, and key 0 of the next packed sequence.  Rows pick their needle column at random (decode:
per token and head), or the column of the needle on or just past their last visible key.  A needle row must return its
needle's V row, any other row the mean of the keys it sees, bit for bit.  Split decode merges the splits' mean rows
through log2f / ex2.approx weights, so those rows are held to one ulp of the dtype plus 2^-14 (the fp32 rounding of up
to 128 weighted partial sums of values of at most 8); their needle rows stay bit-exact."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))  # the helpers and oracles sit next to this file
import attention_ref as ar  # noqa: E402
import exact_attention as ex  # noqa: E402
import kvcache_append_oracle as ko  # noqa: E402
import kvcache_oracle  # noqa: E402
from oracle import oracle  # noqa: E402

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]
EDGES = [0, 1, 15, 16, 63, 64, 127, 128, 129, 191, 192, 255, 256, 383, 384, 511, 512]   # box and tile edges
CHUNK = 1 << 20   # rows per expected-value pass


def _ops():
    from b200k import ops

    return ops


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _i32(x):
    return torch.as_tensor(x).to(device="cuda", dtype=torch.int32)


def _place(L, D, cands, g, lo=0):
    """Local needle key [nb, D] of each column of each block of L[b] keys (-1 in an empty block).  Block b's candidate
    keys cands[b] that lie in [0, L[b]) go to distinct random columns in [lo, D), a random subset when there are more
    candidates than columns; every other column gets a random key."""
    nb = L.numel()
    L = L.view(nb, 1).long()
    cands = cands.long()
    if cands.size(1) > D - lo:
        cands = cands.gather(1, torch.argsort(torch.rand(cands.shape, generator=g, device="cuda"), 1)[:, :D - lo])
    m = cands.size(1)
    hi = (L - 1).clamp(min=0)
    pos = (torch.rand(nb, D, generator=g, device="cuda") * L).long().minimum(hi)
    rnd = (torch.rand(nb, m, generator=g, device="cuda") * L).long().minimum(hi)
    cand = torch.where((cands >= 0) & (cands < L), cands, rnd)
    at = lo + torch.argsort(torch.rand(nb, D - lo, generator=g, device="cuda"), 1)[:, :m]
    pos.scatter_(1, at, cand)
    return torch.where(L > 0, pos, torch.full_like(pos, -1))


def _columns(pos, blk, last, D, g, lo=0):
    """Needle column of each row of block blk[r] whose last visible key is last[r]: half the rows take the column whose
    needle sits on that key or on the one after it, when there is one; the rest a random column in [lo, D)."""
    R = blk.numel()
    cols = lo + torch.randint(0, D - lo, (R,), generator=g, device="cuda")
    nb, top = pos.size(0), int(pos.max()) + 1
    inv = torch.full((nb, top + 4), -1, dtype=torch.long, device="cuda")           # key k -> slot k + 1
    slot = torch.where(pos >= 0, pos + 1, torch.full_like(pos, top + 3))
    inv.scatter_(1, slot, torch.arange(D, device="cuda").expand(nb, D).contiguous())
    inv[:, top + 3] = -1
    inv = torch.where(inv >= lo, inv, torch.full_like(inv, -1))
    d = last.long().clamp(-1, top)
    on, past = inv[blk, d + 1], inv[blk, d + 2]
    coin = torch.rand(R, generator=g, device="cuda") < 0.5
    a, b = torch.where(coin, on, past), torch.where(coin, past, on)
    pick = torch.where(a >= 0, a, b)
    use = (pick >= 0) & (torch.rand(R, generator=g, device="cuda") < 0.5)
    return torch.where(use, pick, cols)


class Spec:
    """Rows of an exact case: flat keys v [T, D]; each row sees keys [first, first + n) and has its needle at flat key
    `needle` (-1: none in its block)."""

    def __init__(self, v, first, n, needle):
        self.v, self.first, self.n, self.needle = v, first, n, needle


def _check(o, spec, dtype, split=False, what="", needles=True):
    """O (rows in the order of spec) against the closed form: bit for bit, or for split decode the mean rows within one
    ulp + 2^-14 (module docstring).  `needles`: at least one row must see its needle."""
    o = o.reshape(-1, o.size(-1))
    R = o.size(0)
    assert spec.n.numel() == R
    bad, nmean = 0, 0
    first_bad = None
    for r0 in range(0, R, CHUNK):
        sl = slice(r0, min(R, r0 + CHUNK))
        want, mean = ex.expected(spec.v, spec.first[sl], spec.n[sl], spec.needle[sl], dtype)
        got = o[sl]
        if split:
            tol = torch.where(mean.view(-1, 1), ex.ulp(want, dtype) + 2.0 ** -14, torch.zeros_like(want, dtype=torch.float))
            wrong = ((got.float() - want.float()).abs() > tol).any(1) | torch.isnan(got).any(1)
        else:
            wrong = (got != want).any(1) | torch.isnan(got).any(1)
        nmean += int(mean.sum())
        if wrong.any():
            bad += int(wrong.sum())
            if first_bad is None:
                first_bad = (r0 + wrong.nonzero()[:4].view(-1)).tolist()
    assert bad == 0, "%s: %d of %d rows differ, first %s" % (what, bad, R, first_bad)
    assert nmean < R or not needles, "%s: no row saw its needle" % what
    return nmean


# ------------------------------------------------------------------------------------------------ dense and FFPA
def _dense(B, H, N, D, dtype, causal, lens, seed, pin=()):
    """(q, k, v, seqlens, spec) for [B,H,N,D]; block = (batch, head), flat key = block * N + key.  Rows r % 8 == 0 take
    the columns in `pin` in turn."""
    g = _gen(seed)
    BH = B * H
    kv = torch.full((B,), N, device="cuda") if lens is None else torch.as_tensor(lens, device="cuda").clamp(1, N)
    kvb = kv.repeat_interleave(H)
    cands = torch.cat([torch.tensor(EDGES, device="cuda").expand(BH, -1),
                       torch.stack([kvb - 2, kvb - 1, kvb, torch.full_like(kvb, N - 1)], 1)], 1)
    pos = _place(torch.full((BH,), N, device="cuda"), D, cands, g)
    r = torch.arange(N, device="cuda").repeat(BH)
    blk = torch.arange(BH, device="cuda").repeat_interleave(N)
    n = kvb[blk]
    if causal:
        n = torch.minimum(n, r + 1)
    cols = _columns(pos, blk, n - 1, D, g)
    if pin:
        pins = torch.tensor(pin, device="cuda")
        cols = torch.where(r % 8 == 0, pins[(r // 8) % len(pin)], cols)
    q = ex.queries(cols, D, dtype).view(B, H, N, D)
    base = torch.arange(BH, device="cuda").view(BH, 1) * N
    k = ex.keys(BH * N, D, (pos + base).view(-1), torch.arange(D, device="cuda").repeat(BH), dtype, "cuda")
    v = ex.values(BH * N, D, dtype, g, "cuda")
    spec = Spec(v, blk * N, n, pos[blk, cols] + blk * N)
    return q, k.view(B, H, N, D), v.view(B, H, N, D), (None if lens is None else _i32(lens)), spec


@pytest.mark.parametrize("lens", [False, True])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("D", [32, 64, 96, 128])
@pytest.mark.parametrize("dtype", DTYPES)
def test_dense_exact(dtype, D, causal, lens):
    """Key-padding lengths around 1, 63, 64, 127, 128, 129 and N; ragged N."""
    ops = _ops()
    for N in (1000, 77):
        L = [1, 63, 64, 127, 128, 129, N] if lens else None
        B = 7 if lens else 2
        q, k, v, sl, spec = _dense(B, 2, N, D, dtype, causal, L, seed=D + 2 * causal + N, pin=(0, D - 1))
        o = torch.full_like(q, float("nan"))
        ops.fa2_fwd(q, k, v, o, causal=causal, seqlens_k=sl)
        _check(o, spec, dtype, what="N=%d" % N)


@pytest.mark.parametrize("lens", [False, True])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("D", [32, 64, 96, 128])
def test_dense_v_stored_dn_exact(D, causal, lens):
    """V [B,H,D,N] (fp16): AttnCfg<0, 64 / 128, 2, 128, true> in the dense mode, with causal, key padding and
    N % 128 != 0."""
    ops = _ops()
    for N in (1000, 72):
        L = [1, 63, 64, 127, 128, 129, N] if lens else None
        B = 7 if lens else 2
        q, k, v, sl, spec = _dense(B, 2, N, D, torch.float16, causal, L, seed=3 * D + causal + N, pin=(0, D - 1))
        o = torch.full_like(q, float("nan"))
        ops.fa2_fwd(q, k, v.transpose(-1, -2).contiguous(), o, v_is_dn=True, causal=causal, seqlens_k=sl)
        _check(o, spec, torch.float16, what="N=%d" % N)


@pytest.mark.parametrize("D", [160, 192, 256, 288, 512, 544, 1024])
def test_ffpa_exact(D):
    """O in column slices of 192 or 256; needle columns in the first 64-column chunk, the last one (half zero-filled when
    D % 64 == 32) and D - 1."""
    ops = _ops()
    last = 64 * ((D - 1) // 64)
    q, k, v, _, spec = _dense(1, 2, 300, D, torch.float16, False, None, seed=D, pin=(0, 63, last, D - 1))
    o = torch.full_like(q, float("nan"))
    ops.ffpa_fwd(q, k, v, o)
    _check(o, spec, torch.float16)


# ------------------------------------------------------------------------------------------------ packed sequences
def _varlen(lq, lk, H, H_kv, D, dtype, causal, seed):
    """(q, k, v, cu_q, cu_k, spec) for a pack; block = (sequence, K/V head), flat key = kv head * total_k + token.
    Columns 0-3 hold their needle at key 0 of every sequence, so a sequence's last tile also reads the next sequence's
    needle for the same column, which it must mask."""
    g = _gen(seed)
    lq, lk = torch.as_tensor(lq, device="cuda").long(), torch.as_tensor(lk, device="cuda").long()
    B, group = lq.numel(), H // H_kv
    cu_q = torch.cat([torch.zeros(1, dtype=torch.long, device="cuda"), lq.cumsum(0)])
    cu_k = torch.cat([torch.zeros(1, dtype=torch.long, device="cuda"), lk.cumsum(0)])
    tq, tk = int(cu_q[-1]), int(cu_k[-1])
    Lb = lk.repeat_interleave(H_kv)
    nb = B * H_kv
    cands = torch.cat([torch.tensor(EDGES, device="cuda").expand(nb, -1), torch.stack([Lb - 2, Lb - 1], 1)], 1)
    pos = _place(Lb, D, cands, g, lo=4)
    pos[:, :4] = torch.where(Lb.view(-1, 1) > 0, 0, -1)
    bb = torch.arange(nb, device="cuda") // H_kv
    start = (torch.arange(nb, device="cuda") % H_kv) * tk + cu_k[bb]             # flat key 0 of each block
    tok = torch.arange(tq, device="cuda").repeat_interleave(H)
    h = torch.arange(H, device="cuda").repeat(tq)
    b = torch.bucketize(tok, cu_q[1:], right=True)
    i, Lq, Lk = tok - cu_q[b], lq[b], lk[b]
    blk = b * H_kv + h // group
    n = (i + Lk - Lq + 1).clamp(min=0).minimum(Lk) if causal else Lk
    cols = _columns(pos, blk, n - 1, D, g)
    cols = torch.where(torch.rand(cols.shape, generator=g, device="cuda") < 0.2, cols % 4, cols)
    p = pos[blk, cols]
    spec = Spec(None, start[blk], n, torch.where(p >= 0, start[blk] + p, torch.full_like(p, -1)))
    ok = pos >= 0
    kf = ex.keys(H_kv * tk, D, (start.view(-1, 1) + pos)[ok], torch.arange(D, device="cuda").expand(nb, D)[ok], dtype, "cuda")
    vf = ex.values(H_kv * tk, D, dtype, g, "cuda")
    spec.v = vf
    q = ex.queries(cols, D, dtype).view(tq, H, D)
    k, v = [t.view(H_kv, tk, D).transpose(0, 1).contiguous() for t in (kf, vf)]
    return q, k, v, _i32(cu_q), _i32(cu_k), spec


LQ = [77, 0, 1, 129, 300, 128, 200, 64, 5]
LK = [300, 5, 0, 128, 129, 1000, 200, 63, 700]


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("D", [32, 64, 96, 128])
@pytest.mark.parametrize("dtype", DTYPES)
def test_varlen_exact(dtype, D, causal):
    """Lq != Lk, empty sequences, group sizes 1 / 2 / 8 / MQA."""
    ops = _ops()
    H = 16
    for group in (1, 2, 8, H):
        q, k, v, cq, ck, spec = _varlen(LQ, LK, H, H // group, D, dtype, causal, seed=D + group + 7 * causal)
        o = torch.full_like(q, float("nan"))
        ops.fa2_fwd_varlen(q, k, v, o, cq, ck, max(LQ), causal=causal)
        _check(o, spec, dtype, what="group %d" % group)


# ------------------------------------------------------------------------------------------------ KV-cache decode
def _splits(B, Lq, H, H_kv, D, cap):
    ws = _ops().fa2_fwd_kvcache_workspace_bytes(B, Lq, H, H_kv, D, cap)
    return ws // (B * Lq * H * (D + 1) * 4) if ws else 1


def _decode_blocks(B, Lq, H, H_kv, D, cap, lens, causal, splits, g, extra=None, lo=0):
    """Needles, row columns and spec (without V) of a decode call; block = (sequence, K/V head), flat key =
    block * cap + key, rows (b, t, h) in Q's order."""
    G, nb = H // H_kv, B * H_kv
    Lk = torch.as_tensor(lens, device="cuda").long().clamp(0, cap)
    Lb = Lk.repeat_interleave(H_kv)
    per = [Lb - 2, Lb - 1, Lb] + [Lb - 1 - t for t in range(min(Lq, 16))]   # the last tokens' causal diagonals
    nt = (Lb + 127) // 128
    for s in range(1, min(splits, 24)):           # tiles of split boundaries
        t = (s * splits // min(splits, 24)) * nt // splits * 128
        per += [t - 1, t]
    if extra is not None:
        per += extra(Lb)
    cands = torch.cat([torch.tensor(EDGES, device="cuda").expand(nb, -1), torch.stack(per, 1)], 1)
    pos = _place(torch.full((nb,), cap, device="cuda"), D, cands, g, lo=lo)
    r = torch.arange(B * Lq * H, device="cuda")
    h, t, b = r % H, (r // H) % Lq, r // (H * Lq)
    blk = b * H_kv + h // G
    n = (t + Lk[b] - Lq + 1).clamp(min=0).minimum(Lk[b]) if causal else Lk[b]
    cols = _columns(pos, blk, n - 1, D, g, lo=lo)
    spec = Spec(None, blk * cap, n, blk * cap + pos[blk, cols])
    return pos, cols, spec


def _page(kc, vc, kind, seed):
    if kind == "contig":
        return kc, vc, None
    kp, vp, table, _ = kvcache_oracle.paged_copy(kc, vc, kind, seed=seed, fill=lambda shape: torch.full(shape, ex.A))
    return kp, vp, table


def _decode(kind, B, Lq, G, H_kv, D, cap, lens, dtype, causal, seed):
    """Builds and runs one decode call; returns (o, spec, splits)."""
    g = _gen(seed)
    H, nb = G * H_kv, B * H_kv
    splits = _splits(B, Lq, H, H_kv, D, cap)
    pos, cols, spec = _decode_blocks(B, Lq, H, H_kv, D, cap, lens, causal, splits, g)
    kf = ex.keys(nb * cap, D, (pos + torch.arange(nb, device="cuda").view(-1, 1) * cap).view(-1),
                 torch.arange(D, device="cuda").repeat(nb), dtype, "cuda")
    spec.v = ex.values(nb * cap, D, dtype, g, "cuda")
    kc, vc = [t.view(B, H_kv, cap, D).transpose(1, 2).contiguous() for t in (kf, spec.v)]
    kc, vc, table = _page(kc, vc, kind, seed)
    q = ex.queries(cols, D, dtype).view(B, Lq, H, D)
    o = torch.full_like(q, float("nan"))
    _ops().fa2_fwd_kvcache(q, kc, vc, o, _i32(lens), table, causal=causal)
    return o, spec, splits


DLENS = [0, 1, 127, 128, 129, 2999, 3072]   # the decoy slot at Lk exists below the capacity 3072


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("kind", ["contig", 16, 32, 64, 128, 256, 384])
def test_decode_pages_exact(kind, causal, dtype):
    """Contiguous caches and every page size the table accepts up to 384 (shuffled table, unlisted pages hold A); one K/V
    head per sequence runs split, 20 fill the SMs and run unsplit."""
    for H_kv in (1, 20):
        o, spec, splits = _decode(kind, len(DLENS), 3, 6, H_kv, 128, 3072, DLENS, dtype, causal, seed=H_kv + causal)
        assert (splits > 1) == (H_kv == 1)
        _check(o, spec, dtype, split=splits > 1, what="H_kv=%d splits=%d" % (H_kv, splits))


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("D", [32, 64, 96, 128])
@pytest.mark.parametrize("dtype", DTYPES)
def test_decode_head_dims_exact(dtype, D, causal):
    for H_kv in (1, 20):
        o, spec, splits = _decode(64, len(DLENS), 3, 6, H_kv, D, 3072, DLENS, dtype, causal, seed=D + H_kv + causal)
        _check(o, spec, dtype, split=splits > 1, what="H_kv=%d splits=%d" % (H_kv, splits))


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("G", [1, 6, 64, 71])
@pytest.mark.parametrize("Lq", [1, 3, 16])
def test_decode_groups_and_query_lengths_exact(Lq, G, causal):
    """Row r of a CTA is token r / hb, head r % hb: G = 6 packs 60 rows, G = 71 takes two head tiles."""
    for kind, H_kv in (("contig", 1), (16, 20)):
        o, spec, splits = _decode(kind, len(DLENS), Lq, G, H_kv, 64, 3072, DLENS, torch.float16, causal,
                                  seed=G * 31 + Lq + causal + H_kv)
        _check(o, spec, torch.float16, split=splits > 1, what="%s H_kv=%d splits=%d" % (kind, H_kv, splits))


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("G", [1, 8])
def test_decode_many_splits_exact(G, causal):
    """MQA, one sequence, a 32K cache: the split rule's top end (109 splits on 132 SMs); short sequences leave most
    splits empty."""
    Lq = 16 if G == 1 else 3      # one CTA of 16 or 24 rows either way
    for i, n in enumerate((1, 129, 5000, 32767, 32768)):
        o, spec, splits = _decode(256, 1, Lq, G, 1, 128, 32768, [n], torch.bfloat16, causal, seed=i + G + causal)
        assert splits >= 64, splits
        _check(o, spec, torch.bfloat16, split=True, what="Lk=%d splits=%d" % (n, splits), needles=n > 1)


# ------------------------------------------------------------------------------------------------ append and rotary
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("Lq,L_new", [(1, 1), (3, 3), (16, 16), (2, 5)])
@pytest.mark.parametrize("kind", ["contig", 16, 64, 384])
def test_append_exact(kind, Lq, L_new, dtype):
    """Needles in the new K rows: they must land at cache_seqlens + i and be read there.  The slots they go to hold A in
    every K column beforehand, so a row that is not written shows.  Rotary over 32 of 64 columns keeps the needles in
    columns 32-63, which rotation leaves alone; rotary over all 64 runs with Q = 0, every row a mean row."""
    ops = _ops()
    B, G, D, cap = 5, 4, 64, 768
    base = [0, 15, 380, 383, cap - L_new]
    for rotary in (None, 32, D):
        for causal in (False, True):
            for H_kv in (1, 24):
                seed = L_new + H_kv + causal + (rotary or 0)
                g = _gen(seed)
                H, nb = G * H_kv, B * H_kv
                splits = _splits(B, Lq, H, H_kv, D, cap)
                lens = [x + L_new for x in base]
                bt = torch.tensor(base, device="cuda").repeat_interleave(H_kv)
                new = lambda Lb: [bt + i for i in range(L_new)]  # noqa: E731
                lo = rotary if rotary and rotary < D else 0
                pos, cols, spec = _decode_blocks(B, Lq, H, H_kv, D, cap, lens, causal, splits, g, extra=new, lo=lo)
                boff = torch.arange(nb, device="cuda").view(-1, 1) * cap
                kf = ex.keys(nb * cap, D, (pos + boff).view(-1), torch.arange(D, device="cuda").repeat(nb), dtype, "cuda")
                spec.v = ex.values(nb * cap, D, dtype, g, "cuda")
                j = bt.view(-1, 1) + torch.arange(L_new, device="cuda").view(1, -1)         # [nb, L_new]
                slots = (boff + j).view(-1)
                k_old, v_old = kf.clone(), spec.v.clone()
                k_old[slots] = ex.A
                v_old[slots] = ex.values(slots.numel(), D, dtype, g, "cuda")
                kn, vn = [t[slots].view(B, H_kv, L_new, D).transpose(1, 2).contiguous() for t in (kf, spec.v)]
                kc, vc = [t.view(B, H_kv, cap, D).transpose(1, 2).contiguous() for t in (k_old, v_old)]
                kc, vc, table = _page(kc, vc, kind, seed)
                q = ex.queries(cols, D, dtype).view(B, Lq, H, D)
                rot = {}
                if rotary:
                    theta = torch.rand(cap, rotary // 2, generator=g, device="cuda") * 2 * math.pi
                    rot = dict(rotary_cos=theta.cos().to(dtype), rotary_sin=theta.sin().to(dtype),
                               rotary_interleaved=causal)
                    if rotary == D:
                        q.zero_()
                        spec.needle = torch.full_like(spec.needle, -1)
                o = torch.full_like(q, float("nan"))
                ops.fa2_fwd_kvcache(q, kc, vc, o, _i32(base), table, causal=causal, k=kn, v=vn, **rot)
                what = "rotary=%s causal=%d H_kv=%d splits=%d" % (rotary, causal, H_kv, splits)
                _check(o, spec, dtype, split=splits > 1, what=what, needles=rotary != D)
                if table is None:
                    vl = vc
                else:
                    jj = torch.arange(cap, device="cuda")
                    vl = vc[table[:, jj // kind].long(), jj % kind]
                assert torch.equal(vl, spec.v.view(B, H_kv, cap, D).transpose(1, 2)), what


# ------------------------------------------------------------------------------------------------ softmax scale
def _scale_case(mode):
    """(D, dtype, q, call(q, scale) -> O, ref(q, scale) -> O on the CPU) for one entry point, random inputs."""
    ops = _ops()
    torch.manual_seed(SCALE_MODES.index(mode))
    rn = lambda *s, dt=torch.float16: torch.randn(*s, device="cuda").to(dt)  # noqa: E731
    if mode in ("dense_f16", "dense_bf16"):
        dt = torch.float16 if mode == "dense_f16" else torch.bfloat16
        D = 64 if dt == torch.float16 else 128
        causal, lens = (True, None) if dt == torch.float16 else (False, [333, 100])
        q, k, v = [rn(2, 2, 333, D, dt=dt) for _ in range(3)]
        sl = None if lens is None else _i32(lens)

        def call(q, scale):
            o = torch.full_like(q, float("nan"))
            ops.fa2_fwd(q, k, v, o, scale=scale, causal=causal, seqlens_k=sl)
            return o
        return D, dt, q, call, lambda q, s: oracle.attention(q, k, v, scale=s, causal=causal, seqlens=lens)
    if mode == "ffpa":
        D = 288
        q, k, v = [rn(1, 2, 300, D) for _ in range(3)]

        def call(q, scale):
            o = torch.full_like(q, float("nan"))
            ops.ffpa_fwd(q, k, v, o, scale=scale)
            return o
        return D, torch.float16, q, call, lambda q, s: oracle.attention(q, k, v, scale=s)
    if mode == "varlen":
        D, lq, lk = 64, [77, 0, 300, 129], [300, 5, 129, 1000]
        q, k, v = rn(sum(lq), 8, D, dt=torch.bfloat16), rn(sum(lk), 2, D, dt=torch.bfloat16), rn(sum(lk), 2, D, dt=torch.bfloat16)
        cq, ck = [_i32([0] + torch.tensor(x).cumsum(0).tolist()) for x in (lq, lk)]

        def call(q, scale):
            o = torch.full_like(q, float("nan"))
            ops.fa2_fwd_varlen(q, k, v, o, cq, ck, max(lq), scale=scale, causal=True)
            return o
        return D, torch.bfloat16, q, call, lambda q, s: ar.packed(q, k, v, cq, ck, scale=s, causal=True)[0].to(q.dtype).cpu()
    if mode in ("decode_split", "decode"):
        B, H, H_kv, D, S = (2, 8, 2, 128, 2048) if mode == "decode_split" else (16, 32, 8, 64, 512)
        assert (_splits(B, 3, H, H_kv, D, S) > 1) == (mode == "decode_split")
        q, kc, vc = rn(B, 3, H, D), rn(B, S, H_kv, D), rn(B, S, H_kv, D)
        lens = ([2000, 700] if B == 2 else torch.randint(0, S + 1, (B,)).tolist())

        def call(q, scale):
            o = torch.full_like(q, float("nan"))
            ops.fa2_fwd_kvcache(q, kc, vc, o, _i32(lens), causal=True, scale=scale)
            return o
        return D, torch.float16, q, call, lambda q, s: ar.kvcache(q, kc, vc, lens, scale=s, causal=True)[0].to(q.dtype)
    assert mode == "append_rotary"
    B, Lq, L_new, H, H_kv, D, S, ps = 3, 2, 2, 8, 2, 64, 256, 64
    kc, vc = rn(B, S, H_kv, D), rn(B, S, H_kv, D)
    kp, vp, table, _ = kvcache_oracle.paged_copy(kc, vc, ps, seed=1)
    q, kn, vn = rn(B, Lq, H, D), rn(B, L_new, H_kv, D), rn(B, L_new, H_kv, D)
    theta = torch.rand(S, 16, device="cuda") * 2 * math.pi
    cos, sin = theta.cos().half(), theta.sin().half()
    lens = [0, 100, S - L_new]

    def call(q, scale):
        o = torch.full_like(q, float("nan"))
        ops.fa2_fwd_kvcache(q, kp.clone(), vp.clone(), o, _i32(lens), table, causal=True, scale=scale, k=kn, v=vn,
                            rotary_cos=cos, rotary_sin=sin, rotary_interleaved=True)
        return o
    return D, torch.float16, q, call, lambda q, s: ko.attention_append(q, kp, vp, lens, kn, vn, table, cos, sin, True,
                                                                        scale=s, causal=True)[0]


SCALE_MODES = ["dense_f16", "dense_bf16", "ffpa", "varlen", "decode_split", "decode", "append_rotary"]


@pytest.mark.parametrize("factor", [0.25, "1.0", 4.0, 16.0])
@pytest.mark.parametrize("mode", SCALE_MODES)
def test_scale_against_the_reference(mode, factor):
    """scale = factor / sqrt(D), or 1.0; 16 / sqrt(D) gives large logits (rescale, combine weights)."""
    D, dt, q, call, ref = _scale_case(mode)
    scale = 1.0 if factor == "1.0" else factor / math.sqrt(D)
    o = call(q, scale)
    assert torch.isfinite(o).all()
    assert torch.allclose(o.cpu().float(), ref(q, scale).float(), **ar.TOL[dt])


@pytest.mark.parametrize("mode", SCALE_MODES)
def test_scale_identities(mode):
    """scale = 2c on Q has the bits of scale = c on 2Q (power-of-two scaling commutes with every rounding in the kernel
    and the rotary arithmetic); scale 0 and -1 have the bits of 1.0f / sqrtf(D)."""
    D, dt, q, call, _ = _scale_case(mode)
    c = 0.7 / math.sqrt(D)
    assert torch.equal(call(q, 2 * c), call((2 * q).contiguous(), c))
    o_default = call(q, float(np.float32(1) / np.sqrt(np.float32(D))))
    assert torch.equal(call(q, None), o_default)
    assert torch.equal(call(q, -1.0), o_default)
    assert not torch.equal(call(q, 2 * float(np.float32(1) / np.sqrt(np.float32(D)))), o_default)


# ------------------------------------------------------------------------------------------------ V [B,H,D,N]
@pytest.mark.parametrize("lens", [None, [1000, 129]])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("D", [32, 64, 96, 128])
def test_v_stored_dn_same_bits_as_v_stored_nd(D, causal, lens):
    """Random inputs: V [B,H,D,N] against the oracle and bit for bit against V [B,H,N,D] (the same products summed in
    the same k16 order)."""
    ops = _ops()
    torch.manual_seed(D + causal)
    q, k, v = [torch.randn(2, 2, 1000, D, dtype=torch.half, device="cuda") for _ in range(3)]
    sl = None if lens is None else _i32(lens)
    o_nd, o_dn = torch.full_like(q, float("nan")), torch.full_like(q, float("nan"))
    ops.fa2_fwd(q, k, v, o_nd, causal=causal, seqlens_k=sl)
    ops.fa2_fwd(q, k, v.transpose(-1, -2).contiguous(), o_dn, v_is_dn=True, causal=causal, seqlens_k=sl)
    assert torch.allclose(o_dn.cpu().float(), oracle.attention(q, k, v, causal=causal, seqlens=lens).float(), **ar.TOL[torch.float16])
    assert torch.equal(o_dn, o_nd)


# ------------------------------------------------------------------------------------------------ limits
def test_dense_and_ffpa_at_65535_heads_exact():
    """B * H = 65535, the largest grid.z the dense and FFPA entry points accept."""
    ops = _ops()
    q, k, v, sl, spec = _dense(3, 21845, 16, 32, torch.float16, True, [16, 5, 1], seed=1)
    o = torch.full_like(q, float("nan"))
    ops.fa2_fwd(q, k, v, o, causal=True, seqlens_k=sl)
    _check(o, spec, torch.float16, what="dense")
    del q, k, v, o, spec
    q, k, v, _, spec = _dense(5, 13107, 8, 160, torch.float16, False, None, seed=2, pin=(0, 159))
    o = torch.full_like(q, float("nan"))
    ops.ffpa_fwd(q, k, v, o)
    _check(o, spec, torch.float16, what="ffpa")


def test_varlen_at_65535_sequence_heads_exact():
    g = torch.Generator(device="cuda").manual_seed(3)
    B, H, H_kv = 4369, 15, 5
    lq, lk = [torch.randint(0, 7, (B,), generator=g, device="cuda") for _ in range(2)]
    lq[0] = 6
    q, k, v, cq, ck, spec = _varlen(lq, lk, H, H_kv, 64, torch.bfloat16, True, seed=4)
    o = torch.full_like(q, float("nan"))
    _ops().fa2_fwd_varlen(q, k, v, o, cq, ck, 6, causal=True)
    _check(o, spec, torch.bfloat16)


@pytest.mark.parametrize("shape", ["pairs", "token_tiles", "head_tiles"])
def test_decode_at_the_largest_grid_exact(shape):
    """B * H_kv = 65535; 65535 token tiles (G = 1, Lq = 65535 * 64); 65535 head tiles (H_kv = 1, H = 65535 * 64)."""
    if shape == "pairs":
        B, Lq, G, H_kv, cap, causal = 13107, 2, 2, 5, 32, True
        lens = torch.randint(0, cap + 1, (B,), generator=torch.Generator().manual_seed(5)).tolist()
    elif shape == "token_tiles":
        B, Lq, G, H_kv, cap, causal, lens = 1, 65535 * 64, 1, 1, 128, False, [100]
    else:
        B, Lq, G, H_kv, cap, causal, lens = 1, 1, 65535 * 64, 1, 128, False, [100]
    o, spec, splits = _decode("contig", B, Lq, G, H_kv, 32, cap, lens, torch.float16, causal, seed=6)
    assert splits == 1
    _check(o, spec, torch.float16)


def _free_gib():
    return torch.cuda.mem_get_info()[0] / 2 ** 30


def test_varlen_q_and_o_past_2_31_elements_exact():
    """[total_q, H, D] Q / O of 2^31 + 8M elements with B * H = 192 CTAs per query tile; not causal, so every row past
    element 2^31 sees keys."""
    if _free_gib() < 20:
        pytest.skip("needs 20 GiB of free device memory")
    lq, lk = [131072, 131072, 1000], [300, 129, 64]
    H, H_kv, D = 64, 8, 128
    assert sum(lq) * H * D > 2 ** 31
    q, k, v, cq, ck, spec = _varlen(lq, lk, H, H_kv, D, torch.float16, False, seed=7)
    o = torch.full_like(q, float("nan"))
    _ops().fa2_fwd_varlen(q, k, v, o, cq, ck, max(lq))
    del q
    _check(o, spec, torch.float16)


def test_paged_decode_cache_past_2_31_elements_exact():
    """Caches of 8200 pages x 256 keys x 8 heads x 128 (2^31 + 2M elements each); the tables list pages on both sides
    of element 2^31, so needles sit past that offset."""
    if _free_gib() < 14:
        pytest.skip("needs 14 GiB of free device memory")
    B, Lq, G, H_kv, D, ps, pps, num_pages = 2, 2, 4, 8, 128, 256, 4, 8200
    assert num_pages * ps * H_kv * D > 2 ** 31
    cap, H, nb = pps * ps, G * H_kv, B * H_kv
    lens = [1000, 777]
    g = _gen(8)
    splits = _splits(B, Lq, H, H_kv, D, cap)
    pos, cols, spec = _decode_blocks(B, Lq, H, H_kv, D, cap, lens, True, splits, g)
    kf = ex.keys(nb * cap, D, (pos + torch.arange(nb, device="cuda").view(-1, 1) * cap).view(-1),
                 torch.arange(D, device="cuda").repeat(nb), torch.bfloat16, "cuda")
    spec.v = ex.values(nb * cap, D, torch.bfloat16, g, "cuda")
    table = _i32([[8199, 8191, 8195, 8197], [8192, 8198, 5, 8194]])
    caches = []
    for t in (kf, spec.v):
        c = torch.zeros(num_pages, ps, H_kv, D, dtype=torch.bfloat16, device="cuda")
        c[table.view(-1).long()] = t.view(B, H_kv, pps, ps, D).permute(0, 2, 3, 1, 4).reshape(B * pps, ps, H_kv, D)
        caches.append(c)
    q = ex.queries(cols, D, torch.bfloat16).view(B, Lq, H, D)
    o = torch.full_like(q, float("nan"))
    _ops().fa2_fwd_kvcache(q, caches[0], caches[1], o, _i32(lens), table, causal=True)
    _check(o, spec, torch.bfloat16, split=splits > 1)
