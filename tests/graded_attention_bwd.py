"""Exact answers for the attention backward (b200k_fa2_bwd), used by test_gpu_attention_bwd_graded.py and proved on the
CPU in test_attention_bwd_graded_cpu.py.  The needle inputs of test_gpu_attention_bwd.py make dS = 0 everywhere; here P is
graded, dS is nonzero, and both are rounded where the dtype makes them.

The backward is a function of Q, K, V, O, lse and dO, consistent or not, so O and lse are chosen freely:
  scores  scale = scale_exact(k), so scale_log2 = 2^-k exactly.  Q row i = 2^k e_c(i), column c of K holds small integer
          grades g, so S * scale_log2 = g.
  lse     row i gets lse_exact(t_i) with fp32(lse * fp32(log2 e)) == t_i, an integer >= every grade the row sees: P =
          ex2(g - t) = 2^(g - t) exactly.  Not every t has such an lse (no_exact_lse); t_i is moved up past those.
  rows    three kinds, per row:
            normal  dO_i two +-1 entries in columns >= 1, O_i and V integers: dP - Delta is a small integer, so dS is
                    exact and so are the sums over long rows;
            round   rows that see at most ROUND_KEYS keys: dO_i integers whose sum of magnitudes is about ROUND_MASS,
                    O_id = -16 sign(dO_id), so dP - Delta = sum_d |dO_id| (16 + sign V_jd) lies near 2^12..2^13 (fp16),
                    2^9..2^10 (bf16) and dS = P (dP - Delta) is rounded to nearest, ties to even, by pack_round;
            frac    lse2 = t + i / 8 with i from graded_attention.fractional_grades, so P~ is a rounded value; dO_i = e_0,
                    O_i0 = 1 and V[:, 0] = 1 make dP = Delta exactly, so dS = 0 whatever ex2.approx gave, and dV[:, 0]
                    (which only frac rows feed: every other dO_i0 is 0) holds P~ bit for bit.
  decoys  DECOY = 250 on every column of the key at seqlens_k, and (causal) on key E of a cliff column that only rows
          i < E read, row E - 1 among them, for E on both sides of the 64-key tile edges.  A mask that lets a row see one
          gives P = 2^(250 - t) = inf and NaN in the output.

closed_form() takes the six inputs as they are, computes P = 2^(S scale_log2 - lse2), dS = P (dP - Delta), P~, dS~ and the
three sums in fp64, asserts each is what fp32 holds (the window: every term of an output element is a multiple of 2^-G
and the sum of their magnitudes is below 2^(24 - G), which keeps every partial sum exact in any order), and stores
dV = dtype(sum), dQ, dK = dtype(fp32(sum * fp32(scale))).  make_forward_case() builds the one consistent case, whose O and
lse come from fa2_fwd.  emulate_bwd() is the three kernels' fp32 arithmetic in numpy, with the mutations the tests must
reject."""
from __future__ import annotations

import math

import numpy as np
import torch

import graded_attention as ga

LOG2E_F32 = ga.LOG2E_F32
FAR, DECOY = ga.FAR, ga.DECOY
LN2_FWD = 0.6931472                   # the forward's fp32 ln 2 in (m + log2f(l)) * 0.6931472f
ROUND_KEYS = 8                        # rows that see at most this many keys take the "round" regime
ROUND_MASS = {torch.float16: 300, torch.bfloat16: 40}   # about sum_d |dO_id| of a round row
CLIFFS = [63, 64, 65, 127, 128, 129, 190, 191, 192, 255, 256, 511, 512, 513, 999]  # cliff keys E (causal)


# ------------------------------------------------------------------------------------------------ exact lse
def lse2_of(lse):
    """What the prep kernel writes: fp32(lse * fp32(log2 e))."""
    return np.float32(lse) * np.float32(LOG2E_F32)


def lse_exact(x: float):
    """The fp32 lse nearest x ln 2 with lse2_of(lse) == x, searched 8 ulps either side; None if there is none."""
    want = np.float32(x)
    assert float(want) == x
    c = np.float32(x * math.log(2))
    cands, lo, hi = [c], c, c
    for _ in range(8):
        lo, hi = np.nextafter(lo, np.float32(-np.inf)), np.nextafter(hi, np.float32(np.inf))
        cands += [lo, hi]
    for lse in sorted(cands, key=lambda v: abs(float(v) - x * math.log(2))):
        if lse2_of(lse) == want:
            return float(lse)
    return None


def no_exact_lse(lo: int, hi: int):
    """The integers t in [lo, hi] that no fp32 lse reaches."""
    return [t for t in range(lo, hi + 1) if lse_exact(t) is None]


_TABLE_LO, _TABLE_HI = -16, 40
_LSE_TABLE: list = []


def _lse_table():
    """fp32 [8 (HI - LO)]: lse_exact(LO + i / 8), NaN where there is none."""
    if not _LSE_TABLE:
        _LSE_TABLE.append(torch.tensor([float("nan") if v is None else v for v in
                                        (lse_exact(e / 8) for e in range(8 * _TABLE_LO, 8 * _TABLE_HI))]))
    return _LSE_TABLE[0]


def exact_lse_of(eighths: torch.Tensor):
    """(eighths moved up by whole units until each has an exact lse, that lse as fp32) for integer tensors of 8 x."""
    table = _lse_table()
    e = eighths.clone()
    while True:
        assert int(e.min()) >= 8 * _TABLE_LO and int(e.max()) < 8 * _TABLE_HI
        v = table[e - 8 * _TABLE_LO]
        if not bool(v.isnan().any()):
            return e, v.float()
        e = torch.where(v.isnan(), e + 8, e)


# ------------------------------------------------------------------------------------------------ inputs
def kv_lens(lens, B, N):
    """seqlens_k clamped to [1, N] as the kernels do, [B] long (N everywhere without seqlens_k)."""
    if lens is None:
        return torch.full((B,), N, dtype=torch.long)
    return torch.as_tensor(lens).long().clamp(1, N)


def visible(B, H, N, causal, lens):
    """[B, H, N, N] bool: row i of (b, h) sees key j."""
    j = torch.arange(N)
    vis = (j.view(1, 1, 1, N) < kv_lens(lens, B, N).view(B, 1, 1, 1)).expand(B, H, N, N)
    return vis & (j.view(1, 1, 1, N) <= j.view(1, 1, N, 1)) if causal else vis


def make_case(dtype, B, H, N, D, causal, lens=None, seed=0, k=0, W=3, nnz=2, frac_rows=2):
    """One graded case on the CPU: dict of q, k, v, o, do (dtype [B, H, N, D]), lse (fp32 [B, H, N]), seqlens (int32 [B]
    or None), scale, causal, and per row: col (the grade column), t (lse2, an integer or t + i / 8), kind (0 normal,
    1 round, 2 frac).  Grades of head (b, h) are beta + [0, W] with beta in [-4, 4], and t = beta + W + {0, 1}, so heads
    differ in t; nnz is the number of +-1 entries of a normal row's dO."""
    g = torch.Generator().manual_seed(seed)
    BH = B * H
    ri = lambda lo, hi, shape: torch.randint(lo, hi, shape, generator=g)  # noqa: E731
    kv = kv_lens(lens, B, N).repeat_interleave(H)                                    # [BH]
    rows = torch.arange(N)
    beta = ri(-4, 5, (BH,))
    K = beta.view(BH, 1, 1) + ri(0, W + 1, (BH, N, D))
    K[rows.view(1, N) == kv.view(BH, 1)] = DECOY                                     # the key at seqlens_k
    col = ri(0, D, (BH, N))
    cliffs = [E for E in CLIFFS if E < N][:D - 1] if causal else []
    if cliffs:
        e_of = torch.full((D,), N + 1)
        for i, E in enumerate(cliffs):
            K[:, E, 1 + i] = DECOY
            e_of[1 + i] = E
        plain = (e_of > N).nonzero().view(-1)
        late = e_of[col] <= rows.view(1, N)                                          # would see its column's decoy
        col = torch.where(late, plain[ri(0, plain.numel(), (BH, N))], col)
        for i, E in enumerate(cliffs):                                               # the last row before E reads it
            col[:, E - 1] = 1 + i
    n = torch.minimum(rows.view(1, N) + 1, kv.view(BH, 1)) if causal else kv.view(BH, 1).expand(BH, N)

    kind = torch.zeros(BH, N, dtype=torch.long)
    kind[n <= ROUND_KEYS] = 1
    F = min(frac_rows, N // 2)
    if F:
        kind.scatter_(1, torch.rand(BH, N, generator=g).argsort(1)[:, :F], 2)

    t = beta.view(BH, 1) + W + ri(0, 2, (BH, N))
    fr = torch.tensor(ga.fractional_grades(dtype))
    eighths, lse = exact_lse_of(8 * t + torch.where(kind == 2, fr[ri(0, fr.numel(), (BH, N))], 0))

    V = ri(-8, 9, (BH, N, D))
    V[..., 0] = 1
    dO, O = row_values(kind.view(-1), D, dtype, nnz, ri)

    q = torch.zeros(BH, N, D)
    q.scatter_(2, col.view(BH, N, 1), 2.0 ** k)
    out = _pack(dtype, (B, H, N, D), dict(q=q, k=K, v=V, o=O, do=dO))
    out.update(lse=lse.view(B, H, N), seqlens=None if lens is None else torch.as_tensor(lens, dtype=torch.int32),
               scale=ga.scale_exact(k), causal=causal, col=col.view(B, H, N), t=(eighths / 8.0).view(B, H, N),
               kind=kind.view(B, H, N))
    return out


def row_values(kind, D, dtype, nnz, ri):
    """(dO, O) long [R, D] for rows of the given kinds (0 normal, 1 round, 2 frac), with V[:, 0] = 1 assumed; ri(lo, hi,
    shape) draws integers."""
    R = kind.numel()
    O = ri(-8, 9, (R, D))
    dO = torch.zeros(R, D, dtype=torch.long)
    dO.scatter_add_(1, ri(1, D, (R, nnz)), 2 * ri(0, 2, (R, nnz)) - 1)              # normal: two +-1 entries
    M = max(1, round(2 * ROUND_MASS[dtype] / (D - 1)))
    big = ri(-M, M + 1, (R, D))
    big[:, 0] = 0
    rnd = (kind == 1).view(R, 1)
    dO = torch.where(rnd, big, dO)
    O = torch.where(rnd & (big != 0), -16 * big.sign(), O)
    e0 = torch.zeros(1, D, dtype=torch.long)
    e0[:, 0] = 1
    dO = torch.where((kind == 2).view(R, 1), e0, dO)
    O[:, 0] = torch.where(kind == 2, 1, O[:, 0])
    return dO, O


def _pack(dtype, shape, ints):
    """The integer tensors in dtype, each asserted to be held exactly."""
    out = {}
    for name, x in ints.items():
        out[name] = x.reshape(shape).to(dtype)
        assert torch.equal(out[name].double(), x.reshape(shape).double()), name
    return out


def make_forward_case(dtype, B, H, N, D, lens=None, seed=0, k=0):
    """The consistent case (non-causal), whose O and lse come from fa2_fwd: in head (b, h) every row sees the n = kv_len
    keys of its column c, of which a = 2^u - x hold the column's top grade m (weight 1), 2x hold m - 1 (weight 1/2) and
    the rest FAR (weight exactly 0), so the row's weights sum to 2^u and its lse is t = m + u, |t| <= 12 (which the
    forward's fp32 (m + log2f(l)) * 0.6931472f carries through lse * log2 e exactly).  u <= 3 keeps P a multiple of
    2^-4, so O, Delta and dS stay within a few bits.  Returns make_case's dict without o and lse, and t per row."""
    g = torch.Generator().manual_seed(seed)
    BH = B * H
    K, top = forward_keys(BH, N, D, kv_lens(lens, B, N).repeat_interleave(H), g)
    col = torch.randint(0, D, (BH, N), generator=g)
    q = torch.zeros(BH, N, D)
    q.scatter_(2, col.view(BH, N, 1), 2.0 ** k)
    V = torch.randint(-8, 9, (BH, N, D), generator=g)
    dO = torch.zeros(BH, N, D, dtype=torch.long)
    dO.scatter_add_(2, torch.randint(0, D, (BH, N, 2), generator=g), 2 * torch.randint(0, 2, (BH, N, 2), generator=g) - 1)
    out = _pack(dtype, (B, H, N, D), dict(q=q, k=K, v=V, do=dO))
    t = top.gather(1, col)
    assert int(t.abs().max()) <= 12
    out.update(seqlens=None if lens is None else torch.as_tensor(lens, dtype=torch.int32), scale=ga.scale_exact(k),
               causal=False, col=col.view(B, H, N), t=t.view(B, H, N).double(), kind=torch.zeros(B, H, N, dtype=torch.long))
    return out


def forward_keys(BH, N, D, kv, g):
    """(K long [BH, N, D], top [BH, D]) of make_forward_case: head bh has kv[bh] keys (DECOY on the key after them when
    kv[bh] < N), and column c of it holds 2^u - x keys at grade m, 2x at m - 1 and FAR elsewhere; top = m + u, the lse2
    of a row that reads column c."""
    K = torch.randint(-4, 5, (BH, N, D), generator=g)
    top = torch.zeros(BH, D, dtype=torch.long)
    for bh in range(BH):
        n = int(kv[bh])
        if n < N:
            K[bh, n] = DECOY
        for c in range(D):
            u = int(torch.randint(0, min(3, int(math.log2(n))) + 1, (1,), generator=g))
            x = int(torch.randint(0, min(2 ** u - 1, n - 2 ** u) + 1, (1,), generator=g))
            m = int(torch.randint(-4, 5, (1,), generator=g))
            perm = torch.randperm(n, generator=g)
            K[bh, :n, c] = FAR
            K[bh, perm[:2 ** u - x], c] = m
            K[bh, perm[2 ** u - x:2 ** u + x], c] = m - 1
            top[bh, c] = m + u
    return K, top


def forward_lse(t):
    """The lse the forward writes for a row whose max is m and whose weights sum to 2^u, t = m + u: fp32(t * 0.6931472f)."""
    return (t.float() * torch.tensor(LN2_FWD, dtype=torch.float32)).float()


# ------------------------------------------------------------------------------------------------ the closed form
def _low_bits(x):
    """G per element of an fp64 tensor: x is a multiple of 2^-G and of no finer power; -10^6 for zeros."""
    m, e = torch.frexp(x.abs())
    M = (m * 2.0 ** 53).long()
    tz = torch.log2((M & -M).double()).round().long()
    return torch.where(x != 0, 53 - tz - e.long(), torch.full_like(tz, -10 ** 6))


def _window(absum, G, what):
    """Every partial sum of terms that are multiples of 2^-G is exact in fp32 when the sum of their magnitudes is below
    2^(24 - G).  Returns the largest absum 2^G / 2^24 (how close the case comes)."""
    r = absum * torch.pow(2.0, G.clamp(min=-200).double()) / 2.0 ** 24
    bad = r >= 1
    assert not bool(bad.any()), "%s: %d sums leave the fp32 window (largest sum x 2^G = 2^%.2f)" % (
        what, int(bad.sum()), math.log2(float(r.max()) * 2 ** 24))
    return float(r.max()) if r.numel() else 0.0


def _maxG(x, dim=None):
    G = _low_bits(x)
    return G.max() if dim is None else G.max(dim, keepdim=True).values


def _window_mm(A, B, what):
    """_window for the sums A @ B: element (i, d) has terms A_ij B_jd; its G is the largest G(A_ij) over the j with
    B_jd != 0, plus the largest G of B (found one level of G(A) at a time)."""
    GA, nzB = _low_bits(A), (B != 0).double()
    G = torch.full(A.shape[:-1] + B.shape[-1:], -10 ** 6, dtype=torch.long, device=A.device)
    for lev in GA[A != 0].unique().tolist():
        hit = ((GA == lev) & (A != 0)).double() @ nzB > 0
        G = torch.where(hit, torch.maximum(G, torch.full_like(G, lev)), G)
    return _window(A.abs() @ B.abs(), G + _maxG(B), what)


def closed_form(q, k, v, o, lse, do, scale, causal, seqlens, rounded=True):
    """((dq, dk, dv) in q's dtype, info) from the six inputs, in fp64 on q's device, every step asserted exact (see the
    module docstring).  rounded=False gives the fp64 gradients of the same P and dS without the dtype roundings and
    with the exact scale (scale_log2 ln 2), for comparison with attention_ref.dense_grads_given."""
    B, H, N, D = q.shape
    vis = visible(B, H, N, causal, None if seqlens is None else seqlens.cpu()).to(q.device)
    lse2 = (lse.float() * torch.tensor(LOG2E_F32, dtype=torch.float32, device=q.device)).double()
    return closed_form_core(*(t.double() for t in (q, k, v, o, do)), lse2, vis, scale, q.dtype, rounded)


def closed_form_core(Q, K, V, O, dO, lse2, vis, scale, dtype, rounded=True, group=1):
    """closed_form on fp64 operands: Q, O, dO [..., H, Lq, D], K, V [..., H / group, Lk, D] (query head h reads K/V head
    h // group), lse2 [..., H, Lq] as the prep writes it, vis [..., H, Lq, Lk] (or broadcastable) the keys each row sees.
    dK and dV sum over the group: their windows are those of the group's G * Lq terms.  info adds ds_group, the keys
    whose dK sums nonzero dS~ from two or more heads."""
    dev = Q.device
    H, Lq, Lk = Q.size(-3), Q.size(-2), K.size(-2)
    vis = vis.expand(*Q.shape[:-1], Lk)
    Kx, Vx = (t.repeat_interleave(group, dim=-3) for t in (K, V))
    sl = float(np.float32(scale) * np.float32(LOG2E_F32))
    S = Q @ Kx.transpose(-1, -2)
    x = torch.where(vis, S * sl - lse2.unsqueeze(-1), torch.full_like(S, float("-inf")))
    xv = x[vis]
    assert bool((xv * 8 == (xv * 8).round()).all()), "a score exponent is not a multiple of 1/8"
    assert not bool(((xv >= -150) & (xv < -126)).any()), "P near the fp32 flush-to-zero threshold"
    P = torch.where(x >= -126, torch.exp2(x), torch.zeros_like(x))
    assert bool(torch.isfinite(P).all()) and float(P.max()) <= 1, "P above 1: a row sees a key above its lse"
    frac = vis & (x != x.floor()) & (x >= -126)
    eighth = ((x.ceil() - x) * 8).round().long()
    assert bool(torch.isin(eighth[frac], torch.tensor(ga.fractional_grades(dtype), device=dev)).all())
    Pr = P.to(dtype).double() if rounded else P

    _window(dO.abs() @ Vx.abs().transpose(-1, -2), _maxG(dO, -1) + _maxG(Vx, -1).transpose(-1, -2), "dP")
    _window((dO * O).abs().sum(-1), _maxG(dO, -1).squeeze(-1) + _maxG(O, -1).squeeze(-1), "Delta")
    dP = dO @ Vx.transpose(-1, -2)
    Delta = (dO * O).sum(-1)
    dd = torch.where(vis, dP - Delta.unsqueeze(-1), torch.zeros_like(dP))
    assert torch.equal(dd.float().double(), dd), "dP - Delta is not an fp32 value"
    assert bool((dd[frac] == 0).all()), "a row with fractional P has nonzero dP - Delta"
    dS = P * dd
    assert torch.equal(torch.where(frac, 0.0, dS).float().double(), torch.where(frac, 0.0, dS)), "dS not fp32"
    dSr = dS.float().to(dtype).double() if rounded else dS

    # the group's heads side by side as G * Lq rows of one K/V head (heads h = kv head * G + g are adjacent)
    fold = lambda t: t.reshape(*t.shape[:-3], H // group, group * Lq, t.size(-1))  # noqa: E731
    dSf, Prf, Qf, dOf = fold(dSr), fold(Pr), fold(Q), fold(dO)
    dq, dk, dv = dSr @ Kx, dSf.transpose(-1, -2) @ Qf, Prf.transpose(-1, -2) @ dOf
    if not rounded:
        return (dq * (sl * math.log(2)), dk * (sl * math.log(2)), dv), {}
    info = dict(
        win_dq=_window_mm(dSr, Kx, "dQ"), win_dk=_window_mm(dSf.transpose(-1, -2), Qf, "dK"),
        win_dv=_window_mm(Prf.transpose(-1, -2), dOf, "dV"),
        ds_group=int(((dSr != 0).any(-2).reshape(*dSr.shape[:-3], H // group, group, Lk).sum(-2) >= 2).sum()))
    for name, t in (("dQ", dq), ("dK", dk), ("dV", dv)):
        assert torch.equal(t.float().double(), t), name + " sum is not an fp32 value"
    s32 = torch.tensor(float(np.float32(scale)), dtype=torch.float32, device=dev)
    outs = [((dq.float() * s32) + 0.0).to(dtype), ((dk.float() * s32) + 0.0).to(dtype), (dv.float() + 0.0).to(dtype)]
    rnd = vis & ~frac & (dSr != dS)
    other = 2 * dS - dSr                                                     # the other neighbour, if dS is a tie
    info.update(ds_rounded=int(rnd.sum()), ds_away=int((rnd & (dSr.abs() > dS.abs())).sum()),
                ds_ties=int((rnd & (other.to(dtype).double() == other)).sum()),
                p_rounded=int((frac & (Pr != P)).sum()), ds_nonzero=int((vis & (dS != 0)).sum()))
    return outs, info


# ------------------------------------------------------------------------------------------------ the kernels' arithmetic
MUTATIONS = ["ds_trunc", "p_trunc", "delta_swap", "lse2_swap", "causal_diag", "causal_next", "len_short", "len_long",
             "scale_dv", "dk_unscaled", "dq_unscaled", "ds_sign", "delta_from_v"]


def emulate_bwd(q, k, v, o, lse, do, scale, causal, seqlens, mut=""):
    """The three kernels in numpy fp32, (dq, dk, dv) as fp32 arrays of dtype values.  The prep kernel's Delta and
    lse2 = lse * log2 e; the masks (keys >= kv_len, causal keys > row); P = ex2(fmaf(S, scale_log2, -lse2)) flushed below
    2^-126; dS = P (dP - Delta); P~, dS~ rounded to the dtype (pack_round); the sums, exact (closed_form asserts the
    window), then the stores: dQ, dK times fp32(scale), dV as is.  `mut` is one of MUTATIONS or "":
      ds_trunc, p_trunc        dS~ / P~ rounded toward zero
      delta_swap, lse2_swap    Delta / lse2 of the thread's other row, r ^ 8 (the row statistics' 0 / +inf past N)
      causal_diag, causal_next the causal mask key >= row, key > row + 1
      len_short, len_long      the length mask one key short, one key long
      scale_dv                 dV stored times scale;  dk_unscaled, dq_unscaled: dK / dQ stored without it
      ds_sign                  dS = P (Delta - dP);  delta_from_v: Delta = dO . V (row i of V) instead of dO . O"""
    f, f64 = np.float32, np.float64
    dtype = q.dtype
    Q, K, V, O, dO = (t.float().cpu().numpy() for t in (q, k, v, o, do))
    B, H, N, D = Q.shape
    with np.errstate(all="ignore"):
        Delta = (dO.astype(f64) * (V if mut == "delta_from_v" else O)).sum(-1).astype(f)
        lse2 = lse.float().cpu().numpy() * f(LOG2E_F32)
        if mut in ("delta_swap", "lse2_swap"):
            r = np.arange(N) ^ 8
            src, fill = (Delta, f(0)) if mut == "delta_swap" else (lse2, f(np.inf))
            src = np.where(r < N, src[..., np.minimum(r, N - 1)], fill)
            Delta, lse2 = (src, lse2) if mut == "delta_swap" else (Delta, src)
        sl = f(f(scale) * f(LOG2E_F32))
        kv = kv_lens(None if seqlens is None else seqlens.cpu(), B, N).numpy() + \
            {"len_short": -1, "len_long": 1}.get(mut, 0)
        j = np.arange(N)
        vis = j.reshape(1, 1, 1, N) < kv.reshape(B, 1, 1, 1)
        if causal:
            vis = vis & (j.reshape(1, 1, 1, N) <= j.reshape(1, 1, N, 1) + {"causal_diag": -1, "causal_next": 1}.get(mut, 0))
        S = np.where(vis, (Q.astype(f64) @ K.astype(f64).swapaxes(-1, -2)).astype(f), f(-np.inf))
        dP = np.where(vis, (dO.astype(f64) @ V.astype(f64).swapaxes(-1, -2)).astype(f), f(0))
        x = (S.astype(f64) * f64(sl) - lse2[..., None]).astype(f)
        P = np.exp2(x.astype(f64)).astype(f)
        P[P < f(2.0 ** -126)] = 0
        dS = P * (dP - Delta[..., None])
        if mut == "ds_sign":
            dS = -dS
        Pr = ga.round_to(P, dtype, trunc=mut == "p_trunc")
        dSr = ga.round_to(dS, dtype, trunc=mut == "ds_trunc")
        dq = (dSr.astype(f64) @ K.astype(f64)).astype(f)
        dk = (dSr.astype(f64).swapaxes(-1, -2) @ Q.astype(f64)).astype(f)
        dv = (Pr.astype(f64).swapaxes(-1, -2) @ dO.astype(f64)).astype(f)
        s = f(scale)
        dq = dq if mut == "dq_unscaled" else dq * s
        dk = dk if mut == "dk_unscaled" else dk * s
        dv = dv * s if mut == "scale_dv" else dv
        return tuple(ga.round_to(t, dtype) + f(0) for t in (dq, dk, dv))


def same_bits(a, b):
    """Two fp32 arrays of dtype values hold the same bits (zeros of either sign are equal)."""
    a, b = (np.asarray(t, np.float32) + np.float32(0) for t in (a, b))
    return np.array_equal(a.view(np.uint32), b.view(np.uint32))


# ------------------------------------------------------------------------------------------------ failures
def describe(case, name, want, got, count=1):
    """The first `count` wrong elements of output `name` (dq: by query row, dk / dv: by key) as text."""
    bad = ((want.float() != got.float()) | torch.isnan(got.float())).nonzero().tolist()[:count]
    kv = kv_lens(None if case["seqlens"] is None else case["seqlens"].cpu(), want.size(0), want.size(2))
    lines = []
    for b, h, r, c in bad:
        if name == "dq":
            where = "row %d (t %s, grade column %d, kind %d)" % (r, float(case["t"][b, h, r]), int(case["col"][b, h, r]),
                                                                 int(case["kind"][b, h, r]))
        else:
            readers = (case["col"][b, h] == c).nonzero().view(-1)[:6].tolist()
            where = "key %d (kv_len %d; rows reading column %d: %s)" % (r, int(kv[b]), c, readers)
        lines.append("%s[b %d, h %d] %s, column %d: expected %r got %r" % (
            name, b, h, where, c, float(want[b, h, r, c]), float(got[b, h, r, c])))
    return "; ".join(lines) + " (%d wrong)" % int(((want.float() != got.float()) | torch.isnan(got.float())).sum())


# ------------------------------------------------------------------------------------------------ the cases the GPU runs
DTYPES = [torch.float16, torch.bfloat16]
HEADDIMS = [32, 64, 96, 128]
NS = [1, 63, 64, 65, 127, 128, 129, 191, 1000]
LENS = ["none", "edges", "clamped"]


def lens_of(kind, N):
    """seqlens_k of a case: none; 1, 64, 65 and N - 1; or the clamped 0, -5, N + 5 beside N / 2."""
    return {"none": None, "edges": (1, 64, 65, N - 1), "clamped": (0, -5, N + 5, (N + 1) // 2)}[kind]


def cases():
    """Every (dtype, D, mask, N) once, the seqlens_k variant rotating with them; B = 2, H = 2 without seqlens_k and
    B = 4, H = 2 with it; k (Q = 2^k) in 0..2."""
    out = []
    for di, dtype in enumerate(DTYPES):
        for Di, D in enumerate(HEADDIMS):
            for causal in (False, True):
                for Ni, N in enumerate(NS):
                    kind = LENS[(Di + 2 * causal + di + Ni) % 3]
                    B = 2 if kind == "none" else 4
                    out.append(dict(dtype=dtype, B=B, H=2, N=N, D=D, causal=causal, lens=lens_of(kind, N),
                                    seed=1000 * di + 100 * Di + 10 * causal + Ni, k=(Di + Ni) % 3))
    return out


def case_id(c):
    if c["B"] * c["H"] == 65535:
        return "grid65535"
    return "%s-D%d-%s-N%d-%s" % ("f16" if c["dtype"] == torch.float16 else "bf16", c["D"],
                                 "causal" if c["causal"] else "full", c["N"],
                                 "none" if c["lens"] is None else "sl" + "_".join(map(str, c["lens"]))) + \
        ("-long" if c.get("nnz") else "")


def long_cases():
    """One long row per dtype near the window's limit: 2048 keys, 16 +-1 entries per dO row, grades spread over 6, so
    the largest dQ sum comes within a factor of two of 2^(24 - G)."""
    return [dict(dtype=dt, B=1, H=2, N=2048, D=64, causal=False, lens=None, seed=7 + i, k=1, W=6, nnz=16)
            for i, dt in enumerate(DTYPES)]


def all_cases():
    return cases() + long_cases()


def grid_case():
    """B * H = 65535, the largest grid y of the dK/dV kernel and grid z of the dQ kernel, at N = 3 with seqlens_k from -1
    to 4 (clamped to [1, 3])."""
    lens = tuple((torch.arange(257) % 6 - 1).tolist())
    return dict(dtype=torch.float16, B=257, H=255, N=3, D=32, causal=True, lens=lens, seed=65535, k=2)


def forward_cases():
    return [dict(dtype=dt, B=2, H=2, N=N, D=D, lens=lens, seed=s, k=1)
            for s, (dt, N, D, lens) in enumerate([(torch.float16, 200, 64, None), (torch.bfloat16, 200, 128, None),
                                                  (torch.float16, 333, 96, (333, 70)),
                                                  (torch.bfloat16, 129, 32, (1, 100))])]
