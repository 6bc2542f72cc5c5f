"""Exact and bounded answers for the attention softmax itself, shared by every mode (dense, FFPA, packed, KV-cache decode,
append); used by test_gpu_attention_graded.py and proved on the CPU in test_attention_graded_cpu.py.  exact_attention.py
makes every P 0 or 1; here the weights are fractional and the running max moves.

Graded weights.  The launcher forms scale_log2 = scale * 1.4426950408889634f in fp32.  For scale = fp32(ln 2) * 2^-k that
product is exactly 2^-k (scale_exact asserts it).  Q row r is 2^k * e_c and column c of K holds small integers g_c(j), the
column's *profile*, so the score times scale_log2 is exactly g_c(j), fmaf(s, scale_log2, -max) is the integer g - max and
P = 2^(g - max) is exact in fp16 and bf16.  With grades in [0, W], V integers in [-8, 8] and W + log2(keys) + 4 <= 24,
every partial sum of o and l at every running max is an integer multiple of 2^-W below 2^(24 - W): fp32 holds it exactly
whatever the tile size and the order of summation (window asserts the condition, expected asserts the sums).  Two more
levels sit outside the window: FAR = -256, whose weight is exactly 0 next to a graded key whichever is seen first, and
DECOY = 250, put on keys a row must not see: a max moved by 250 flushes every weight of the row to 0.  (A max that is too
high by a small amount scales o and l alike and cannot be seen in O; only a decoy that underflows P can.)

Expected value of a row that sees keys S of its column: m = max g, w_j = dtype(2^(g_j - m)), o = sum w_j V_j, l = sum w_j in
fp64, both asserted to be fp32 values, O = dtype(fp32(o) * fp32(1 / fp32(l))), the kernel's o * (1.f / l); no key: O = 0.

Fractional weights.  Grades in eighths, max on key 0 so alpha is 0 once and 1 afterwards: P = dtype(2^(-i / 8)) is a rounded,
not a representable, number, and ex2.approx's 2^-22 cannot move it because fractional_grades keeps only eighths whose power
sits 2^-16 or more (relative) from a rounding boundary and from a representable value.  This is the case that tells a
truncating pack from a rounding one, and a row sum of unrounded P from one of rounded P, bit for bit.

Constant V (const_v).  V[:, d] = c_d gives O[:, d] = c_d * sum(P) / l; l sums the P the tensor core multiplied, so o and
l differ by fp32 summation order only and O == c_d exactly while keys <= CONST_V_MAX_KEYS.

fp64 bound (reference, bound).  For random inputs, O against the exact fp64 softmax and against the ideal 16-bit-P model.

emulate() is the kernel's loop in numpy fp32, with the mutations the tests must reject."""
from __future__ import annotations

import math

import numpy as np
import torch

from exact_attention import values

LN2_F32 = 0.6931471824645996          # fp32(ln 2)
LOG2E_F32 = 1.4426950408889634        # the launcher's constant, rounded to fp32 when it multiplies
FAR, DECOY = -256, 250
# fp32 roundings of a row: one per 16-key wgmma step into o, one per key pair per thread into l, 1 / l and the product:
# relative keys * 2^-26 + 2^-22 at most, which must stay below half an ulp of the dtype at a power of two from below.
CONST_V_MAX_KEYS = {torch.float16: 4096, torch.bfloat16: 32768}
U_P = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}   # unit roundoff of P


def scale_exact(k: int) -> float:
    """The softmax scale whose fp32 product with log2(e) is exactly 2^-k."""
    s = LN2_F32 * 2.0 ** -k
    assert np.float32(s) == s and np.float32(s) * np.float32(LOG2E_F32) == np.float32(2.0 ** -k)
    return s


def window(keys: int) -> int:
    """The largest spread W <= 14 (no fp16 P subnormal) with W + log2(keys) + 4 <= 24."""
    W = min(14, 24 - 4 - max(1, math.ceil(math.log2(max(keys, 2)))))
    assert W >= 2, "too many keys (%d) for exact fp32 sums" % keys
    return W


def profile_names(edges):
    """The profiles, in column order; columns past the list repeat it with other random draws."""
    peaks = [e for e in edges if e > 0 and e % 64 in (0, 63)][:4]
    cliffs = [e for e in edges if e in (16, 64, 128, 129, 192, 512)]
    return (["asc1", "asc2", "asc3", "ascmix", "desc1", "desc3", "mid", "last", "saw", "rand", "far_first", "far_last",
             "far_mix", "islands", "decoy"] + ["peak%d" % e for e in peaks] + ["cliff%d" % e for e in cliffs])


def grades(nb, L, last, D, W, edges, g, lo=0):
    """int16 [nb, L, D]: column c of block b holds profile names[(c - lo) % len(names)] over the block's L key slots, of
    which [0, last[b]] are valid (a row may see fewer).  Tile edges are multiples of 64, so a staircase steps at every
    tile boundary of the 64-key (FFPA) and the 128-key configurations.
      asc1-3    min(W, s * tile): the max rises by s at every tile until it reaches W (alpha = 2^-s)
      ascmix    the same with a period-4 dip inside the tile
      desc1, 3  max(0, W - s * tile): alpha = 1 throughout, P shrinks
      mid       W on the middle valid key, below W elsewhere;  last: W on the last valid key
      peakE     W on key E (first and last keys of tiles, from `edges`)
      saw       j mod (W + 1);  rand: uniform in [0, W]
      far_first FAR on the first half of the valid keys, graded after;  far_last: the reverse;  far_mix: half at random
      islands   FAR but for 16 keys at W from key 2 and 8 keys at W - 1 in the last valid 128-key tile
      decoy     DECOY on the key after the last valid one
      cliffE    DECOY on key E: rows that stop before E must not see it, rows that reach it return V[E]"""
    dev = last.device
    names = profile_names(edges)
    j = torch.arange(L, device=dev).view(1, L)
    last = last.view(nb, 1).long()
    tile = j // 64

    def rnd(hi):
        return torch.randint(0, hi + 1, (nb, L), generator=g, device=dev)

    def spike(key, top, base):
        return torch.where(j == key, torch.full_like(base, top), base)

    out = torch.zeros(nb, L, D, dtype=torch.int16, device=dev)
    for c in range(lo, D):
        name = names[(c - lo) % len(names)]
        if name.startswith("asc"):
            x = (tile * int(name[3] if name[3].isdigit() else 2)).clamp(max=W).expand(nb, L)
            if name == "ascmix":
                x = (x - (j * 7) % 4).clamp(min=0)
        elif name.startswith("desc"):
            x = (W - tile * int(name[4])).clamp(min=0).expand(nb, L)
        elif name == "mid":
            x = spike((last + 1) // 2, W, rnd(W - 1))
        elif name == "last":
            x = spike(last, W, rnd(W - 1))
        elif name.startswith("peak"):
            x = spike(int(name[4:]), W, rnd(W - 1))
        elif name == "saw":
            x = (j % (W + 1)).expand(nb, L)
        elif name == "rand":
            x = rnd(W)
        elif name in ("far_first", "far_last"):
            first = j < (last + 1) // 2
            x = torch.where(first == (name == "far_first"), torch.full((1, 1), FAR, device=dev), rnd(W))
        elif name == "far_mix":
            x = torch.where(rnd(1) == 0, torch.full((1, 1), FAR, device=dev), rnd(W))
        elif name == "islands":
            t2 = (last // 128) * 128
            x = torch.full((nb, L), FAR, device=dev)
            x = torch.where((j >= 2) & (j < 18), torch.full_like(x, W), x)
            x = torch.where((t2 >= 128) & (j >= t2) & (j < t2 + 8) & (j <= last), torch.full_like(x, W - 1), x)
        elif name == "decoy":
            x = spike(last + 1, DECOY, rnd(W))
        else:
            x = spike(int(name[5:]), DECOY, rnd(W))
        out[:, :, c] = x.to(torch.int16)
    return out


def fractional_grades(dtype):
    """The i in 1..8 for which dtype(2^(-i / 8)) is a safe rounded value: 2^-16 or more (relative) from the rounding
    boundary, and 2^-16 or more from the nearest representable value (so truncation and rounding differ)."""
    mant = 11 if dtype == torch.float16 else 8
    keep = []
    for i in range(1, 9):
        x = 2.0 ** (-i / 8.0) * 2.0 ** mant        # in [2^(mant-1), 2^mant): integers are the representable values
        frac = x - math.floor(x)
        if min(abs(frac - 0.5), frac, 1 - frac) * 2.0 ** -mant >= 2.0 ** -16 and frac > 0.5:
            keep.append(i)
    return keep


def columns(R, D, edges, g, device, lo=0, special=0.3):
    """The profile column of each row: uniform over [lo, D), but `special` of the rows take a decoy or cliff column."""
    names = profile_names(edges)
    sp = torch.tensor([c for c in range(lo, D) if names[(c - lo) % len(names)][:5] in ("decoy", "cliff")], device=device)
    cols = lo + torch.randint(0, D - lo, (R,), generator=g, device=device)
    pick = sp[torch.randint(0, sp.numel(), (R,), generator=g, device=device)]
    return torch.where(torch.rand(R, generator=g, device=device) < special, pick, cols)


def expected(G, V, blk, n, col, dtype, bn=None, unit=1.0):
    """(O [R, D] in dtype, info) for rows that see keys [0, n[r]) of block blk[r] and read column col[r]; G [nb, L, D]
    grades (in units of `unit`), V [nb, L, D].  With `bn`, P is rounded relative to the running max after its bn-key tile
    (as the kernel does) instead of the final max; the two differ only when some P is not representable.  info: m, l, o
    (fp64) and `decoyed`, rows whose next key slot holds a grade above their max."""
    dev = V.device
    blk, n, col = (t.to(dev).long().view(-1) for t in (blk, n, col))
    R, L, D = blk.numel(), G.size(1), V.size(2)
    g = G[blk, :, col].double() * unit                                       # [R, L]
    j = torch.arange(L, device=dev).view(1, L)
    vis = j < n.view(-1, 1)
    nxt = g.gather(1, n.clamp(max=L - 1).view(-1, 1)).view(-1)
    g = torch.where(vis, g, torch.full_like(g, float("-inf")))
    m = g.max(1).values if L else torch.full((R,), float("-inf"), device=dev, dtype=torch.float64)
    ref = m.view(-1, 1)
    if bn is not None:
        pad = (-L) % bn
        gt = torch.nn.functional.pad(g, (0, pad), value=float("-inf")).view(R, -1, bn).max(2).values.cummax(1).values
        ref = gt.repeat_interleave(bn, 1)[:, :L]
    w = torch.exp2(g - ref).to(dtype).double() * torch.exp2(ref - m.view(-1, 1))
    w = torch.where(vis & (ref > float("-inf")), w, torch.zeros_like(w))
    l = w.sum(1)
    o = torch.zeros(R, D, dtype=torch.float64, device=dev)
    order = torch.argsort(blk, stable=True)
    ids, counts = torch.unique_consecutive(blk[order], return_counts=True)
    at = 0
    for b, cnt in zip(ids.tolist(), counts.tolist()):
        rows = order[at:at + cnt]
        at += cnt
        top = int(n[rows].max())
        o[rows] = w[rows, :top] @ V[b, :top].double()
    assert bool((o.float().double() == o).all()) and bool((l.float().double() == l).all()), \
        "a row's sums are not fp32 values: the window condition is broken"
    lf = l.float()
    inv = torch.where(lf > 0, torch.ones_like(lf) / lf.clamp(min=1e-30), torch.zeros_like(lf))
    decoyed = (n > 0) & (n < L) & (nxt > m)
    return (o.float() * inv.view(-1, 1)).to(dtype), dict(m=m, l=l, o=o, decoyed=decoyed)


def describe(G, blk, n, col, want, got, info, edges, W, lo=0, rows=4):
    """The first failing rows as text: row, block, column, profile, visible keys, max, and expected / got in units of 2^-W."""
    names = profile_names(edges)
    bad = ((want != got).any(1) | torch.isnan(got.float()).any(1)).nonzero().view(-1)[:rows].tolist()
    lines = []
    for r in bad:
        c = int(col[r])
        d = int((want[r] != got[r]).nonzero()[0])
        lines.append("row %d block %d column %d (%s) sees %d keys, max %s, l %s, O[%d] expected %s got %s (x 2^-%d)" % (
            r, int(blk[r]), c, names[(c - lo) % len(names)], int(n[r]), float(info["m"][r]), float(info["l"][r]), d,
            float(want[r, d]) * 2.0 ** W, float(got[r, d]) * 2.0 ** W, W))
    return "; ".join(lines)


def ulp(x: torch.Tensor, dtype) -> torch.Tensor:
    """One ulp of dtype at |x| (the subnormal spacing below the smallest normal)."""
    mant, emin = (10, -14) if dtype == torch.float16 else (7, -126)
    e = torch.floor(torch.log2(x.double().abs().clamp(min=2.0 ** emin)))
    return torch.pow(2.0, e - mant)


def subnormal_case(device):
    """The fp16 case of subnormal and vanishing P (test_subnormal_and_vanishing_fp16_weights_by_running_max): one block of
    256 keys, (G, V, n, cols, raw scores [R, L]) at scale_log2 = 1."""
    g = torch.Generator(device=device).manual_seed(11)
    L, D, R = 256, 64, 128
    G = torch.zeros(1, L, D, dtype=torch.int16, device=device)
    spread = torch.tensor([15, 16, 17, 18, 19, 20, 21, 22, 23, 25, 26, 27, 30], device=device)
    G[0, 128:] = (26 - spread[torch.randint(0, spread.numel(), (128, D), generator=g, device=device)]).to(torch.int16)
    G[0, 128 + torch.arange(D, device=device) % D, torch.arange(D, device=device)] = 26
    V = values(L, D, torch.float16, g, device).view(1, L, D)
    V[0, 128:128 + D] = 0                      # the rows of the max keys
    cols = torch.arange(R, device=device) % D
    n = torch.where(torch.arange(R, device=device) % 4 == 3, 128, 256)
    s = G[0][:, cols].t().float()
    return G, V, n, cols, (s.cpu().numpy() if device == "cpu" else s)


# ------------------------------------------------------------------------------------------------ constant V
def const_v(shape, kind, dtype, device):
    """V of `shape` [..., D] with V[..., d] = c_d: all ones, or the integers d % 17 - 8.  Returns (V, c [D])."""
    D = shape[-1]
    c = torch.ones(D, device=device) if kind == "ones" else (torch.arange(D, device=device) % 17 - 8).float()
    return c.to(dtype).expand(shape).contiguous(), c.to(dtype)


def check_const_v(o, c, seen, keys, dtype):
    """O [R, D] must be c in every row that sees a key and 0 in the others; returns the number of wrong rows and the
    largest deviation."""
    assert keys <= CONST_V_MAX_KEYS[dtype], "%d keys: fp32 summation order could show in %s" % (keys, dtype)
    want = torch.where(seen.view(-1, 1), c.view(1, -1).expand(o.shape), torch.zeros_like(o))
    wrong = (o != want).any(1) | torch.isnan(o.float()).any(1)
    return int(wrong.sum()), float((o.float() - want.float()).abs().nan_to_num(nan=float("inf")).max()) if o.numel() else 0.0


# ------------------------------------------------------------------------------------------------ fp64 reference and bound
def reference(q, k, v, n, scale, dtype):
    """One block in fp64: q [R, D], k / v [L, D], row r sees keys [0, n[r]).  Returns O64, O_model (weights rounded to dtype
    relative to the row's final max), A = sum p |v| / sum p, T = the largest sum_d |q_d k_jd| * scale * log2(e) of a row
    (what the rounding of a score's exponent scales with) and the rows' tile counts at 64 keys a tile."""
    q, k, v = q.double(), k.double(), v.double()
    L = k.size(0)
    x = (q @ k.t()) * (scale * LOG2E_F32)
    vis = torch.arange(L, device=q.device).view(1, L) < n.view(-1, 1)
    x = torch.where(vis, x, torch.full_like(x, float("-inf")))
    m = x.max(1, keepdim=True).values
    p = torch.where(vis, torch.exp2(x - m), torch.zeros_like(x))
    pm = p.to(dtype).double()
    den, denm = p.sum(1, keepdim=True).clamp(min=1e-300), pm.sum(1, keepdim=True).clamp(min=1e-300)
    T = (torch.where(vis, q.abs() @ k.abs().t(), torch.zeros_like(x)) * (scale * LOG2E_F32)).max(1).values
    return (p @ v) / den, (pm @ v) / denm, (p @ v.abs()) / den, T, (n + 63) // 64


def bound(o64, A, T, tiles, D, dtype):
    """Elementwise bound on |O - O64|: the first-order effect of a relative error e in every weight is at most 2 e A, with
    e = u_P (P rounded to dtype) + ln 2 * 2^-23 * (D / 16 + 3) * T (fp32 score: one rounding per 16-column wgmma step,
    the scale product and the fma) + 2^-22 * (1 + tiles) (ex2.approx in P and in each tile's alpha) + 2^-20 (fp32 sums of
    o and l); then half an ulp of the dtype at the result for the store."""
    e = U_P[dtype] + math.log(2) * 2.0 ** -23 * (D / 16 + 3) * T + 2.0 ** -22 * (1 + tiles.double()) + 2.0 ** -20
    first = 2 * e.view(-1, 1) * A
    return first + ulp(o64.abs() + first, dtype) / 2


# ------------------------------------------------------------------------------------------------ the kernel's loop
def round_to(x, dtype, trunc=False):
    """fp32 array -> the nearest (ties to even) or the next-toward-zero fp16 / bf16 value, as fp32."""
    x = np.asarray(x, dtype=np.float32)
    if dtype == torch.float16:
        r = x.astype(np.float16)
        if trunc:
            over = np.abs(r.astype(np.float32)) > np.abs(x)
            r = np.where(over, np.nextafter(r, np.float16(0)), r)
        return r.astype(np.float32)
    b = x.view(np.uint32).astype(np.uint64)
    if not trunc:
        b = b + 0x7FFF + ((b >> 16) & 1)
    return (b & 0xFFFF0000).astype(np.uint32).view(np.float32)


MUTATIONS = ["rowsum_unrounded", "trunc", "alpha_skips_l", "alpha_swapped", "decoy_moves_max", "no_renorm"]


def emulate(s, v, n, scale_log2, dtype, bn, mut="", splits=1):
    """The kernel's online softmax in fp32: s [R, L] raw scores, v [L, D], row r sees keys [0, n[r]).  Tiles of bn keys,
    `splits` contiguous tile ranges merged as attn_combine_kernel does.  `mut` is one of MUTATIONS or ""."""
    f = np.float32
    s, v, sl = np.asarray(s, f), np.asarray(v, f), f(scale_log2)
    (R, L), D = s.shape, v.shape[1]
    nt = -(-L // bn)
    parts = []
    with np.errstate(all="ignore"):
        for sp in range(splits):
            m, l, o = np.full(R, -np.inf, f), np.zeros(R, f), np.zeros((R, D), f)
            for t in range(sp * nt // splits, (sp + 1) * nt // splits):
                j = np.arange(t * bn, min(L, (t + 1) * bn))
                x = np.where(j[None] < n[:, None], s[:, j], f(-np.inf))
                xm = np.where(j[None] <= n[:, None], s[:, j], f(-np.inf)) if mut == "decoy_moves_max" else x
                m_new = np.maximum(m, xm.max(1) * sl)
                mu = np.where(m_new == -np.inf, f(0), m_new)
                alpha = np.where(m == -np.inf, f(0), np.exp2(m - mu))
                if mut == "alpha_swapped":
                    alpha = alpha[np.arange(R) ^ 8]                    # the thread's other row
                m = m_new
                if mut != "alpha_skips_l":
                    l = l * alpha
                p = np.exp2((x.astype(np.float64) * np.float64(sl) - mu[:, None]).astype(f))
                p[p < f(2.0 ** -126)] = 0                             # ex2.approx.ftz
                pr = round_to(p, dtype, trunc=mut == "trunc")
                l = l + (p if mut == "rowsum_unrounded" else pr).sum(1, dtype=f)
                o = o * alpha[:, None] + pr @ v[j]
            inv = np.where(l > 0, f(1) / l, f(0))
            parts.append((o * inv[:, None], np.where(l > 0, m + np.log2(l), f(-np.inf)), l))
        if splits == 1:
            return round_to(parts[0][0], dtype)
        lse = np.stack([p[1] for p in parts])
        mx = lse.max(0)
        x, den = np.zeros((R, D), f), np.zeros(R, f)
        for part, ls, _ in parts:
            w = np.where(mx == -np.inf, f(0), np.exp2(ls - mx))
            w[w < f(2.0 ** -126)] = 0
            x, den = x + w[:, None] * part, den + w
        inv = np.where(den > 0, f(1) / den, f(0))
        if mut == "no_renorm":
            inv = np.where(den > 0, f(1), f(0))
        return round_to(x * inv[:, None], dtype)
