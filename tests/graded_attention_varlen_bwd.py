"""Exact answers for the packed attention backward (b200k_fa2_bwd_varlen, ops.fa2_bwd_varlen, ops.attention_varlen), used
by test_gpu_attention_varlen_bwd_graded.py and proved on the CPU in test_attention_varlen_bwd_graded_cpu.py.  Within a
sequence the inputs are graded_attention_bwd.py's: Q rows 2^k e_c, grades beta + [0, W] with beta per (sequence, K/V
head), lse exact for an integer or eighth t, normal, round and frac rows, integer V and O.  What is added is what the
packed layout can get wrong:
  groups      the G query heads of a K/V head choose their columns, t and row kinds independently, so dK / dV of a key
              sum nonzero dS~ / P~ from several heads; the fp32 window is checked on the group sum (G * Lq terms);
  cliffs      (causal) row r sees key j iff j <= r + shift, shift = Lk - Lq.  DECOY on key E of a cliff column, which row
              E - shift - 1 (the last row that must not see E) reads; E runs over CLIFFS and over the keys that put that
              row on a 64-row edge (CLIFF_ROWS), so both the key and the row sit on tile edges;
  no key      (causal, Lq > Lk) rows r < Lq - Lk get lse = -inf, as the forward writes it, and dQ = +0: the prep must
              turn that lse into lse2 = +inf;
  boundaries  key Lk of sequence b is physically the next token: the key 0 of the next sequence that has keys, which
              holds DECOY in the two boundary columns of b's parity (sequences with keys alternate parity).  Rows of b
              read those columns, rows of the next sequence never do.  Keys past cu_k[B] hold DECOY in every column;
  outside     tokens before cu_q[0] / cu_k[0] and past cu_q[B] hold finite junk Q, dO, O and lse = JUNK_LSE, so a kernel
              that took their lse2 in place of the +inf of padding gets P = 2^144 = inf against a zeroed row: NaN.
closed_form() is graded_attention_bwd.closed_form_core one sequence at a time, every exactness assertion included;
emulate_bwd() is the three kernels' fp32 arithmetic at tile granularity, with the mutations the tests must reject."""
from __future__ import annotations

import numpy as np
import torch

import attention_ref as ar
import graded_attention as ga
import graded_attention_bwd as gb

LOG2E_F32 = ga.LOG2E_F32
DECOY = ga.DECOY
JUNK_LSE = -100.0
BOUNDARY = ([1, 2], [3, 4])           # the boundary columns of each parity
CLIFF0 = 5                            # cliff columns from here; column 0 and those after the cliffs are plain
CLIFFS = [63, 64, 65, 127, 128, 129, 191, 192, 255, 256, 511, 512, 513, 999]
CLIFF_ROWS = [63, 64, 127, 128, 191, 192]


# ------------------------------------------------------------------------------------------------ inputs
def make_case(dtype, D, causal, H, H_kv, lens, pre=(0, 0), post=(0, 0), seed=0, k=0, W=3, nnz=2, frac_rows=2, ncol=None,
              push=0, **_):
    """One packed call on the CPU: q, o, do dtype [total_q, H, D], k, v dtype [total_k, H_kv, D], lse fp32 [total_q, H],
    cu_q, cu_k int32 [B + 1], max_q, max_k, scale, causal, and per (token, head) of q: col (grade column), t (lse2; NaN
    where the row sees no key or lies outside every sequence) and kind (0 normal, 1 round, 2 frac).  lens: (Lq, Lk) per
    sequence; pre / post: (query, key) tokens before cu[0] and after cu[B].  The long case's knobs: ncol, rows read only
    the first ncol plain columns, so a column's dK sums more rows; push, O = -push sign(dO) where a normal row's dO is
    nonzero, so Delta = -push * nnz and dP - Delta lies in [0, 2 push nnz]."""
    g = torch.Generator().manual_seed(seed)
    ri = lambda lo, hi, shape: torch.randint(lo, hi, shape, generator=g)  # noqa: E731
    G = H // H_kv
    cu_q = np.cumsum([pre[0]] + [a for a, _ in lens]).tolist()
    cu_k = np.cumsum([pre[1]] + [b for _, b in lens]).tolist()
    Tq, Tk = cu_q[-1] + post[0], cu_k[-1] + post[1]
    K = ri(-4, 5, (Tk, H_kv, D))                                   # junk before cu_k[0]
    K[cu_k[-1]:] = DECOY
    V = ri(-8, 9, (Tk, H_kv, D))
    V[..., 0] = 1
    Q, dO, O = ri(-2, 3, (Tq, H, D)).double(), ri(-2, 3, (Tq, H, D)), ri(-8, 9, (Tq, H, D))   # junk outside
    lse = torch.full((Tq, H), JUNK_LSE)
    col = torch.full((Tq, H), -1, dtype=torch.long)
    t = torch.full((Tq, H), float("nan"), dtype=torch.float64)
    kind = torch.zeros(Tq, H, dtype=torch.long)
    fr = torch.tensor(ga.fractional_grades(dtype))
    par = np.cumsum([0] + [int(b > 0) for _, b in lens]) % 2       # parity of each sequence among those with keys
    for b, (Lq, Lk) in enumerate(lens):
        q0, k0, shift = cu_q[b], cu_k[b], Lk - Lq
        beta = ri(-4, 5, (H_kv,))
        K[k0:k0 + Lk] = beta.view(1, H_kv, 1) + ri(0, W + 1, (Lk, H_kv, D))
        cl = []
        if causal:
            cand = sorted(set(CLIFFS) | {r + shift + 1 for r in CLIFF_ROWS})
            cl = [E for E in cand if 1 <= E < Lk and 0 <= E - shift - 1 < Lq][:D - 8]
        for i, E in enumerate(cl):
            K[k0 + E, :, CLIFF0 + i] = DECOY
        if Lq == 0:
            continue
        rows = torch.arange(Lq)
        n = (rows + shift + 1).clamp(0, max(Lk, 0)) if causal else torch.full((Lq,), Lk)
        plain = torch.tensor([0] + list(range(CLIFF0 + len(cl), D)))[:ncol]
        allowed = torch.cat([plain, torch.tensor(BOUNDARY[par[b]] if ncol is None else []).long(),
                             torch.arange(CLIFF0, CLIFF0 + len(cl))])
        c = allowed[ri(0, allowed.numel(), (Lq, H))]
        e_of = torch.full((D,), Lk + 1)
        e_of[CLIFF0:CLIFF0 + len(cl)] = torch.tensor(cl, dtype=torch.long)
        late = e_of[c] <= (rows + shift).view(Lq, 1)                             # would see its column's decoy
        c = torch.where(late, plain[ri(0, plain.numel(), (Lq, H))], c)
        for i, E in enumerate(cl):                                                # the last row before E reads it
            c[E - shift - 1] = CLIFF0 + i
        c[Lq - 1, ::G] = BOUNDARY[par[b]][0]                                      # the last row sees key Lk - 1
        kd = torch.zeros(Lq, H, dtype=torch.long)
        kd[(n <= gb.ROUND_KEYS) & (n > 0)] = 1
        F = min(frac_rows, Lq // 2)
        if F:
            pick = torch.rand(Lq, H, generator=g).argsort(0)[:F]
            kd.scatter_(0, pick, torch.where(n[pick] > 0, 2, kd.gather(0, pick)))
        tt = beta[torch.arange(H) // G].view(1, H) + W + ri(0, 2, (Lq, H))
        eighths, lv = gb.exact_lse_of(8 * tt + torch.where(kd == 2, fr[ri(0, fr.numel(), (Lq, H))], 0))
        seen = (n > 0).view(Lq, 1)
        d_o, o = gb.row_values(kd.view(-1), D, dtype, nnz, ri)
        if push:
            o = torch.where((kd.view(-1, 1) == 0) & (d_o != 0), -push * d_o.sign(), o)
        Q[q0:q0 + Lq] = torch.zeros(Lq, H, D, dtype=torch.float64).scatter_(2, c.view(Lq, H, 1), 2.0 ** k)
        dO[q0:q0 + Lq], O[q0:q0 + Lq] = d_o.view(Lq, H, D), o.view(Lq, H, D)
        lse[q0:q0 + Lq] = torch.where(seen, lv.view(Lq, H), float("-inf"))
        col[q0:q0 + Lq], kind[q0:q0 + Lq] = c, kd
        t[q0:q0 + Lq] = torch.where(seen, eighths / 8.0, float("nan"))
    for b, (_, Lk) in enumerate(lens):                                            # after every sequence's grades
        if Lk and cu_k[b + 1] < cu_k[-1]:
            K[cu_k[b + 1], :, BOUNDARY[par[b]]] = DECOY
    out = gb._pack(dtype, (Tq, H, D), dict(q=Q, o=O, do=dO))
    out.update(gb._pack(dtype, (Tk, H_kv, D), dict(k=K, v=V)))
    out.update(lse=lse.float(), cu_q=torch.tensor(cu_q, dtype=torch.int32), cu_k=torch.tensor(cu_k, dtype=torch.int32),
               max_q=max(1, max(a for a, _ in lens)), max_k=max(1, max(b for _, b in lens)), scale=ga.scale_exact(k),
               causal=causal, col=col, t=t, kind=kind)
    return out


def make_forward_case(dtype, lens, H, H_kv, D, seed=0, k=1, **_):
    """The consistent packed case (non-causal, GQA), whose O and lse come from fa2_fwd_varlen: the keys of each
    (sequence, K/V head) are graded_attention_bwd.forward_keys', so a row that reads column c sees weights summing to a
    power of two and its lse is t = top of c exactly (as fp32(t * 0.6931472f)).  make_case's dict without o and lse;
    t is -inf for rows of a sequence without keys."""
    g = torch.Generator().manual_seed(seed)
    G = H // H_kv
    cu_q = np.cumsum([0] + [a for a, _ in lens]).tolist()
    cu_k = np.cumsum([0] + [b for _, b in lens]).tolist()
    K = torch.zeros(cu_k[-1], H_kv, D, dtype=torch.long)
    col = torch.randint(0, D, (cu_q[-1], H), generator=g)
    t = torch.full((cu_q[-1], H), float("-inf"), dtype=torch.float64)
    for b, (Lq, Lk) in enumerate(lens):
        if Lk == 0:
            continue
        kb, top = gb.forward_keys(H_kv, Lk, D, torch.full((H_kv,), Lk), g)
        K[cu_k[b]:cu_k[b + 1]] = kb.transpose(0, 1)
        c = col[cu_q[b]:cu_q[b + 1]]
        t[cu_q[b]:cu_q[b + 1]] = top[torch.arange(H) // G].t().gather(0, c).double()
    assert float(t.abs().nan_to_num(posinf=0).max()) <= 12
    Q = torch.zeros(cu_q[-1], H, D).scatter_(2, col.view(-1, H, 1), 2.0 ** k)
    V = torch.randint(-8, 9, (cu_k[-1], H_kv, D), generator=g)
    dO = torch.zeros(cu_q[-1], H, D, dtype=torch.long)
    dO.scatter_add_(2, torch.randint(0, D, (cu_q[-1], H, 2), generator=g),
                    2 * torch.randint(0, 2, (cu_q[-1], H, 2), generator=g) - 1)
    out = gb._pack(dtype, (cu_q[-1], H, D), dict(q=Q, do=dO))
    out.update(gb._pack(dtype, (cu_k[-1], H_kv, D), dict(k=K, v=V)))
    out.update(cu_q=torch.tensor(cu_q, dtype=torch.int32), cu_k=torch.tensor(cu_k, dtype=torch.int32),
               max_q=max(a for a, _ in lens), max_k=max(b for _, b in lens), scale=ga.scale_exact(k), causal=False,
               col=col, t=t, kind=torch.zeros(cu_q[-1], H, dtype=torch.long))
    return out


def forward_outputs(case):
    """(O, lse) the forward computes for make_forward_case: the weights 2^(g - t) sum to 1 (those below 2^-126 flush to
    0, as ex2.approx.ftz does), so O is the exact P V rounded once, and lse = fp32(t * 0.6931472f)."""
    q, k, v = case["q"], case["k"], case["v"]
    G = q.size(1) // k.size(1)
    sl = float(np.float32(case["scale"]) * np.float32(LOG2E_F32))
    o = torch.zeros(q.shape, dtype=torch.float64)
    for q0, q1, k0, k1 in ar.seqs(case["cu_q"], case["cu_k"]):
        if q1 > q0 and k1 > k0:
            kk, vv = (x[k0:k1].double().repeat_interleave(G, dim=1) for x in (k, v))
            x = torch.einsum("qhd,khd->hqk", q[q0:q1].double(), kk) * sl - case["t"][q0:q1].t().unsqueeze(-1)
            p = torch.where(x >= -126, torch.exp2(x), 0)     # FAR weighs exactly 0 (not 2^-260: O would be -0)
            assert torch.equal(p.sum(-1), torch.ones_like(p[..., 0])), "weights do not sum to 1"
            o[q0:q1] = torch.einsum("hqk,khd->qhd", p, vv)
    return o.to(q.dtype), gb.forward_lse(case["t"])


def lse2_of(lse):
    """What the packed prep writes: fp32(lse * fp32(log2 e)), and +inf for lse = -inf."""
    l2 = lse.float() * torch.tensor(LOG2E_F32, dtype=torch.float32, device=lse.device)
    return torch.where(lse == float("-inf"), float("inf"), l2)


# ------------------------------------------------------------------------------------------------ the closed form
def closed_form(case, rounded=True):
    """((dq, dk, dv), info): graded_attention_bwd.closed_form_core one sequence at a time on the case's device, K/V
    expanded over the group and dK / dV summed back, bottom-right causal mask; everything outside the sequences, keys of
    an empty query sequence and rows of an empty key sequence +0.  rounded=False: the fp64 gradients (as in
    closed_form_core) for comparison with attention_ref.packed_grads_given.  info: counts summed, windows maximised."""
    q, k, v, o, do = (case[n] for n in ("q", "k", "v", "o", "do"))
    H, H_kv = q.size(1), k.size(1)
    out_dt = q.dtype if rounded else torch.float64
    dq, dk, dv = (torch.zeros(t.shape, dtype=out_dt, device=q.device) for t in (q, k, v))
    l2 = lse2_of(case["lse"]).double()
    info: dict = {}
    for q0, q1, k0, k1 in ar.seqs(case["cu_q"].cpu(), case["cu_k"].cpu()):
        if q1 == q0 or k1 == k0:
            continue
        seq = lambda t, a, b: t[a:b].double().transpose(0, 1)  # noqa: E731
        (a, b, c), inf = gb.closed_form_core(
            seq(q, q0, q1), seq(k, k0, k1), seq(v, k0, k1), seq(o, q0, q1), seq(do, q0, q1), l2[q0:q1].t(),
            ar.visible(q1 - q0, k1 - k0, k1 - k0 - (q1 - q0) if case["causal"] else None, q.device), case["scale"],
            q.dtype, rounded, group=H // H_kv)
        dq[q0:q1], dk[k0:k1], dv[k0:k1] = a.transpose(0, 1), b.transpose(0, 1), c.transpose(0, 1)
        for key, val in inf.items():
            info[key] = max(info.get(key, 0), val) if key.startswith("win") else info.get(key, 0) + val
    return (dq, dk, dv), info


# ------------------------------------------------------------------------------------------------ the kernels' arithmetic
MUTATIONS = gb.MUTATIONS + ["group_first_only", "group_interleaved", "top_left", "first_tile_late", "q_tail_stats",
                            "lse_head_major", "no_key_lse", "kv_tail_len"]


def emulate_bwd(case, mut=""):
    """The three kernels in numpy fp32, (dq, dk, dv) as fp32 arrays of dtype values.
      prep   Delta = dO . O, lse2 = lse * log2 e (+inf for lse = -inf), zeros outside every sequence;
      dK/dV  per (sequence, K/V head, 64-key tile): for each query head of the group, the 64-row query tiles from
             first = max(k0 - shift, 0) / 64 (causal; else 0) to end = max(ceil(Lq / 64), first); rows past Lq read the
             next tokens with Q and dO zeroed (zero_q_tail) and row_stats' +inf / 0; keys past Lk or after a row's
             diagonal r + shift masked (S = -inf, dP = 0); P = ex2(fmaf(S, scale_log2, -lse2)) flushed below 2^-126,
             dS = P (dP - Delta), P~ and dS~ rounded; dV += P~^T dO, dK += dS~^T Q over the group; keys < Lk stored;
      dQ     per (sequence, head, 128-row tile): key tiles 0 .. min(ceil(Lk / 64), (q0 + shift + 127) / 64 + 1), K past Lk
             zeroed (zero_kv_tail), the same masks, dQ += dS~ K; rows < Lq stored;
    dQ and dK times fp32(scale), then rounded to the dtype.  `mut` is one of MUTATIONS or "": graded_attention_bwd's
    (swaps pair row r with r ^ 8 of the sequence; the length and diagonal mutations act in both kernels) and
      group_first_only   dK / dV sum only the group's first head
      group_interleaved  query head h reads K/V head h % H_kv instead of h / G (both kernels)
      top_left           the causal shift is 0 instead of Lk - Lq (both kernels)
      first_tile_late    first = ceil((k0 - shift) / 64): the partial first query tile is skipped
      q_tail_stats       rows past Lq in the dK/dV kernel take the next token's lse2 / Delta instead of +inf / 0
      lse_head_major     the row statistics are read at h * total_q + token instead of token * H + h
      no_key_lse         lse2 = lse * log2 e for lse = -inf too: 2^(-inf + inf) = NaN
      kv_tail_len        the dQ kernel's Lk (its key mask, K tail zeroing and tile count) is the next sequence's"""
    f, f64 = np.float32, np.float64
    dtype = case["q"].dtype
    Q, K, V, O, dO = (case[n].float().cpu().numpy() for n in ("q", "k", "v", "o", "do"))
    lse = case["lse"].float().cpu().numpy()
    Tq, H, D = Q.shape
    Tk, H_kv = K.shape[:2]
    G = H // H_kv
    cq, ck = case["cu_q"].tolist(), case["cu_k"].tolist()
    B, causal = len(cq) - 1, case["causal"]
    sl, s = f(f(case["scale"]) * f(LOG2E_F32)), f(case["scale"])
    off = {"causal_diag": -1, "causal_next": 1}.get(mut, 0)
    dlen = {"len_short": -1, "len_long": 1}.get(mut, 0)
    kv_of = np.arange(H) % H_kv if mut == "group_interleaved" else np.arange(H) // G
    members = [np.nonzero(kv_of == j)[0][:1 if mut == "group_first_only" else H] for j in range(H_kv)]
    dq, dk, dv = np.zeros((Tq, H, D), f), np.zeros((Tk, H_kv, D), f), np.zeros((Tk, H_kv, D), f)

    def rows_of(X, toks):  # tokens past the tensor read as zeros (TMA)
        return np.where((toks < len(X)).reshape(-1, 1, 1), X[np.minimum(toks, len(X) - 1)], f(0))

    def bmm(a, b):
        return np.matmul(a.astype(f64), b.astype(f64))

    with np.errstate(all="ignore"):
        src = O
        if mut == "delta_from_v":
            Vf, i = V.reshape(-1, D), np.arange(Tq * H)
            src = np.where((i < len(Vf))[:, None], Vf[np.minimum(i, len(Vf) - 1)], f(0)).reshape(Tq, H, D)
        Delta = (dO.astype(f64) * src).sum(-1).astype(f)
        lse2 = (lse * f(LOG2E_F32)).astype(f)
        if mut != "no_key_lse":
            lse2 = np.where(lse == -np.inf, f(np.inf), lse2)
        if mut == "lse_head_major":
            lse2, Delta = (x.reshape(H, Tq).T.copy() for x in (lse2, Delta))
        if mut in ("delta_swap", "lse2_swap"):
            x, fill = (Delta, f(0)) if mut == "delta_swap" else (lse2, f(np.inf))
            x = x.copy()
            for b in range(B):
                Lq = cq[b + 1] - cq[b]
                r = np.arange(Lq) ^ 8
                x[cq[b]:cq[b + 1]] = np.where((r < Lq)[:, None], x[cq[b] + np.minimum(r, Lq - 1)], fill)
            Delta, lse2 = (x, lse2) if mut == "delta_swap" else (Delta, x)

        def stats(q0, Lq, r, tail):
            """lse2, Delta [R, H] of rows r of the sequence at q0 (+inf, 0 past Lq)."""
            inside = r < Lq
            if tail and mut == "q_tail_stats":
                inside = q0 + r < Tq
            tok = np.minimum(q0 + r, Tq - 1)
            return (np.where(inside[:, None], lse2[tok], f(np.inf)), np.where(inside[:, None], Delta[tok], f(0)))

        def grads(S, dP, l2, dl):
            """P~, dS~ [H, R, keys] from S, dP [H, R, keys] and l2, dl [R, H]."""
            x = (S.astype(f64) * f64(sl) - l2.T[:, :, None]).astype(f)
            P = np.exp2(x.astype(f64)).astype(f)
            P[P < f(2.0 ** -126)] = 0
            dS = P * (dP - dl.T[:, :, None])
            if mut == "ds_sign":
                dS = -dS
            return ga.round_to(P, dtype, trunc=mut == "p_trunc"), ga.round_to(dS, dtype, trunc=mut == "ds_trunc")

        def scores(Qt, dOt, Kt, Vt, vis):
            """S, dP [H, R, keys] of rows Qt, dOt [R, H, D] against keys Kt, Vt [keys, H_kv, D], masked by vis."""
            S = bmm(Qt.transpose(1, 0, 2), Kt[:, kv_of].transpose(1, 2, 0)).astype(f)
            dP = bmm(dOt.transpose(1, 0, 2), Vt[:, kv_of].transpose(1, 2, 0)).astype(f)
            return np.where(vis, S, f(-np.inf)), np.where(vis, dP, f(0))

        for b in range(B):
            q0, k0, Lq, Lk = cq[b], ck[b], cq[b + 1] - cq[b], ck[b + 1] - ck[b]
            shift = 0 if mut == "top_left" else Lk - Lq
            kvl = Lk + dlen
            for t0 in range(0, Lk, 64):                                            # the dK/dV kernel
                first = 0
                if causal:
                    first = max(-(-(t0 - shift) // 64), 0) if mut == "first_tile_late" else max(t0 - shift, 0) // 64
                end = max(-(-Lq // 64), first)
                if first >= end:
                    continue
                r, keys = np.arange(first * 64, end * 64), t0 + np.arange(64)
                Qt, dOt = rows_of(Q, q0 + r), rows_of(dO, q0 + r)
                Qt[r >= Lq], dOt[r >= Lq] = 0, 0
                vis = (keys < kvl)[None, :] & ((keys[None, :] <= r[:, None] + shift + off) if causal else True)
                S, dP = scores(Qt, dOt, rows_of(K, k0 + keys), rows_of(V, k0 + keys), vis)
                Pr, dSr = grads(S, dP, *stats(q0, Lq, r, True))
                cv = bmm(Pr.transpose(0, 2, 1), dOt.transpose(1, 0, 2))                # [H, 64 keys, D]
                ckk = bmm(dSr.transpose(0, 2, 1), Qt.transpose(1, 0, 2))
                n = min(64, Lk - t0)
                for j in range(H_kv):
                    sk = ckk[members[j]].sum(0).astype(f)[:n]
                    sv = cv[members[j]].sum(0).astype(f)[:n]
                    dk[k0 + t0:k0 + t0 + n, j] = ga.round_to(sk if mut == "dk_unscaled" else sk * s, dtype)
                    dv[k0 + t0:k0 + t0 + n, j] = ga.round_to(sv * s if mut == "scale_dv" else sv, dtype)
            kvq = kvl
            if mut == "kv_tail_len":
                kvq = ck[b + 2] - ck[b + 1] if b + 1 < B else 0
            for t0 in range(0, Lq, 128):                                           # the dQ kernel
                r = np.arange(t0, min(t0 + 128, Lq))
                nt = max(-(-kvq // 64), 0)
                if causal:
                    last = t0 + shift + 127
                    nt = min(nt, 0 if last < 0 else last // 64 + 1)
                if nt == 0:
                    continue
                keys = np.arange(nt * 64)
                Kt = rows_of(K, k0 + keys)
                Kt[keys >= kvq] = 0
                vis = (keys < kvq)[None, :] & ((keys[None, :] <= r[:, None] + shift + off) if causal else True)
                S, dP = scores(rows_of(Q, q0 + r), rows_of(dO, q0 + r), Kt, rows_of(V, k0 + keys), vis)
                _, dSr = grads(S, dP, *stats(q0, Lq, r, False))
                x = bmm(dSr, Kt[:, kv_of].transpose(1, 0, 2)).astype(f).transpose(1, 0, 2)
                dq[q0 + r] = ga.round_to(x if mut == "dq_unscaled" else x * s, dtype)
    return dq, dk, dv


# ------------------------------------------------------------------------------------------------ failures
def describe(case, name, want, got, count=3):
    """The first `count` wrong elements of output `name` (dq by query token, dk / dv by key token) as text, naming the
    sequence, head, token and column."""
    want, got = want.float().cpu(), got.float().cpu()
    wrong = (want != got) | torch.isnan(got)
    cu = (case["cu_q"] if name == "dq" else case["cu_k"]).cpu().tolist()
    lines = []
    for tok, h, c in wrong.nonzero().tolist()[:count]:
        b = int(np.searchsorted(cu, tok, side="right")) - 1
        if b < 0 or b >= len(cu) - 1:
            where = "token %d (outside every sequence)" % tok
        elif name == "dq":
            where = "seq %d head %d row %d (token %d; t %s, grade column %d, kind %d)" % (
                b, h, tok - cu[b], tok, float(case["t"][tok, h]), int(case["col"][tok, h]), int(case["kind"][tok, h]))
        else:
            cq = case["cu_q"].cpu().tolist()
            G = case["q"].size(1) // case["k"].size(1)
            heads = case["col"][cq[b]:cq[b + 1], h * G:(h + 1) * G]
            readers = (heads == c).nonzero()[:6].tolist()
            where = "seq %d K/V head %d key %d of %d (token %d; (row, g) reading column %d: %s)" % (
                b, h, tok - cu[b], cu[b + 1] - cu[b], tok, c, readers)
        lines.append("%s %s, column %d: expected %r got %r" % (name, where, c, float(want[tok, h, c]),
                                                              float(got[tok, h, c])))
    return "; ".join(lines) + " (%d wrong)" % int(wrong.sum())


# ------------------------------------------------------------------------------------------------ the cases the GPU runs
DTYPES = gb.DTYPES
HEADDIMS = gb.HEADDIMS
GROUPS = [(3, 3), (4, 2), (16, 2), (6, 1)]         # (H, H_kv): G = 1, 2, 8 and MQA
# (Lq, Lk) per sequence, (query, key) tokens before cu[0], after cu[B].  Shifts 0, +-1, +-63, +-64, +-65, +936, -809;
# empty query sequences first, middle and last, empty key sequences first, middle and last.
LENSETS = [([(0, 65), (64, 64), (127, 128), (1, 64)], (3, 5), (7, 64)),
           ([(129, 128), (65, 0), (127, 64), (63, 128)], (0, 0), (40, 0)),
           ([(65, 129), (0, 127), (192, 128), (1, 1)], (64, 1), (0, 17)),
           ([(129, 64), (191, 192), (63, 0)], (1, 0), (100, 3)),
           ([(192, 191), (64, 1000), (0, 63)], (5, 9), (65, 0)),
           ([(1000, 191), (128, 65), (64, 0), (191, 191)], (2, 2), (1, 1)),
           ([(1, 0), (65, 65), (63, 127), (128, 192)], (0, 3), (130, 2))]


def cases():
    """Every (dtype, D, mask, length set) once, the group rotating with them; k (Q = 2^k) in 0..2."""
    out = []
    for di, dtype in enumerate(DTYPES):
        for Di, D in enumerate(HEADDIMS):
            for causal in (False, True):
                for li, (lens, pre, post) in enumerate(LENSETS):
                    H, H_kv = GROUPS[(di + Di + 2 * causal + li) % 4]
                    out.append(dict(dtype=dtype, D=D, causal=causal, H=H, H_kv=H_kv, lens=lens, pre=pre, post=post,
                                    seed=1000 * di + 100 * Di + 10 * causal + li, k=(Di + li) % 3))
    return out


def long_cases():
    """One 2048-key sequence at G = 8 per dtype, whose dK sums come within a factor of two of the fp32 window."""
    return [dict(dtype=dt, D=32, causal=False, H=8, H_kv=1, lens=[(2048, 2048)], pre=(1, 0), post=(3, 1), seed=7 + i,
                 k=1, W=3, nnz=28, ncol=1, push=18, name="long") for i, dt in enumerate(DTYPES)]


def all_cases():
    return cases() + long_cases()


def grid_case():
    """B * H = 65535 (B = 257, H = 255, H_kv = 15): the largest dQ grid z and the most dK/dV CTAs, causal, lengths 0 - 5."""
    lens = [(b % 6, (5 * b + 2) % 6) for b in range(257)]
    return dict(dtype=torch.float16, D=32, causal=True, H=255, H_kv=15, lens=lens, pre=(2, 1), post=(3, 2), seed=65535,
                k=2, name="grid65535")


def big_core():
    """The graded sequences of the call past 2^31 elements (H = 16, H_kv = 2, D = 128): the first is placed across
    element 2^31 of Q / dQ, the second last."""
    return dict(dtype=torch.bfloat16, D=128, causal=True, H=16, H_kv=2, lens=[(1000, 700), (129, 300)], seed=31, k=1,
                name="past2_31")


def forward_cases():
    return [dict(dtype=dt, lens=lens, H=H, H_kv=H_kv, D=D, seed=s, k=1)
            for s, (dt, lens, H, H_kv, D) in enumerate([
                (torch.float16, [(200, 333), (1, 64), (129, 65), (50, 0), (64, 1)], 8, 2, 64),
                (torch.bfloat16, [(65, 1000), (300, 129)], 6, 1, 128),
                (torch.float16, [(333, 70), (0, 40), (128, 128)], 4, 4, 96),
                (torch.bfloat16, [(100, 2), (70, 191)], 16, 2, 32)])]


def case_id(c):
    if "name" in c:
        return "%s-%s" % (c["name"], "f16" if c["dtype"] == torch.float16 else "bf16")
    return "%s-D%d-%s-G%s-L%d" % ("f16" if c["dtype"] == torch.float16 else "bf16", c["D"],
                                  "causal" if c["causal"] else "full",
                                  "MQA" if c["H_kv"] == 1 else str(c["H"] // c["H_kv"]),
                                  [lens for lens, _, _ in LENSETS].index(c["lens"]))
