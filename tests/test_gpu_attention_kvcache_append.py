"""GPU: KV-cache decode with append and rotary (ops.fa2_fwd_kvcache with k / v / rotary_cos / rotary_sin).  Without
rotary the call has the bits of the two-step path (rows scattered into the cache, then fa2_fwd_kvcache on lengths +
L_new); with rotary, the cache rows and O match the CPU reference (kvcache_append_oracle.py) and Q and K go through the
same arithmetic.  Then isolation and memory safety with poisoned pages and guard buffers, overflow past the capacity,
CUDA graph replay of a decode loop, and a full-size run."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))  # the oracles sit next to this file
import attention_ref as ar  # noqa: E402
import kvcache_append_oracle as ko  # noqa: E402
import kvcache_oracle  # noqa: E402

pytestmark = pytest.mark.gpu
MANTISSA = {torch.float16: 10, torch.bfloat16: 7}


def _ops():
    from b200k import ops

    return ops


def _rand(*shape, dtype=torch.float16):
    return torch.randn(*shape, device="cuda").to(dtype)


def _caches(kind, B, S, H_kv, D, dtype, seed):
    """(k_cache, v_cache, table) of `kind` ("contig" or a page size) holding random keys, the pages under a shuffled
    table with spare pages."""
    torch.manual_seed(seed)
    kc, vc = _rand(B, S, H_kv, D, dtype=dtype), _rand(B, S, H_kv, D, dtype=dtype)
    if kind == "contig":
        return kc, vc, None
    kp, vp, table, _ = kvcache_oracle.paged_copy(kc, vc, kind, seed=seed, fill=lambda shape: torch.randn(shape))
    return kp, vp, table


def _rope(n, rd, dtype, base=10000.0):
    """cos / sin [n, rd / 2] for positions 0 .. n - 1, computed in fp32 on the GPU and rounded to dtype."""
    inv = base ** (-torch.arange(0, rd, 2, device="cuda", dtype=torch.float32) / rd)
    ang = torch.arange(n, device="cuda", dtype=torch.float32).view(n, 1) * inv.view(1, -1)
    return ang.cos().to(dtype), ang.sin().to(dtype)


def _bits(t):
    return t.contiguous().view(torch.int16)


def _lens(lens):
    return torch.tensor(lens, dtype=torch.int32, device="cuda")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("Lq,L_new", [(1, 1), (3, 3), (16, 16), (2, 5)])
@pytest.mark.parametrize("kind", ["contig", 16, 64, 256])
def test_no_rotary_same_bits_as_scatter_then_decode(kind, Lq, L_new, causal, dtype):
    """Both sides of the split rule: 7 sequences x 2 K/V heads are split, 7 x 16 fill the SMs and run unsplit."""
    ops = _ops()
    S, D = 512, 64
    lens_l = [0, 15, 16, 127, 128, 255, S - L_new]
    B = len(lens_l)
    for H_kv, split in ((2, True), (16, False)):
        H = 4 * H_kv
        assert (ops.fa2_fwd_kvcache_workspace_bytes(B, Lq, H, H_kv, D, S) > 0) == split
        kc, vc, table = _caches(kind, B, S, H_kv, D, dtype, seed=L_new + H_kv)
        q, kn, vn = _rand(B, Lq, H, D, dtype=dtype), _rand(B, L_new, H_kv, D, dtype=dtype), _rand(B, L_new, H_kv, D, dtype=dtype)
        lens = _lens(lens_l)
        # the two-step path: scatter, then decode on lens + L_new
        k2 = ko.write(kc, kn, lens_l, table).cuda()
        v2 = ko.write(vc, vn, lens_l, table).cuda()
        o2 = torch.full_like(q, float("nan"))
        ops.fa2_fwd_kvcache(q, k2, v2, o2, lens + L_new, table, causal=causal)
        o = torch.full_like(q, float("nan"))
        ops.fa2_fwd_kvcache(q, kc, vc, o, lens, table, causal=causal, k=kn, v=vn)
        assert torch.equal(_bits(o), _bits(o2)), (H_kv, split)
        assert torch.equal(_bits(kc), _bits(k2)) and torch.equal(_bits(vc), _bits(v2)), (H_kv, split)
        assert torch.equal(lens, _lens(lens_l))   # cache_seqlens is not updated


def _ulp(x, dtype):
    e = torch.floor(torch.log2(x.abs().clamp(min=2.0 ** -14 if dtype == torch.float16 else 2.0 ** -126)))
    return torch.pow(2.0, e - MANTISSA[dtype])


def _rotary_cases():
    for D in (32, 64, 96, 128):
        for rd in sorted({16, (D // 32) * 16, D}):
            yield D, rd


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("interleaved", [False, True])
@pytest.mark.parametrize("D,rd", list(_rotary_cases()))
def test_rotary_against_the_reference(D, rd, interleaved, causal, dtype):
    ops = _ops()
    B, Lq, L_new, H, H_kv, S, ps = 4, 3, 3, 8, 2, 256, 64
    lens_l = [0, 15, 100, S - L_new]
    kc, vc, table = _caches(ps, B, S, H_kv, D, dtype, seed=D + rd)
    q, kn, vn = _rand(B, Lq, H, D, dtype=dtype), _rand(B, L_new, H_kv, D, dtype=dtype), _rand(B, L_new, H_kv, D, dtype=dtype)
    g = torch.Generator().manual_seed(rd)
    theta = torch.rand(S + 5, rd // 2, generator=g, dtype=torch.float64) * 2 * math.pi
    cos, sin = theta.cos().to(dtype).cuda(), theta.sin().to(dtype).cuda()
    want_o, want_k, want_v = ko.attention_append(q, kc, vc, lens_l, kn, vn, table, cos, sin, interleaved, causal=causal)
    q0 = q.clone()
    o = torch.full_like(q, float("nan"))
    ops.fa2_fwd_kvcache(q, kc, vc, o, _lens(lens_l), table, causal=causal, k=kn, v=vn, rotary_cos=cos, rotary_sin=sin,
                        rotary_interleaved=interleaved)
    assert torch.equal(q, q0)                                         # Q is not modified
    assert torch.equal(_bits(vc.cpu()), _bits(want_v))                # V copied bit for bit
    kg = kc.cpu()
    # rotated columns of the new rows within 1 ulp of the fp64 rotation rounded to the dtype; every other value exact
    sel = torch.zeros(kg.shape[:2] + (1, 1), dtype=torch.bool)
    for b, n in enumerate(lens_l):
        for i in range(L_new):
            p = n + i
            sel[table[b, p // ps].item(), p % ps] = True
    rot_cols = torch.zeros(D, dtype=torch.bool)
    rot_cols[:rd] = True
    rot = sel & rot_cols.view(1, 1, 1, D)
    assert torch.equal(_bits(kg[~rot.expand_as(kg)]), _bits(want_k[~rot.expand_as(kg)]))
    a, w = kg[rot.expand_as(kg)].float(), want_k[rot.expand_as(kg)].float()
    assert bool(((a - w).abs() <= _ulp(w, dtype)).all())
    assert torch.isfinite(o).all()
    assert torch.allclose(o.cpu().float(), want_o.float(), **ar.TOL[dtype])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("interleaved", [False, True])
def test_q_and_k_are_rotated_by_the_same_arithmetic(interleaved, dtype):
    """MHA, Lq = L_new, causal, q = k_new: O has the bits of fa2_fwd_kvcache with Q read back from the rotated K rows
    the call wrote into the cache."""
    ops = _ops()
    B, L_new, H, D, S, ps = 3, 4, 8, 128, 512, 64
    lens_l = [0, 61, 300]
    kc, vc, table = _caches(ps, B, S, H, D, dtype, seed=11)
    kn, vn = _rand(B, L_new, H, D, dtype=dtype), _rand(B, L_new, H, D, dtype=dtype)
    cos, sin = _rope(S, D, dtype)
    o = torch.full_like(kn, float("nan"))
    ops.fa2_fwd_kvcache(kn, kc, vc, o, _lens(lens_l), table, causal=True, k=kn, v=vn, rotary_cos=cos, rotary_sin=sin,
                        rotary_interleaved=interleaved)
    j = torch.tensor(lens_l, device="cuda").view(B, 1) + torch.arange(L_new, device="cuda").view(1, L_new)
    qk = kc[table.gather(1, j // ps).long(), j % ps]                  # [B, L_new, H, D]
    o2 = torch.full_like(kn, float("nan"))
    ops.fa2_fwd_kvcache(qk.contiguous(), kc, vc, o2, _lens(lens_l) + L_new, table, causal=True)
    assert torch.equal(_bits(o), _bits(o2))


def _poison(shape):
    vals = torch.tensor([float("nan"), float("inf"), float("-inf")])
    return vals[torch.randint(0, 3, shape)]


@pytest.mark.parametrize("kind", ["contig", 16])
def test_isolation_guards_and_overflow(kind):
    """Caches and O sit in sentinel-filled guard buffers; slots past each length and the spare pages hold NaN / +-Inf,
    and table entries past each sequence's last touched page point at a poison page.  Only the new rows' slots change,
    nothing is written at or past the capacity (the last sequence overflows it), and O is finite, inside its guards and
    equal to the reference over the clipped cache.  NeoX rotary with rotary_seqlen = capacity, so the overflowing
    sequence's queries use the last cos / sin row."""
    ops = _ops()
    B, Lq, L_new, H, H_kv, D = 4, 5, 5, 8, 2, 64
    cap = 128
    lens_l = [0, 14, 60, cap - 3]
    torch.manual_seed(5)
    guard, sentinel = 4096, 7.0
    if kind == "contig":
        num_pages, ps, pps, table = B, cap, 1, None
    else:
        ps, pps, spare = kind, cap // kind, 3
        num_pages = B * pps + spare + 1
        poison_page = num_pages - 1
        perm = torch.randperm(B * pps + spare)
        table = perm[:B * pps].view(B, pps).to(torch.int32)
        for b, n in enumerate(lens_l):
            last = (min(n + L_new, cap) - 1) // ps
            table[b, last + 1:] = poison_page
    shape = (num_pages, ps, H_kv, D)
    n_el = math.prod(shape)
    bufs = []
    for _ in range(2):
        buf = torch.full((guard + n_el + guard,), sentinel, dtype=torch.half)
        c = buf[guard:guard + n_el].view(shape)
        c.copy_(torch.randn(shape).half())
        if table is not None:
            listed = set(table.view(-1).tolist()) - {num_pages - 1}
            for p in range(num_pages):
                if p not in listed:
                    c[p] = _poison(c[p].shape).half()
        for b, n in enumerate(lens_l):                       # slots past the length, in pages the sequence lists
            for pos in range(n, cap):
                if table is None:
                    c[b, pos] = _poison((H_kv, D)).half()
                elif table[b, pos // ps] != num_pages - 1:
                    c[table[b, pos // ps], pos % ps] = _poison((H_kv, D)).half()
        bufs.append(buf.cuda())
    kb, vb = bufs
    kc, vc = [b[guard:guard + n_el].view(shape) for b in bufs]
    before_k, before_v = kb.cpu().clone(), vb.cpu().clone()
    q, kn, vn = torch.randn(B, Lq, H, D).half(), torch.randn(B, L_new, H_kv, D).half(), torch.randn(B, L_new, H_kv, D).half()
    cos, sin = _rope(cap, D, torch.float16)
    tcuda = table.cuda() if table is not None else None
    n_o = B * Lq * H * D
    ob = torch.full((guard + n_o + guard,), sentinel, dtype=torch.half, device="cuda")
    o = ob[guard:guard + n_o].view(B, Lq, H, D)
    want_o, want_k, want_v = ko.attention_append(q, kc, vc, lens_l, kn, vn, table, cos, sin, False, causal=True)
    ops.fa2_fwd_kvcache(q.cuda(), kc, vc, o, _lens(lens_l), tcuda, causal=True, k=kn.cuda(), v=vn.cuda(),
                        rotary_cos=cos, rotary_sin=sin, rotary_interleaved=False)
    torch.cuda.synchronize()
    for buf, before, want in ((kb, before_k, want_k), (vb, before_v, want_v)):
        got = buf.cpu()
        exp = before.clone()
        exp[guard:guard + n_el] = want.reshape(-1)
        assert torch.equal(_bits(got), _bits(exp))            # guards, poison, spare pages and slots >= capacity unchanged
    assert bool((ob[:guard] == sentinel).all()) and bool((ob[guard + n_o:] == sentinel).all())
    assert torch.isfinite(o).all()
    assert torch.allclose(o.cpu().float(), want_o.float(), **ar.TOL[torch.float16])


def test_cuda_graph_replay_of_a_decode_loop():
    """"Append, then lens += L_new" captured once and replayed for 40 steps on pages of 16 keys (steps cross page
    boundaries); fresh q / k / v go into the static inputs before each replay.  Each step's O and the final caches have
    the bits of the same steps run eagerly from the same state."""
    ops = _ops()
    B, Lq, L_new, H, H_kv, D, ps, pps, steps = 2, 3, 3, 16, 4, 128, 16, 16, 40
    cap = ps * pps
    torch.manual_seed(17)
    num_pages = B * pps
    kp0, vp0 = _rand(num_pages, ps, H_kv, D), _rand(num_pages, ps, H_kv, D)
    table = torch.randperm(num_pages, device="cuda").to(torch.int32).view(B, pps)
    lens0 = _lens([5, 100])
    cos, sin = _rope(cap, D, torch.float16)
    inputs = [(_rand(B, Lq, H, D), _rand(B, L_new, H_kv, D), _rand(B, L_new, H_kv, D)) for _ in range(steps)]

    def step(q, k, v, kp, vp, o, lens):
        ops.fa2_fwd_kvcache(q, kp, vp, o, lens, table, causal=True, k=k, v=v, rotary_cos=cos, rotary_sin=sin,
                            rotary_interleaved=False)
        lens.add_(L_new)

    kp, vp, lens = kp0.clone(), vp0.clone(), lens0.clone()
    eager = []
    for q, k, v in inputs:
        o = torch.empty_like(q)
        step(q, k, v, kp, vp, o, lens)
        eager.append(o)
    eager_k, eager_v = kp, vp

    sq, sk, sv = torch.empty_like(inputs[0][0]), torch.empty_like(inputs[0][1]), torch.empty_like(inputs[0][2])
    gk, gv, glens, go = kp0.clone(), vp0.clone(), lens0.clone(), torch.empty_like(inputs[0][0])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step(sq, sk, sv, gk, gv, go, glens)                         # warm-up: tensor maps, shared-memory attribute
    torch.cuda.current_stream().wait_stream(s)
    gk.copy_(kp0)
    gv.copy_(vp0)
    glens.copy_(lens0)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step(sq, sk, sv, gk, gv, go, glens)
    for i, (q, k, v) in enumerate(inputs):
        sq.copy_(q)
        sk.copy_(k)
        sv.copy_(v)
        go.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(_bits(go), _bits(eager[i])), i
    assert torch.equal(glens, lens0 + steps * L_new)
    assert torch.equal(_bits(gk), _bits(eager_k)) and torch.equal(_bits(gv), _bits(eager_v))
    assert bool(torch.isfinite(go).all())


def test_full_size_paged_gqa_rotary():
    """B = 8, H = 64, H_kv = 8, D = 128, a 32K cache paged at 256, NeoX rotary over all 128 columns, two new tokens,
    causal: sampled rows match an fp32 reference computed on the GPU from the cache before the call."""
    ops = _ops()
    B, Lq, L_new, H, H_kv, D, S, ps = 8, 2, 2, 64, 8, 128, 32768, 256
    G = H // H_kv
    torch.manual_seed(23)
    pps = S // ps
    num_pages = B * pps
    kp, vp = _rand(num_pages, ps, H_kv, D), _rand(num_pages, ps, H_kv, D)
    table = torch.randperm(num_pages, device="cuda").to(torch.int32).view(B, pps)
    lens_l = [S - L_new, 32000, 0, 129, 20000, 8191, 31000, 5]
    q, kn, vn = _rand(B, Lq, H, D), _rand(B, L_new, H_kv, D), _rand(B, L_new, H_kv, D)
    cos, sin = _rope(S, D, torch.float16)
    old = {}
    for b in (0, 2, 4, 6):
        j = torch.arange(lens_l[b], device="cuda")
        pg = table[b, j // ps].long()
        old[b] = (kp[pg, j % ps].float(), vp[pg, j % ps].float())
    o = torch.full_like(q, float("nan"))
    ops.fa2_fwd_kvcache(q, kp, vp, o, _lens(lens_l), table, causal=True, k=kn, v=vn, rotary_cos=cos, rotary_sin=sin,
                        rotary_interleaved=False)
    assert torch.isfinite(o).all()

    def rot(x, pos):   # [L, heads, D] at positions pos [L], fp32, rounded to half
        c, s = cos[pos].float().unsqueeze(1), sin[pos].float().unsqueeze(1)
        x0, x1 = x[..., :D // 2].float(), x[..., D // 2:].float()
        return torch.cat([x0 * c - x1 * s, x0 * s + x1 * c], -1).half().float()

    for b in (0, 2, 4, 6):
        n = lens_l[b]
        pos = n + torch.arange(L_new, device="cuda")
        ks = torch.cat([old[b][0], rot(kn[b], pos)])
        vs = torch.cat([old[b][1], vn[b].float()])
        qs = rot(q[b], n + torch.arange(Lq, device="cuda"))           # [Lq, H, D]
        lk = n + L_new
        j = torch.arange(lk, device="cuda")
        for h in (0, 13, H - 1):
            s = (qs[:, h] @ ks[:, h // G].t()) / D ** 0.5
            s = s.masked_fill(j.view(1, lk) > torch.arange(Lq, device="cuda").view(Lq, 1) + lk - Lq, float("-inf"))
            want = torch.softmax(s, -1) @ vs[:, h // G]
            assert torch.allclose(o[b, :, h].float(), want, **ar.TOL[torch.float16]), (b, h)
