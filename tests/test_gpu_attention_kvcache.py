"""GPU: KV-cache decode attention (ops.fa2_fwd_kvcache) against the CPU reference (attention_ref.py), both sides of
the split rule, bit equality with fa2_fwd_varlen / between paged and contiguous caches / between repeated calls,
isolation from whatever the cache holds past each length, stores that stay inside O, CUDA graph replay while the
cache grows, and a full-size run.  Tolerances are those of test_gpu_attention_varlen.py."""
import ctypes
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))  # kvcache_oracle.py sits next to this file
import attention_ref as ar  # noqa: E402
import kvcache_oracle  # noqa: E402

pytestmark = pytest.mark.gpu
LENS = [0, 1, 127, 128, 129, 3000]


def _inputs(B, Lq, H, H_kv, D, S, dtype, seed):
    torch.manual_seed(seed)
    q = torch.randn(B, Lq, H, D, device="cuda").to(dtype)
    kc, vc = [torch.randn(B, S, H_kv, D, device="cuda").to(dtype) for _ in range(2)]
    return q, kc, vc


def _lens(lens):
    return torch.tensor(lens, dtype=torch.int32, device="cuda")


def _run(q, kc, vc, lens, table=None, causal=False, fill=float("nan")):
    from b200k import ops

    o = torch.full_like(q, fill)
    ops.fa2_fwd_kvcache(q, kc, vc, o, lens, table, causal=causal)
    return o


def _ws(B, Lq, H, H_kv, D, cap):
    from b200k import ops

    return ops.fa2_fwd_kvcache_workspace_bytes(B, Lq, H, H_kv, D, cap)


def _check(o, q, kc, vc, lens, table, causal, dtype):
    assert torch.isfinite(o).all()
    want = ar.kvcache(q, kc, vc, lens, table, causal=causal)[0].to(q.dtype)
    assert torch.allclose(o.cpu().float(), want.float(), **ar.TOL[dtype])


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("D", [32, 64, 96, 128])
def test_head_dims_paged_vs_reference(D, dtype, causal):
    B, H, H_kv, S, ps = len(LENS), 16, 2, 3008, 64
    q, kc, vc = _inputs(B, 1, H, H_kv, D, S, dtype, seed=D + causal)
    kp, vp, table, _ = kvcache_oracle.paged_copy(kc, vc, ps, seed=D)
    lens = _lens(LENS)
    _check(_run(q, kp, vp, lens, table, causal), q, kp, vp, lens, table, causal, dtype)


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("Lq", [1, 3, 16])
@pytest.mark.parametrize("G", [1, 4, 6, 8, 16, 64, 71])
def test_groups_and_query_lengths_contiguous_vs_reference(G, Lq, causal):
    """G = 6 packs a Q box of 60 rows; G = 71 takes two head tiles, the second reading heads of no output."""
    B, H_kv, D, S = len(LENS), 2, 128, 3100
    q, kc, vc = _inputs(B, Lq, G * H_kv, H_kv, D, S, torch.float16, seed=G * 31 + Lq + causal)
    lens = _lens(LENS)
    o = _run(q, kc, vc, lens, causal=causal)
    _check(o, q, kc, vc, lens, None, causal, torch.float16)
    if causal:   # rows that see no key are exactly 0: token t of sequence b with t + Lk_b - Lq < 0
        for b, n in enumerate(LENS):
            assert (o[b, :max(0, Lq - n)] == 0).all(), b


@pytest.mark.parametrize("page_size", [16, 32, 64, 128, 256])
def test_page_sizes_shuffled_table_same_bits_as_contiguous(page_size):
    B, Lq, H, H_kv, D, S = len(LENS), 3, 8, 2, 64, 3072
    q, kc, vc = _inputs(B, Lq, H, H_kv, D, S, torch.bfloat16, seed=page_size)
    kp, vp, table, _ = kvcache_oracle.paged_copy(kc, vc, page_size, seed=page_size)
    assert table.view(-1).tolist() != sorted(table.view(-1).tolist())
    lens = _lens(LENS)
    o = _run(q, kp, vp, lens, table, causal=True)
    _check(o, q, kp, vp, lens, table, True, torch.bfloat16)
    assert torch.equal(o, _run(q, kc, vc, lens, causal=True))


def test_split_rule_both_sides_and_short_workspace():
    """Sixteen sequences x 8 K/V heads fill the SMs and run unsplit; one sequence with a long cache is split.  On the
    split shape a workspace one byte short is refused before anything runs, and O is left as it was."""
    from b200k import _loader as L

    assert _ws(16, 1, 32, 8, 128, 4096) == 0
    need = _ws(1, 1, 32, 8, 128, 32768)
    assert need > 0
    B, H, H_kv, D, S = 1, 32, 8, 128, 32768
    q, kc, vc = _inputs(B, 1, H, H_kv, D, S, torch.float16, seed=3)
    lens = _lens([30000])
    o = _run(q, kc, vc, lens)
    _check(o, q, kc, vc, lens, None, False, torch.float16)
    ws = torch.empty(need - 1, dtype=torch.uint8, device="cuda")
    o2 = torch.full_like(q, 7.0)
    rc = L.lib.b200k_fa2_fwd_kvcache(q.data_ptr(), kc.data_ptr(), vc.data_ptr(), o2.data_ptr(), lens.data_ptr(), None,
                                     B, 1, H, H_kv, D, B, S, 1, 0.0, L.F16, 0, ws.data_ptr(), need - 1,
                                     torch.cuda.current_stream().cuda_stream)
    assert rc == L.EARG
    rc = L.lib.b200k_fa2_fwd_kvcache(q.data_ptr(), kc.data_ptr(), vc.data_ptr(), o2.data_ptr(), lens.data_ptr(), None,
                                     B, 1, H, H_kv, D, B, S, 1, 0.0, L.F16, 0, None, 0, None)
    assert rc == L.EARG
    torch.cuda.synchronize()
    assert (o2 == 7.0).all()


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("Lq", [1, 3])
def test_one_split_same_bits_as_varlen(Lq, causal):
    """One split and a contiguous cache: each row goes through the arithmetic of fa2_fwd_varlen on the same tokens."""
    from b200k import ops

    B, H, H_kv, D, S = 16, 32, 8, 128, 1500
    assert _ws(B, Lq, H, H_kv, D, S) == 0
    q, kc, vc = _inputs(B, Lq, H, H_kv, D, S, torch.float16, seed=Lq + causal)
    lens_l = [0, 1, 127, 128, 129, 1500, 777, 3, 256, 1000, 1499, 64, 2, 900, 385, 1200]
    lens = _lens(lens_l)
    o = _run(q, kc, vc, lens, causal=causal)
    pk = torch.cat([kc[b, :n] for b, n in enumerate(lens_l)])
    pv = torch.cat([vc[b, :n] for b, n in enumerate(lens_l)])
    cu_k = torch.tensor([0] + torch.tensor(lens_l).cumsum(0).tolist(), dtype=torch.int32, device="cuda")
    cu_q = torch.arange(B + 1, dtype=torch.int32, device="cuda") * Lq
    pq = q.reshape(B * Lq, H, D)
    ov = torch.full_like(pq, float("nan"))
    ops.fa2_fwd_varlen(pq, pk, pv, ov, cu_q, cu_k, Lq, causal=causal)
    assert torch.equal(o.view(B * Lq, H, D), ov)


@pytest.mark.parametrize("B", [1, 16])   # split / unsplit
def test_paged_same_bits_as_contiguous_and_repeatable(B):
    H, H_kv, D, S, Lq = 32, 8, 128, 8192, 2
    assert (_ws(B, Lq, H, H_kv, D, S) > 0) == (B == 1)
    q, kc, vc = _inputs(B, Lq, H, H_kv, D, S, torch.float16, seed=B)
    lens = _lens(([8192, 5000, 129, 1] * 4)[:B])
    kp, vp, table, _ = kvcache_oracle.paged_copy(kc, vc, 256, seed=B)
    for causal in (False, True):
        o = _run(q, kc, vc, lens, causal=causal)
        assert torch.equal(_run(q, kp, vp, lens, table, causal=causal), o)
        assert torch.equal(_run(q, kc, vc, lens, causal=causal), o)
    _check(o, q, kc, vc, lens, None, True, torch.float16)


def _poison(shape):
    vals = torch.tensor([float("nan"), float("inf"), float("-inf"), 1e4, -1e4])
    return vals[torch.randint(0, 5, shape)]


@pytest.mark.parametrize("B", [1, 16])   # split / unsplit
@pytest.mark.parametrize("page_size", [16, 256])
def test_isolation_from_slots_past_the_length_and_unlisted_pages(B, page_size):
    """Every slot at or past Lk_b, every unlisted page, and every table entry past a sequence's last valid page (pointed
    at such a page) holds NaN / +-Inf / +-1e4: O stays finite and has the bits of the clean run."""
    H, H_kv, D, S, Lq = 32, 8, 128, 4096, 3
    q, kc, vc = _inputs(B, Lq, H, H_kv, D, S, torch.float16, seed=page_size + B)
    lens_l = ([4096, 1, 129, 0, 1000, 4000, 255, 2049] * 2)[:B] if B > 1 else [2500]
    lens = _lens(lens_l)
    kp, vp, table, spare = kvcache_oracle.paged_copy(kc, vc, page_size, spare_pages=5, seed=B,
                                                     fill=lambda shape: torch.zeros(shape))
    for causal in (False, True):
        clean = _run(q, kp, vp, lens, table, causal=causal)
        kd, vd, td = kp.clone(), vp.clone(), table.clone()
        for b, n in enumerate(lens_l):
            j = torch.arange(n, S, device="cuda")   # slots past the length, including whole pages past the last valid one
            pg, sl = table[b, j // page_size].long(), j % page_size
            kd[pg, sl] = _poison((S - n, H_kv, D)).half().cuda()
            vd[pg, sl] = _poison((S - n, H_kv, D)).half().cuda()
            first_unused = (n + page_size - 1) // page_size
            td[b, first_unused:] = int(spare[b % len(spare)])
        for s in spare.tolist():
            kd[s] = _poison(kd[s].shape).half().cuda()
            vd[s] = _poison(vd[s].shape).half().cuda()
        o = _run(q, kd, vd, lens, td, causal=causal)
        assert torch.isfinite(o).all()
        assert torch.equal(o, clean)


@pytest.mark.parametrize("G", [6, 71])
def test_stores_stay_inside_o(G):
    """O is a slice of a sentinel-filled buffer; the Q boxes of G = 6 and G = 71 read rows that belong to no output."""
    from b200k import ops

    for B, Lq in ((1, 5), (16, 3)):   # split and unsplit
        H_kv, D, S, guard = 2, 64, 2048, 4096
        H = G * H_kv
        q, kc, vc = _inputs(B, Lq, H, H_kv, D, S, torch.float16, seed=G + B)
        n = B * Lq * H * D
        buf = torch.full((guard + n + guard,), 7.0, dtype=torch.half, device="cuda")
        o = buf[guard:guard + n].view(B, Lq, H, D)
        lens = _lens(([2048, 1, 700, 0] * 4)[:B])
        for causal in (False, True):
            ops.fa2_fwd_kvcache(q, kc, vc, o, lens, causal=causal)
            torch.cuda.synchronize()
            assert bool((buf[:guard] == 7.0).all()) and bool((buf[guard + n:] == 7.0).all()), (B, causal)
            _check(o, q, kc, vc, lens, None, causal, torch.float16)


def test_cuda_graph_replay_while_the_cache_grows():
    """Captured once; before each replay the lengths grow, pages are appended to the table and their K/V written.  Each
    replay equals the eager call on the same state."""
    from b200k import ops

    B, Lq, H, H_kv, D, ps, pps = 2, 1, 32, 8, 128, 64, 50
    num_pages = B * pps + 1
    torch.manual_seed(9)
    q = torch.randn(B, Lq, H, D, device="cuda").half()
    kp, vp = [torch.randn(num_pages, ps, H_kv, D, device="cuda").half() for _ in range(2)]
    order = torch.randperm(num_pages - 1).to(torch.int32).cuda()
    table = torch.full((B, pps), num_pages - 1, dtype=torch.int32, device="cuda")   # unused entries: a spare page
    lens = _lens([100, 1000])
    used = [2, 16]   # pages listed so far
    for b in range(B):
        table[b, :used[b]] = order[b * pps:b * pps + used[b]]
    o = torch.empty_like(q)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.fa2_fwd_kvcache(q, kp, vp, o, lens, table, causal=True)     # warm-up: tensor maps, shared-memory attribute
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.fa2_fwd_kvcache(q, kp, vp, o, lens, table, causal=True)
    for step in (1, 63, 64, 700, 1000):
        for b in range(B):
            n = int(lens[b]) + step
            need = (n + ps - 1) // ps
            while used[b] < need:
                table[b, used[b]] = order[b * pps + used[b]]
                used[b] += 1
            lens[b] = n
        for b in range(B):   # new K/V for the appended tokens
            j = torch.arange(int(lens[b]) - step, int(lens[b]), device="cuda")
            pg = table[b, j // ps].long()
            kp[pg, j % ps] = torch.randn(step, H_kv, D, device="cuda").half()
            vp[pg, j % ps] = torch.randn(step, H_kv, D, device="cuda").half()
        q.copy_(torch.randn_like(q.float()).half())
        o.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(o, _run(q, kp, vp, lens, table, causal=True)), step
    _check(o, q, kp, vp, lens, table, True, torch.float16)


def test_full_size_paged_gqa_properties():
    """B = 8, H = 64, H_kv = 8, D = 128, a 32K paged cache: V = 1 gives O = 1, and sampled rows match an fp32 reference
    computed on the GPU."""
    B, Lq, H, H_kv, D, S, ps = 8, 2, 64, 8, 128, 32768, 256
    torch.manual_seed(21)
    q = torch.randn(B, Lq, H, D, device="cuda").half()
    pps = S // ps
    num_pages = B * pps
    kp = torch.randn(num_pages, ps, H_kv, D, device="cuda").half()
    table = torch.randperm(num_pages, device="cuda").to(torch.int32).view(B, pps)
    lens_l = [32768, 32767, 1, 129, 20000, 8192, 31000, 5]
    lens = _lens(lens_l)
    ones = torch.ones_like(kp)
    o1 = _run(q, kp, ones, lens, table, causal=True)
    assert (o1[[b for b in range(B) if lens_l[b] >= Lq]].float() - 1.0).abs().max().item() <= 1e-3
    assert (o1[2, 0] == 0).all() and (o1[2, 1].float() - 1.0).abs().max().item() <= 1e-3   # Lk = 1: token 0 sees no key
    del ones
    vp = torch.randn(num_pages, ps, H_kv, D, device="cuda").half()
    o = _run(q, kp, vp, lens, table, causal=True)
    assert torch.isfinite(o).all()
    for b in (0, 4, 6):
        n = lens_l[b]
        j = torch.arange(n, device="cuda")
        pg = table[b, j // ps].long()
        for h in (0, 13, H - 1):
            ks, vs = kp[pg, j % ps, h // (H // H_kv)].float(), vp[pg, j % ps, h // (H // H_kv)].float()
            qs = q[b, :, h].float()                                           # [Lq, D]
            s = (qs @ ks.t()) / D ** 0.5
            s = s.masked_fill(j.view(1, n) > torch.arange(Lq, device="cuda").view(Lq, 1) + n - Lq, float("-inf"))
            want = torch.softmax(s, -1) @ vs
            assert torch.allclose(o[b, :, h].float(), want, **ar.TOL[torch.float16]), (b, h)
