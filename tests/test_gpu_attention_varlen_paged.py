"""GPU: packed attention over paged caches (ops.fa2_fwd_varlen with block_table).  The kernel is the packed mode's main
loop with the decode mode's page addressing, so O and lse must have the bits of ops.fa2_fwd_varlen on K / V gathered
through the table, whatever the slots outside the valid keys hold; plus table shapes, clipped stores, exact answers,
agreement with KV-cache decode and CUDA graph replay."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))  # the oracles sit next to this file
import attention_ref as ar  # noqa: E402
import varlen_paged_oracle as vpo  # noqa: E402

pytestmark = pytest.mark.gpu
LQ = [77, 0, 1, 129, 300, 128, 5]
LK = [300, 5, 0, 128, 129, 1000, 700]   # Lk < Lq, Lk = 0, an empty query sequence, Lk not a multiple of any page


def _ops():
    from b200k import ops
    return ops


def _pack(lq, lk, H, H_kv, D, dtype, seed, extra_q=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(sum(lq) + extra_q, H, D, device="cuda", generator=g).to(dtype)
    k, v = [torch.randn(sum(lk), H_kv, D, device="cuda", generator=g).to(dtype) for _ in range(2)]
    return q, k, v, ar.cu(lq, "cuda"), ar.cu(lk, "cuda")


def _paged(q, kc, vc, cq, ck, table, max_q, causal, fill=float("nan")):
    o = torch.full_like(q, fill)
    lse = torch.full(q.shape[:2], fill, device="cuda")
    _ops().fa2_fwd_varlen(q, kc, vc, o, cq, ck, max_q, causal=causal, lse=lse, block_table=table)
    return o, lse


def _gathered(q, kc, vc, cq, ck, table, max_q, causal, fill=float("nan")):
    """ops.fa2_fwd_varlen on the keys the paged call reads, gathered into contiguous K / V."""
    k, v, cg = vpo.gather(kc, vc, ck, table)
    if k.size(0) == 0:
        k, v = kc[:1, 0].clone(), vc[:1, 0].clone()   # every sequence empty: one key no sequence reads
    o = torch.full_like(q, fill)
    lse = torch.full(q.shape[:2], fill, device="cuda")
    _ops().fa2_fwd_varlen(q, k.cuda(), v.cuda(), o, cq, cg.cuda(), max_q, causal=causal, lse=lse)
    return o, lse


def _same_bits(a, b):
    assert torch.equal(a[0].view(torch.int16), b[0].view(torch.int16)), "O differs"
    assert torch.equal(a[1].view(torch.int32), b[1].view(torch.int32)), "lse differs"


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("D", [32, 64, 96, 128])
@pytest.mark.parametrize("page_size", [16, 32, 64, 128, 256])
def test_same_bits_as_gathered(page_size, D, dtype, causal):
    H = 16
    for group in (1, 2, 8, 16):
        q, k, v, cq, ck = _pack(LQ, LK, H, H // group, D, dtype, seed=page_size + D + group + causal)
        kc, vc, table = vpo.to_pages(k, v, ck, page_size, seed=group)
        got = _paged(q, kc, vc, cq, ck, table, max(LQ), causal)
        assert torch.isfinite(got[0]).all(), group
        _same_bits(got, _gathered(q, kc, vc, cq, ck, table, max(LQ), causal))
        if group == 8 and D == 64:
            want = ar.packed(q, k, v, cq, ck, causal=causal)[0].to(q.dtype).cpu()
            assert torch.allclose(got[0].cpu().float(), want.float(), **ar.TOL[dtype])


@pytest.mark.parametrize("poison", [float("nan"), float("inf"), float("-inf")])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("page_size", [16, 32, 64, 128, 256])
def test_poisoned_caches(page_size, dtype, causal, poison):
    """Slots past Lk in each last page, listed pages past the length and pages no table row names all hold NaN or Inf.
    The result is finite and has the bits of the clean cache; a missing or racing V tail zeroing fails here."""
    H, D = 16, 128
    for group, d in ((8, D), (2, 64)):
        q, k, v, cq, ck = _pack(LQ, LK, H, H // group, d, dtype, seed=page_size + group)
        clean = vpo.to_pages(k, v, ck, page_size, pages_per_seq=1024 // page_size + 1, seed=1)
        dirty = vpo.to_pages(k, v, ck, page_size, pages_per_seq=1024 // page_size + 1, seed=1, fill=poison)
        a = _paged(q, clean[0], clean[1], cq, ck, clean[2], max(LQ), causal)
        b = _paged(q, dirty[0], dirty[1], cq, ck, dirty[2], max(LQ), causal)
        assert torch.isfinite(b[0]).all()
        _same_bits(a, b)
        _same_bits(b, _gathered(q, dirty[0], dirty[1], cq, ck, dirty[2], max(LQ), causal))


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("page_size", [16, 64, 256])
def test_table_shapes(page_size, causal):
    """Shared prefix pages, Lq > Lk (rows that see no key: 0 and lse -inf under causal), Lk past the capacity (clamped),
    Lk = 0 and an empty query sequence."""
    ops = _ops()
    H, H_kv, D, dtype = 8, 2, 64, torch.float16
    lq, lk = [40, 50, 300, 0, 7, 20], [512, 600, 100, 40, 0, 2000]
    q, k, v, cq, ck = _pack(lq, lk, H, H_kv, D, dtype, seed=page_size)
    k[512:1024], v[512:1024] = k[:512], v[:512]       # sequence 1 starts with sequence 0's 512 keys
    pps = 1024 // page_size                           # capacity 1024 < 2000: the last sequence is clamped
    kc, vc, table = vpo.to_pages(k, v, ck, page_size, pages_per_seq=pps, share=512 // page_size, seed=2,
                                 fill=float("nan"))
    got = _paged(q, kc, vc, cq, ck, table, max(lq), causal)
    _same_bits(got, _gathered(q, kc, vc, cq, ck, table, max(lq), causal))
    c = cq.tolist()
    if causal:                                       # sequence 2: rows r < 200 see no key
        assert (got[0][c[2]:c[2] + 200] == 0).all() and torch.isneginf(got[1][c[2]:c[2] + 200]).all()
    assert (got[0][c[4]:c[5]] == 0).all() and torch.isneginf(got[1][c[4]:c[5]]).all()     # Lk = 0
    # the clamped sequence equals its first 1024 keys given explicitly
    cut = ar.cu([lq[5]], "cuda"), ar.cu([1024], "cuda")
    o2 = torch.empty_like(q[c[5]:c[6]])
    ops.fa2_fwd_varlen(q[c[5]:c[6]], kc, vc, o2, cut[0], cut[1], lq[5], causal=causal, block_table=table[5:6].clone())
    assert torch.equal(o2.view(torch.int16), got[0][c[5]:c[6]].view(torch.int16))


def test_stores_stay_inside_o():
    """O and lse inside larger buffers with sentinel rows before and after, and tokens past the last sequence."""
    ops = _ops()
    H, H_kv, D, dtype = 8, 2, 128, torch.bfloat16
    lq, lk, extra = [100, 3, 129], [200, 64, 129], 50
    q, k, v, cq, ck = _pack(lq, lk, H, H_kv, D, dtype, seed=11, extra_q=extra)
    kc, vc, table = vpo.to_pages(k, v, ck, 64, seed=4, fill=float("nan"))
    T = q.size(0)
    for causal in (False, True):
        obuf = torch.full((T + 2 * 64, H, D), 7.0, dtype=dtype, device="cuda")
        lbuf = torch.full((T + 2 * 64, H), 7.0, device="cuda")
        o, lse = obuf[64:64 + T], lbuf[64:64 + T]
        ops.fa2_fwd_varlen(q, kc, vc, o, cq, ck, max(lq), causal=causal, lse=lse, block_table=table)
        n = sum(lq)
        for t in (obuf[:64], obuf[64 + n:], lbuf[:64], lbuf[64 + n:]):
            assert (t == 7.0).all()
        assert torch.isfinite(o[:n]).all()


def test_exact_answers_through_pages():
    """Exact-answer inputs of the packed mode (exact_attention.py) scattered into shuffled pages with NaN elsewhere."""
    from test_gpu_attention_exact import LK as ELK, LQ as ELQ, _check, _varlen
    ops = _ops()
    for dtype in (torch.float16, torch.bfloat16):
        for causal in (False, True):
            for page_size, D, group in ((16, 128, 8), (64, 64, 1), (256, 32, 2), (128, 96, 16)):
                H = 16
                q, k, v, cq, ck, spec = _varlen(ELQ, ELK, H, H // group, D, dtype, causal, seed=D + group)
                kc, vc, table = vpo.to_pages(k, v, ck, page_size, seed=D, fill=float("nan"))
                o = torch.full_like(q, float("nan"))
                ops.fa2_fwd_varlen(q, kc, vc, o, cq, ck, max(ELQ), causal=causal, block_table=table)
                _check(o, spec, dtype, what="page %d D %d group %d" % (page_size, D, group))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("B,Lq,H,H_kv", [(8, 128, 32, 8), (1, 4, 8, 2)])
def test_agrees_with_decode(B, Lq, H, H_kv, dtype, causal):
    """Equal query lengths over a contiguous cache [B, S, H_kv, D], which is also a paged cache of B pages of S keys.
    fa2_fwd_kvcache unsplit has the packed mode's bits; split, it agrees within the usual tolerance."""
    ops = _ops()
    S, D = 1024, 128
    g = torch.Generator(device="cuda").manual_seed(B + Lq)
    q = torch.randn(B, Lq, H, D, device="cuda", generator=g).to(dtype)
    kc, vc = [torch.randn(B, S, H_kv, D, device="cuda", generator=g).to(dtype) for _ in range(2)]
    lens = torch.tensor([S - 37 * b for b in range(B)], dtype=torch.int32, device="cuda")
    o_dec = torch.empty_like(q)
    ops.fa2_fwd_kvcache(q, kc, vc, o_dec, lens, causal=causal)
    o = torch.empty_like(q).view(B * Lq, H, D)
    table = torch.arange(B, dtype=torch.int32, device="cuda").view(B, 1)
    ck = torch.cat([torch.zeros(1, dtype=torch.int32, device="cuda"), lens.cumsum(0).int()])
    ops.fa2_fwd_varlen(q.view(B * Lq, H, D), kc, vc, o, ar.cu([Lq] * B, "cuda"), ck, Lq, causal=causal, block_table=table)
    if ops.fa2_fwd_kvcache_workspace_bytes(B, Lq, H, H_kv, D, S) > 0:   # decode splits the keys across CTAs
        assert torch.allclose(o.view_as(q).float(), o_dec.float(), **ar.TOL[dtype])
    else:
        assert torch.equal(o.view_as(q).view(torch.int16), o_dec.view(torch.int16))


def test_cuda_graph_replays_new_lengths_and_tables():
    ops = _ops()
    H, H_kv, D, dtype, ps = 16, 4, 128, torch.float16, 64
    lq, lk = [100, 30, 200, 1], [300, 30, 900, 700]
    q, k, v, cq, ck = _pack(lq, lk, H, H_kv, D, dtype, seed=21)
    kc, vc, table = vpo.to_pages(k, v, ck, ps, pages_per_seq=16, spare_pages=20, seed=5)
    o, lse = torch.zeros_like(q), torch.zeros(q.shape[:2], device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.fa2_fwd_varlen(q, kc, vc, o, cq, ck, 256, causal=True, lse=lse, block_table=table)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.fa2_fwd_varlen(q, kc, vc, o, cq, ck, 256, causal=True, lse=lse, block_table=table)
    for seed, (nq, nk) in enumerate([([50, 80, 150, 51], [1000, 80, 64, 1]), ([0, 256, 74, 1], [5, 1024, 700, 0])]):
        cq.copy_(ar.cu(nq, "cuda"))
        ck.copy_(ar.cu(nk, "cuda"))
        g = torch.Generator().manual_seed(seed)
        table.copy_(torch.randperm(kc.size(0), generator=g)[:table.numel()].view_as(table).int())
        o.fill_(float("nan"))
        graph.replay()
        want = _paged(q, kc, vc, cq, ck, table, 256, True)
        torch.cuda.synchronize()
        n = sum(nq)
        assert torch.equal(o[:n].view(torch.int16), want[0][:n].view(torch.int16))
        assert torch.equal(lse[:n].view(torch.int32), want[1][:n].view(torch.int32))


def _placed_call(offsets):
    """The paged call with each named tensor copied to its byte offset from a 256-byte boundary (others at 0), inside
    0xFF guard bytes.  Returns (error or None, o, lse, placed, inputs)."""
    from test_gpu_attention_align import Placed
    H, H_kv, D, dtype = 8, 2, 64, torch.float16
    lq, lk = [70, 3, 130], [200, 0, 129]
    q, k, v, cq, ck = _pack(lq, lk, H, H_kv, D, dtype, seed=31)
    kc, vc, table = vpo.to_pages(k, v, ck, 32, seed=6, fill=float("nan"))
    at = Placed()
    t = dict(Q=q, K_cache=kc, V_cache=vc, cu_seqlens_q=cq, cu_seqlens_k=ck, block_table=table)
    t = {n: at(x, offsets.get(n, 0)) for n, x in t.items()}
    o = at((q.shape, dtype), offsets.get("O", 0))
    lse = at((q.shape[:2], torch.float32), offsets.get("lse", 0))
    o_in, lse_in = o.clone(), lse.clone()
    try:
        _ops().fa2_fwd_varlen(t["Q"], t["K_cache"], t["V_cache"], o, t["cu_seqlens_q"], t["cu_seqlens_k"], max(lq),
                              causal=True, lse=lse, block_table=t["block_table"])
        err = None
    except RuntimeError as e:
        err = str(e)
    torch.cuda.synchronize()
    return err, o, lse, at, (o_in, lse_in, q, kc, vc, cq, ck, table, max(lq))


ACCEPTED = [("O", 4), ("O", 8), ("O", 12), ("lse", 4), ("cu_seqlens_q", 4), ("cu_seqlens_k", 4), ("block_table", 4),
            ("Q", 16), ("Q", 48), ("K_cache", 16), ("V_cache", 48)]
# lse and the int32 arrays cannot be placed below 4 bytes through a tensor; the CPU tests refuse them through the ABI
REFUSED = [("O", 2), ("O", 6), ("O", 14), ("Q", 2), ("Q", 8), ("K_cache", 4), ("K_cache", 8), ("V_cache", 2),
           ("V_cache", 8)]


@pytest.mark.parametrize("name,off", ACCEPTED)
def test_accepted_offsets_give_the_same_bits(name, off):
    err, o, lse, at, (_, _, q, kc, vc, cq, ck, table, max_q) = _placed_call({name: off})
    assert err is None, err
    want = _paged(q, kc, vc, cq, ck, table, max_q, True, fill=0.0)
    n = int(cq[-1])
    _same_bits((o[:n], lse[:n]), (want[0][:n], want[1][:n]))
    assert at.guards_kept()


@pytest.mark.parametrize("name,off", REFUSED)
def test_refused_offsets_name_the_pointer_and_write_nothing(name, off):
    err, o, lse, at, (o_in, lse_in, *_) = _placed_call({name: off})
    need = 16 if name in ("Q", "K_cache", "V_cache") else 4
    assert err is not None and "%s must be %d-byte aligned" % (name, need) in err, err
    assert torch.equal(o.view(torch.uint8), o_in.view(torch.uint8))
    assert torch.equal(lse.view(torch.uint8), lse_in.view(torch.uint8))
    assert at.guards_kept()
