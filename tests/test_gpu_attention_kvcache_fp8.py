"""GPU: KV-cache attention over fp8 caches (ops.fa2_fwd_kvcache and ops.fa2_fwd_varlen(block_table=) with
float8_e4m3fn / float8_e5m2 caches).  With unit or power-of-two scales, O and lse must have the bits of the 16-bit call
on the dequantized caches (kvcache_fp8_oracle.dequantize); with arbitrary scales O is held to the tolerance
test_gpu_attention_kvcache.py uses against the CPU reference.  Also: isolation from NaN / Inf bytes past each length
and in unlisted pages, append (bytes equal the reference quantisation, nothing else written, O equal to decode on the
updated cache), paged prefill, and CUDA-graph replay while lengths, table and scales change."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attention_ref as ar  # noqa: E402
import kvcache_fp8_oracle as fo  # noqa: E402
import kvcache_oracle  # noqa: E402

pytestmark = pytest.mark.gpu
NAN8 = 0x7F  # NaN in both formats


def _ops():
    from b200k import ops

    return ops


def _caches(B, S, H_kv, D, fmt, seed, k_scale=None, v_scale=None):
    """fp8 caches [B, S, H_kv, D] on the device, quantised from randn, and their dequantized 16-bit twins per dtype."""
    g = torch.Generator().manual_seed(seed)
    k = torch.randn(B, S, H_kv, D, generator=g) * 2
    v = torch.randn(B, S, H_kv, D, generator=g) * 2
    k8, v8 = fo.quantize(k, fmt, k_scale), fo.quantize(v, fmt, v_scale)
    return k8.cuda(), v8.cuda()


def _dq(x8, dtype, scale=None):
    return fo.dequantize(x8.cpu(), dtype, scale).cuda()


def _page(k8, v8, page_size, seed, fill=None):
    """Paged copies of fp8 caches (through their bytes) under a shuffled table; unlisted pages hold `fill` bytes."""
    f = None if fill is None else (lambda shape: torch.full(shape, fill, dtype=torch.uint8))
    kp, vp, table, spare = kvcache_oracle.paged_copy(k8.view(torch.uint8), v8.view(torch.uint8), page_size, seed=seed,
                                                     fill=f)
    return kp.view(k8.dtype), vp.view(v8.dtype), table, spare


def _scales(kind, H_kv, seed):
    if kind == "unit":
        return None, None
    g = torch.Generator().manual_seed(seed)
    if kind == "pow2":
        e = torch.randint(-2, 3, (2, H_kv), generator=g).float()
        return (2.0 ** e[0]).cuda(), (2.0 ** e[1]).cuda()
    return (0.3 + torch.rand(H_kv, generator=g)).cuda(), (0.3 + torch.rand(H_kv, generator=g)).cuda()


def _pair(q, k8, v8, lens, table, causal, ks, vs):
    """(fp8 call, 16-bit call on the dequantized caches), each as (O, lse)."""
    ops = _ops()
    B, Lq, H, D = q.shape
    o8, l8 = torch.full_like(q, float("nan")), torch.full((B, Lq, H), float("nan"), device="cuda")
    ops.fa2_fwd_kvcache(q, k8, v8, o8, lens, table, causal=causal, lse=l8, k_scale=ks, v_scale=vs)
    o16, l16 = torch.full_like(q, float("nan")), torch.full((B, Lq, H), float("nan"), device="cuda")
    ops.fa2_fwd_kvcache(q, _dq(k8, q.dtype, ks), _dq(v8, q.dtype, vs), o16, lens, table, causal=causal, lse=l16)
    return (o8, l8), (o16, l16)


def _same_bits(a, b):
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int16) if x.dtype != torch.float32 else x.view(torch.int32),
                           y.view(torch.int16) if y.dtype != torch.float32 else y.view(torch.int32))


LAYOUT = {32: None, 64: 16, 96: 64, 128: 256}  # contiguous, then pages of 16, 64, 256


@pytest.mark.parametrize("scales", ["unit", "pow2"])
@pytest.mark.parametrize("D", [32, 64, 96, 128])
@pytest.mark.parametrize("fmt", fo.FORMATS, ids=["e4m3", "e5m2"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_same_bits_as_16_bit_call_on_dequantized_cache(dtype, fmt, D, scales):
    page_size = LAYOUT[D]
    causal = D in (64, 128)
    Lq = 1 if D in (32, 64) else 3
    B, H, H_kv, S = 5, 8, 2, 1024
    torch.manual_seed(D)
    q = torch.randn(B, Lq, H, D, device="cuda").to(dtype)
    ks, vs = _scales(scales, H_kv, seed=D)
    k8, v8 = _caches(B, S, H_kv, D, fmt, seed=D, k_scale=ks, v_scale=vs)
    table = None
    if page_size:
        k8, v8, table, _ = _page(k8, v8, page_size, seed=D)
    lens = torch.tensor([0, 1, 129, 700, 1024], dtype=torch.int32, device="cuda")
    got, want = _pair(q, k8, v8, lens, table, causal, ks, vs)
    assert torch.isfinite(got[0]).all()
    _same_bits(got, want)


@pytest.mark.parametrize("B", [2, 64])  # 2: split grid, 64 sequences x 2 K/V heads: one split
@pytest.mark.parametrize("H,H_kv", [(8, 8), (8, 2), (16, 1)], ids=["mha", "gqa", "mqa"])
def test_groups_and_both_sides_of_the_split_rule(B, H, H_kv):
    ops = _ops()
    D, S = 128, 2048
    torch.manual_seed(B + H_kv)
    q = torch.randn(B, 2, H, D, device="cuda").to(torch.bfloat16)
    ks, vs = _scales("pow2", H_kv, seed=B)
    k8, v8 = _caches(B, S, H_kv, D, torch.float8_e4m3fn, seed=B, k_scale=ks, v_scale=vs)
    lens = torch.randint(1, S + 1, (B,), dtype=torch.int32).cuda()
    splits = ops.fa2_fwd_kvcache_fp8_workspace_bytes(B, 2, H, H_kv, D, S) > 0
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert splits == (B * H_kv * 5 < sms * 4)
    got, want = _pair(q, k8, v8, lens, None, True, ks, vs)
    _same_bits(got, want)


@pytest.mark.parametrize("fmt", fo.FORMATS, ids=["e4m3", "e5m2"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_arbitrary_scales_against_the_reference(dtype, fmt):
    ops = _ops()
    B, Lq, H, H_kv, D, S, ps = 4, 2, 16, 4, 128, 1536, 64
    torch.manual_seed(7)
    q = torch.randn(B, Lq, H, D, device="cuda").to(dtype)
    ks, vs = _scales("any", H_kv, seed=7)
    k8, v8 = _caches(B, S, H_kv, D, fmt, seed=7, k_scale=ks, v_scale=vs)
    k8, v8, table, _ = _page(k8, v8, ps, seed=7)
    lens = torch.tensor([1, 64, 1000, 1536], dtype=torch.int32, device="cuda")
    o = torch.empty_like(q)
    ops.fa2_fwd_kvcache(q, k8, v8, o, lens, table, causal=True, k_scale=ks, v_scale=vs)
    want = ar.kvcache(q, fo.dequantize(k8.cpu(), torch.float32, ks), fo.dequantize(v8.cpu(), torch.float32, vs), lens,
                      table, causal=True)[0].to(q.dtype)
    assert torch.allclose(o.cpu().float(), want.float(), **ar.TOL[dtype])


@pytest.mark.parametrize("fmt", fo.FORMATS, ids=["e4m3", "e5m2"])
@pytest.mark.parametrize("page_size", [None, 16, 256])
def test_nan_and_inf_bytes_past_the_length_and_in_unlisted_pages_change_nothing(fmt, page_size):
    ops = _ops()
    B, H, H_kv, D, S = 3, 8, 2, 64, 512
    torch.manual_seed(3)
    q = torch.randn(B, 1, H, D, device="cuda").to(torch.float16)
    k8, v8 = _caches(B, S, H_kv, D, fmt, seed=3)
    lens = torch.tensor([5, 130, 300], dtype=torch.int32, device="cuda")
    outs = []
    for fill in (0x00, NAN8, 0x7C if fmt == torch.float8_e5m2 else 0xFF):  # zeros, NaN, Inf (e5m2) / -NaN (e4m3)
        kf, vf = k8.clone(), v8.clone()
        for b, n in enumerate(lens.tolist()):
            kf.view(torch.uint8)[b, n:] = fill
            vf.view(torch.uint8)[b, n:] = fill
        table = None
        if page_size:
            kf, vf, table, _ = _page(kf, vf, page_size, seed=3, fill=fill)
        o, lse = torch.empty_like(q), torch.empty(B, 1, H, device="cuda")
        ops.fa2_fwd_kvcache(q, kf, vf, o, lens, table, lse=lse)
        outs.append((o, lse))
    assert torch.isfinite(outs[0][0]).all()
    for other in outs[1:]:
        _same_bits(other, outs[0])


@pytest.mark.parametrize("rotary", [False, True])
@pytest.mark.parametrize("fmt", fo.FORMATS, ids=["e4m3", "e5m2"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_append_quantises_on_write_and_attends_over_the_new_keys(dtype, fmt, rotary):
    ops = _ops()
    B, Lq, H, H_kv, D, ps, pps, L_new = 3, 2, 8, 2, 128, 64, 4, 2
    torch.manual_seed(11)
    q = torch.randn(B, Lq, H, D, device="cuda").to(dtype)
    k_new = (torch.randn(B, L_new, H_kv, D, device="cuda") * 3).to(dtype)
    v_new = (torch.randn(B, L_new, H_kv, D, device="cuda") * 3).to(dtype)
    k_new[0, 0, 0, :2] = torch.tensor([6e4, -6e4], dtype=dtype)  # past both formats' largest value: saturates
    ks, vs = _scales("any", H_kv, seed=11)
    num_pages = B * pps + 2
    table = torch.randperm(num_pages)[:B * pps].view(B, pps).to(torch.int32).cuda()
    k8 = fo.quantize(torch.randn(num_pages, ps, H_kv, D), fmt, ks).cuda()
    v8 = fo.quantize(torch.randn(num_pages, ps, H_kv, D), fmt, vs).cuda()
    lens = torch.tensor([0, 100, ps * pps - 1], dtype=torch.int32, device="cuda")  # the last one overflows by one
    cos = sin = None
    if rotary:
        ang = torch.rand(ps * pps, D // 4) * 6.28
        cos, sin = ang.cos().to(dtype).cuda(), ang.sin().to(dtype).cuda()
    # x16: what the 16-bit append writes into a 16-bit cache, rotary included
    k16, v16 = torch.zeros(num_pages, ps, H_kv, D, dtype=dtype, device="cuda"), torch.zeros(num_pages, ps, H_kv, D, dtype=dtype, device="cuda")
    ops.fa2_fwd_kvcache(q, k16, v16, torch.empty_like(q), lens, table, k=k_new, v=v_new, rotary_cos=cos, rotary_sin=sin,
                        rotary_interleaved=True)
    k8_before, v8_before = k8.clone(), v8.clone()
    o = torch.full_like(q, float("nan"))
    # the C call with a workspace of our own: its rotated Q (header: lengths [B], then Q [B, Lq, H, D], 256-aligned)
    # is what the decode below must see
    from b200k import _loader as L
    nbytes = ops.fa2_fwd_kvcache_fp8_workspace_bytes(B, Lq, H, H_kv, D, ps * pps, True, rotary)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    ptr = (lambda t: t.data_ptr() if t is not None else None)
    L.check(L.lib.b200k_fa2_kvcache_fp8(
        q.data_ptr(), k8.data_ptr(), v8.data_ptr(), o.data_ptr(), None, lens.data_ptr(), table.data_ptr(), ks.data_ptr(),
        vs.data_ptr(), L.FP8_E4M3 if fmt == torch.float8_e4m3fn else L.FP8_E5M2, k_new.data_ptr(), v_new.data_ptr(),
        L_new, ptr(cos), ptr(sin), cos.size(0) if rotary else 0, D // 2 if rotary else 0, 1, B, Lq, H, H_kv, D,
        num_pages, ps, pps, 0.0, L.BF16 if dtype == torch.bfloat16 else L.F16, 0, ws.data_ptr(), nbytes,
        torch.cuda.current_stream().cuda_stream))
    want_k, want_v = k8_before.clone(), v8_before.clone()
    tab = table.cpu()
    for b, base in enumerate(lens.tolist()):
        for i in range(L_new):
            p = base + i
            if p >= ps * pps:
                continue
            pg, sl = tab[b, p // ps], p % ps
            want_k[pg, sl] = fo.quantize(k16[pg, sl].cpu()[None], fmt, ks)[0].cuda()
            want_v[pg, sl] = fo.quantize(v16[pg, sl].cpu()[None], fmt, vs)[0].cuda()
    assert torch.equal(k8.view(torch.uint8), want_k.view(torch.uint8))
    assert torch.equal(v8.view(torch.uint8), want_v.view(torch.uint8))
    # O: the decode call on the updated cache over the new lengths, with the rotated q
    assert torch.equal(ws[:4 * B].view(torch.int32), (lens + L_new).clamp(max=2 ** 31 - 1))
    q_rot = ws[256:256 + q.numel() * 2].view(dtype).view_as(q) if rotary else q
    o_dec = torch.empty_like(q)
    ops.fa2_fwd_kvcache(q_rot, k8, v8, o_dec, (lens + L_new).clamp(max=ps * pps), table, k_scale=ks, v_scale=vs)
    assert torch.equal(o.view(torch.int16), o_dec.view(torch.int16))


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("page_size", [16, 64, 256])
@pytest.mark.parametrize("fmt", fo.FORMATS, ids=["e4m3", "e5m2"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_paged_prefill_same_bits_as_varlen_on_gathered_dequantized_kv(dtype, fmt, page_size, causal):
    ops = _ops()
    H, H_kv, D = 8, 2, 128 if page_size != 64 else 64
    lq, lk = [1, 100, 300], [200, 100, 1000]
    B, S = len(lq), 1024
    torch.manual_seed(page_size)
    cu_q = torch.tensor([0] + torch.tensor(lq).cumsum(0).tolist(), dtype=torch.int32, device="cuda")
    cu_k = torch.tensor([0] + torch.tensor(lk).cumsum(0).tolist(), dtype=torch.int32, device="cuda")
    q = torch.randn(sum(lq), H, D, device="cuda").to(dtype)
    ks, vs = _scales("pow2", H_kv, seed=page_size)
    k8, v8 = _caches(B, S, H_kv, D, fmt, seed=page_size, k_scale=ks, v_scale=vs)
    kp, vp, table, _ = _page(k8, v8, page_size, seed=page_size, fill=NAN8)
    o8, l8 = torch.full_like(q, float("nan")), torch.full((sum(lq), H), float("nan"), device="cuda")
    ops.fa2_fwd_varlen(q, kp, vp, o8, cu_q, cu_k, max(lq), causal=causal, lse=l8, block_table=table, k_scale=ks,
                       v_scale=vs)
    kg, vg, _ = kvcache_oracle.gather(_dq(kp, dtype, ks), _dq(vp, dtype, vs), torch.tensor(lk), table)
    o16, l16 = torch.full_like(q, float("nan")), torch.full((sum(lq), H), float("nan"), device="cuda")
    ops.fa2_fwd_varlen(q, kg.cuda(), vg.cuda(), o16, cu_q, cu_k, max(lq), causal=causal, lse=l16)
    _same_bits((o8, l8), (o16, l16))


def test_graph_replay_follows_new_lengths_table_and_scales():
    ops = _ops()
    B, H, H_kv, D, ps, pps = 4, 8, 2, 128, 64, 8
    torch.manual_seed(5)
    q = torch.randn(B, 1, H, D, device="cuda").to(torch.float16)
    num_pages = B * pps + 4
    k8 = fo.quantize(torch.randn(num_pages, ps, H_kv, D), torch.float8_e4m3fn).cuda()
    v8 = fo.quantize(torch.randn(num_pages, ps, H_kv, D), torch.float8_e4m3fn).cuda()
    table = torch.randperm(num_pages)[:B * pps].view(B, pps).to(torch.int32).cuda()
    lens = torch.tensor([1, 100, 300, 512], dtype=torch.int32, device="cuda")
    ks, vs = torch.ones(H_kv, device="cuda"), torch.ones(H_kv, device="cuda")
    o = torch.empty_like(q)
    ops.fa2_fwd_kvcache(q, k8, v8, o, lens, table, k_scale=ks, v_scale=vs)  # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.fa2_fwd_kvcache(q, k8, v8, o, lens, table, k_scale=ks, v_scale=vs)
    for step in range(3):
        lens.copy_(torch.tensor([1 + 50 * step, 100 + step, 300 - 7 * step, 512 - step], dtype=torch.int32))
        table.copy_(torch.randperm(num_pages)[:B * pps].view(B, pps).to(torch.int32))
        ks.copy_(torch.tensor([0.5, 2.0]) * (step + 1))
        vs.copy_(torch.tensor([1.5, 0.75]) / (step + 1))
        o.fill_(float("nan"))
        g.replay()
        want = torch.empty_like(q)
        ops.fa2_fwd_kvcache(q, k8, v8, want, lens, table, k_scale=ks, v_scale=vs)
        assert torch.equal(o.view(torch.int16), want.view(torch.int16))


@pytest.mark.parametrize("fmt", fo.FORMATS, ids=["e4m3", "e5m2"])
def test_append_keeps_nan_and_saturates_inf(fmt):
    """cvt.rn.satfinite: a NaN element is stored as NaN, +-Inf as the format's largest finite value."""
    ops = _ops()
    B, H, H_kv, D, S = 2, 4, 2, 64, 128
    torch.manual_seed(13)
    q = torch.randn(B, 1, H, D, device="cuda").to(torch.float16)
    k_new = torch.randn(B, 1, H_kv, D, device="cuda").to(torch.float16)
    v_new = torch.randn(B, 1, H_kv, D, device="cuda").to(torch.float16)
    special = torch.tensor([float("nan"), -float("nan"), float("inf"), -float("inf"), 7e4], dtype=torch.float16)
    k_new[0, 0, 1, :5] = special.cuda()
    v_new[1, 0, 0, 3:8] = special.cuda()
    ks = torch.tensor([0.5, 2.0], device="cuda")
    k8 = torch.zeros(B, S, H_kv, D, dtype=torch.uint8, device="cuda").view(fmt)
    v8 = torch.zeros(B, S, H_kv, D, dtype=torch.uint8, device="cuda").view(fmt)
    lens = torch.tensor([3, 100], dtype=torch.int32, device="cuda")
    ops.fa2_fwd_kvcache(q, k8, v8, torch.empty_like(q), lens, k=k_new, v=v_new, k_scale=ks)
    for cache, new, scale in ((k8, k_new, ks), (v8, v_new, None)):
        for b, p in enumerate(lens.tolist()):
            got = cache[b, p].cpu()
            want = fo.quantize(new[b, 0].cpu(), fmt, scale)
            nan = torch.isnan(want.float())
            assert torch.equal(torch.isnan(got.float()), nan)
            assert torch.equal(got.view(torch.uint8)[~nan], want.view(torch.uint8)[~nan])
    assert torch.isnan(k8[0, 3, 1, :2].float().cpu()).all() and torch.isnan(v8[1, 100, 0, 3:5].float().cpu()).all()
    assert k8[0, 3, 1, 2:5].float().tolist() == [fo.FMAX[fmt], -fo.FMAX[fmt], fo.FMAX[fmt]]
