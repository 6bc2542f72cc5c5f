"""GPU: every kernel of libb200k.so launched by a public call and checked.  One case per case id of
kernel_inventory.COVERAGE: the case runs a small call under torch.profiler, requires the library kernels it launched to
be exactly kernel_inventory.launched(case), then checks what the call wrote.

  - Outputs go into NaN-filled buffers with guards, and the guards must keep their NaNs.
  - Attention forward: O against fp64 by the suite's rule (at most twice the error of the same math in the dtype, plus
    one ulp of the dtype), lse within 2e-3 of fp64 wherever it is written; and, where an exact identity exists, the bits:
    paged prefill against the packed call on the gathered K / V, fp8 caches with power-of-two per-head scales against
    the 16-bit call on the dequantized caches, unsplit decode against fa2_fwd_varlen, split decode against its own
    unsplit rows within the fp64 rule.
  - Append: the cache bytes are the reference rotation (and quantisation) of the new rows, O is the decode call on
    the updated cache.
  - Backward: attention_ref in fp64 by the same rule.  GEMM: integer operands, so the answer is exact.  Bandwidth
    kernels: the CPU oracle (oracle/oracle.py), exact where the operation is."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attention_ref as ar  # noqa: E402
import exact_attention as ea  # noqa: E402
import kernel_inventory as ki  # noqa: E402
import kvcache_append_oracle as kao  # noqa: E402
import kvcache_fp8_oracle as fo  # noqa: E402
import kvcache_oracle  # noqa: E402
import varlen_paged_oracle as vpo  # noqa: E402

pytestmark = pytest.mark.gpu
CASES = sorted(set(ki.COVERAGE.values()))
TORCH = {"f16": torch.float16, "bf16": torch.bfloat16, "f32": torch.float32, "tf32": torch.float32,
         "e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2, "i8": torch.int8}
GUARD = 64  # elements on each side of an output: 128 or 256 bytes, so the output keeps 16-byte alignment
LSE_ATOL = 2e-3


def _ops():
    from b200k import ops

    return ops


class _TraceLost(Exception):
    """torch.profiler returned a session without a single CUDA kernel, though the block launched some."""


class _Record:
    """The library kernels (normalised names) launched inside the block, via torch.profiler's CUDA activities."""

    def __enter__(self):
        from torch.profiler import ProfilerActivity, profile

        torch.cuda.synchronize()
        self.prof = profile(activities=[ProfilerActivity.CUDA])
        self.prof.__enter__()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.prof.__exit__(*exc)
        if exc[0] is not None:
            return False
        names = [e.name for e in self.prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        kernels = [n for n in names if not n.startswith(("Memcpy", "Memset"))]
        if not kernels:
            raise _TraceLost
        self.names = {ki.normalize(n) for n in kernels}
        self.names = {n for n in self.names if n.startswith("b200k::")}
        return False


@pytest.fixture(scope="module", autouse=True)
def _profiler_warm():
    """One profiled launch before the first case: the first session of a process can miss its kernels."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]):
        torch.ones(8, device="cuda").add_(1)
        torch.cuda.synchronize()


def _out(shape, dtype, fill=float("nan")):
    """(view of `shape` in a `fill`-filled buffer with GUARD elements on each side, the buffer)."""
    n = math.prod(shape)
    buf = torch.full((n + 2 * GUARD,), fill, dtype=dtype, device="cuda")
    return buf[GUARD:GUARD + n].view(shape), buf


def _guards(*bufs):
    for b in bufs:
        for g in (b[:GUARD], b[-GUARD:]):
            assert torch.isnan(g.float()).all(), "a guard element was written"


def _bits(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


def _same_bits(a, b, what):
    bad = _bits(a) != _bits(b)
    assert not bool(bad.any()), "%s: %d elements differ, first at %s" % (what, int(bad.sum()), bad.nonzero()[0].tolist())


# ------------------------------------------------------------------------------------------------ attention references
def _rule(got, ref, o64, what):
    """max|got - o64| <= 2 max|ref - o64| + one ulp of the dtype at max|o64| (ref: the same math in got's dtype)."""
    assert bool(torch.isfinite(got).all()), "%s: non-finite output" % what
    err, err_ref = (got.double() - o64).abs().max().item(), (ref.double() - o64).abs().max().item()
    eps = ea.ulp(o64.abs().max().view(1).cpu(), got.dtype).item()
    assert err <= 2 * err_ref + eps, (what, err, err_ref, eps)


def _lse_close(got, want, what):
    assert torch.equal(torch.isinf(got), torch.isinf(want.float())), "%s: -inf rows differ" % what
    fin = torch.isfinite(want)
    err = (got.double()[fin] - want[fin]).abs().max().item() if bool(fin.any()) else 0.0
    assert err <= LSE_ATOL, (what, err)


def _scale_pair(H_kv, seed, pow2=True):
    g = torch.Generator().manual_seed(seed)
    if pow2:  # distinct per head (where there are several), so a wrong head index shows
        e = torch.randperm(5, generator=g)[:2 * H_kv].float() - 2 if H_kv <= 2 else torch.randint(-2, 3, (2 * H_kv,), generator=g).float()
        return (2.0 ** e[:H_kv]).cuda(), (2.0 ** e[H_kv:]).cuda()
    return (0.3 + torch.rand(H_kv, generator=g)).cuda(), (0.3 + torch.rand(H_kv, generator=g)).cuda()


# ------------------------------------------------------------------------------------------------ attention forward
def _dense(toks, dt, D, lse):
    ops = _ops()
    vdn = "vdn" in toks
    B, H, N = 2, 3, 200
    causal = D in (64, 128)
    g = torch.Generator(device="cuda").manual_seed(D)
    q, k, v = (torch.randn(B, H, N, D, generator=g, device="cuda").to(dt) for _ in range(3))
    (o, ob), (l, lb) = _out((B, H, N, D), dt), _out((B, H, N), torch.float32)
    vin = v.transpose(-1, -2).contiguous() if vdn else v
    with _Record() as r:
        ops.fa2_fwd(q, k, vin, o, v_is_dn=vdn, causal=causal, lse=l if lse else None)
    _guards(ob, *([lb] if lse else []))
    if not lse:
        assert torch.isnan(l).all()
    o64, l64 = ar.dense(q, k, v, causal=causal)
    od = ar.dense(q, k, v, causal=causal, dtype=dt)[0]
    for b in range(B):
        _rule(o[b], od[b], o64[b], "dense O")
        if lse:
            _lse_close(l[b], l64[b], "dense lse")
    return r.names


def _ffpa(D):
    ops = _ops()
    B, H, N = 1, 2, 200
    g = torch.Generator(device="cuda").manual_seed(D)
    q, k, v = (torch.randn(B, H, N, D, generator=g, device="cuda").half() for _ in range(3))
    o, ob = _out((B, H, N, D), torch.float16)
    with _Record() as r:
        ops.ffpa_fwd(q, k, v, o)
    _guards(ob)
    for h in range(H):
        args = (q[0, h][:, None], k[0, h][:, None], v[0, h][:, None], 1 / math.sqrt(D))
        _rule(o[0, h][:, None], ar.sequence(*args, dtype=torch.float16)[0], ar.sequence(*args)[0], "ffpa O")
    return r.names


LQ, LK = [1, 130, 70, 0], [200, 130, 50, 77]  # a one-token sequence, Lq = Lk, Lq > Lk (causal: rows with no key), empty


def _packed_inputs(dt, D, H, H_kv, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    cu_q = torch.tensor([0] + torch.tensor(LQ).cumsum(0).tolist(), dtype=torch.int32, device="cuda")
    cu_k = torch.tensor([0] + torch.tensor(LK).cumsum(0).tolist(), dtype=torch.int32, device="cuda")
    q = torch.randn(sum(LQ), H, D, generator=g, device="cuda").to(dt)
    k, v = (torch.randn(sum(LK), H_kv, D, generator=g, device="cuda").to(dt) for _ in range(2))
    return q, k, v, cu_q, cu_k


def _check_packed(o, l, lse, q, k, v, cu_q, cu_k, causal, what):
    o64, l64 = ar.packed(q, k, v, cu_q, cu_k, causal=causal)
    _rule(o, ar.packed(q, k, v, cu_q, cu_k, causal=causal, dtype=q.dtype)[0], o64, what + " O")
    if lse:
        _lse_close(l, l64, what + " lse")


def _packed(toks, dt, D, lse):
    ops = _ops()
    H, H_kv, causal = 4, 2, lse
    q, k, v, cu_q, cu_k = _packed_inputs(dt, D, H, H_kv, D)
    (o, ob), (l, lb) = _out(q.shape, dt), _out(q.shape[:2], torch.float32)
    with _Record() as r:
        ops.fa2_fwd_varlen(q, k, v, o, cu_q, cu_k, max(LQ), causal=causal, lse=l if lse else None)
    _guards(ob, lb)
    _check_packed(o, l, lse, q, k, v, cu_q, cu_k, causal, "packed")
    return r.names


def _paged(toks, dt, D, lse, fmt):
    """Paged prefill over a shuffled table; every slot past a sequence's length in its listed pages, and every unlisted
    page, holds NaN.  16-bit: the bits of the packed call on the gathered K / V.  fp8 (distinct power-of-two scales per
    K/V head): the bits of the 16-bit paged call on the dequantized caches."""
    ops = _ops()
    H = 8
    H_kv = {32: 1, 64: 2, 96: 8, 128: 4}[D]  # MQA, G = 4, G = 1, G = 2
    page_size = {32: 16, 64: 64, 96: 32, 128: 256}[D]
    causal = D in (64, 96)
    q, k, v, cu_q, cu_k = _packed_inputs(dt, D, H, H_kv, 10 + D)
    ks = vs = None
    if fmt:
        ks, vs = _scale_pair(H_kv, D)
        k8, v8 = fo.quantize(k.cpu(), TORCH[fmt], ks), fo.quantize(v.cpu(), TORCH[fmt], vs)
        kc, vc, table = vpo.to_pages(k8.view(torch.uint8), v8.view(torch.uint8), cu_k.cpu(), page_size, fill=0x7F, seed=D)
        kc, vc, table = kc.view(TORCH[fmt]).cuda(), vc.view(TORCH[fmt]).cuda(), table.cuda()
        k, v = fo.dequantize(k8, dt, ks).cuda(), fo.dequantize(v8, dt, vs).cuda()  # what the cache holds, in dt
    else:
        kc, vc, table = vpo.to_pages(k, v, cu_k, page_size, fill=float("nan"), seed=D)
    (o, ob), (l, lb) = _out(q.shape, dt), _out(q.shape[:2], torch.float32)
    with _Record() as r:
        ops.fa2_fwd_varlen(q, kc, vc, o, cu_q, cu_k, max(LQ), causal=causal, lse=l if lse else None, block_table=table,
                           k_scale=ks, v_scale=vs)
    _guards(ob, lb)
    (o2, _), (l2, _) = _out(q.shape, dt), _out(q.shape[:2], torch.float32)
    if fmt:
        kd, vd = fo.dequantize(kc.cpu(), dt, ks).cuda(), fo.dequantize(vc.cpu(), dt, vs).cuda()  # NaN bytes stay NaN
        ops.fa2_fwd_varlen(q, kd, vd, o2, cu_q, cu_k, max(LQ), causal=causal, lse=l2 if lse else None, block_table=table)
        what = "fp8 paged vs 16-bit paged on the dequantized caches"
    else:
        ops.fa2_fwd_varlen(q, k, v, o2, cu_q, cu_k, max(LQ), causal=causal, lse=l2 if lse else None)
        what = "paged vs packed on the gathered K / V"
    _same_bits(o, o2, what + ": O")
    if lse:
        _same_bits(l, l2, what + ": lse")
    _check_packed(o, l, lse, q, k, v, cu_q, cu_k, causal, "paged")
    return r.names


def _decode(toks, dt, D, lse, fmt):
    """Unsplit: 64 sequences x 2 K/V heads fill the SMs; split: 2 sequences.  16-bit unsplit: the bits of
    fa2_fwd_varlen on the same tokens; fp8 (distinct power-of-two scales): the bits of the 16-bit call on the
    dequantized caches, workspace included; every case: O and lse against fp64."""
    ops = _ops()
    split = "split" in toks
    B, Lq, H, H_kv, S = (2, 2, 8, 2, 1024) if split else (64, 1, 8, 2, 256)
    nbytes = (ops.fa2_fwd_kvcache_fp8_workspace_bytes if fmt else ops.fa2_fwd_kvcache_workspace_bytes)(B, Lq, H, H_kv, D, S)
    assert (nbytes > 0) == split, "this shape was meant to run %s" % ("split" if split else "unsplit")
    g = torch.Generator(device="cuda").manual_seed(D + 7 * split)
    q = torch.randn(B, Lq, H, D, generator=g, device="cuda").to(dt)
    kc, vc = (torch.randn(B, S, H_kv, D, generator=g, device="cuda").to(dt) for _ in range(2))
    lens = torch.randint(1, S + 1, (B,), generator=torch.Generator().manual_seed(D)).to(torch.int32)
    lens[0] = 0 if not split else lens[0]
    lens = lens.cuda()
    ks = vs = None
    if fmt:
        ks, vs = _scale_pair(H_kv, D + 1)
        k8, v8 = fo.quantize(kc.cpu(), TORCH[fmt], ks).cuda(), fo.quantize(vc.cpu(), TORCH[fmt], vs).cuda()
        kc, vc = fo.dequantize(k8.cpu(), dt, ks).cuda(), fo.dequantize(v8.cpu(), dt, vs).cuda()
    causal = Lq > 1
    (o, ob), (l, lb) = _out(q.shape, dt), _out(q.shape[:3], torch.float32)
    with _Record() as r:
        ops.fa2_fwd_kvcache(q, k8 if fmt else kc, v8 if fmt else vc, o, lens, causal=causal, lse=l if lse else None,
                            k_scale=ks, v_scale=vs)
    _guards(ob, lb)
    if not lse:
        assert torch.isnan(l).all()
    # the exact identity
    (o2, _), (l2, _) = _out(q.shape, dt), _out(q.shape[:3], torch.float32)
    if fmt:
        ops.fa2_fwd_kvcache(q, kc, vc, o2, lens, causal=causal, lse=l2 if lse else None)
        _same_bits(o, o2, "fp8 decode vs 16-bit decode on the dequantized caches: O")
    kg, vg, cu_k = kvcache_oracle.gather(kc, vc, lens.cpu())
    kg, vg, cu_k = kg.cuda(), vg.cuda(), cu_k.cuda()
    cu_q = torch.arange(B + 1, dtype=torch.int32, device="cuda") * Lq
    if not split and not fmt:
        ov = torch.full((B * Lq, H, D), float("nan"), dtype=dt, device="cuda")
        ops.fa2_fwd_varlen(q.view(B * Lq, H, D), kg, vg, ov, cu_q, cu_k, Lq, causal=causal)
        _same_bits(o.view(B * Lq, H, D), ov, "unsplit decode vs fa2_fwd_varlen: O")
    if lse and fmt:
        _same_bits(l, l2, "fp8 decode vs 16-bit decode: lse")
    o64, l64 = ar.packed(q.view(B * Lq, H, D), kg, vg, cu_q, cu_k, causal=causal)
    _rule(o.view(B * Lq, H, D), ar.packed(q.view(B * Lq, H, D), kg, vg, cu_q, cu_k, causal=causal, dtype=dt)[0], o64,
          "decode O")
    if lse:
        _lse_close(l.view(B * Lq, H), l64, "decode lse")
    return r.names


def _append(toks, dt, fmt):
    """Append two tokens per sequence (one sequence overflows its capacity by one) into paged caches with NeoX rotary
    over rotary_dim = D, interleaved over D / 2, or none, then decode (unsplit: 256 keys per sequence).  16-bit caches: V rows copied bit for bit,
    rotated K columns within one ulp of the fp64 rotation, every other byte unchanged.  fp8 caches (arbitrary per-head
    scales): every byte equals the reference quantisation of what the 16-bit append writes.  O: the decode call on the
    updated cache (its bits without rotary; with rotary, the fp64 rule on the reference-rotated Q)."""
    ops = _ops()
    rot = toks[-1]
    B, Lq, H, H_kv, D, ps, pps, L_new = 3, 2, 8, 2, 128, 64, 4, 2
    g = torch.Generator(device="cuda").manual_seed(len(rot))
    q = torch.randn(B, Lq, H, D, generator=g, device="cuda").to(dt)
    k_new, v_new = ((torch.randn(B, L_new, H_kv, D, generator=g, device="cuda") * 2).to(dt) for _ in range(2))
    num_pages = B * pps + 2
    table = torch.randperm(num_pages, generator=torch.Generator().manual_seed(3))[:B * pps].view(B, pps).to(torch.int32)
    table = table.cuda()
    lens = torch.tensor([0, 100, ps * pps - 1], dtype=torch.int32, device="cuda")
    cos = sin = None
    if rot != "plain":
        rd = D if rot == "neox" else D // 2
        ang = torch.rand(ps * pps, rd // 2, generator=torch.Generator().manual_seed(5)) * 6.28
        cos, sin = ang.cos().to(dt).cuda(), ang.sin().to(dt).cuda()
    kw = dict(k=k_new, v=v_new, rotary_cos=cos, rotary_sin=sin, rotary_interleaved=rot == "inter")
    ks = vs = None
    if fmt:
        ks, vs = _scale_pair(H_kv, 9, pow2=False)
        kc = fo.quantize(torch.randn(num_pages, ps, H_kv, D), TORCH[fmt], ks).cuda()
        vc = fo.quantize(torch.randn(num_pages, ps, H_kv, D), TORCH[fmt], vs).cuda()
    else:
        kc, vc = (torch.randn(num_pages, ps, H_kv, D, generator=g, device="cuda").to(dt) for _ in range(2))
    k_before, v_before = kc.cpu(), vc.cpu()
    o, ob = _out(q.shape, dt)
    with _Record() as r:
        ops.fa2_fwd_kvcache(q, kc, vc, o, lens, table, causal=True, k_scale=ks, v_scale=vs, **kw)
    _guards(ob)
    kpos = lens.cpu().long().view(B, 1) + torch.arange(L_new).view(1, L_new)
    if fmt:  # the rows the 16-bit append writes, quantised by the reference
        k16, v16 = (torch.zeros(num_pages, ps, H_kv, D, dtype=dt, device="cuda") for _ in range(2))
        ops.fa2_fwd_kvcache(q, k16, v16, torch.empty_like(q), lens, table, causal=True, **kw)
        tab = table.cpu().long()
        rows = [[k16[tab[b, p // ps], p % ps] for p in kpos[b].tolist() if p < ps * pps] for b in range(B)]
        vrows = [[v16[tab[b, p // ps], p % ps] for p in kpos[b].tolist() if p < ps * pps] for b in range(B)]
        k_rows = torch.stack([torch.stack(x + [x[0]] * (L_new - len(x))) for x in rows]).cpu()
        v_rows = torch.stack([torch.stack(x + [x[0]] * (L_new - len(x))) for x in vrows]).cpu()
        want_k = kao.write(k_before.view(torch.uint8), fo.quantize(k_rows, TORCH[fmt], ks).view(torch.uint8), lens, table)
        want_v = kao.write(v_before.view(torch.uint8), fo.quantize(v_rows, TORCH[fmt], vs).view(torch.uint8), lens, table)
        _same_bits(kc.cpu().view(torch.uint8), want_k, "fp8 K cache after append")
        _same_bits(vc.cpu().view(torch.uint8), want_v, "fp8 V cache after append")
    else:
        k_rot = kao.rotate(k_new, cos, sin, kpos, rot == "inter") if cos is not None else k_new.cpu()
        want_k, want_v = kao.write(k_before, k_rot, lens, table), kao.write(v_before, v_new, lens, table)
        _same_bits(vc.cpu(), want_v, "V cache after append")
        err = (kc.cpu().double() - want_k.double()).abs()
        assert bool((err <= ea.ulp(want_k.double().abs(), dt)).all()), "K cache after append: %g" % err.max().item()
        if cos is None:
            _same_bits(kc.cpu(), want_k, "K cache after append")
    new_lens = (lens + L_new).clamp(max=ps * pps)
    if cos is None:
        o_dec = torch.empty_like(q)
        ops.fa2_fwd_kvcache(q, kc, vc, o_dec, new_lens, table, causal=True, k_scale=ks, v_scale=vs)
        _same_bits(o, o_dec, "append O vs decode on the updated cache")
    qpos = lens.cpu().long().view(B, 1) + torch.arange(Lq).view(1, Lq)
    q_rot = (kao.rotate(q, cos, sin, qpos, rot == "inter") if cos is not None else q.cpu()).cuda()
    kd = fo.dequantize(kc.cpu(), dt, ks) if fmt else kc.cpu()
    vd = fo.dequantize(vc.cpu(), dt, vs) if fmt else vc.cpu()
    kg, vg, cu_k = (t.cuda() for t in kvcache_oracle.gather(kd, vd, new_lens.cpu(), table.cpu()))
    cu_q = torch.arange(B + 1, dtype=torch.int32, device="cuda") * Lq
    q_rot = q_rot.view(B * Lq, H, D)
    _rule(o.view(B * Lq, H, D), ar.packed(q_rot, kg, vg, cu_q, cu_k, causal=True, dtype=dt)[0],
          ar.packed(q_rot, kg, vg, cu_q, cu_k, causal=True)[0], "append O")
    return r.names


def _merge(toks, dt, lse):
    ops = _ops()
    S, rows, D = 3, 50, 64
    g = torch.Generator(device="cuda").manual_seed(S)
    parts = torch.randn(S, rows, D, generator=g, device="cuda").to(dt)
    lp = torch.randn(S, rows, generator=g, device="cuda") * 3
    lp[1, :5] = float("-inf")
    lp[:, 7] = float("-inf")  # a row no part saw a key for
    parts[1, :5] = float("nan")  # skipped parts: whatever they hold never reaches the result
    (o, ob), (l, lb) = _out((rows, D), dt), _out((rows,), torch.float32)
    with _Record() as r:
        ops.attn_merge(parts, lp, o, l if lse else None)
    _guards(ob, lb)
    import lse_oracle
    o64, l64 = lse_oracle.merge(parts, lp)
    assert torch.equal(o[7].float().cpu(), torch.zeros(D))
    err = (o.double().cpu() - o64).abs().max().item()
    assert err <= ea.ulp(o64.abs().max().view(1), dt).item() * 2, err
    if lse:
        _lse_close(l, l64.cuda(), "merge lse")
    else:
        assert torch.isnan(l).all()
    return r.names


def _bwd(toks, dt, D):
    ops = _ops()
    packed = toks[1] == "packed"
    g = torch.Generator(device="cuda").manual_seed(D + packed)
    if not packed:
        B, H, N = 2, 2, 150
        q, k, v, do = (torch.randn(B, H, N, D, generator=g, device="cuda").to(dt) for _ in range(4))
        sl = torch.tensor([150, 77], dtype=torch.int32, device="cuda")
        o, lse = torch.empty_like(q), torch.empty(B, H, N, device="cuda")
        ops.fa2_fwd(q, k, v, o, causal=True, seqlens_k=sl, lse=lse)
        outs = [_out(q.shape, dt) for _ in range(3)]
        with _Record() as r:
            ops.fa2_bwd(q, k, v, o, lse, do, *(t for t, _ in outs), causal=True, seqlens_k=sl)
        _guards(*(b for _, b in outs))
        g64 = ar.dense_grads(q, k, v, do, None, True, sl)[:3]
        qa, ka, va = (t.clone().requires_grad_() for t in (q, k, v))
        ar.dense(qa, ka, va, None, True, sl, dt)[0].backward(do)
        ref = (qa.grad, ka.grad, va.grad)
    else:
        H, H_kv = 4, 2
        lq, lk = [70, 130], [90, 150]
        cu_q = torch.tensor([0, 70, 200], dtype=torch.int32, device="cuda")
        cu_k = torch.tensor([0, 90, 240], dtype=torch.int32, device="cuda")
        q, do = (torch.randn(200, H, D, generator=g, device="cuda").to(dt) for _ in range(2))
        k, v = (torch.randn(240, H_kv, D, generator=g, device="cuda").to(dt) for _ in range(2))
        o, lse = torch.empty_like(q), torch.empty(200, H, device="cuda")
        ops.fa2_fwd_varlen(q, k, v, o, cu_q, cu_k, 130, causal=True, lse=lse)
        outs = [_out(q.shape, dt), _out(k.shape, dt), _out(k.shape, dt)]
        with _Record() as r:
            ops.fa2_bwd_varlen(q, k, v, o, lse, do, *(t for t, _ in outs), cu_q, cu_k, 130, 150, causal=True)
        _guards(*(b for _, b in outs))
        g64, ref = [torch.zeros_like(t, dtype=torch.float64) for t in (q, k, v)], [torch.zeros_like(t) for t in (q, k, v)]
        for (q0, q1), (k0, k1) in zip(((0, 70), (70, 200)), ((0, 90), (90, 240))):
            parts = [t[a:b].transpose(0, 1)[None] for t, a, b in ((q, q0, q1), (k, k0, k1), (v, k0, k1), (do, q0, q1))]
            rep = [parts[0], parts[1].repeat_interleave(H // H_kv, 1), parts[2].repeat_interleave(H // H_kv, 1), parts[3]]
            off = (k1 - k0) - (q1 - q0)
            mask = torch.ones(q1 - q0, k1 - k0, dtype=torch.bool, device="cuda").tril(off)
            for cd, dst in ((torch.float64, g64), (dt, ref)):
                a = [t.to(cd).detach().requires_grad_() for t in rep[:3]]
                torch.nn.functional.scaled_dot_product_attention(*a, attn_mask=mask).backward(rep[3].to(cd))
                grads = [a[0].grad, a[1].grad.view(1, H_kv, H // H_kv, k1 - k0, D).sum(2),
                         a[2].grad.view(1, H_kv, H // H_kv, k1 - k0, D).sum(2)]
                for t, gr, x0, x1 in zip(dst, grads, (q0, k0, k0), (q1, k1, k1)):
                    t[x0:x1] = gr[0].transpose(0, 1).to(t.dtype)
    for name, a, rf, w in zip(("dq", "dk", "dv"), (t for t, _ in outs), ref, g64):
        _rule(a, rf, w.to(a.device), "bwd " + name)
    return r.names


def _gemm(toks, dt):
    """Operands in {-1, 0, 1}: every partial sum is an integer of magnitude <= K, exact in each dtype, so C must be
    the exact product."""
    ops = _ops()
    layout = toks[2]
    M, N, K = 200, 264, 136
    t = TORCH[dt]
    g = torch.Generator(device="cuda").manual_seed(len(layout))
    a = torch.randint(-1, 2, (M, K), generator=g, device="cuda").to(t)
    b = torch.randint(-1, 2, (K, N), generator=g, device="cuda").to(t)
    c, cb = _out((M, N), t)
    a_in = a.t().contiguous().t() if layout.startswith("km") else a
    b_in = b if layout.endswith("nn") else b.t().contiguous().t()
    with _Record() as r:
        ops.gemm(a_in, b_in, c, tn=not layout.endswith("nn"), a_km=layout.startswith("km"))
    _guards(cb)
    _same_bits(c, (a.double() @ b.double()).to(t), "gemm C")
    return r.names


# ------------------------------------------------------------------------------------------------ bandwidth kernels
def _support(toks, fam):
    from oracle import oracle

    ops = _ops()
    dt = next((x for x in toks[1:] if x in TORCH), None)
    t = TORCH.get(dt)
    g = torch.Generator(device="cuda").manual_seed(len(toks[0]) + len(toks))
    if fam in ("softmax", "rmsnorm", "layernorm"):
        H = int(toks[-1][1:])
        x = torch.randn(40, H, generator=g, device="cuda").to(t)
        y, yb = _out(x.shape, t)
        tol = dict(rtol=1e-3, atol=1e-5) if t == torch.float32 else dict(rtol=2e-3, atol=4e-3)
        if toks[2:3] == ["m0"]:
            tol = dict(rtol=1e-3, atol=1e-10)
        with _Record() as r:
            if fam == "softmax":
                ops.softmax(x, y, int(toks[2][1]))
            elif fam == "rmsnorm":
                ops.rms_norm(x, y, 1.5, acc_f16="acc16" in toks)
            else:
                ops.layer_norm(x, y, 1.5, 0.25)
        _guards(yb)
        if fam == "softmax":
            want = oracle.softmax_all(x) if toks[2] == "m0" else torch.softmax(x.double().cpu(), -1)
        elif fam == "rmsnorm":
            want = oracle.rms_norm(x.double(), 1.5)
            if "acc16" in toks:
                tol = dict(rtol=2e-2, atol=2e-2)
        else:
            want = oracle.layer_norm(x, 1.5, 0.25)
        assert torch.allclose(y.double().cpu(), want.double(), **tol), (y.double().cpu() - want.double()).abs().max()
        return r.names
    if fam == "reduce":
        n = 1 << 16
        if dt == "i8":
            x = torch.randint(-100, 100, (n,), generator=g, device="cuda").to(torch.int8)
        else:
            x = (torch.randn(n, generator=g, device="cuda") * 4).to(t)
        with _Record() as r:
            got = ops.block_all_reduce_sum(x, acc_f16="acc16" in toks)
        want = oracle.reduce_sum(x)
        if dt == "i8":
            assert int(got.item()) == want
        else:
            tol = 0.5 + 1e-2 * float(x.float().abs().sum()) if "acc16" in toks else 1e-4 * float(x.float().abs().sum())
            assert abs(float(got.item()) - want) <= tol, (float(got.item()), want)
        return r.names
    if fam == "add":
        n = 10007
        off = 1 if toks[2] == "scalar" else 0  # one element in: not 16-byte aligned
        a, b = (torch.randn(n + 1, generator=g, device="cuda").to(t)[off:off + n] for _ in range(2))
        cbuf = torch.full((n + 2 * GUARD + 1,), float("nan"), dtype=t, device="cuda")
        c = cbuf[GUARD + off:GUARD + off + n]
        with _Record() as r:
            ops.elementwise_add(a, b, c)
        assert torch.isnan(cbuf[:GUARD + off].float()).all() and torch.isnan(cbuf[GUARD + off + n:].float()).all()
        _same_bits(c.cpu(), oracle.elementwise_add(a, b), "add")
        return r.names
    if fam == "hist":
        a = torch.randint(0, 9000 if toks[1] == "global" else 300, (50000,), generator=g, device="cuda").to(torch.int32)
        nb = None if toks[1] == "auto" else 10000
        with _Record() as r:
            h = ops.histogram_i32(a, nb)
        want = torch.bincount(a.cpu().long(), minlength=nb or 0).to(torch.int32)
        assert torch.equal(h.cpu(), want)
        return r.names
    if fam == "embedding":
        w = torch.randn(500, 96, generator=g, device="cuda")
        idx = torch.randint(0, 500, (300,), generator=g, device="cuda").to(torch.int32)
        out, ob = _out((300, 96), torch.float32)
        with _Record() as r:
            ops.embedding(idx, w, out)
        _guards(ob)
        assert torch.equal(out.cpu(), oracle.embedding(idx, w))
        return r.names
    if fam == "rope":
        x = torch.randn(64, 128, generator=g, device="cuda")
        out, ob = _out(x.shape, torch.float32)
        with _Record() as r:
            ops.rope_f32(x, out, ref_quirk=False)
        _guards(ob)
        assert torch.allclose(out.cpu(), oracle.rope(x, False), rtol=1e-3, atol=1e-3)
        return r.names
    if fam == "dot":
        a, b = (torch.randn(30001, generator=g, device="cuda").to(t) for _ in range(2))
        with _Record() as r:
            got = ops.dot_prod(a, b)
        want = oracle.dot_prod(a, b)
        assert abs(float(got.item()) - want) <= 1e-5 * float((a.double() * b.double()).abs().sum()), (float(got.item()), want)
        return r.names
    if fam == "gemv":
        a = torch.randn(333, 1032, generator=g, device="cuda").to(t)
        x = torch.randn(1032, generator=g, device="cuda").to(t)
        y, yb = _out((333,), t)
        with _Record() as r:
            ops.gemv(a, x, y)
        _guards(yb)
        want = oracle.gemv(a, x).view(-1)
        bound = 1e-5 * (a.double().abs() @ x.double().abs()).cpu()
        if t != torch.float32:
            bound = bound + ea.ulp(want.abs(), t)
        assert bool(((y.double().cpu() - want).abs() <= bound).all())
        return r.names
    if fam == "transpose":
        if toks[1] == "u16":
            x = torch.randn(3, 70, 130, generator=g, device="cuda").half()
            y, yb = _out((3, 130, 70), torch.float16)
            with _Record() as r:
                ops.transpose_16bit_batched(x, y)
            want = x.transpose(-1, -2)
        else:
            M, N = (200, 132) if toks[1] == "f32x4" else (201, 133)
            x = torch.randn(M, N, generator=g, device="cuda")
            y, yb = _out((N, M), torch.float32)
            with _Record() as r:
                ops.mat_transpose(x, y)
            want = x.t()
        _guards(yb)
        _same_bits(y, want.contiguous(), "transpose")
        return r.names
    if fam == "act":
        op = toks[2]
        x = (torch.randn(10003, generator=g, device="cuda") * 6).to(t)
        x[:4] = torch.tensor([-100.0, 100.0, 0.5, -0.5], device="cuda").to(t)
        y, yb = _out(x.shape, t)
        with _Record() as r:
            ops.activation(x, y, op, ref_clamp="clamp" in toks)
        _guards(yb)
        want = oracle.activation(x, op, ref_clamp="clamp" in toks)
        tol = dict(rtol=1e-4, atol=1e-6) if t == torch.float32 else dict(rtol=2e-3, atol=2e-3)
        assert torch.allclose(y.double().cpu(), want, **tol), (y.double().cpu() - want).abs().max()
        return r.names
    raise KeyError(fam)


def _run(case):
    toks = case.split("-")
    fam = toks[0]
    dt = TORCH.get(next((x for x in toks[1:] if x in ("f16", "bf16")), "f16"))
    fmt = next((x for x in toks[2:] if x in ki.FMT), None)
    D = next((int(x[1:]) for x in toks[1:] if x[0] == "d" and x[1:].isdigit()), None)
    lse = "lse" in toks
    if fam == "dense":
        return _dense(toks, dt, D, lse)
    if fam == "ffpa":
        return _ffpa(D)
    if fam == "packed":
        return _packed(toks, dt, D, lse)
    if fam == "paged":
        return _paged(toks, dt, D, lse, fmt)
    if fam == "decode":
        return _decode(toks, dt, D, lse, fmt)
    if fam == "append":
        return _append(toks, dt, fmt)
    if fam == "merge":
        return _merge(toks, dt, lse)
    if fam == "bwd":
        return _bwd(toks, dt, D)
    if fam == "gemm":
        return _gemm(toks, toks[1])
    return _support(toks, fam)


@pytest.mark.parametrize("case", CASES)
def test_case_launches_exactly_its_kernels_and_is_right(case):
    # Now and then a short profiler session comes back empty.  Each case builds its own inputs, so it runs once more;
    # a second empty session fails the case rather than skipping its launch check.
    try:
        got = _run(case)
    except _TraceLost:
        try:
            got = _run(case)
        except _TraceLost:
            pytest.fail("torch.profiler recorded no CUDA kernel in two runs: the launch check cannot run")
    want = ki.launched(case)
    assert got == want, "launched %s\nexpected %s" % (sorted(got - want), sorted(want - got))
