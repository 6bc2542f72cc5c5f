"""GPU: attention at pointer offsets.  Every tensor of these tests sits inside a byte buffer, at a chosen offset from a
256-byte boundary, with GUARD bytes of 0xFF (NaN in fp16, bf16 and fp32) on each side.

  - accepted offsets (O at +4, +8, +12; lse and the int32 arrays at +4; Q, K, V, the caches, the new rows, cos and sin
    at +16 and +48; the workspace at +16) give the bits of the same call on fresh tensors, in every mode, and that
    fresh call gives its exact answer (exact_attention.py); no byte outside an output changes;
  - refused offsets (O at +2, +6, +10, +14; a split call's workspace at +4, +8; Q and the caches at +2, +4, +8) return
    B200K_EALIGN through the C ABI and raise through ops, naming the pointer, before anything runs: O, lse, the caches
    and the block table keep every bit and the stream stays clean;
  - the Python drop-ins refuse an O one fp16 element into a buffer and accept one two elements in."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))  # the helpers sit next to this file
import exact_attention as ex  # noqa: E402
import test_gpu_attention_exact as gx  # noqa: E402

from b200k import _loader as L  # noqa: E402

pytestmark = pytest.mark.gpu
GUARD = 4096          # bytes of 0xFF on each side: more than one row of any O below
DT = {torch.float16: L.F16, torch.bfloat16: L.BF16}


def _ops():
    from b200k import ops

    return ops


class Placed:
    """Tensors placed at byte offsets inside 0xFF-filled buffers; guards_kept() checks every buffer outside its tensor."""

    def __init__(self):
        self.items = []

    def __call__(self, t, off):
        """A copy of t at byte `off` from a 256-byte boundary (t = (shape, dtype): an output, all 0xFF)."""
        shape, dtype = (t.shape, t.dtype) if isinstance(t, torch.Tensor) else t
        n = math.prod(shape) * torch.empty((), dtype=dtype).element_size()
        buf = torch.full((GUARD + off + n + GUARD,), 0xFF, dtype=torch.uint8, device="cuda")
        assert buf.data_ptr() % 256 == 0
        view = buf[GUARD + off:GUARD + off + n].view(dtype).view(shape)
        if isinstance(t, torch.Tensor):
            view.copy_(t)
        assert view.data_ptr() % 256 == off
        self.items.append((view, buf, GUARD + off, n))
        return view

    def guards_kept(self):
        torch.cuda.synchronize()
        return all(bool((b[:s] == 0xFF).all()) and bool((b[s + n:] == 0xFF).all()) for _, b, s, n in self.items)


def _same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------ cases
# Each case builds fresh inputs once and offers fresh(): (outputs...) through ops, check(outputs) against the exact
# answer, and placed(offsets, P): the same call through the C ABI with each tensor placed by P at offsets[name]
# (default 16 for inputs, 4 for outputs and int32 arrays), returning (rc, outputs).

class Dense:
    def __init__(self, dtype, causal, lens, v_dn=False, D=64, ffpa=False, seed=0):
        B = len(lens) if lens else 2
        N = 200 if not ffpa else 300
        pin = (0, 63, 64 * ((D - 1) // 64), D - 1) if ffpa else (0, D - 1)
        self.q, self.k, v, self.sl, self.spec = gx._dense(B, 2, N, D, dtype, causal, lens, seed, pin=pin)
        self.v = v.transpose(-1, -2).contiguous() if v_dn else v
        self.dtype, self.causal, self.v_dn, self.ffpa = dtype, causal, v_dn, ffpa
        self.lse = not ffpa
        self.names = ["Q", "K", "V", "O"] + (["lse"] if self.lse else []) + (["seqlens_k"] if self.sl is not None else [])

    def fresh(self):
        o = torch.full_like(self.q, float("nan"))
        lse = torch.full(self.q.shape[:-1], float("nan"), device="cuda") if self.lse else None
        if self.ffpa:
            _ops().ffpa_fwd(self.q, self.k, self.v, o)
        else:
            _ops().fa2_fwd(self.q, self.k, self.v, o, v_is_dn=self.v_dn, causal=self.causal, seqlens_k=self.sl, lse=lse)
        return o, lse

    def check(self, out):
        gx._check(out[0], self.spec, self.dtype)

    def placed(self, offs, P):
        q, k, v = (P(t, offs.get(n, 16)) for t, n in ((self.q, "Q"), (self.k, "K"), (self.v, "V")))
        o = P((self.q.shape, self.dtype), offs.get("O", 4))
        lse = P((self.q.shape[:-1], torch.float32), offs.get("lse", 4)) if self.lse else None
        sl = P(self.sl, offs.get("seqlens_k", 4)) if self.sl is not None else None
        B, H, N, D = self.q.shape
        if self.ffpa:
            rc = L.lib.b200k_ffpa_fwd_f16(_p(q), _p(k), _p(v), _p(o), B, H, N, D, 0.0, 0, _stream())
        else:
            rc = L.lib.b200k_fa2_fwd_lse(_p(q), _p(k), _p(v), _p(o), _p(lse), B, H, N, D, 0.0, int(self.v_dn),
                                         DT[self.dtype], int(self.causal), _p(sl), 0, _stream())
        return rc, (o, lse)

    def via_ops(self, offs, P):
        q, k, v = (P(t, offs.get(n, 16)) for t, n in ((self.q, "Q"), (self.k, "K"), (self.v, "V")))
        o = P((self.q.shape, self.dtype), offs.get("O", 4))
        if self.ffpa:
            _ops().ffpa_fwd(q, k, v, o)
        else:
            _ops().fa2_fwd(q, k, v, o, v_is_dn=self.v_dn, causal=self.causal, seqlens_k=self.sl)


class Packed:
    def __init__(self, dtype, causal, seed=0):
        self.q, self.k, self.v, self.cq, self.ck, self.spec = gx._varlen(gx.LQ, gx.LK, 8, 2, 64, dtype, causal, seed)
        self.dtype, self.causal = dtype, causal
        self.names = ["Q", "K", "V", "O", "lse", "cu_seqlens_q", "cu_seqlens_k"]

    def fresh(self):
        o = torch.full_like(self.q, float("nan"))
        lse = torch.full(self.q.shape[:-1], float("nan"), device="cuda")
        _ops().fa2_fwd_varlen(self.q, self.k, self.v, o, self.cq, self.ck, max(gx.LQ), causal=self.causal, lse=lse)
        return o, lse

    def check(self, out):
        gx._check(out[0], self.spec, self.dtype)

    def placed(self, offs, P):
        q, k, v = (P(t, offs.get(n, 16)) for t, n in ((self.q, "Q"), (self.k, "K"), (self.v, "V")))
        o = P((self.q.shape, self.dtype), offs.get("O", 4))
        lse = P((self.q.shape[:-1], torch.float32), offs.get("lse", 4))
        cq, ck = P(self.cq, offs.get("cu_seqlens_q", 4)), P(self.ck, offs.get("cu_seqlens_k", 4))
        tq, H, D = self.q.shape
        rc = L.lib.b200k_fa2_fwd_varlen_lse(_p(q), _p(k), _p(v), _p(o), _p(lse), _p(cq), _p(ck), self.cq.numel() - 1,
                                            max(gx.LQ), tq, self.k.size(0), H, self.k.size(1), D, 0.0, DT[self.dtype],
                                            int(self.causal), _stream())
        return rc, (o, lse)

    def via_ops(self, offs, P):
        q, k, v = (P(t, offs.get(n, 16)) for t, n in ((self.q, "Q"), (self.k, "K"), (self.v, "V")))
        o = P((self.q.shape, self.dtype), offs.get("O", 4))
        _ops().fa2_fwd_varlen(q, k, v, o, self.cq, self.ck, max(gx.LQ), causal=self.causal)


class Decode:
    """KV-cache decode (append=False: gx._decode's inputs) or append with NeoX rotary over 32 of 64 columns (append=True:
    test_append_exact's inputs with Lq = 2, L_new = 5)."""

    def __init__(self, kind, H_kv, dtype, causal, append, seed=0):
        g = gx._gen(seed)
        self.dtype, self.causal, self.append = dtype, causal, append
        if not append:
            B, Lq, G, D, cap, lens = len(gx.DLENS), 3, 6, 128, 3072, gx.DLENS
        else:
            B, Lq, G, D, cap, L_new = 5, 2, 4, 64, 768, 5
            base = [0, 15, 380, 383, cap - L_new]
            lens = [x + L_new for x in base]
        H, nb = G * H_kv, B * H_kv
        self.splits = gx._splits(B, Lq, H, H_kv, D, cap)
        assert (self.splits > 1) == (H_kv == 1)
        boff = torch.arange(nb, device="cuda").view(-1, 1) * cap
        if not append:
            pos, cols, self.spec = gx._decode_blocks(B, Lq, H, H_kv, D, cap, lens, causal, self.splits, g)
            kf = ex.keys(nb * cap, D, (pos + boff).view(-1), torch.arange(D, device="cuda").repeat(nb), dtype, "cuda")
            self.spec.v = ex.values(nb * cap, D, dtype, g, "cuda")
            k_old, v_old = kf, self.spec.v
            self.lens, self.kn = gx._i32(lens), None
        else:
            bt = torch.tensor(base, device="cuda").repeat_interleave(H_kv)
            new = lambda Lb: [bt + i for i in range(L_new)]  # noqa: E731
            pos, cols, self.spec = gx._decode_blocks(B, Lq, H, H_kv, D, cap, lens, causal, self.splits, g, extra=new,
                                                     lo=32)
            kf = ex.keys(nb * cap, D, (pos + boff).view(-1), torch.arange(D, device="cuda").repeat(nb), dtype, "cuda")
            self.spec.v = ex.values(nb * cap, D, dtype, g, "cuda")
            slots = (boff + bt.view(-1, 1) + torch.arange(L_new, device="cuda").view(1, -1)).view(-1)
            k_old, v_old = kf.clone(), self.spec.v.clone()
            k_old[slots] = ex.A
            v_old[slots] = ex.values(slots.numel(), D, dtype, g, "cuda")
            self.kn, self.vn = [t[slots].view(B, H_kv, L_new, D).transpose(1, 2).contiguous() for t in (kf, self.spec.v)]
            theta = torch.rand(cap, 16, generator=g, device="cuda") * 2 * math.pi
            self.cos, self.sin = theta.cos().to(dtype), theta.sin().to(dtype)
            self.lens = gx._i32(base)
        kc, vc = [t.view(B, H_kv, cap, D).transpose(1, 2).contiguous() for t in (k_old, v_old)]
        self.kc, self.vc, self.table = gx._page(kc, vc, kind, seed)
        self.q = ex.queries(cols, D, dtype).view(B, Lq, H, D)
        self.names = ["Q", "K_cache", "V_cache", "O", "lse", "cache_seqlens", "workspace"]
        self.names += ["block_table"] if self.table is not None else []
        self.names += ["K_new", "V_new", "rotary_cos", "rotary_sin"] if append else []

    def _ws_bytes(self):
        B, Lq, H, D = self.q.shape
        cap = self.kc.size(1) * (self.table.size(1) if self.table is not None else 1)
        if self.append:
            return _ops().fa2_fwd_kvcache_append_workspace_bytes(B, Lq, H, self.kc.size(2), D, cap, True)
        return _ops().fa2_fwd_kvcache_workspace_bytes(B, Lq, H, self.kc.size(2), D, cap)

    def _rot(self):
        return dict(k=self.kn, v=self.vn, rotary_cos=self.cos, rotary_sin=self.sin, rotary_interleaved=False) \
            if self.append else {}

    def fresh(self):
        o = torch.full_like(self.q, float("nan"))
        lse = torch.full(self.q.shape[:-1], float("nan"), device="cuda")
        kc, vc = self.kc.clone(), self.vc.clone()
        _ops().fa2_fwd_kvcache(self.q, kc, vc, o, self.lens, self.table, causal=self.causal, lse=lse, **self._rot())
        return o, lse, kc, vc

    def check(self, out):
        gx._check(out[0], self.spec, self.dtype, split=self.splits > 1)

    def placed(self, offs, P):
        q, kc, vc = (P(t, offs.get(n, 16)) for t, n in ((self.q, "Q"), (self.kc, "K_cache"), (self.vc, "V_cache")))
        o = P((self.q.shape, self.dtype), offs.get("O", 4))
        lse = P((self.q.shape[:-1], torch.float32), offs.get("lse", 4))
        lens = P(self.lens, offs.get("cache_seqlens", 4))
        table = P(self.table, offs.get("block_table", 4)) if self.table is not None else None
        nbytes = self._ws_bytes()
        ws = P(((max(nbytes, 16),), torch.uint8), offs.get("workspace", 16))
        B, Lq, H, D = self.q.shape
        num_pages, ps, H_kv = self.kc.shape[:3]
        pps = self.table.size(1) if self.table is not None else 1
        tail = (B, Lq, H, H_kv, D, num_pages, ps, pps, 0.0, DT[self.dtype], int(self.causal), _p(ws), nbytes, _stream())
        if not self.append:
            rc = L.lib.b200k_fa2_fwd_kvcache_lse(_p(q), _p(kc), _p(vc), _p(o), _p(lse), _p(lens), _p(table), *tail)
        else:
            kn, vn, cos, sin = (P(t, offs.get(n, 16)) for t, n in ((self.kn, "K_new"), (self.vn, "V_new"),
                                                                   (self.cos, "rotary_cos"), (self.sin, "rotary_sin")))
            rc = L.lib.b200k_fa2_fwd_kvcache_append_lse(_p(q), _p(kc), _p(vc), _p(o), _p(lse), _p(lens), _p(table),
                                                        _p(kn), _p(vn), kn.size(1), _p(cos), _p(sin), cos.size(0),
                                                        2 * cos.size(1), 0, *tail)
        return rc, (o, lse, kc, vc)

    def via_ops(self, offs, P):
        q = P(self.q, offs.get("Q", 16))
        kc, vc = P(self.kc, offs.get("K_cache", 16)), P(self.vc, offs.get("V_cache", 16))
        o = P((self.q.shape, self.dtype), offs.get("O", 4))
        _ops().fa2_fwd_kvcache(q, kc, vc, o, self.lens, self.table, causal=self.causal, **self._rot())


CASES = {
    "dense_f16_causal_lens": lambda: Dense(torch.float16, True, [1, 129, 200], seed=1),
    "dense_bf16_causal": lambda: Dense(torch.bfloat16, True, None, seed=2),
    "dense_bf16_lens": lambda: Dense(torch.bfloat16, False, [63, 200, 128], D=128, seed=3),
    "dense_v_dn": lambda: Dense(torch.float16, True, [1, 129, 200], v_dn=True, seed=4),
    "ffpa_d192": lambda: Dense(torch.float16, False, None, D=192, ffpa=True, seed=5),
    "ffpa_d512": lambda: Dense(torch.float16, False, None, D=512, ffpa=True, seed=6),
    "packed_gqa_f16": lambda: Packed(torch.float16, True, seed=7),
    "packed_gqa_bf16": lambda: Packed(torch.bfloat16, False, seed=8),
    "decode_split_contig": lambda: Decode("contig", 1, torch.float16, True, False, seed=9),
    "decode_unsplit_contig": lambda: Decode("contig", 20, torch.bfloat16, False, False, seed=10),
    "decode_split_pages16": lambda: Decode(16, 1, torch.bfloat16, False, False, seed=11),
    "decode_unsplit_pages16": lambda: Decode(16, 20, torch.float16, True, False, seed=12),
    "append_split_contig": lambda: Decode("contig", 1, torch.float16, True, True, seed=13),
    "append_unsplit_pages16": lambda: Decode(16, 24, torch.bfloat16, False, True, seed=14),
    "append_split_pages16": lambda: Decode(16, 1, torch.bfloat16, True, True, seed=15),
}

INPUTS = ("Q", "K", "V", "K_cache", "V_cache", "K_new", "V_new", "rotary_cos", "rotary_sin")


@pytest.mark.parametrize("case", list(CASES))
def test_accepted_offsets_give_the_bits_of_fresh_tensors(case):
    """Three placements: O at +4, +8, +12, the inputs at +16, +48, +16; lse, the int32 arrays at +4, the workspace at
    +16.  Each has the bits of the fresh call, whose O is the exact answer; no guard byte changes."""
    c = CASES[case]()
    want = c.fresh()
    c.check(want)
    for o_off, in_off in ((4, 16), (8, 48), (12, 16)):
        P = Placed()
        offs = {n: in_off for n in INPUTS}
        offs.update(O=o_off, lse=4, seqlens_k=4, cu_seqlens_q=4, cu_seqlens_k=4, cache_seqlens=4, block_table=4,
                    workspace=16)
        rc, got = c.placed(offs, P)
        assert rc == L.OK, L.last_error()
        for i, (a, b) in enumerate(zip(got, want)):
            if b is not None:
                assert _same_bits(a, b), (case, o_off, i)
        assert P.guards_kept(), (case, o_off)


def _refused(c):
    """(pointer, offset) pairs each call must refuse."""
    out = [("O", off) for off in (2, 6, 10, 14)]
    out += [(n, off) for n in ("Q", "K", "V", "K_cache", "V_cache") if n in c.names for off in (2, 4, 8)]
    if isinstance(c, Decode) and c.splits > 1:
        out += [("workspace", 4), ("workspace", 8)]
    return out


REFUSED = ["dense_f16_causal_lens", "ffpa_d512", "packed_gqa_bf16", "decode_split_pages16", "decode_unsplit_contig",
           "append_split_pages16", "append_unsplit_pages16"]


@pytest.mark.parametrize("case", REFUSED)
def test_refused_offsets_change_nothing(case):
    """B200K_EALIGN naming the pointer, through the C ABI and through ops; O and lse stay 0xFF, the caches and the block
    table keep their bits, and the stream is clean afterwards."""
    c = CASES[case]()
    table = c.table.clone() if isinstance(c, Decode) and c.table is not None else None
    for name, off in _refused(c):
        P = Placed()
        rc, got = c.placed({name: off}, P)
        assert rc == L.EALIGN, (name, off, rc, L.last_error())
        need = 4 if name == "O" else 16
        assert ": %s must be %d-byte aligned" % (name, need) in L.last_error(), L.last_error()
        torch.cuda.synchronize()
        for t in got[:2]:
            if t is not None:
                assert bool((t.contiguous().view(torch.uint8) == 0xFF).all()), (name, off)
        if isinstance(c, Decode):
            assert _same_bits(got[2], c.kc) and _same_bits(got[3], c.vc), (name, off)
            if table is not None:
                assert torch.equal(c.table, table)
        assert P.guards_kept()
        if name != "workspace":
            P = Placed()
            with pytest.raises(L.B200KError, match="%s must be %d-byte aligned" % (name, need)):
                c.via_ops({name: off}, P)
            torch.cuda.synchronize()
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ Python drop-ins
def _o_at(like, elems):
    """An O of `like`'s shape `elems` fp16 / bf16 elements into a NaN-filled buffer (a contiguous view)."""
    buf = torch.full((like.numel() + 8,), float("nan"), dtype=like.dtype, device="cuda")
    return buf[elems:elems + like.numel()].view(like.shape)


def test_drop_ins_refuse_an_o_one_element_in_and_accept_two():
    """ops, flash_attn_lib and ffpa_attn with o = buf[1:] raise an error naming O's alignment and write nothing; with
    buf[2:] (4 bytes) they give the bits of a fresh O.  attn_merge stores 16-byte vectors: buf[1:] and buf[2:] are
    refused, buf[8:] matches."""
    from b200k import flash_attn_lib
    import ffpa_attn
    ops = _ops()
    d = Dense(torch.float16, False, None, seed=20)
    f = Dense(torch.float16, False, None, D=256, ffpa=True, seed=21)
    p = Packed(torch.float16, True, seed=22)
    k = Decode(16, 1, torch.float16, True, False, seed=23)
    calls = [
        ("fa2_fwd", d.q, lambda o: ops.fa2_fwd(d.q, d.k, d.v, o)),
        ("flash_attn_lib", d.q, lambda o: flash_attn_lib.flash_attn_mma_stages_split_q_shared_kv(d.q, d.k, d.v, o, 2)),
        ("ffpa_fwd", f.q, lambda o: ops.ffpa_fwd(f.q, f.k, f.v, o)),
        ("flash_attn_lib_d256", f.q, lambda o: flash_attn_lib.flash_attn_mma_stages_split_q_tiling_qk(f.q, f.k, f.v, o, 2)),
        ("ffpa_attn", f.q, lambda o: ffpa_attn.ffpa(f.q, f.k, f.v, o)),
        ("fa2_fwd_varlen", p.q, lambda o: ops.fa2_fwd_varlen(p.q, p.k, p.v, o, p.cq, p.ck, max(gx.LQ), causal=True)),
        ("fa2_fwd_kvcache", k.q, lambda o: ops.fa2_fwd_kvcache(k.q, k.kc, k.vc, o, k.lens, k.table, causal=True)),
    ]
    for what, like, call in calls:
        o1 = _o_at(like, 1)
        with pytest.raises(RuntimeError, match="O must be 4-byte aligned"):
            call(o1)
        torch.cuda.synchronize()
        assert bool(torch.isnan(o1).all()), what
        fresh, o2 = torch.full_like(like, float("nan")), _o_at(like, 2)
        call(fresh)
        call(o2)
        assert _same_bits(o2, fresh), what
    parts, lp = torch.randn(3, 5, 2, 64, device="cuda").half(), torch.randn(3, 5, 2, device="cuda")
    like = parts[0]
    for elems in (1, 2):
        o = _o_at(like, elems)
        with pytest.raises(RuntimeError, match="O must be 16-byte aligned"):
            ops.attn_merge(parts, lp, o)
        torch.cuda.synchronize()
        assert bool(torch.isnan(o).all())
    fresh, o8 = torch.full_like(like, float("nan")), _o_at(like, 8)
    ops.attn_merge(parts, lp, fresh)
    ops.attn_merge(parts, lp, o8)
    assert _same_bits(o8, fresh)
