"""GPU: packed variable-length attention with grouped-query K/V heads (ops.fa2_fwd_varlen) against the CPU reference
(attention_ref.py), bit equality with the dense kernel and with repeated K/V, isolation of the sequences of a pack, clipped
stores, CUDA graph capture, and full-size properties.  Tolerances are those of test_gpu_attention.py."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))  # attention_ref.py sits next to this file
import attention_ref as ar  # noqa: E402

pytestmark = pytest.mark.gpu


def _pack(lq, lk, H, H_kv, D, dtype, seed):
    torch.manual_seed(seed)
    q = torch.randn(sum(lq), H, D, device="cuda").to(dtype)
    k, v = [torch.randn(sum(lk), H_kv, D, device="cuda").to(dtype) for _ in range(2)]
    return q, k, v, ar.cu(lq, "cuda"), ar.cu(lk, "cuda")


def _run(q, k, v, cq, ck, max_q, causal=False, fill=float("nan")):
    from b200k import ops

    o = torch.full_like(q, fill)
    ops.fa2_fwd_varlen(q, k, v, o, cq, ck, max_q, causal=causal)
    return o


def _covered(o, cq):
    """The rows of o that belong to a sequence (the kernel writes no others)."""
    c = cq.tolist()
    return torch.cat([o[c[b]:c[b + 1]] for b in range(len(c) - 1)])


@pytest.mark.parametrize("group", [1, 2, 8, 16])   # H / H_kv: MHA, GQA, GQA, MQA
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("D", [32, 64, 96, 128])
def test_varlen_vs_oracle_dims(D, dtype, causal, group):
    H = 16
    lq, lk = [77, 0, 1, 129, 128, 300], [77, 5, 1, 128, 200, 300]
    q, k, v, cq, ck = _pack(lq, lk, H, H // group, D, dtype, seed=D + group + 7 * causal)
    o = _run(q, k, v, cq, ck, max(lq), causal)
    assert torch.isfinite(o).all()
    want = ar.packed(q, k, v, cq, ck, causal=causal)[0].to(q.dtype).cpu()
    assert torch.allclose(o.cpu().float(), want.float(), **ar.TOL[dtype])


@pytest.mark.parametrize("lq,lk", [
    ([0, 1, 77, 128, 129, 1000], [0, 1, 77, 128, 129, 1000]),          # equal lengths, including 0 and 1
    ([1000, 129, 1, 77, 0, 128], [1000, 129, 1, 77, 0, 128]),
    ([1, 77, 128, 5, 129], [1000, 129, 300, 128, 1000]),               # Lq < Lk (chunked prefill, decode)
    ([1000, 129, 128, 77, 3], [77, 1, 128, 0, 1000]),                  # Lq > Lk: leading rows see no key under causal
])
@pytest.mark.parametrize("causal", [False, True])
def test_varlen_packs_vs_oracle(lq, lk, causal):
    D, H, H_kv = 64, 4, 2
    q, k, v, cq, ck = _pack(lq, lk, H, H_kv, D, torch.float16, seed=sum(lq) + 3 * sum(lk) + causal)
    o = _run(q, k, v, cq, ck, max(lq), causal)
    assert torch.isfinite(o).all()
    want = ar.packed(q, k, v, cq, ck, causal=causal)[0].to(q.dtype).cpu()
    assert torch.allclose(o.cpu().float(), want.float(), **ar.TOL[torch.float16])
    # rows that see no key are exactly 0
    c = cq.tolist()
    for b in range(len(lq)):
        Lq, Lk = lq[b], lk[b]
        blind = Lq if Lk == 0 else (max(0, Lq - Lk) if causal else 0)
        assert (o[c[b]:c[b] + blind] == 0).all(), b


@pytest.mark.parametrize("D", [32, 64, 96, 128])
@pytest.mark.parametrize("causal", [False, True])
def test_varlen_equal_lengths_same_bits_as_dense(D, causal):
    """[B*N, H, D] packed with equal lengths and H_kv == H runs the same main loop as the dense [B,H,N,D] kernel."""
    from b200k import ops

    B, H, N = 3, 4, 1000
    torch.manual_seed(D + causal)
    q, k, v = [torch.randn(B, H, N, D, dtype=torch.half, device="cuda") for _ in range(3)]
    dense = torch.empty_like(q)
    ops.fa2_fwd(q, k, v, dense, causal=causal)
    pq, pk, pv = [t.transpose(1, 2).contiguous().view(B * N, H, D) for t in (q, k, v)]
    cu = ar.cu([N] * B, "cuda")
    o = _run(pq, pk, pv, cu, cu, N, causal)
    assert torch.equal(o.view(B, N, H, D).transpose(1, 2), dense)
    # bf16 too
    qb, kb, vb = [t.bfloat16() for t in (q, k, v)]
    dense_b = torch.empty_like(qb)
    ops.fa2_fwd(qb, kb, vb, dense_b, causal=causal)
    ob = _run(*[t.transpose(1, 2).contiguous().view(B * N, H, D) for t in (qb, kb, vb)], cu, cu, N, causal)
    assert torch.equal(ob.view(B, N, H, D).transpose(1, 2), dense_b)


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("group", [2, 8])
@pytest.mark.parametrize("causal", [False, True])
def test_gqa_same_bits_as_repeated_kv(D, group, causal):
    H = 8
    lq, lk = [300, 1, 129, 77], [500, 128, 129, 10]
    q, k, v, cq, ck = _pack(lq, lk, H, H // group, D, torch.float16, seed=group * D + causal)
    o = _run(q, k, v, cq, ck, max(lq), causal)
    kr, vr = [t.repeat_interleave(group, dim=1).contiguous() for t in (k, v)]
    assert torch.equal(_covered(o, cq), _covered(_run(q, kr, vr, cq, ck, max(lq), causal), cq))


@pytest.mark.parametrize("causal", [False, True])
def test_sequences_are_isolated(causal):
    """Each sequence alone gives the same bits as inside the pack, and overwriting every other sequence's tokens with
    +-1e4 leaves its output bit-identical (neighbouring keys read by a sequence's last tile are masked exactly)."""
    D, H, H_kv = 128, 8, 2
    lq, lk = [200, 77, 129, 1, 500], [300, 77, 128, 64, 129]
    q, k, v, cq, ck = _pack(lq, lk, H, H_kv, D, torch.float16, seed=5 + causal)
    o = _run(q, k, v, cq, ck, max(lq), causal)
    c, ckl = cq.tolist(), ck.tolist()
    for b in range(len(lq)):
        qs, ks, vs = q[c[b]:c[b + 1]].contiguous(), k[ckl[b]:ckl[b + 1]].contiguous(), v[ckl[b]:ckl[b + 1]].contiguous()
        alone = _run(qs, ks, vs, ar.cu([lq[b]], "cuda"), ar.cu([lk[b]], "cuda"), lq[b], causal)
        assert torch.equal(alone, o[c[b]:c[b + 1]]), b
        q2, k2, v2 = q.clone(), k.clone(), v.clone()
        for t, lo, hi in ((q2, c[b], c[b + 1]), (k2, ckl[b], ckl[b + 1]), (v2, ckl[b], ckl[b + 1])):
            keep = t[lo:hi].clone()
            t.copy_(torch.where(torch.rand(t.shape, device="cuda") < 0.5, 1e4, -1e4).to(t.dtype))
            t[lo:hi] = keep
        o2 = _run(q2, k2, v2, cq, ck, max(lq), causal)
        assert torch.equal(o2[c[b]:c[b + 1]], o[c[b]:c[b + 1]]), b


def test_stores_stay_inside_o():
    """O is a slice of a larger sentinel-filled buffer: a normal call, and calls whose cu_seqlens_q runs past total_q or
    starts before token 0, write only rows [0, total_q) of O.  A store that escaped the clip would land in the guard
    regions of this same buffer, where the test sees it."""
    from b200k import ops

    D, H, H_kv, total_q, guard = 64, 4, 2, 1000, 512
    torch.manual_seed(2)
    q = torch.randn(total_q, H, D, dtype=torch.half, device="cuda")
    k, v = [torch.randn(total_q, H_kv, D, dtype=torch.half, device="cuda") for _ in range(2)]
    buf = torch.full(((guard + total_q + guard) * H * D,), 7.0, dtype=torch.half, device="cuda")
    o = buf[guard * H * D:(guard + total_q) * H * D].view(total_q, H, D)
    before, after = buf[:guard * H * D], buf[(guard + total_q) * H * D:]
    for causal in (False, True):
        cq = ar.cu([600, 400], "cuda")
        ops.fa2_fwd_varlen(q, k, v, o, cq, cq, 600, causal=causal)
        want = ar.packed(q, k, v, cq, cq, causal=causal)[0].to(q.dtype).cpu()
        assert torch.allclose(o.cpu().float(), want.float(), **ar.TOL[torch.float16])
        # sequence 1 claims tokens [600, 1200): rows past total_q are dropped
        bad = torch.tensor([0, 600, 1200], dtype=torch.int32, device="cuda")
        ops.fa2_fwd_varlen(q, k, v, o, bad, cq, 600, causal=causal)
        # sequence 0 claims tokens [-300, 300): rows before token 0 are dropped
        bad = torch.tensor([-300, 300, 1000], dtype=torch.int32, device="cuda")
        ops.fa2_fwd_varlen(q, k, v, o, bad, cq, 700, causal=causal)
        torch.cuda.synchronize()
        assert bool((before == 7.0).all()) and bool((after == 7.0).all()), causal
        assert torch.isfinite(o).all()


def test_cuda_graph_capture_and_replay():
    """The call reads no length back to the host, so it can be captured and replayed; a replay after new inputs are
    copied in gives the eager result for those inputs."""
    from b200k import ops

    lq, lk = [300, 1, 129], [500, 1, 77]
    q, k, v, cq, ck = _pack(lq, lk, 8, 2, 128, torch.bfloat16, seed=12)
    o = torch.empty_like(q)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.fa2_fwd_varlen(q, k, v, o, cq, ck, max(lq), causal=True)   # warm-up: tensor maps, shared-memory attribute
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.fa2_fwd_varlen(q, k, v, o, cq, ck, max(lq), causal=True)
    for seed in (1, 2):
        q2, k2, v2, _, _ = _pack(lq, lk, 8, 2, 128, torch.bfloat16, seed=seed)
        q.copy_(q2)
        k.copy_(k2)
        v.copy_(v2)
        o.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(o, _run(q2, k2, v2, cq, ck, max(lq), causal=True))


def test_full_size_gqa_causal_properties():
    """4 x 8192 tokens, H = 64, H_kv = 8, D = 128, causal: V = 1 gives O = 1 (within 1e-3 at this size; the contract, bit
    equality, is held by test_gpu_attention_graded.py), and sampled rows match an fp32 reference
    computed on the GPU from the full K/V of their sequence and K/V head."""
    B, N, H, H_kv, D = 4, 8192, 64, 8, 128
    torch.manual_seed(21)
    q = torch.randn(B * N, H, D, dtype=torch.half, device="cuda")
    k, v = [torch.randn(B * N, H_kv, D, dtype=torch.half, device="cuda") for _ in range(2)]
    cu = ar.cu([N] * B, "cuda")
    ones = torch.ones_like(v)
    assert (_run(q, k, ones, cu, cu, N, causal=True).float() - 1.0).abs().max().item() <= 1e-3
    o = _run(q, k, v, cu, cu, N, causal=True)
    rows = torch.tensor([0, 1, 127, 128, 4095, 4096, 8191], device="cuda")
    for b in (0, B - 1):
        for h in (0, 13, H - 1):
            qs = q[b * N + rows, h].float()                                  # [R, D]
            ks, vs = k[b * N:(b + 1) * N, h // (H // H_kv)].float(), v[b * N:(b + 1) * N, h // (H // H_kv)].float()
            s = (qs @ ks.t()) / D ** 0.5
            s = s.masked_fill(torch.arange(N, device="cuda").view(1, N) > rows.view(-1, 1), float("-inf"))
            want = torch.softmax(s, -1) @ vs
            assert torch.allclose(o[b * N + rows, h].float(), want, **ar.TOL[torch.float16]), (b, h)
