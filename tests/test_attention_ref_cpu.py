"""CPU: attention_ref.py against torch, per layout.  Dense and packed O against scaled_dot_product_attention in fp64 with
an explicit mask and lse against torch.logsumexp of the masked scores; the KV-cache and paged layouts equal the packed
one on the keys the cache holds, for contiguous caches and shuffled tables.  Gradients against torch.autograd and
gradcheck are in test_attention_bwd_cpu.py and test_attention_varlen_bwd_cpu.py, poison in test_attention_poison_cpu.py."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attention_ref as ar  # noqa: E402
import kvcache_oracle  # noqa: E402
import varlen_paged_oracle as vpo  # noqa: E402


def _torch_sequence(q, k, v, scale, mask):
    """(o, lse) of one sequence [L, H, D] by SDPA and logsumexp, K/V heads repeated; rows with no visible key 0 / -inf."""
    G = q.size(1) // k.size(1)
    qh, kh, vh = (t.transpose(0, 1) for t in (q, k.repeat_interleave(G, 1), v.repeat_interleave(G, 1)))
    s = (qh @ kh.transpose(-1, -2) * scale).masked_fill(~mask, float("-inf"))
    seen = mask.any(-1).view(-1, 1)
    o = F.scaled_dot_product_attention(qh, kh, vh, attn_mask=mask, scale=scale).nan_to_num(0.0) * seen
    return o.transpose(0, 1), torch.logsumexp(s, -1).transpose(0, 1)


@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
def test_dense_is_sdpa_and_logsumexp(causal):
    B, H, N, D = 6, 2, 23, 8
    g = torch.Generator().manual_seed(int(causal))
    q, k, v = (torch.randn(B, H, N, D, generator=g, dtype=torch.float64) for _ in range(3))
    sl = torch.tensor([-3, 0, 1, N - 1, N, N + 4], dtype=torch.int32)
    o, lse = ar.dense(q, k, v, 0.3, causal, sl)
    for b, n in enumerate((1, 1, 1, N - 1, N, N)):
        mask = torch.arange(N).view(1, N) < n
        if causal:
            mask = mask & torch.ones(N, N, dtype=torch.bool).tril()
        want = _torch_sequence(*(t[b].transpose(0, 1) for t in (q, k, v)), 0.3, mask.expand(N, N))
        assert torch.allclose(o[b].transpose(0, 1), want[0], rtol=1e-12, atol=1e-12)
        assert torch.allclose(lse[b].transpose(0, 1), want[1], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("H,H_kv", [(4, 4), (4, 2), (6, 1)])
def test_packed_is_sdpa_and_logsumexp(H, H_kv, causal):
    """Empty query and key sequences, Lq > Lk (causal: rows that see no key), and tokens past cu[B] (0 and -inf)."""
    lq, lk, D = [5, 0, 9, 4, 3], [7, 3, 2, 0, 3], 8
    g = torch.Generator().manual_seed(H + causal)
    q = torch.randn(sum(lq) + 2, H, D, generator=g, dtype=torch.float64)
    k, v = (torch.randn(sum(lk) + 2, H_kv, D, generator=g, dtype=torch.float64) for _ in range(2))
    o, lse = ar.packed(q, k, v, ar.cu(lq), ar.cu(lk), None, causal)
    for q0, q1, k0, k1 in ar.seqs(ar.cu(lq), ar.cu(lk)):
        Lq, Lk = q1 - q0, k1 - k0
        mask = torch.arange(Lk).view(1, Lk) <= torch.arange(Lq).view(Lq, 1) + (Lk - Lq if causal else Lk)
        want = _torch_sequence(q[q0:q1], k[k0:k1], v[k0:k1], D ** -0.5, mask)
        assert torch.allclose(o[q0:q1], want[0], rtol=1e-12, atol=1e-12)
        assert torch.allclose(lse[q0:q1], want[1], rtol=1e-12, atol=1e-12)
    assert (o[-2:] == 0).all() and (lse[-2:] == float("-inf")).all()


@pytest.mark.parametrize("page_size", [None, 16, 64])
def test_kvcache_and_paged_are_packed_on_the_cached_keys(page_size):
    B, Lq, H, H_kv, D, S = 3, 4, 4, 2, 8, 128
    g = torch.Generator().manual_seed(page_size or 0)
    q = torch.randn(B, Lq, H, D, generator=g).half()
    kc, vc = (torch.randn(B, S, H_kv, D, generator=g).half() for _ in range(2))
    lens = [0, 2, 100]
    k, v = (torch.cat([c[b, :n] for b, n in enumerate(lens)]) for c in (kc, vc))
    want = ar.packed(q.view(B * Lq, H, D), k, v, ar.cu([Lq] * B), ar.cu(lens), None, True)
    table = None
    if page_size:
        kc, vc, table, _ = kvcache_oracle.paged_copy(kc, vc, page_size, seed=page_size)
    got = ar.kvcache(q, kc, vc, torch.tensor(lens, dtype=torch.int32), table, causal=True)
    assert torch.equal(got[0].view(B * Lq, H, D), want[0]) and torch.equal(got[1].view(B * Lq, H), want[1])
    if page_size:
        kp, vp, table = vpo.to_pages(k, v, ar.cu(lens), page_size, fill=float("nan"), seed=page_size)
        got = ar.paged(q.view(B * Lq, H, D), kp, vp, ar.cu([Lq] * B), ar.cu(lens), table, causal=True)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
