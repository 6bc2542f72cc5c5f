"""CPU: the exact-answer construction of exact_attention.py against attention_ref.packed (fp64, rounded once)
on packed sequences with grouped K/V heads, empty sequences, Lq != Lk, causal and decoy needles in the
next sequence's first key.  Needle rows and rows that see no key agree bit for bit; rows that average their keys agree
within one ulp of the dtype (the reference's weights are 1 / n rounded, summed in its own order) plus 2^-20
for sums that cancel to 0."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))  # the helpers sit next to this file
import attention_ref as ar  # noqa: E402
import exact_attention as ex  # noqa: E402


def pack(lq, lk, H, H_kv, D, dtype, causal, seed):
    """(q, k, v, cu_q, cu_k, want, mean): a needle pack and the closed-form answer.  Column c of K/V head g of sequence
    b has its needle at a random key of b, or at key 0 of sequence b + 1 (then none in b)."""
    g = torch.Generator().manual_seed(seed)
    B, group = len(lq), H // H_kv
    cu_q = torch.tensor([0] + torch.tensor(lq).cumsum(0).tolist())
    cu_k = torch.tensor([0] + torch.tensor(lk).cumsum(0).tolist())
    tq, tk = int(cu_q[-1]), int(cu_k[-1])
    needle = torch.full((B, H_kv, D), -1, dtype=torch.long)           # flat key (kv head g, token t) = g * tk + t
    for b in range(B):
        for h in range(H_kv):
            for c in range(D):
                r = torch.randint(0, 4, (1,), generator=g).item()
                if r == 0 and b + 1 < B and lk[b + 1] > 0:
                    needle[b + 1, h, c] = h * tk + int(cu_k[b + 1])     # key 0 of the next sequence, none in b
                elif lk[b] > 0 and needle[b, h, c] < 0:
                    needle[b, h, c] = h * tk + int(cu_k[b]) + torch.randint(0, lk[b], (1,), generator=g).item()
    placed = needle >= 0
    v = ex.values(H_kv * tk, D, dtype, g)
    k = ex.keys(H_kv * tk, D, needle[placed], torch.arange(D).expand(B, H_kv, D)[placed], dtype)
    cols = torch.randint(0, D, (tq, H), generator=g)
    q = ex.queries(cols.view(-1), D, dtype).view(tq, H, D)
    tok = torch.arange(tq).view(tq, 1).repeat(1, H)
    b_of = torch.bucketize(tok, cu_q[1:], right=True)
    i = tok - cu_q[b_of]
    Lq, Lk = cu_q[b_of + 1] - cu_q[b_of], cu_k[b_of + 1] - cu_k[b_of]
    n = (i + Lk - Lq + 1).clamp(min=0).minimum(Lk) if causal else Lk
    kvh = torch.arange(H).view(1, H).expand(tq, H) // group
    first = kvh * tk + cu_k[b_of]
    nd = needle[b_of, kvh, cols]
    want, mean = ex.expected(v, first, n, nd, dtype)
    return (q, k.view(H_kv, tk, D).transpose(0, 1).contiguous(), v.view(H_kv, tk, D).transpose(0, 1).contiguous(),
            cu_q, cu_k, want.view(tq, H, D), mean.view(tq, H))


@pytest.mark.parametrize("D", [32, 128, 1024])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("causal", [False, True])
def test_closed_form_matches_the_varlen_oracle(D, dtype, causal):
    lq, lk = [5, 0, 40, 1, 33, 7], [9, 3, 0, 70, 33, 2]
    H, H_kv = 4, 2
    q, k, v, cu_q, cu_k, want, mean = pack(lq, lk, H, H_kv, D, dtype, causal, seed=D + causal)
    ref = ar.packed(q, k, v, cu_q, cu_k, causal=causal)[0].to(dtype)
    assert ref.dtype == dtype
    exact = ~mean
    assert int(exact.sum()) > 0 and int(mean.sum()) > 0
    assert torch.equal(ref[exact], want[exact])
    d = (ref[mean].float() - want[mean].float()).abs()
    assert bool((d <= ex.ulp(want[mean], dtype) + 2.0 ** -20).all())


def test_needles_and_means_are_what_they_claim():
    """Each (sequence, K/V head, column) has at most one needle; a needle row's value is its needle's V row; a row with
    no visible needle gets the mean of its prefix; a row with no visible key gets 0."""
    lq, lk = [3, 4], [5, 0]
    q, k, v, cu_q, cu_k, want, mean = pack(lq, lk, 2, 1, 32, torch.float16, False, seed=1)
    for b in range(2):
        blk = k[int(cu_k[b]):int(cu_k[b + 1]), 0]
        assert bool(((blk == ex.A).sum(0) <= 1).all())
    assert (want[3:] == 0).all() and not mean[3:].any()                # sequence 1 has no key
    for t in range(3):
        for h in range(2):
            c = int(q[t, h].nonzero())
            j = (k[:5, 0, c] == ex.A).nonzero().view(-1)
            expect = v[int(j), 0] if j.numel() else v[:5, 0].float().sum(0) * (torch.tensor(1.0) / 5)
            assert torch.equal(want[t, h], expect.half()), (t, h)
