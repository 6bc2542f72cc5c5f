"""CPU: the regions of attention_poison.py, and attention_ref under poison.

  - on clean inputs the dense reference equals oracle.attention;
  - poisoning the elements a call does not own leaves attention_ref unchanged and finite, and turns the masking
    reference oracle.attention NaN: the same 0 * NaN hazard the kernels have;
  - poisoning one owned element at each boundary (key kv_len - 1, key 0 when seqlens_k <= 0, token cu[B] - 1, the first
    token of the next sequence) makes the owned outputs non-finite, so the regions are no wider than the contract."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attention_poison as ap  # noqa: E402
import attention_ref as ar  # noqa: E402
from oracle import oracle  # noqa: E402

LENS = [1, 63, 64, 65, 99, 100, 0, -5]     # N = 100: N - 1 and N, and the clamped 0 and -5
N = 100


def _dense(D=32, seed=0):
    g = torch.Generator().manual_seed(seed)
    B = len(LENS)
    q, k, v, do = (torch.randn(B, 2, N, D, generator=g, dtype=torch.float64) for _ in range(4))
    return q, k, v, do, torch.tensor(LENS, dtype=torch.int32)


LQ, LK = (65, 0, 64, 63, 1), (40, 7, 129, 63, 200)
PAD = 9                                     # tokens past cu[B] on both sides


def _packed(H=4, H_kv=2, D=16, seed=1):
    g = torch.Generator().manual_seed(seed)
    q, do = (torch.randn(sum(LQ) + PAD, H, D, generator=g, dtype=torch.float64) for _ in range(2))
    k, v = (torch.randn(sum(LK) + PAD, H_kv, D, generator=g, dtype=torch.float64) for _ in range(2))
    cu = lambda L: torch.tensor([0] + torch.tensor(L).cumsum(0).tolist(), dtype=torch.int32)  # noqa: E731
    return q, k, v, do, cu(LQ), cu(LK)


def _finite(*ts):
    return all(bool(torch.isfinite(t).all()) for t in ts)


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


# ------------------------------------------------------------------------------------------------ clean inputs
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
def test_dense_references_agree_on_clean_inputs(causal):
    q, k, v, do, sl = _dense()
    # oracle.attention does not clamp seqlens_k: give it the clamped lengths
    o64 = ar.dense(q, k, v, None, causal, sl)[0]
    ref = oracle.attention(q.half(), k.half(), v.half(), causal=causal, seqlens=ap.kv_lens(sl, len(LENS), N))
    assert torch.allclose(o64.half().float(), ref.float(), rtol=2e-3, atol=2e-3)


# ------------------------------------------------------------------------------------------------ poisoned inputs
def test_dense_masks():
    k = torch.zeros(len(LENS), 2, N, 8)
    m = ap.dense_kv_mask(k.shape, torch.tensor(LENS))
    for b, n in enumerate(LENS):
        n = min(max(n, 1), N)
        assert not m[b, :, :n].any() and m[b, :, n:].all()
    assert torch.equal(ap.dense_kv_mask((len(LENS), 2, 8, N), torch.tensor(LENS), v_dn=True), m.transpose(-1, -2))
    assert not ap.dense_kv_mask(k.shape, None).any()


@pytest.mark.parametrize("value", ap.VALUES, ids=ap.VALUE_IDS)
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
def test_dense_poison_leaves_slicing_references_unchanged(causal, value):
    q, k, v, do, sl = _dense(seed=2)
    clean = ar.dense_grads(q, k, v, do, None, causal, sl)
    m = ap.dense_kv_mask(k.shape, sl)
    kp, vp = ap.poison(k, m, value), ap.poison(v, m, value)
    got = ar.dense_grads(q, kp, vp, do, None, causal, sl)
    assert _finite(*got) and _same(got, clean)
    o, lse = clean[3], clean[4]
    assert _same(ar.dense_grads_given(q, kp, vp, o, lse, do, None, causal, sl), clean[:3])
    # the masking reference reads the poison: O of every batch with a padded key goes NaN
    pad = [b for b, n in enumerate(LENS) if min(max(n, 1), N) < N]
    bad = oracle.attention(q, kp, vp, causal=causal, seqlens=ap.kv_lens(sl, len(LENS), N)).float()
    assert torch.isnan(bad[pad]).any() and not torch.isnan(bad[[b for b in range(len(LENS)) if b not in pad]]).any()


@pytest.mark.parametrize("value", ap.VALUES, ids=ap.VALUE_IDS)
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
def test_packed_poison_leaves_references_unchanged(causal, value):
    q, k, v, do, cq, ck = _packed(seed=3)
    clean = ar.packed_grads(q, k, v, do, cq, ck, None, causal)
    mq, mk = ap.packed_masks(cq, ck, q.shape, k.shape)
    assert mq[:int(cq[-1])].logical_not().all() and mq[int(cq[-1]):].all() and mk[int(ck[-1]):].all()
    got = ar.packed_grads(*(ap.poison(t, m, value) for t, m in ((q, mq), (k, mk), (v, mk), (do, mq))), cq, ck, None, causal)
    assert _same(got, clean) and _finite(*got[:4])
    o, lse = clean[3], clean[4]
    lse_m = ap.packed_masks(cq, ck, lse.shape, k.shape)[0]
    given = ar.packed_grads_given(ap.poison(q, mq, value), ap.poison(k, mk, value), ap.poison(v, mk, value),
                                   ap.poison(o, mq, value), ap.poison(lse, lse_m, value), ap.poison(do, mq, value), cq, ck,
                                   None, causal)
    assert _same(given, clean[:3])
    # isolation: sequence 2 (after the 65-token one, with an empty one between) poisoned whole; the others keep theirs
    for b in range(len(LQ)):
        sq, sk = ap.sequence_masks(cq, ck, b, q.shape, k.shape)
        other = ar.packed_grads(*(ap.poison(t, m, value) for t, m in ((q, sq), (k, sk), (v, sk), (do, sq))), cq, ck, None,
                                causal)
        q0, q1, k0, k1 = ar.seqs(cq, ck)[b]
        for got_t, want_t, lo, hi in zip(other, clean, (q0, k0, k0, q0, q0), (q1, k1, k1, q1, q1)):
            assert torch.equal(got_t[lo:hi], want_t[lo:hi])


# ------------------------------------------------------------------------------------------------ boundaries
def test_dense_boundary_keys_are_owned():
    """Key kv_len - 1 of each batch (key 0 where seqlens_k <= 0 clamps to 1) is read: NaN there reaches every row."""
    q, k, v, do, sl = _dense(seed=4)
    m = ap.dense_kv_mask(k.shape, sl)
    for b, n in enumerate(ap.kv_lens(sl, len(LENS), N)):
        assert not m[b, :, n - 1].any()
        vp = v.clone()
        vp[b, 0, n - 1, 0] = float("nan")
        o = ar.dense(q, k, vp, None, False, sl)[0]
        assert torch.isnan(o[b, 0, :, 0]).all() and _finite(o[b, 1]) and _finite(o[:b], o[b + 1:])
        kp = k.clone()
        kp[b, 1, n - 1, 3] = float("nan")
        dq, dk, dv, o, lse = ar.dense_grads(q, kp, v, do, None, False, sl)
        assert not _finite(o[b, 1]) and _finite(o[b, 0])


def test_packed_boundary_tokens_are_owned():
    """Token cu[B] - 1 on each side belongs to the last sequence, and the first token of each sequence to it alone."""
    q, k, v, do, cq, ck = _packed(seed=5)
    mq, mk = ap.packed_masks(cq, ck, q.shape, k.shape)
    tq, tk = int(cq[-1]), int(ck[-1])
    assert not mq[tq - 1].any() and not mk[tk - 1].any()
    # the query side through dO: dQ of that row and dV of its sequence's keys go NaN
    dop, kp = do.clone(), k.clone()
    dop[tq - 1, 0, 0] = float("nan")
    kp[tk - 1, 0, 0] = float("nan")
    dq, dk, dv = ar.packed_grads(q, k, v, dop, cq, ck)[:3]
    assert torch.isnan(dq[tq - 1, 0]).all() and _finite(dq[:tq - 1])
    assert torch.isnan(dv[int(ck[-2]):tk, 0]).any() and _finite(dv[:int(ck[-2])])
    o = ar.packed(q, kp, v, cq, ck)[0]
    assert not _finite(o[int(cq[-2]):tq, :2]) and _finite(o[:int(cq[-2])], o[int(cq[-2]):tq, 2:])
    seqs = ar.seqs(cq, ck)
    for b in range(len(LQ) - 1):
        nxt = next((s for s in seqs[b + 1:] if s[3] > s[2] and s[1] > s[0]), None)
        sq, sk = ap.sequence_masks(cq, ck, b, q.shape, k.shape)
        if seqs[b][1] > seqs[b][0]:
            assert sq[seqs[b][1]:].all() and not sq[seqs[b][0]:seqs[b][1]].any()
        if nxt is None:
            continue
        assert sk[nxt[2]].all() and not ap.sequence_masks(cq, ck, seqs.index(nxt), q.shape, k.shape)[1][nxt[2]].any()
        vp = v.clone()
        vp[nxt[2], 0, 0] = float("nan")  # key 0 of the next sequence with keys: its rows see it, causal or not
        o = ar.packed(q, k, vp, cq, ck, None, True)[0]
        assert torch.isnan(o[nxt[0]:nxt[1], 0, 0]).all() and _finite(o[:nxt[0]], o[nxt[1]:])
