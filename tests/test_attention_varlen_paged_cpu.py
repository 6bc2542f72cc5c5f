"""CPU: argument validation of packed attention over paged caches (b200k_fa2_varlen_paged) before any CUDA call, the
Python wrapper's checks for ops.fa2_fwd_varlen(..., block_table=), and the paged layout of the reference
(attention_ref.paged, which gathers through the table) against the packed layout on the keys the pages were made from."""
import ctypes
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))  # the oracles sit next to this file
import attention_ref as ar  # noqa: E402
import varlen_paged_oracle as vpo  # noqa: E402

from b200k import _loader as L

ONE = ctypes.c_void_p(16)  # never dereferenced: validation fails first
NAMES = ["Q", "K_cache", "V_cache", "O", "lse", "cu_seqlens_q", "cu_seqlens_k", "block_table"]


def _call(ptrs=(ONE,) * 8, B=2, max_q=64, total_q=100, H=8, H_kv=2, D=64, num_pages=10, page_size=64, pps=4,
          dtype=L.F16, causal=0):
    return L.lib.b200k_fa2_varlen_paged(*ptrs, B, max_q, total_q, H, H_kv, D, num_pages, page_size, pps, 0.0, dtype,
                                        causal, None)


def _msg():
    return L.lib.b200k_last_error().decode()


@pytest.mark.parametrize("null_at", [i for i in range(8) if NAMES[i] != "lse"])
def test_null_pointers_are_refused(null_at):
    ptrs = [ONE] * 8
    ptrs[null_at] = None
    assert _call(ptrs=ptrs) == L.EARG
    assert "b200k_fa2_varlen_paged: null pointer" in _msg()


@pytest.mark.parametrize("dtype", [L.F32, L.I8, L.FP8_E4M3, 99])
def test_unsupported_dtypes_are_refused(dtype):
    assert _call(dtype=dtype) == L.EDTYPE


@pytest.mark.parametrize("D", [0, 16, 48, 80, 160, 256])
def test_unsupported_head_dims_are_refused(D):
    assert _call(D=D) == L.EHEADDIM
    assert "headdim not support!" in _msg()


@pytest.mark.parametrize("kw,text", [
    (dict(B=0), "H %% H_kv"), (dict(B=-1), "H %% H_kv"),
    (dict(H=0), "H %% H_kv"), (dict(H_kv=0), "H %% H_kv"), (dict(H=8, H_kv=3), "H %% H_kv"),
    (dict(H=2, H_kv=4), "H %% H_kv"),
    (dict(num_pages=0), ">= 1"), (dict(page_size=0), ">= 1"), (dict(pps=0), ">= 1"), (dict(page_size=-16), ">= 1"),
    (dict(num_pages=2 ** 25, page_size=64), "2^31 - 1"),          # cache rows overflow int32
    (dict(pps=2 ** 25, page_size=64), "2^31 - 1"),                # a sequence's capacity overflows int32
    (dict(page_size=1), "page_size 1"), (dict(page_size=8), "page_size 8"), (dict(page_size=48), "page_size 48"),
    (dict(page_size=96), "page_size 96"), (dict(page_size=200), "page_size 200"),
    (dict(max_q=0), "max_seqlen_q"), (dict(max_q=101), "max_seqlen_q"),  # max_seqlen_q outside [1, total_q]
    (dict(total_q=0, max_q=1), "total_q"), (dict(total_q=2 ** 31, max_q=1), "total_q"),
    (dict(B=65536, H=1, H_kv=1), "65535"), (dict(B=2, H=32768, H_kv=1), "65535"),   # grid z
])
def test_bad_shapes_are_refused(kw, text):
    assert _call(**kw) == L.ESHAPE
    assert text.replace("%%", "%") in _msg()


@pytest.mark.parametrize("at", range(8))
def test_misaligned_pointers_are_refused_by_name(at):
    need = 16 if NAMES[at] in ("Q", "K_cache", "V_cache") else 4
    for off in sorted({need // 2, 2, 1} - {0}):
        if off % need == 0:
            continue
        ptrs = [ctypes.c_void_p(4096)] * 8
        ptrs[at] = ctypes.c_void_p(4096 + off)
        assert _call(ptrs=ptrs) == L.EALIGN, (NAMES[at], off)
        assert "b200k_fa2_varlen_paged: %s must be %d-byte aligned" % (NAMES[at], need) in _msg()


def test_valid_arguments_reach_the_device():
    """Validation passes; without a GPU the call then fails loudly at the device query instead of doing anything else."""
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lse_null = [ONE] * 4 + [None] + [ONE] * 3
    for kw in (dict(), dict(ptrs=lse_null), dict(page_size=16), dict(page_size=32), dict(page_size=128),
               dict(page_size=384), dict(total_q=2 ** 31 - 1, max_q=2 ** 31 - 1), dict(B=65535, H=1, H_kv=1),
               dict(dtype=L.BF16, D=128, causal=1), dict(D=32), dict(D=96)):
        assert _call(**kw) in (L.ECUDA, L.EARCH), kw


def test_python_wrapper_checks():
    from b200k import ops

    q = torch.zeros(10, 4, 64, dtype=torch.half)
    kc = torch.zeros(6, 16, 2, 64, dtype=torch.half)
    cu = torch.tensor([0, 4, 10], dtype=torch.int32)
    cuk = torch.tensor([0, 20, 40], dtype=torch.int32)
    bt = torch.tensor([[0, 1], [2, 3]], dtype=torch.int32)

    def run(q=q, k=kc, v=kc, o=q, cu=cu, cuk=cuk, bt=bt, lse=None):
        ops.fa2_fwd_varlen(q, k, v, o, cu, cuk, 6, lse=lse, block_table=bt)

    with pytest.raises(RuntimeError, match="values must be torch::kHalf"):
        run(k=kc.float())
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        run(k=kc[0])                                                  # a 3-D cache
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        run(v=kc[:, :8].contiguous())                                 # V pages differ from K pages
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        run(k=torch.zeros(6, 16, 3, 64, dtype=torch.half), v=torch.zeros(6, 16, 3, 64, dtype=torch.half))  # H % H_kv
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        run(k=torch.zeros(6, 16, 2, 32, dtype=torch.half), v=torch.zeros(6, 16, 2, 32, dtype=torch.half))  # D differs
    with pytest.raises(RuntimeError, match="headdim not support!"):
        q48 = torch.zeros(10, 4, 48, dtype=torch.half)
        k48 = torch.zeros(6, 16, 2, 48, dtype=torch.half)
        run(q=q48, o=q48, k=k48, v=k48)
    with pytest.raises(RuntimeError, match="values must be torch::kInt"):
        run(bt=bt.long())
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        run(bt=bt[:1])                                                # one table row for two sequences
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        run(bt=bt.view(-1))                                           # not [B, pages_per_seq]
    with pytest.raises(RuntimeError, match="contiguous"):
        run(bt=torch.zeros(2, 4, dtype=torch.int32)[:, ::2])          # non-contiguous table
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        run(lse=torch.zeros(10, 3))
    with pytest.raises(RuntimeError):
        run()                                                         # CPU tensors: refused before any launch


def _pack(lq, lk, H, H_kv, D, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(sum(lq), H, D, generator=g).half()
    k, v = [torch.randn(sum(lk), H_kv, D, generator=g).half() for _ in range(2)]
    cu = lambda n: torch.tensor([0] + torch.tensor(n).cumsum(0).tolist(), dtype=torch.int32)  # noqa: E731
    return q, k, v, cu(lq), cu(lk)


@pytest.mark.parametrize("page_size", [16, 64])
@pytest.mark.parametrize("causal", [False, True])
def test_paged_reference_reads_the_packed_keys_through_the_table(page_size, causal):
    """Shuffled tables with unlisted pages, Lk not a multiple of the page size, Lk = 0, an empty query sequence, Lq > Lk,
    and a length past the table's capacity (clamped): the paged reference is the packed one on the keys the pages were
    made from, the last sequence's cut to the capacity."""
    lq, lk = [7, 0, 20, 5, 9], [40, 3, 0, 5, 100]
    q, k, v, cq, ck = _pack(lq, lk, 4, 2, 32, seed=page_size + causal)
    kc, vc, table = vpo.to_pages(k, v, ck, page_size, pages_per_seq=80 // page_size, fill=float("nan"), seed=3)
    cap = table.size(1) * page_size
    assert vpo.lengths(ck, cap)[-1] == cap
    cut = ar.cu(lk[:-1] + [cap])
    want = ar.packed(q, k[:int(cut[-1])], v[:int(cut[-1])], cq, cut, causal=causal)[0].half().double()
    ref, lse = ar.paged(q, kc, vc, cq, ck, table, causal=causal)
    assert torch.isfinite(ref).all()
    assert torch.allclose(want, ref, rtol=1e-2, atol=1e-3)
    if causal:
        assert torch.isinf(lse[cq[2]:cq[2] + 15]).all()   # Lk = 0
        assert (ref[cq[3]:cq[4]] != 0).any()


def test_shared_prefix_pages():
    """Two sequences whose tables share their first pages read the same prefix keys."""
    lq, lk = [5, 6], [70, 90]
    q, k, v, cq, ck = _pack(lq, lk, 2, 1, 32, seed=5)
    k[70:70 + 64], v[70:70 + 64] = k[:64], v[:64]                 # sequence 1 starts with sequence 0's first 64 keys
    kc, vc, table = vpo.to_pages(k, v, ck, 32, share=2, seed=1)
    assert (table[0, :2] == table[1, :2]).all()
    kg, vg, cg = vpo.gather(kc, vc, ck, table)
    assert torch.equal(kg, k) and torch.equal(vg, v)
    want = ar.packed(q, k, v, cq, ck)[0].half().double()
    ref, _ = ar.paged(q, kc, vc, cq, ck, table)
    assert torch.allclose(want, ref, rtol=1e-2, atol=1e-3)
