"""The GEMM's TMA-store epilogue: C is written through shared memory and clipped to [M, N] by the tensor map.

Four ragged shapes (M, N and K not multiples of the tile) with tile counts from just under one wave to just over two
on this GPU's SM count, for every dtype; the row past C must stay untouched.  C must be 16-byte aligned."""
import ctypes

import pytest
import torch

from b200k import _loader as L
from oracle import oracle


def test_unaligned_c_is_rejected_before_cuda():
    lib = L.lib
    one, odd = ctypes.c_void_p(16), ctypes.c_void_p(18)  # never dereferenced: validation fails first
    assert lib.b200k_hgemm_f16(one, one, odd, 8, 8, 8, 0, 0, None) == L.EALIGN
    assert b"16-byte aligned" in lib.b200k_last_error()
    for dt in (L.F16, L.BF16, L.F32):
        assert lib.b200k_gemm(one, one, odd, 8, 8, 8, 0, dt, 0, None) == L.EALIGN


def _sm_count():
    n = ctypes.c_int(0)
    assert L.lib.b200k_device_info(ctypes.byref(n), None, None) == L.OK, L.lib.b200k_last_error()
    return n.value


def _shape(tiles):
    """Ragged M and N with `tiles` 128 x 256 tiles (two column tiles), ragged K."""
    assert tiles % 2 == 0
    return 128 * (tiles // 2) - 56, 392, 200


def _check(c, a, b, dtype):
    if dtype == torch.float32:
        exact, bound = oracle.gemm_tf32_bound(a.cpu(), b.cpu())
        assert ((c.double().cpu() - exact).abs() <= bound + 1e-6 * bound).all()
        return
    exact = a.double().cpu() @ b.double().cpu()
    mag = a.double().abs().cpu() @ b.double().abs().cpu()
    eps = 2.0 ** -10 if dtype == torch.float16 else 2.0 ** -8
    assert ((c.double().cpu() - exact).abs() <= eps * exact.abs() + 1e-5 * mag + 1e-30).all()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
@pytest.mark.parametrize("where", ["below", "equal", "multiple", "above"])
def test_tile_counts_around_the_sm_count(where, dtype):
    from b200k import ops

    sm = _sm_count()
    tiles = {"below": sm - 2, "equal": sm, "multiple": 2 * sm, "above": 2 * sm + 2}[where]
    tiles += tiles % 2
    M, N, K = _shape(tiles)
    torch.manual_seed(M + K)
    a = torch.randn(M, K, device="cuda").to(dtype)
    b = torch.randn(K, N, device="cuda").to(dtype)
    # one row past C: the clipped stores of the last row tile must not reach it
    buf = torch.full((M + 1, N), float("nan"), device="cuda").to(dtype)
    c = buf[:M]
    ops.gemm(a, b, c)
    torch.cuda.synchronize()
    assert torch.isnan(buf[M].float()).all()
    assert torch.isfinite(c.float()).all()
    _check(c, a, b, dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_column_parts_at_other_tile_offsets_are_bit_equal(dtype):
    """C(A, [B1 | B2]) cut at column 520, not a multiple of the 256-column tile: an element of B2 sits at a different
    column of its tile and staging slice than in the whole product.  Every element is still summed over K in the same
    order and rounded once, so the parts equal the whole bit for bit."""
    from b200k import ops

    sm = _sm_count()
    M, N, K = 128 * (sm + 1) - 40, 1024, 4160
    torch.manual_seed(11)
    a = torch.randn(M, K, device="cuda").to(dtype)
    b = torch.randn(K, N, device="cuda").to(dtype)
    c = torch.empty(M, N, device="cuda").to(dtype)
    ops.gemm(a, b, c)
    for lo, hi in ((0, 520), (520, N)):
        h = torch.empty(M, hi - lo, device="cuda").to(dtype)
        ops.gemm(a, b[:, lo:hi].contiguous(), h)
        assert torch.equal(h, c[:, lo:hi]), (lo, hi)
