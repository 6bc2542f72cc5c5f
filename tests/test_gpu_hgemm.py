"""GPU parity: wgmma HGEMM (through the C ABI) vs the CPU oracle, golden fixture, edge shapes, and full-size
(BASELINE config #2) property checks.  Tolerance: the north star's rtol=1e-2 / atol=1e-3 applies to fp16 outputs of
O(1) magnitude; GEMM outputs are O(sqrt(K)), so atol is scaled by sqrt(K/64) (what fp16 output rounding alone needs,
SURVEY.md §7.2-1).  Written in each assert."""
import numpy as np
import pytest
import torch

from oracle import oracle

pytestmark = pytest.mark.gpu


def _tol(K):
    return dict(rtol=1e-2, atol=1e-3 * max(1.0, (K / 64.0) ** 0.5))


@pytest.mark.parametrize("variant", [0, 1, 2, 3])
@pytest.mark.parametrize("tn", [False, True])
@pytest.mark.parametrize("shape", [(128, 256, 64), (256, 256, 256), (300, 520, 264), (1, 8, 8), (129, 264, 8), (1000, 72, 1000)])
def test_hgemm_vs_oracle(variant, tn, shape):
    from b200k import ops

    M, N, K = shape
    torch.manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(M, K, dtype=torch.half, device="cuda")
    b = torch.randn(K, N, dtype=torch.half, device="cuda")
    c = torch.full((M, N), float("nan"), dtype=torch.half, device="cuda")
    bb = b.t().contiguous().t() if tn else b  # [K,N] view over B^T storage, like the reference's as_col_major
    ops.hgemm(a, bb, c, tn=tn, variant=variant)
    ref = oracle.hgemm(a, b)
    assert torch.isfinite(c).all()
    assert torch.allclose(c.cpu().float(), ref.float(), **_tol(K))


def test_hgemm_golden_fixture(golden):
    from b200k import ops

    g = golden("seeded_hgemm.npz")
    a = torch.from_numpy(g["a"]).cuda()
    b = torch.from_numpy(g["b"]).cuda()
    c = torch.empty(a.size(0), b.size(1), dtype=torch.half, device="cuda")
    ops.hgemm(a, b, c)
    want = torch.from_numpy(g["c"]).float()
    # fp32-accumulating tensor core vs exact accumulate + one rounding: at most 1 fp16 ulp apart
    assert torch.allclose(c.cpu().float(), want, rtol=2 ** -10, atol=2 ** -10)


def test_hgemm_drop_in_names_route_to_kernel():
    import toy_hgemm

    torch.manual_seed(5)
    a = torch.randn(256, 128, dtype=torch.half, device="cuda")
    b = torch.randn(128, 384, dtype=torch.half, device="cuda")
    ref = oracle.hgemm(a, b).float()
    b_col_major = b.t().contiguous().t()
    for name in toy_hgemm.HGEMM_NAMES:
        c = torch.zeros(256, 384, dtype=torch.half, device="cuda")
        fn = getattr(toy_hgemm, name)
        bb = b_col_major if ("_tn" in name) else b
        if name.endswith("_tn_cute"):  # the reference script's own spelling: contiguous [K,N]-shaped buffer of B^T
            bb = b.t().reshape(b.shape).contiguous()
        if "stages" in name:
            fn(a, bb, c, 3, True, 2048)
        else:
            fn(a, bb, c)
        assert torch.allclose(c.cpu().float(), ref, **_tol(128)), name


@pytest.mark.parametrize("n", [2048, 4096, 8192])
def test_hgemm_full_size_sampled_entries_and_linearity(n):
    """BASELINE config #2 sizes: (1) 512 sampled entries against fp64 dot products of the same fp16 inputs,
    (2) structure: C(A, [B1 | B2]) column blocks equal C(A, B1), C(A, B2): every output tile is summed over K in the same
    order whatever the grid, so the halves agree bit for bit, (3) run-to-run determinism, also through a legacy variant
    value (every variant selects the same kernel)."""
    from b200k import ops

    torch.manual_seed(n)
    a = torch.randn(n, n, dtype=torch.half, device="cuda")
    b = torch.randn(n, n, dtype=torch.half, device="cuda")
    c = torch.empty(n, n, dtype=torch.half, device="cuda")
    ops.hgemm(a, b, c)
    idx = torch.randint(0, n, (512, 2), device="cuda")
    want = (a[idx[:, 0]].double() * b[:, idx[:, 1]].t().double()).sum(-1)
    got = c[idx[:, 0], idx[:, 1]].double()
    assert torch.allclose(got, want, **_tol(n))
    half = n // 2
    bh = b[:, :half].contiguous()
    c1 = torch.empty(n, half, dtype=torch.half, device="cuda")
    ops.hgemm(a, bh, c1)
    # one fp16 ulp of the value; near zero the fp32 summation-order difference (~ sqrt(K) * 2^-24 per add) dominates
    assert torch.equal(c1, c[:, :half])
    c2 = torch.empty_like(c)
    ops.hgemm(a, b, c2)
    assert torch.equal(c2, c)                                                               # deterministic
    LEGACY = 2 | (1 << 20)      # a variant value of the old ABI: accepted, same kernel, same bits
    ops.hgemm(a, b, c2, variant=LEGACY)
    assert torch.equal(c2, c)


def test_hgemm_16384_smoke_and_stream():
    """Largest sweep size (3 x 512 MiB operands) on a side stream: sampled entries only."""
    from b200k import ops

    n = 16384
    torch.manual_seed(2)
    a = torch.randn(n, n, dtype=torch.half, device="cuda")
    b = torch.randn(n, n, dtype=torch.half, device="cuda")
    c = torch.empty(n, n, dtype=torch.half, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.hgemm(a, b, c)
    s.synchronize()
    idx = torch.randint(0, n, (128, 2), device="cuda")
    want = (a[idx[:, 0]].double() * b[:, idx[:, 1]].t().double()).sum(-1)
    assert torch.allclose(c[idx[:, 0], idx[:, 1]].double(), want, **_tol(n))


@pytest.mark.parametrize("tn", [False, True])
@pytest.mark.parametrize("shape", [(256, 256, 256), (1024, 512, 768), (300, 264, 200), (2048, 2048, 2048)])
def test_bf16_gemm_vs_float64(shape, tn):
    """bf16 build of the GEMM kernel (SURVEY 8f-4): fp32 accumulation, one rounding to bf16 (2^-9 relative)."""
    from b200k import ops

    M, N, K = shape
    torch.manual_seed(M + N + K)
    a = torch.randn(M, K, device="cuda").bfloat16()
    b = torch.randn(K, N, device="cuda").bfloat16()
    c = torch.full((M, N), float("nan"), device="cuda").bfloat16()
    bb = b.t().contiguous().t() if tn else b
    ops.gemm(a, bb, c, tn=tn)
    exact = a.double().cpu() @ b.double().cpu()
    mag = a.double().abs().cpu() @ b.double().abs().cpu()
    assert torch.isfinite(c).all()
    assert ((c.double().cpu() - exact).abs() <= 2.0 ** -8 * exact.abs() + 1e-6 * mag + 1e-30).all()


@pytest.mark.parametrize("tn", [False, True])
@pytest.mark.parametrize("shape", [(256, 256, 256), (1024, 512, 768), (300, 260, 204), (2048, 2048, 2048)])
def test_tf32_gemm_within_the_truncation_bound(shape, tn):
    """TF32 build (fp32 in / out): every entry within the rigorous bound of 13 ignored mantissa bits per operand plus
    fp32 accumulation, and on average far better (random signs cancel)."""
    from b200k import ops

    M, N, K = shape
    torch.manual_seed(M * 3 + N + K)
    a = torch.randn(M, K, device="cuda")
    b = torch.randn(K, N, device="cuda")
    c = torch.full((M, N), float("nan"), device="cuda")
    bb = b.t().contiguous().t() if tn else b
    ops.gemm(a, bb, c, tn=tn)
    exact, bound = oracle.gemm_tf32_bound(a, b)
    err = (c.double().cpu() - exact).abs()
    assert torch.isfinite(c).all()
    assert (err <= bound + 1e-6 * bound).all(), float((err / bound).max())
    assert float(err.mean()) < 2e-3 * float(exact.abs().mean())


def test_gemm_f16_entry_is_the_hgemm_kernel():
    from b200k import ops

    torch.manual_seed(3)
    a = torch.randn(512, 256, dtype=torch.half, device="cuda")
    b = torch.randn(256, 384, dtype=torch.half, device="cuda")
    c0, c1 = torch.empty(512, 384, dtype=torch.half, device="cuda"), torch.empty(512, 384, dtype=torch.half, device="cuda")
    ops.hgemm(a, b, c0)
    ops.gemm(a, b, c1)
    assert torch.equal(c0, c1)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
def test_ragged_n_epilogue_staging_buffers(dtype):
    """Ragged N (not a multiple of the 256-column tile) with short K, so the run is epilogue-bound: the clipped stores of
    the last column tile must write every valid column and nothing else, for every dtype; repeated ten times."""
    from b200k import ops

    torch.manual_seed(7)
    for (M, N, K) in ((2048, 264, 64), (1024, 384, 64), (4096, 296, 32), (512, 328, 128)):
        a = torch.randn(M, K, device="cuda").to(dtype)
        b = torch.randn(K, N, device="cuda").to(dtype)
        want = a.double().cpu() @ b.double().cpu()
        mag = a.double().abs().cpu() @ b.double().abs().cpu()
        tol = 2.0 ** -9 if dtype == torch.float32 else 2.0 ** -7
        for rep in range(10):
            c = torch.full((M, N), float("nan"), device="cuda").to(dtype)
            ops.gemm(a, b, c)
            assert ((c.double().cpu() - want).abs() <= tol * mag + 1e-30).all(), (dtype, M, N, K, rep)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("tn", [False, True])
@pytest.mark.parametrize("shape", [(256, 256, 256), (1024, 512, 768), (264, 520, 200), (2048, 2048, 2048), (4096, 4096, 1024)])
def test_gemm_a_stored_transposed_nt_tt(shape, tn, dtype):
    """SURVEY 8(f)-4: A stored as [K,M] ("NT"; with tn also "TT"), consumed in place as an MN-major operand."""
    from b200k import ops

    M, N, K = shape
    torch.manual_seed(M + N + K)
    at = torch.randn(K, M, device="cuda").to(dtype)          # storage of A^T
    b = torch.randn(K, N, device="cuda").to(dtype)
    c = torch.full((M, N), float("nan"), device="cuda").to(dtype)
    bb = b.t().contiguous().t() if tn else b
    ops.gemm(at.t(), bb, c, tn=tn, a_km=True)
    want = at.t().double() @ b.double()
    eps = 2.0 ** -10 if dtype == torch.float16 else 2.0 ** -7
    assert torch.isfinite(c).all()
    assert (c.double() - want).abs().max() <= want.abs().max() * eps
    # same numbers as the NN call on a materialised A
    c2 = torch.empty_like(c)
    ops.gemm(at.t().contiguous(), b, c2, variant=2 | (1 << 20))
    ops.gemm(at.t(), bb, c, tn=tn, a_km=True, variant=2 | (1 << 20))
    assert torch.equal(c, c2)


@pytest.mark.parametrize("K", [64, 128, 192, 256, 320, 1024])
@pytest.mark.parametrize("mn", [(512, 256), (1024, 768), (1000, 520), (2048, 2048)])
def test_short_k_fills_the_stage_ring_partly_and_exactly(mn, K):
    """Short K (1 ... 16 k-blocks of 64, so the 4-stage ring is filled partly, exactly and many times over), one and
    several 128 x 256 tiles, ragged M / N, NN and TN storage of B; variant values 4 and 2 of the old ABI are accepted and
    give the same bits as each other and as the TN product (same kernel, same K order)."""
    from b200k import ops

    M, N = mn
    torch.manual_seed(M + K)
    a = torch.randn(M, K, dtype=torch.half, device="cuda")
    b = torch.randn(K, N, dtype=torch.half, device="cuda")
    c = torch.full((M, N), float("nan"), dtype=torch.half, device="cuda")
    ops.hgemm(a, b, c, variant=4)
    want = a.double() @ b.double()
    assert torch.isfinite(c).all()
    assert (c.double() - want).abs().max() <= want.abs().max() * 2.0 ** -10
    c2 = torch.empty_like(c)
    ops.hgemm(a, b, c2, variant=2 | (1 << 20))     # legacy variant value: same kernel, same bits
    assert torch.equal(c, c2)
    ops.hgemm(a, b.t().contiguous().t(), c2, tn=True, variant=4)
    assert torch.equal(c, c2)


@pytest.mark.parametrize("shape", [(4096, 4096, 1024), (2304, 3072, 512)])
def test_gemm_launch_replays_under_cuda_graph(shape):
    """One GEMM launch (one 128 x 256 tile per CTA) captured into a CUDA graph and replayed with new contents of A:
    nothing launch-specific may be frozen into the graph, so every replay equals an eager call on the same operands,
    bit for bit."""
    from b200k import _loader as L
    from b200k import ops

    M, N, K = shape
    torch.manual_seed(7)
    a = torch.randn(M, K, dtype=torch.half, device="cuda")
    b = torch.randn(K, N, dtype=torch.half, device="cuda")
    c = torch.empty(M, N, dtype=torch.half, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            ops.hgemm(a, b, c, variant=L.HGEMM_2CTA_256x256)
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        ops.hgemm(a, b, c, variant=L.HGEMM_2CTA_256x256)
    for rep in range(4):
        a.copy_(torch.randn(M, K, dtype=torch.half, device="cuda"))
        torch.cuda.synchronize()
        c.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        eager = torch.empty_like(c)
        ops.hgemm(a, b, eager, variant=L.HGEMM_2CTA_256x256)
        torch.cuda.synchronize()
        assert torch.equal(c, eager), rep                      # same kernel, same fixed summation order
        want = a.double() @ b.double()
        assert (c.double() - want).abs().max() <= want.abs().max() * 2.0 ** -9, rep
