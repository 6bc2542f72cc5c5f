"""GPU parity: FA-2 / FFPA forward (through the C ABI) vs the CPU oracle, the reference's known-answer fixtures,
golden vectors, ragged / tiny shapes, and full-size (BASELINE configs #3, #4) property checks.
Tolerance = the north star's rtol=1e-2 / atol=1e-3 on fp16 outputs (the reference's own --check uses atol=1e-2,
flash_attn_mma.py:L421)."""
import pytest
import torch

from oracle import oracle

pytestmark = pytest.mark.gpu
TOL = dict(rtol=1e-2, atol=1e-3)


def _run(q, k, v):
    from b200k import ops

    o = torch.full_like(q, float("nan"))
    (ops.fa2_fwd if q.size(-1) <= 128 else ops.ffpa_fwd)(q, k, v, o)
    assert torch.isfinite(o).all()
    return o


@pytest.mark.parametrize("shape", [(1, 2, 256, 64), (1, 1, 128, 64), (2, 3, 1000, 64), (1, 1, 77, 64), (1, 1, 1, 64),
                                   (1, 2, 384, 128), (2, 2, 1000, 128), (1, 2, 512, 32), (1, 2, 333, 32),
                                   (1, 2, 512, 96), (1, 2, 333, 96), (1, 2, 256, 256), (1, 2, 1000, 256),
                                   (1, 2, 512, 512), (1, 1, 384, 320), (1, 1, 300, 192), (1, 1, 256, 1024), (1, 1, 200, 768),
                                   # one and two KV tiles, ragged, for every FA-2 layout (D = 128 shares one S buffer)
                                   (1, 1, 1, 128), (1, 1, 100, 128), (1, 2, 128, 128), (1, 2, 129, 128), (1, 1, 257, 128),
                                   (1, 1, 64, 96), (1, 1, 65, 96), (1, 1, 5, 32), (1, 1, 130, 32), (1, 1, 3, 256), (1, 1, 129, 512)])
def test_attention_vs_oracle(shape):
    B, H, N, D = shape
    torch.manual_seed(N + D)
    q, k, v = [torch.randn(B, H, N, D, dtype=torch.half, device="cuda") for _ in range(3)]
    o = _run(q, k, v)
    assert torch.allclose(o.cpu().float(), oracle.attention(q, k, v).float(), **TOL)


@pytest.mark.parametrize("D", [32, 64, 96, 128, 256, 320])
def test_attention_golden_vectors(golden, D):
    g = golden("seeded_attention_d%d.npz" % D)
    q, k, v = [torch.from_numpy(g[n]).cuda() for n in ("q", "k", "v")]
    o = _run(q, k, v)
    assert torch.allclose(o.cpu().float(), torch.from_numpy(g["o"]).float(), **TOL)


@pytest.mark.parametrize("D", [64, 128, 512])
def test_reference_known_answer_fixtures(golden, D):
    # --no-rand-qkv: all ones -> O == 1 exactly;  --range-k fixture (flash_attn_mma.py:L23-26, L353-369)
    ones = torch.ones(1, 2, 512, D, dtype=torch.half, device="cuda")
    assert torch.equal(_run(ones, ones, ones), ones)
    if D == 64:
        g = golden("kat_attention_range_k.npz")
        q, k, v = [torch.from_numpy(g[n]).cuda() for n in ("q", "k", "v")]
        assert torch.allclose(_run(q, k, v).cpu().float(), torch.from_numpy(g["o"]).float(), **TOL)


def test_large_logits_exercise_lazy_rescale():
    """Scores grow along the key axis so the running max moves by > 2^8 several times (the O-rescale path)."""
    torch.manual_seed(9)
    B, H, N, D = 1, 2, 1024, 64
    q = torch.randn(B, H, N, D, dtype=torch.half, device="cuda")
    k = torch.randn(B, H, N, D, dtype=torch.half, device="cuda")
    ramp = torch.linspace(0, 6, N, device="cuda").half()[None, None, :, None]
    k = (k + ramp * q.mean(dim=2, keepdim=True).sign()).contiguous()
    v = torch.randn(B, H, N, D, dtype=torch.half, device="cuda")
    q = (q * 4).contiguous()
    assert torch.allclose(_run(q, k, v).cpu().float(), oracle.attention(q, k, v).float(), **TOL)
    D = 256
    q, k, v = [(torch.randn(1, 1, 640, D, dtype=torch.half, device="cuda") * s) for s in (3.0, 3.0, 1.0)]
    assert torch.allclose(_run(q, k, v).cpu().float(), oracle.attention(q, k, v).float(), **TOL)


@pytest.mark.parametrize("variant", [0x1C000, 0x8000, 0x10000, 0x1000, 0x2000, 0x3000, 0x400, 0x20000])
@pytest.mark.parametrize("D", [64, 128])
def test_fa2_experiment_builds_agree_with_oracle(D, variant):
    """The variant values of the old ABI are still accepted (each runs the one FA-2 configuration of its head dim) and
    give the oracle's answer; the band of keys with huge |scores| drives exp2 arguments far below -126, which must
    flush to zero, not to NaN or denormal garbage, at a ragged N."""
    from b200k import ops

    torch.manual_seed(D + variant)
    B, H, N = 1, 2, 777
    q, k, v = [torch.randn(B, H, N, D, dtype=torch.half, device="cuda") for _ in range(3)]
    k[:, :, 100:140] *= 24.0  # a band of keys with huge |scores|: exp2 arguments far below -126 for most rows
    o = torch.full_like(q, float("nan"))
    ops.fa2_fwd(q, k, v, o, variant=variant)
    assert torch.isfinite(o).all()
    assert torch.allclose(o.cpu().float(), oracle.attention(q, k, v).float(), **TOL)


@pytest.mark.parametrize("D,variant", [(256, 32), (256, 2), (256, 4), (256, 8), (512, 1), (512, 2), (512, 33), (320, 32),
                                       (512, 0x400), (256, 0x200), (512, 0x200)])
def test_ffpa_selectable_builds_agree_with_oracle(D, variant):
    """The FFPA variant values of the old ABI are still accepted and give the oracle's answer at a ragged N, for head
    dims with one (256) and two (320, 512) column slices of O."""
    from b200k import ops

    torch.manual_seed(D + variant)
    q, k, v = [torch.randn(1, 2, 700, D, dtype=torch.half, device="cuda") for _ in range(3)]
    o = torch.full_like(q, float("nan"))
    ops.ffpa_fwd(q, k, v, o, variant=variant)
    assert torch.isfinite(o).all()
    assert torch.allclose(o.cpu().float(), oracle.attention(q, k, v).float(), **TOL)


def test_flash_attn_lib_and_ffpa_drop_in_entry_points():
    import ffpa_attn
    from b200k import flash_attn_lib

    torch.manual_seed(4)
    q, k, v = [torch.randn(1, 2, 256, 64, dtype=torch.half, device="cuda") for _ in range(3)]
    ref = oracle.attention(q, k, v).float()
    for name in flash_attn_lib.NAMES:
        o = torch.zeros_like(q)
        short = name[len("flash_attn_mma_stages_"):]
        vv = v.transpose(-2, -1).contiguous() if short in flash_attn_lib._V_TRANSPOSED else v
        getattr(flash_attn_lib, name)(q, k, vv, o, 2)
        assert torch.allclose(o.cpu().float(), ref, **TOL), name
    q, k, v = [torch.randn(1, 2, 256, 320, dtype=torch.half, device="cuda") for _ in range(3)]
    ref = oracle.attention(q, k, v).float()
    o = ffpa_attn.ffpa(q, k, v)
    assert torch.allclose(o.cpu().float(), ref, **TOL)
    o2 = torch.zeros_like(q)
    assert ffpa_attn.ffpa(q, k, v, o2, num_stages=3, level=ffpa_attn.L1, acc=ffpa_attn.FP16) is o2
    assert torch.allclose(o2.cpu().float(), ref, **TOL)
    ffpa_attn.ffpa_mma_acc_f32_L1(q, k, v, o2, 2)
    assert torch.allclose(o2.cpu().float(), ref, **TOL)


@pytest.mark.parametrize("shape", [(4, 48, 8192, 64), (1, 32, 4096, 512), (4, 64, 8192, 128)])
def test_full_size_properties(shape):
    """BASELINE configs #3 / #4 / #5-shard.  Size-independent properties:
       (1) V = ones  =>  O == 1 within 1e-3 at full size (test_gpu_attention_graded.py holds constant V to bit equality);
       (2) linearity in V: O(V1 + V2) == O(V1) + O(V2) within tolerance;
       (3) sampled query rows recomputed on the CPU oracle from the full K/V of their head."""
    B, H, N, D = shape
    torch.manual_seed(11)
    q, k, v1 = [torch.randn(B, H, N, D, dtype=torch.half, device="cuda") for _ in range(3)]
    o1 = _run(q, k, v1)
    ones = torch.ones_like(v1)
    assert (_run(q, k, ones).float() - 1.0).abs().max().item() <= 1e-3
    v2 = torch.randn_like(v1)
    o2 = _run(q, k, v2)
    o12 = _run(q, k, (v1.float() + v2.float()).half())
    assert torch.allclose(o12.float(), o1.float() + o2.float(), rtol=1e-2, atol=4e-3)
    for (b, h) in ((0, 0), (B - 1, H - 1)):
        rows = torch.tensor([0, 1, N // 2 + 3, N - 1], device="cuda")
        ref = oracle.attention(q[b, h, rows][None, None], k[b, h][None, None], v1[b, h][None, None])[0, 0]
        assert torch.allclose(o1[b, h, rows].cpu().float(), ref.float(), **TOL)


# ------------------------------------------------------------------------------------------------ SURVEY 8(f)-4 options
@pytest.mark.parametrize("shape", [(1, 2, 256, 64), (2, 3, 1000, 64), (1, 2, 513, 128), (1, 1, 77, 32), (1, 2, 640, 96),
                                   (1, 1, 1, 64), (1, 2, 2048, 128), (1, 1, 255, 64), (1, 1, 257, 64)])
def test_causal_mask_vs_oracle_and_sdpa(shape):
    from b200k import ops

    B, H, N, D = shape
    torch.manual_seed(N * 3 + D)
    q, k, v = [torch.randn(B, H, N, D, dtype=torch.half, device="cuda") for _ in range(3)]
    o = torch.full_like(q, float("nan"))
    ops.fa2_fwd(q, k, v, o, causal=True)
    assert torch.isfinite(o).all()
    assert torch.allclose(o.cpu().float(), oracle.attention(q, k, v, causal=True).float(), **TOL)
    sd = torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=True)
    assert torch.allclose(o.float(), sd.float(), **TOL)
    # row 0 sees only key 0: O[0] == V[0] exactly (softmax of one element, fp16 round trip of V)
    assert torch.equal(o[:, :, 0], v[:, :, 0])


@pytest.mark.parametrize("shape,lens", [((3, 2, 512, 64), [512, 100, 1]), ((2, 2, 1000, 128), [999, 129]),
                                        ((2, 1, 300, 32), [300, 37])])
@pytest.mark.parametrize("causal", [False, True])
def test_key_padding_seqlens_vs_oracle(shape, lens, causal):
    from b200k import ops

    B, H, N, D = shape
    torch.manual_seed(N + D + causal)
    q, k, v = [torch.randn(B, H, N, D, dtype=torch.half, device="cuda") for _ in range(3)]
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    o = torch.full_like(q, float("nan"))
    ops.fa2_fwd(q, k, v, o, causal=causal, seqlens_k=sl)
    want = oracle.attention(q, k, v, causal=causal, seqlens=lens).float()
    assert torch.isfinite(o).all()
    assert torch.allclose(o.cpu().float(), want, **TOL)
    # keys past the length must not influence anything: poison them and recompute
    k2, v2 = k.clone(), v.clone()
    for b, n in enumerate(lens):
        k2[b, :, n:] = 1e4
        v2[b, :, n:] = -1e4
    o2 = torch.empty_like(o)
    ops.fa2_fwd(q, k2, v2, o2, causal=causal, seqlens_k=sl)
    assert torch.equal(o, o2)


@pytest.mark.parametrize("shape", [(1, 2, 256, 64), (2, 2, 1000, 128), (1, 2, 333, 32), (1, 2, 512, 96), (1, 4, 4096, 64)])
@pytest.mark.parametrize("causal", [False, True])
def test_bf16_attention_vs_oracle(shape, causal):
    """bf16 Q/K/V/O and P (SURVEY 8f-4): fp32 statistics and accumulators; P and O carry bf16's 2^-9 relative rounding."""
    from b200k import ops

    B, H, N, D = shape
    torch.manual_seed(N + D)
    q, k, v = [torch.randn(B, H, N, D, device="cuda").bfloat16() for _ in range(3)]
    o = torch.full_like(q, float("nan"))
    ops.fa2_fwd(q, k, v, o, causal=causal)
    want = oracle.attention(q, k, v, causal=causal).float()
    assert o.dtype == torch.bfloat16 and torch.isfinite(o).all()
    # tolerance: the north star's rtol with bf16's 8x coarser mantissa: rtol 1e-2 -> 2e-2, atol 1e-3 -> 8e-3 / sqrt(keys) scale
    assert torch.allclose(o.cpu().float(), want, rtol=2e-2, atol=4e-3)
    sd = torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=causal)
    assert (o.float() - want.cuda()).abs().max() <= 2.0 * (sd.float() - want.cuda()).abs().max() + 2e-3


def test_causal_config3_full_size_properties():
    """(4,48,8192,64) causal: sampled rows against an fp32 reference on the GPU, and tile skipping must not change rows."""
    from b200k import ops

    B, H, N, D = 2, 8, 8192, 64
    torch.manual_seed(8)
    q, k, v = [torch.randn(B, H, N, D, dtype=torch.half, device="cuda") for _ in range(3)]
    o = torch.empty_like(q)
    ops.fa2_fwd(q, k, v, o, causal=True)
    rows = torch.tensor([0, 1, 127, 128, 255, 256, 4095, 4096, 8191], device="cuda")
    s = (q[:, :, rows].float() @ k.float().transpose(-1, -2)) / D ** 0.5
    s = s.masked_fill(torch.arange(N, device="cuda").view(1, 1, 1, N) > rows.view(1, 1, -1, 1), float("-inf"))
    want = torch.softmax(s, -1) @ v.float()
    assert torch.allclose(o[:, :, rows].float(), want, **TOL)
    # the first 1024 rows only depend on the first 1024 keys: a shorter problem gives the same bits
    o2 = torch.empty(B, H, 1024, D, dtype=torch.half, device="cuda")
    ops.fa2_fwd(q[:, :, :1024].contiguous(), k[:, :, :1024].contiguous(), v[:, :, :1024].contiguous(), o2, causal=True)
    assert torch.equal(o2, o[:, :, :1024])


@pytest.mark.parametrize("D", [192, 256, 320, 384, 448, 512, 576, 640, 704, 768, 832, 896, 960, 1024])
def test_ffpa_every_ladder_rung(D):
    """Every head dim of the reference's ladder (ffpa-attn-mma/csrc/cuffpa/launch_templates.cuh:L529-551), ragged N."""
    torch.manual_seed(D)
    q, k, v = [torch.randn(1, 2, 300, D, dtype=torch.half, device="cuda") for _ in range(3)]
    o = _run(q, k, v)
    assert torch.allclose(o.cpu().float(), oracle.attention(q, k, v).float(), **TOL)


@pytest.mark.parametrize("D", [160, 224, 288, 352, 480, 544, 736, 992])
def test_ffpa_step32_head_dims(D):
    """The reference's ENABLE_FFPA_ALL_HEADDIM rungs (ffpa-attn-mma/csrc/cuffpa/launch_templates.cuh:L483-552): head dims
    that are multiples of 32 but not of 64.  The last 64-wide chunk of Q / K / V is half outside the tensor (TMA zero fill)
    and the last chunk of O is clipped by the TMA store; memory after O's last row must stay untouched."""
    from b200k import ops

    torch.manual_seed(D)
    N = 300
    q, k, v = [torch.randn(1, 2, N, D, dtype=torch.half, device="cuda") for _ in range(3)]
    buf = torch.full((1 * 2 * N * D + 4096,), 7.0, dtype=torch.half, device="cuda")
    o = buf[:2 * N * D].view(1, 2, N, D)
    ops.ffpa_fwd(q, k, v, o)
    torch.cuda.synchronize()
    assert torch.allclose(o.cpu().float(), oracle.attention(q, k, v).float(), **TOL)
    assert bool((buf[2 * N * D:] == 7.0).all())
    ones = torch.ones_like(v)
    ops.ffpa_fwd(q, k, ones, o)
    assert torch.allclose(o.float(), torch.ones_like(o).float(), atol=1e-3)


@pytest.mark.parametrize("D", [256, 512])
@pytest.mark.parametrize("N", [1, 63, 128, 255, 256, 257, 511, 1000, 2304])
def test_ffpa_otrans_kernel_shapes(D, N):
    """One, two and many 64-key tiles, ragged N, several heads, one (D = 256) and two (D = 512) column slices of O, against
    the oracle; two legacy variant values give the same answer; V = 1 gives O = 1 exactly (row sums of the rounded P)."""
    from b200k import ops

    torch.manual_seed(N * 7 + D)
    q, k, v = [torch.randn(2, 3, N, D, dtype=torch.half, device="cuda") for _ in range(3)]
    o = torch.full_like(q, float("nan"))
    ops.ffpa_fwd(q, k, v, o, variant=0x200)
    assert torch.isfinite(o).all()
    assert torch.allclose(o.cpu().float(), oracle.attention(q, k, v).float(), **TOL)
    o2 = torch.empty_like(o)
    ops.ffpa_fwd(q, k, v, o2, variant=0x400 if D == 512 else 0)
    assert torch.allclose(o.float(), o2.float(), rtol=1e-2, atol=1e-3)
    ones = torch.ones_like(v)
    ops.ffpa_fwd(q, k, ones, o, variant=0x200)
    assert torch.equal(o, ones)


@pytest.mark.parametrize("D", [256, 512])
def test_ffpa_otrans_cross_cta_rescale(D):
    """Scores that grow along the key axis move the running max of the rows by large steps in many tiles (the O rescale
    path of the online softmax): first only rows 0-63 of every 128 (every other 64-row query block), then all rows."""
    from b200k import ops

    torch.manual_seed(11 + D)
    B, H, N = 1, 2, 1536
    q = torch.randn(B, H, N, D, dtype=torch.half, device="cuda")
    v = torch.randn(B, H, N, D, dtype=torch.half, device="cuda")
    base = torch.randn(B, H, N, D, device="cuda") * 0.1
    qdir = q[:, :, :1].float() / q[:, :, :1].float().norm(dim=-1, keepdim=True)
    ramp = torch.linspace(0, 90, N, device="cuda").view(1, 1, N, 1)
    k = (base + ramp * qdir * 0.4).half()
    for rows in ("all", "first_half_of_each_tile"):
        qq = q.clone()
        if rows == "first_half_of_each_tile":
            idx = torch.arange(N, device="cuda")
            qq[:, :, (idx % 128) >= 64] *= 0.01          # these rows see flat scores: only the other blocks' rows move
        qq[:, :, :, :] = qq + 4.0 * qdir.half()           # every active row is pulled along the ramp direction
        o = torch.full_like(qq, float("nan"))
        ops.ffpa_fwd(qq, k, v, o, variant=0x200)
        want = oracle.attention(qq, k, v).float()
        assert torch.isfinite(o).all()
        assert torch.allclose(o.cpu().float(), want, **TOL), rows
