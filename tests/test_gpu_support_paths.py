"""Every launch path of the bandwidth kernels (csrc/support_kernels.cu, csrc/support_kernels2.cu) against exact answers
or fp64 bounds, at shapes taken from the launch rules (tests/support_paths.py) for the SM count of this card: both
sides of every path switch, exactly one pass of each grid-stride loop, one pass plus one row, and several passes
ending on a partial CTA.

Every output is pre-filled with NaN and followed by a guard element, so a skipped element fails and a write past the
end is caught.  Every 16-byte path is also run on views offset by one element, which sends it to the scalar path.
Reductions, dot products, GEMV, elementwise add, relu / hardshrink and the transposes are checked bit for bit on inputs
whose answer is exact; the row kernels and the other activations against fp64 references with a bound derived from the
kernel's arithmetic, written next to each check."""
import math

import pytest
import torch

import support_paths as P
from oracle import oracle

pytestmark = pytest.mark.gpu

U = 2.0 ** -24        # unit roundoff of fp32
U16 = 2.0 ** -11      # unit roundoff of fp16 (the one rounding of an f16 output)
SUB16 = 2.0 ** -25    # half the smallest fp16 subnormal: the rounding of a tiny f16 output
GUARD = -7.0          # exact in every dtype used here; no kernel here writes it
EPS = 9.999999747378752e-06  # 1e-5 as the fp32 the kernels receive
DT = {torch.float32: "f32", torch.float16: "f16", torch.bfloat16: "bf16", torch.int8: "i8",
      torch.float8_e4m3fn: "fp8", torch.float8_e5m2: "fp8"}


@pytest.fixture(scope="module")
def sm():
    from b200k import _loader as L

    return L.device_info()["sm_count"]  # b200k_device_info: the count the launchers size their grids from


def _placed(x, off):
    """x copied to a fresh buffer at element offset `off` (1: not 16-byte aligned, so every launcher takes its scalar
    path)."""
    buf = torch.empty(x.numel() + 1, dtype=x.dtype, device=x.device)
    v = buf[off:off + x.numel()].view(x.shape)
    v.copy_(x)
    return v


def _out(n, dtype, off):
    """(buffer, output view of n elements at offset `off`): NaN everywhere, GUARD right after the view."""
    buf = torch.full((n + 2,), float("nan"), dtype=dtype, device="cuda")
    buf[off + n] = GUARD
    return buf, buf[off:off + n]


def _guard_ok(buf, n, off, what):
    assert buf[off + n].item() == GUARD, "%s: wrote past the end of its output" % what
    if off:
        assert math.isnan(buf[0].item()), "%s: wrote before the start of its output" % what


def _first_bad(ok):
    bad = (~ok).nonzero()
    return None if bad.numel() == 0 else [int(v) for v in bad[0]]


# ------------------------------------------------------------------------------------------------ row kernels
NEEDLE = {"softmax": 4.0, "rms_norm": 32.0, "layer_norm": 32.0}
LN_SHIFT = 16.0  # layer-norm rows are 16 +- 1, so the mean matters: dividing by K - 1 moves y by ~16 / K


def _row_input(rows, H, dtype, kind, positions, seed):
    """+-1 values (16 +- 1 for layer norm) with one needle per row at a position drawn from `positions`, so rows in
    different CTAs and passes carry it at different places; softmax rows also hold a -inf in every third row.  Every
    value is exact in fp16."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randint(0, 2, (rows, H), generator=g, device="cuda", dtype=torch.int8).float() * 2 - 1
    where = torch.tensor(positions, device="cuda")[torch.randint(0, len(positions), (rows,), generator=g, device="cuda")]
    r = torch.arange(rows, device="cuda")
    x[r, where] = NEEDLE[kind]
    if kind == "layer_norm":
        x += LN_SHIFT
    if kind == "softmax":
        x[r[::3], (where[::3] + H // 2) % H] = float("-inf")
    return x.to(dtype), where


def _row_depth(H, plan):
    """Longest chain of fp32 additions behind one row sum: the values one thread adds in turn (at least the 32 a
    thread holds in registers), then the 5 warp shuffle levels and up to 8 per-warp partials."""
    per_thread = -(-H // (plan.R or P.THREADS)) + P.VN["f32"]
    return max(32, per_thread) + 13


def _total_depth(n, sm):
    """The chain behind softmax mode 0's whole-tensor total: one thread's share of the n values (the scalar loop's is
    the longest), the CTA's shuffle tree, one thread's share of at most 2048 partials and the final tree."""
    return -(-n // P.reduce("f32", n, sm, aligned=False).per_pass) + 40


def _softmax_ref(x64, mode, depth):
    """fp64 softmax and its bound.  Kernel: exp(x - m) as ex2.approx(fma(x, log2e, -m log2e)) (argument rounding
    |t| u <= 12 u, i.e. 9 u relative after exp; ex2.approx 2 u), a sum of positive terms with relative error <= depth u,
    one IEEE division, one product: relative error <= (depth + 16) u."""
    if mode == 0:
        e = torch.exp(x64)
        want = e / e.sum()
    else:
        want = torch.softmax(x64, dim=-1)
    return want, (depth + 16) * U * want.abs()


def _rms_ref(x64, g, inside, H):
    """fp64 RMS norm and its bound.  The sum of squares of these integers is exact in fp32 and in the half
    accumulation (per-thread partials <= 32^2 + 31 <= 2048); then two roundings in the denominator, rsqrtf (2 ulp =
    4 u), the product with g and with x: relative error <= 10 u; 16 u written."""
    s = (x64 * x64).sum(-1, keepdim=True)
    denom = s / (H + EPS) if inside else s / H + EPS
    want = x64 * (g / denom.sqrt())
    return want, 16 * U * want.abs()


def _ln_ref(x64, g, b, inside, K, depth):
    """fp64 layer norm and its bound.  The row sum of these integers is exact; the mean is one rounding off
    (u |mean|), each d = x - mean one more (u (|d| + |mean|)), the sum of squares (depth + 2) u relative, then two
    roundings, rsqrtf (4 u) and the product with g for a = g / std (half the q error + 7 u), and one fma for y:
    |dy| <= |a| (|d| (depth / 2 + 9) + 2 |mean|) u + u |y| < (depth + 16) u |a| (|d| + |mean|) + u |y|."""
    mean = x64.mean(-1, keepdim=True)
    d = x64 - mean
    q = (d * d).sum(-1, keepdim=True)
    var = q / (K + EPS) if inside else q / K + EPS
    a = g / var.sqrt()
    want = d * a + b
    return want, (depth + 16) * U * a * (d.abs() + mean.abs()) + U * want.abs()


def _row_ops(kind, dtype, H, depth, sm):
    """(label, run(x, y), reference(x64) -> (want, bound)) for every variant of one row kernel."""
    from b200k import ops

    if kind == "softmax":
        modes = [ops.SOFTMAX_PER_TOKEN, ops.SOFTMAX_SAFE, ops.SOFTMAX_ONLINE] + ([ops.SOFTMAX_ALL] if dtype == torch.float32 else [])
        return [("softmax mode %d" % m, (lambda x, y, m=m: ops.softmax(x, y, m)),
                 (lambda x64, m=m: _softmax_ref(x64, m, depth + (_total_depth(x64.numel(), sm) if m == 0 else 0))))
                for m in modes]
    if kind == "rms_norm":
        combos = [(a, i) for a in ((False, True) if dtype == torch.float16 else (False,)) for i in (False, True)]
        return [("rms_norm acc_f16=%d eps_inside_k=%d" % (a, i),
                 (lambda x, y, a=a, i=i: ops.rms_norm(x, y, 1.5, EPS, acc_f16=a, eps_inside_k=i)),
                 (lambda x64, i=i: _rms_ref(x64, 1.5, i, H))) for a, i in combos]
    return [("layer_norm eps_inside_k=%d" % i, (lambda x, y, i=i: ops.layer_norm(x, y, 1.25, -0.5, EPS, eps_inside_k=i)),
             (lambda x64, i=i: _ln_ref(x64, 1.25, -0.5, i, H, depth))) for i in (True, False)]


def _check_rows(y, want, bound, dtype, label, where, plan, rows):
    if dtype == torch.float16:  # one rounding to fp16 on top: 2^-11 relative, 2^-25 absolute below the normal range
        bound = bound + U16 * want.abs() + SUB16
    ok = (y.double() - want).abs() <= bound
    bad = _first_bad(ok)
    if bad is not None:
        r, c = bad
        raise AssertionError("%s %s H=%d rows=%d (%s path, R=%s, cached=%s, %d rows per pass): row %d (pass %d) col %d "
                             "is %r, want %r +- %.3g; this row's needle is at col %d"
                             % (label, DT[dtype], want.shape[1], rows, "16-byte" if plan.vector else "scalar", plan.R,
                                plan.cached, plan.per_pass, r, r // plan.per_pass, c, float(y[r, c]), float(want[r, c]),
                                float(bound[r, c]), int(where[r])))


ROW_WIDTHS = ["1024", "1024+VN", "4096", "4096+VN", "8192", "8192+VN", "H%VN!=0"]


@pytest.mark.parametrize("kind", ["softmax", "rms_norm", "layer_norm"])
@pytest.mark.parametrize("width", ROW_WIDTHS)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_row_kernels_every_path(dtype, width, kind, sm):
    """Softmax in all four modes, rms_norm in every acc_f16 / eps_inside_k combination, layer_norm both eps forms, at
    H on both sides of each switch and at one pass, one pass + 1 row and two passes + a partial CTA of rows; the
    longest case also offset by one element (scalar path)."""
    dt = DT[dtype]
    H = P.row_widths(dt)[ROW_WIDTHS.index(width)]
    plan = P.full_rows(dt, H, sm)
    counts = P.pass_counts(plan, P.THREADS // plan.R if plan.R else 1)
    x, where = _row_input(counts["two+"], H, dtype, kind, P.row_positions(dt, H, plan), seed=H + len(kind))
    x64 = x.double()
    for label, run, ref in _row_ops(kind, dtype, H, _row_depth(H, plan), sm):
        full = None if "mode 0" in label else ref(x64)  # row-wise: the reference of a prefix of rows is a prefix
        for cname, rows in counts.items():
            for off in ((0, 1) if cname == "two+" else (0,)):
                p = P.row(dt, rows, H, sm, aligned=off == 0)
                want, bound = ref(x64[:rows]) if full is None else (full[0][:rows], full[1][:rows])
                buf, y = _out(rows * H, dtype, off)
                run(_placed(x[:rows], off), y.view(rows, H))
                _check_rows(y.view(rows, H), want, bound, dtype, label, where, p, rows)
                _guard_ok(buf, rows * H, off, label)


# ------------------------------------------------------------------------------------------------ reductions, dot product
def _reduce_digits(dtype):
    """How many needles 4^0 .. 4^(d-1) the dtype holds exactly (e4m3 tops out at 448, fp16 at 65504, int8 at 127)."""
    return {torch.float32: 12, torch.bfloat16: 12, torch.float16: 8, torch.float8_e5m2: 8, torch.float8_e4m3fn: 5,
            torch.int8: 4}[dtype]


def _needle_groups(positions, digits, vn):
    """Positions split into calls of at most `digits` needles with at most one needle per 16-byte pack, so a pack
    summed in half precision holds one power of two and stays exact."""
    groups = []
    for p in positions:
        for g in groups:
            if len(g) < digits and all(q // vn != p // vn for q in g):
                g.append(p)
                break
        else:
            groups.append([p])
    return groups


def _decode(total, group, what):
    """The sum of needles 4^k at group[k] written in base 4: digit k says how often group[k] was counted."""
    want = sum(4 ** k for k in range(len(group)))
    assert math.isfinite(total), "%s: sum %r" % (what, total)
    if total != want:
        counts = [(int(total) // 4 ** k) % 4 for k in range(len(group))]
        wrong = ["position %d counted %d times" % (p, c) for p, c in zip(group, counts) if c != 1]
        raise AssertionError("%s: sum %r, want %d: %s" % (what, total, want, ", ".join(wrong) or "carry out of range"))


REDUCE_NAMES = ["f32_f32", "f32x4_f32", "f16_f16", "f16_f32", "f16x2_f16", "f16x2_f32", "f16x8_pack_f16",
                "f16x8_pack_f32", "bf16_bf16", "bf16_f32", "bf16x2_bf16", "bf16x2_f32", "bf16x8_pack_bf16",
                "bf16x8_pack_f32", "fp8_e4m3_f16", "fp8_e4m3x16_pack_f16", "fp8_e5m2_f16", "fp8_e5m2x16_pack_f16",
                "i8_i32", "i8x16_pack_i32"]


@pytest.mark.parametrize("name", REDUCE_NAMES)
def test_block_all_reduce_needles_and_exact_sums(name, sm):
    """All 20 block_all_reduce_sum names.  Needles at the pack edges, CTA shares, pass starts (including the 4-way
    unrolled body and its remainder loop) and the scalar tail of a 5-pass input, aligned and offset by one; then dense
    small integers whose every partial sum is exact, bit for bit against the integer sum."""
    from b200k import support_libs

    dtype = support_libs._REDUCE[name][0]
    fn = getattr(support_libs.reduce_lib, "block_all_reduce_sum_" + name)
    vn = P.VN[DT[dtype]]
    stride = P.reduce(DT[dtype], 1 << 40, sm).per_pass
    n = (5 * stride + 77) * vn + vn - 1
    for off in (0, 1):
        plan = P.reduce(DT[dtype], n, sm, aligned=off == 0)
        positions = P.reduce_positions(DT[dtype], n, plan)
        for group in _needle_groups(positions, _reduce_digits(dtype), vn):
            x = torch.zeros(n, dtype=torch.float32, device="cuda")
            x[group] = torch.tensor([4.0 ** k for k in range(len(group))], device="cuda")
            got = fn(_placed(x.to(dtype), off))
            _decode(got.item(), group, "%s n=%d offset %d (%d per pass)" % (name, n, off, plan.per_pass))
    # dense: values in [-3, 3], |every partial| <= 3 n < 2^24, so the fp32 (and half-pack) sums are exact
    n = min(2 * stride * vn + vn - 1, (1 << 24) // 3 - 1)
    g = torch.Generator(device="cuda").manual_seed(n)
    ints = torch.randint(-3, 4, (n,), generator=g, device="cuda")
    want = int(ints.sum())
    for off in (0, 1):
        got = fn(_placed(ints.to(torch.float32).to(dtype), off))
        assert got.item() == want, (name, off, got.item(), want)


@pytest.mark.parametrize("name", ["dot_prod_f32_f32", "dot_prod_f32x4_f32", "dot_prod_f16_f32", "dot_prod_f16x2_f32",
                                  "dot_prod_f16x8_pack_f32"])
def test_dot_product_needles_and_exact_sums(name, sm):
    """All 5 dot_prod names: a holds needles +-4^k, b the matching sign (+-1 elsewhere), at the same positions as the
    reduction, aligned and offset by one; then dense small integers with an exact sum."""
    from b200k import support_libs

    dtype = torch.float16 if "f16" in name else torch.float32
    fn = getattr(support_libs.dot_product_lib, name)
    vn = P.VN[DT[dtype]]
    stride = P.dot(DT[dtype], 1 << 40, sm).per_pass
    n = (5 * stride + 77) * vn + vn - 1
    g = torch.Generator(device="cuda").manual_seed(7)
    sign = torch.randint(0, 2, (n,), generator=g, device="cuda").float() * 2 - 1
    for off in (0, 1):
        plan = P.dot(DT[dtype], n, sm, aligned=off == 0)
        for group in _needle_groups(P.reduce_positions(DT[dtype], n, plan), 8 if dtype == torch.float16 else 12, 1):
            a = torch.zeros(n, device="cuda")
            a[group] = torch.tensor([4.0 ** k for k in range(len(group))], device="cuda") * sign[group]
            got = fn(_placed(a.to(dtype), off), _placed(sign.to(dtype), off))
            _decode(got.item(), group, "%s n=%d offset %d (%d per pass)" % (name, n, off, plan.per_pass))
    n = 2 * stride * vn + vn - 1  # |a b| <= 2: every partial <= 2 n < 2^24
    a = torch.randint(-1, 2, (n,), generator=g, device="cuda")
    b = torch.randint(-2, 3, (n,), generator=g, device="cuda")
    want = int((a * b).sum())
    for off in (0, 1):
        got = fn(_placed(a.to(dtype), off), _placed(b.to(dtype), off))
        assert got.item() == want, (name, off, got.item(), want)


# ------------------------------------------------------------------------------------------------ GEMV
@pytest.mark.parametrize("kidx", range(6))
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_gemv_exact_across_vector_counts_and_passes(dtype, kidx, sm):
    """K at 32 / 33 / 64 / 65 / 129 vectors and with a tail, M over two passes of warps plus a partial CTA; +-1
    entries make y an integer with |y| <= K <= 2048, exact in fp16.  The widest K also runs with A offset by one."""
    from b200k import ops

    dt = DT[dtype]
    K = P.gemv_widths(dt)[kidx]
    M = 2 * P.gemv(dt, 1 << 30, K, sm).per_pass + 5
    g = torch.Generator(device="cuda").manual_seed(K)
    a = (torch.randint(0, 2, (M, K), generator=g, device="cuda") * 2 - 1).to(dtype)
    x = (torch.randint(0, 2, (K, 1), generator=g, device="cuda") * 2 - 1).to(dtype)
    want = a.double() @ x.double()
    for off in ((0, 1) if kidx == 4 else (0,)):
        plan = P.gemv(dt, M, K, sm, aligned=off == 0)
        buf, y = _out(M, dtype, 0)
        ops.gemv(_placed(a, off), x, y.view(M, 1))
        ok = y.view(M, 1).double() == want
        bad = _first_bad(ok)
        assert bad is None, ("gemv %s K=%d M=%d (%s path, %d rows per pass): row %d is %r, want %r"
                             % (dt, K, M, "16-byte" if plan.vector else "scalar", plan.per_pass, bad[0],
                                float(y[bad[0]]), float(want[bad[0], 0])))
        _guard_ok(buf, M, 0, "gemv")


# ------------------------------------------------------------------------------------------------ activations, add
ACTS = ["relu", "sigmoid", "gelu", "swish", "elu", "hardswish", "hardshrink"]


def _act_input(n, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, generator=g, device="cuda") * 4.0
    special = torch.tensor([0.0, -0.0, 0.5, -0.5, 3.0, -3.0, 11.09375, 12.0, -9.703125, -12.0, 60.0, -100.0],
                           device="cuda")
    x[:special.numel()] = special
    x[-special.numel():] = special  # the tail too
    return x.to(dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("op", ACTS)
def test_activations_across_passes_and_tails(op, dtype, sm):
    """A full pass of 1024-vector chunks plus a partial chunk and a VN - 1 tail, aligned and offset by one (the scalar
    loop, many passes), then every tail 1 .. VN - 1 on a short input."""
    from b200k import ops

    dt = DT[dtype]
    vn = P.VN[dt]
    big = (P.activation(dt, 1 << 40, sm).per_pass + 2 * 1024 + 5) * vn + vn - 1
    cases = [(big, 0), (big, 1)] + [(3 * 1024 * vn + t, 0) for t in range(1, vn)]
    clamps = (True, False) if op in ("sigmoid", "gelu") else (True,)
    base = _act_input(big + 1, dtype, seed=len(op))
    for clamp in clamps:
        want_all = oracle.activation(base, op, ref_clamp=clamp).cuda()
        for n, off in cases:
            x = base[off:off + n]
            want = want_all[off:off + n]
            buf, y = _out(n, dtype, off)
            ops.activation(x, y, op, ref_clamp=clamp)
            got = y.double()
            if op in ("relu", "hardshrink"):
                ok = got == want
            elif dtype == torch.float32:  # ex2.approx / rcp.approx: 2^-22 relative each; gelu multiplies by |x| <= 100
                ok = (got - want).abs() <= 2e-6 * want.abs() + 1e-6
            else:  # one rounding to fp16 (2^-11 relative) on top of the fp32 evaluation
                ok = (got - want).abs() <= 1e-3 * want.abs() + 1e-6
            bad = _first_bad(ok)
            plan = P.activation(dt, n, sm, aligned=off == 0)
            assert bad is None, ("%s %s n=%d offset %d clamp=%s (%d %s per pass): element %d is %r, want %r"
                                 % (op, dt, n, off, clamp, plan.per_pass, plan.unit, bad[0], float(got[bad[0]]),
                                    float(want[bad[0]])))
            _guard_ok(buf, n, off, op)


def _add_cases(dtype, sm):
    vn = P.VN[DT[dtype]]
    stride = P.add(DT[dtype], 1 << 40, sm).per_pass
    big = (5 * stride + 77) * vn + vn - 1  # the 4-way unrolled body once, its remainder loop, then the tail
    return [(big, 0), (big, 1)] + [(2 * stride * vn + t, 0) for t in range(1, vn)]


def _check_add(fn, dtype, n, off, what, sm):
    g = torch.Generator(device="cuda").manual_seed(n)
    a = torch.randn(n + 1, generator=g, device="cuda").to(dtype)
    b = torch.randn(n + 1, generator=g, device="cuda").to(dtype)
    a, b = a[off:off + n], b[off:off + n]
    want = a + b if dtype == torch.float32 else (a.float() + b.float()).to(dtype)  # one IEEE rounding, like __hadd
    buf, c = _out(n, dtype, off)
    fn(a, b, c)
    bad = _first_bad(c == want)
    plan = P.add(DT[dtype], n, sm, aligned=off == 0)
    assert bad is None, ("%s n=%d offset %d (%d %s per pass): element %d is %r, want %r"
                         % (what, n, off, plan.per_pass, plan.unit, bad[0], float(c[bad[0]]), float(want[bad[0]])))
    _guard_ok(buf, n, off, what)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_elementwise_add_across_passes_and_tails(dtype, sm):
    from b200k import ops

    for n, off in _add_cases(dtype, sm):
        _check_add(ops.elementwise_add, dtype, n, off, "elementwise_add %s" % DT[dtype], sm)


# ------------------------------------------------------------------------------------------------ transposes
@pytest.mark.parametrize("shape", ["vec4", "ragged", "vec4 offset"])
def test_transpose_f32_across_tile_passes(shape, sm):
    """More than two passes of 64 x 64 tiles with ragged last tiles: 16-byte (M, N multiples of 4), scalar (ragged),
    and the 16-byte shape offset by one (scalar).  Bit for bit."""
    from b200k import ops

    M, N = P.tiles_past_passes(sm, 2, (5, 3) if shape == "ragged" else (4, 60))
    off = 1 if "offset" in shape else 0
    g = torch.Generator(device="cuda").manual_seed(M)
    x = _placed(torch.randn(M, N, generator=g, device="cuda"), off)
    buf, y = _out(M * N, torch.float32, off)
    ops.mat_transpose(x, y.view(N, M))
    assert P.transpose_f32(M, N, sm, aligned=off == 0).vector == (shape == "vec4")
    bad = _first_bad(y.view(N, M) == x.t())
    assert bad is None, "transpose %dx%d (%s): y[%d, %d] wrong" % (M, N, shape, bad[0], bad[1])
    _guard_ok(buf, M * N, off, "transpose")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_transpose_16bit_batched_across_tile_passes(dtype, sm):
    """Three batch entries of ragged 21 x tn tiles, more than two passes of the grid in all; every bit pattern (NaN
    payloads included) must come through, so the check compares raw 16-bit words."""
    from b200k import ops

    batch, M = 3, 20 * 64 + 5
    tn = -(-(2 * P.transpose_u16(1, 1 << 20, 1 << 20, sm).per_pass + 1) // (batch * 21))
    N = (tn - 1) * 64 + 3
    assert P.transpose_u16(batch, M, N, sm).passes(batch * 21 * tn) >= 3
    g = torch.Generator(device="cuda").manual_seed(N)
    bits = torch.randint(-32768, 32768, (batch, M, N), generator=g, device="cuda", dtype=torch.int32).to(torch.int16)
    buf, y = _out(batch * M * N, dtype, 0)
    ops.transpose_16bit_batched(bits.view(dtype), y.view(batch, N, M))
    bad = _first_bad(y.view(torch.int16).view(batch, N, M) == bits.transpose(1, 2))
    assert bad is None, "transpose_16bit_batched %s [%d, %d, %d]: y%s wrong" % (DT[dtype], batch, M, N, bad)
    assert buf.view(torch.int16)[batch * M * N] == torch.tensor(GUARD, dtype=dtype).view(torch.int16).item()


# ------------------------------------------------------------------------------------------------ drop-in names
RMS_NAMES = {"rms_norm_f32": (torch.float32, False, False), "rms_norm_f32x4": (torch.float32, False, False),
             "rms_norm_f16_f16": (torch.float16, True, True), "rms_norm_f16x2_f16": (torch.float16, True, True),
             "rms_norm_f16x8_f16": (torch.float16, True, True), "rms_norm_f16x8_f32": (torch.float16, False, True),
             "rms_norm_f16_f32": (torch.float16, False, True), "rms_norm_f16x8_pack_f16": (torch.float16, True, True),
             "rms_norm_f16x8_pack_f32": (torch.float16, False, True)}


@pytest.mark.parametrize("name", sorted(RMS_NAMES))
def test_rms_norm_lib_names(name, sm):
    """Each rms_norm_lib name at H = 4096 + VN (R = 256, cached) and one pass plus one row: the half-accumulating
    names (acc_f16) and the reference's rsqrt(sum / (K + eps)) form, against the fp64 bound."""
    from b200k import support_libs

    dtype, _, inside = RMS_NAMES[name]
    dt = DT[dtype]
    H = 4096 + P.VN[dt]
    plan = P.full_rows(dt, H, sm)
    rows = plan.per_pass + 1
    x, where = _row_input(rows, H, dtype, "rms_norm", P.row_positions(dt, H, plan), seed=len(name))
    buf, y = _out(rows * H, dtype, 0)
    getattr(support_libs.rms_norm_lib, name)(x, y.view(rows, H), 1.5)
    want, bound = _rms_ref(x.double(), 1.5, inside, H)
    _check_rows(y.view(rows, H), want, bound, dtype, name, where, plan, rows)
    _guard_ok(buf, rows * H, 0, name)


SOFTMAX_NAMES = ["softmax_f32", "softmax_f32x4", "softmax_f32_per_token", "softmax_f32x4_per_token",
                 "safe_softmax_f32_per_token", "safe_softmax_f32x4_per_token", "safe_softmax_f16_f32_per_token",
                 "safe_softmax_f16x2_f32_per_token", "safe_softmax_f16x8_pack_f32_per_token",
                 "online_safe_softmax_f32_per_token", "online_safe_softmax_f32x4_pack_per_token"]


@pytest.mark.parametrize("name", SOFTMAX_NAMES)
def test_softmax_lib_names(name, sm):
    """Each softmax_lib name at H = 1024 + VN (R = 128) and one pass plus one row; softmax_f32 / softmax_f32x4 are
    the whole-tensor mode."""
    from b200k import support_libs

    dtype = torch.float16 if "f16" in name else torch.float32
    dt = DT[dtype]
    H = 1024 + P.VN[dt]
    plan = P.full_rows(dt, H, sm)
    rows = plan.per_pass + 1
    x, where = _row_input(rows, H, dtype, "softmax", P.row_positions(dt, H, plan), seed=len(name))
    buf, y = _out(rows * H, dtype, 0)
    getattr(support_libs.softmax_lib, name)(x, y.view(rows, H))
    whole = name in ("softmax_f32", "softmax_f32x4")
    want, bound = _softmax_ref(x.double(), 0 if whole else 1, _row_depth(H, plan) + (_total_depth(x.numel(), sm) if whole else 0))
    _check_rows(y.view(rows, H), want, bound, dtype, name, where, plan, rows)
    _guard_ok(buf, rows * H, 0, name)


@pytest.mark.parametrize("name", ["elementwise_add_f32", "elementwise_add_f32x4", "elementwise_add_f16",
                                  "elementwise_add_f16x2", "elementwise_add_f16x8", "elementwise_add_f16x8_pack"])
def test_elementwise_lib_names(name, sm):
    """Each elementwise_lib name over two passes of the 16-byte loop plus a VN - 1 tail, and offset by one."""
    from b200k import support_libs

    dtype = torch.float16 if "f16" in name else torch.float32
    vn = P.VN[DT[dtype]]
    n = 2 * P.add(DT[dtype], 1 << 40, sm).per_pass * vn + vn - 1
    for off in (0, 1):
        _check_add(getattr(support_libs.elementwise_lib, name), dtype, n, off, name, sm)


@pytest.mark.parametrize("name", ["embedding_f32", "embedding_f32x4", "embedding_f32x4_pack", "embedding_f16",
                                  "embedding_f16x8", "embedding_f16x8_pack"])
def test_embedding_lib_names(name, sm):
    """Each embedding_lib name over one pass of warps plus five rows, with 16-byte rows (100 fp32, 104 fp16) and
    2-byte rows (100 fp16), and indices out of range (-1, rows), which give zero rows.  Bit for bit."""
    from b200k import support_libs

    dtype = torch.float16 if "f16" in name else torch.float32
    fn = getattr(support_libs.embedding_lib, name)
    for emb in ((100, 104) if dtype == torch.float16 else (100,)):
        plan = P.embedding(1 << 30, emb * (2 if dtype == torch.float16 else 4), sm)
        n, rows = plan.per_pass + 5, 1000
        g = torch.Generator(device="cuda").manual_seed(emb)
        w = torch.randn(rows, emb, generator=g, device="cuda").to(dtype)
        idx = torch.randint(0, rows, (n,), generator=g, device="cuda", dtype=torch.int32)
        idx[[0, plan.per_pass - 1, plan.per_pass, n - 1]] = torch.tensor([-1, rows, 7, rows - 1], dtype=torch.int32,
                                                                         device="cuda")
        want = torch.where(((idx >= 0) & (idx < rows))[:, None], w[idx.clamp(0, rows - 1).long()], torch.zeros_like(w[:1]))
        buf, out = _out(n * emb, dtype, 0)
        fn(idx, w, out.view(n, emb))
        bad = _first_bad(out.view(n, emb) == want)
        assert bad is None, "%s emb=%d n=%d (%d rows per pass): out[%d, %d] wrong" % (name, emb, n, plan.per_pass, *bad)
        _guard_ok(buf, n * emb, 0, name)
