"""GPU: the GEMM against exact answers (gemm_exact.py) in every storage order and dtype, at every tile, k-block and
epilogue edge, through every entry point; 64-bit offsets and grids of more than 65,535 tiles; the fp32 NN path (B
transposed into a stream-ordered scratch buffer) on a side stream and in a CUDA graph; and the alignment and variant
errors.  Every comparison is bit for bit, and a failure names the (m, n) that went wrong and where its value came from."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))  # the helpers sit next to this file
import gemm_exact as ex  # noqa: E402

pytestmark = pytest.mark.gpu
KINDS = ("column", "row", "dense")
ENUM = {"f16": 1, "bf16": 2, "f32": 0}   # B200K_F16, B200K_BF16, B200K_F32


def _ops():
    from b200k import ops

    return ops


def _lib():
    from b200k import _loader as L

    return L


def _bits(t, dt):
    return t.contiguous().view(ex.INT_VIEW[dt])


def _run(path, case, spelling, variant=0):
    """C's guarded buffer after ops.gemm on guarded copies of the case's operands, in the path's storage order."""
    M, K = case.a.shape
    N = case.b.size(1)
    _, a_st = ex.guarded(case.a.t().contiguous() if path.a_km else case.a)
    _, b_st = ex.guarded(case.b.t().contiguous() if path.b_nk else case.b)
    cbuf, c = ex.c_buffer(M, N, path.dt, "cuda")
    a = a_st.t() if path.a_km else a_st
    b = {"nn": b_st, "view": b_st.t() if path.b_nk else None, "contiguous": b_st.view(K, N)}[spelling]
    _ops().gemm(a, b, c, tn=bool(path.b_nk), variant=variant, a_km=bool(path.a_km))
    torch.cuda.synchronize()
    return cbuf


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("path", ex.PATHS, ids=str)
def test_exact_at_every_edge(path, kind):
    errs = []
    for s in ex.shapes(path.dt, path.a_km, path.b_nk):
        case = ex.construct(kind, path.dt, s.M, s.N, s.K, ex.salt_of(kind, str(path), s.M, s.N, s.K), "cuda")
        for sp in path.spellings:
            errs += ex.check(case, _run(path, case, sp), "%s %s %s %s" % (path, kind, sp, s))
    assert not errs, "\n".join(errs[:20])


def test_every_entry_point_spelling_and_variant_gives_the_same_bits():
    """b200k_hgemm_f16, b200k_gemm, b200k_gemm_ex, ops.hgemm, ops.gemm and toy_hgemm on one ragged f16 product, NN and
    both TN spellings, every variant 0 .. 4 with high bits set: all equal the exact answer."""
    import toy_hgemm

    L, ops = _lib(), _ops()
    M, N, K = 300, 520, 264
    case = ex.construct("dense", "f16", M, N, K, 5, "cuda")
    a, b = case.a, case.b
    bt = b.t().contiguous()
    stream = torch.cuda.current_stream().cuda_stream
    runs = {
        "b200k_hgemm_f16": lambda c, tn: L.lib.b200k_hgemm_f16(a.data_ptr(), (bt if tn else b).data_ptr(), c.data_ptr(),
                                                               M, N, K, tn, 0, stream),
        "b200k_gemm": lambda c, tn: L.lib.b200k_gemm(a.data_ptr(), (bt if tn else b).data_ptr(), c.data_ptr(), M, N, K,
                                                     tn, L.F16, 0, stream),
        "b200k_gemm_ex": lambda c, tn: L.lib.b200k_gemm_ex(a.data_ptr(), (bt if tn else b).data_ptr(), c.data_ptr(), M,
                                                           N, K, 0, tn, L.F16, 0, stream),
    }
    calls = []
    for name, fn in runs.items():
        for tn in (0, 1):
            calls.append(("%s tn=%d" % (name, tn), lambda c, fn=fn, tn=tn: L.check(fn(c, tn))))
    for v in range(5):
        hv = v | (0x5A5A << 8)
        calls.append(("ops.hgemm variant %#x" % hv, lambda c, hv=hv: ops.hgemm(a, b, c, variant=hv)))
        calls.append(("ops.hgemm TN view variant %#x" % hv, lambda c, hv=hv: ops.hgemm(a, bt.t(), c, tn=True, variant=hv)))
        calls.append(("ops.gemm TN contiguous variant %#x" % hv,
                      lambda c, hv=hv: ops.gemm(a, bt.view(K, N), c, tn=True, variant=hv)))
    calls.append(("toy_hgemm NN", lambda c: toy_hgemm.hgemm_mma_m16n8k16_mma2x4_warp4x4x2_stages_dsmem(a, b, c, 3, True,
                                                                                                      2048)))
    calls.append(("toy_hgemm TN view", lambda c: toy_hgemm.hgemm_mma_m16n8k16_mma2x4_warp4x4_stages_dsmem_tn(
        a, bt.t(), c, 3, True, 2048)))
    calls.append(("toy_hgemm TN contiguous", lambda c: toy_hgemm.hgemm_mma_stages_block_swizzle_tn_cute(
        a, bt.view(K, N), c, 3, True, 2048)))
    for name, call in calls:
        cbuf, c = ex.c_buffer(M, N, "f16", "cuda")
        call(c)
        torch.cuda.synchronize()
        errs = ex.check(case, cbuf, name)
        assert not errs, "\n".join(errs)


# ------------------------------------------------------------------------------------------------ large cases
def _coded_rows(rows, cols, dt, salt):
    """ex.coded of a large matrix, built in row chunks so the index tensor stays small."""
    out = torch.empty(rows, cols, dtype=ex.TORCH[dt], device="cuda")
    step = max(1, (1 << 27) // cols)
    for r0 in range(0, rows, step):
        r1 = min(rows, r0 + step)
        out[r0:r1] = ex.coded(r1 - r0, cols, dt, salt, "cuda", row0=r0)
    return out


def _equal_in_chunks(c, want_rows, dt, what):
    """None when C == want_rows(r0, r1) for every chunk of rows (so the reference never holds a second full C), else
    the first difference."""
    M, N = c.shape
    step = max(1, (1 << 28) // N)
    for r0 in range(0, M, step):
        r1 = min(M, r0 + step)
        bad = (_bits(c[r0:r1], dt) != _bits(want_rows(r0, r1), dt)).nonzero()
        if bad.numel():
            m, n = r0 + int(bad[0, 0]), int(bad[0, 1])
            return "%s: %d elements differ, first at (m, n) = (%d, %d) [%s]" % (what, bad.size(0), m, n,
                                                                                ex.locate(dt, m, n))
    return None


def _large(case):
    """Runs case(), which returns an error message or None, and frees its tensors of several GB before asserting: an
    exception becomes a message, so no traceback keeps the case's frames (and their tensors) alive into the next case."""
    try:
        msg = case()
    except Exception as e:  # noqa: BLE001  reported below, after the memory is released
        msg = "%s: %s" % (type(e).__name__, e)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    assert msg is None, msg


def _column_selector(K, N, dt):
    idx = torch.tensor(ex.affine(K, N, 3), device="cuda")
    b = torch.zeros(K, N, dtype=ex.TORCH[dt], device="cuda")
    b[idx, torch.arange(N, device="cuda")] = 1
    return b, idx


def _column_selector_case(M, N, K, dt, salt, what):
    """C = A[:, pi] for a coded A [M, K]: the large cases of A and C."""
    def case():
        a = _coded_rows(M, K, dt, salt)
        b, idx = _column_selector(K, N, dt)
        c = torch.full((M, N), float("nan"), dtype=ex.TORCH[dt], device="cuda")
        _ops().gemm(a, b, c)
        return _equal_in_chunks(c, lambda r0, r1: a[r0:r1][:, idx], dt, what)

    return case


def test_c_above_2_31_elements_and_65535_tiles():
    M, N, K = 40000, 54000, 64
    tm, tn, _ = ex.geometry("f16", M, N, K)
    assert M * N > 2 ** 31 and tm * tn > 65535
    _large(_column_selector_case(M, N, K, "f16", 1, "C [40000, 54000]"))


def test_a_above_2_31_elements():
    M, N, K = 33000, 256, 65536
    assert M * K > 2 ** 31
    _large(_column_selector_case(M, N, K, "f16", 2, "A [33000, 65536]"))


def test_b_stored_k_major_above_2_31_elements():
    M, N, K = 256, 33000, 65536
    assert N * K > 2 ** 31

    def case():
        bt = _coded_rows(N, K, "bf16", 4)                   # storage of B^T [N, K]
        idx = torch.tensor(ex.affine(K, M, 5), device="cuda")
        a = torch.zeros(M, K, dtype=torch.bfloat16, device="cuda")
        a[torch.arange(M, device="cuda"), idx] = 1
        c = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device="cuda")
        _ops().gemm(a, bt.t(), c, tn=True)
        return _equal_in_chunks(c, lambda r0, r1: bt[:, idx[r0:r1]].t(), "bf16", "B^T [33000, 65536]")

    _large(case)


def test_f32_nn_transpose_above_2_31_elements():
    M, N, K = 128, 32832, 65536
    assert K * N > 2 ** 31
    _large(_column_selector_case(M, N, K, "f32", 6, "fp32 NN, B [65536, 32832]"))


# ------------------------------------------------------------------------------------------------ streams and graphs
F32_NN = ex.Path("f32", 0, 0)


def test_f32_nn_scratch_path_on_a_side_stream():
    ops = _ops()
    M, N, K = 300, 516, 260
    case = ex.construct("column", "f32", M, N, K, 7, "cuda")
    s = torch.cuda.Stream()
    cbuf, c = ex.c_buffer(M, N, "f32", "cuda")
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.gemm(case.a, case.b, c)
    s.synchronize()
    errs = ex.check(case, cbuf, "fp32 NN on a side stream")
    assert not errs, "\n".join(errs)


def test_f32_nn_scratch_path_replays_under_cuda_graph():
    """The scratch buffer's cudaMallocAsync / cudaFreeAsync are captured as graph nodes: every replay after new values
    are written into A and B equals an eager call and the exact answer."""
    ops = _ops()
    M, N, K = 300, 516, 260
    first = ex.construct("column", "f32", M, N, K, 8, "cuda")
    a, b = first.a.clone(), first.b.clone()
    c = torch.full((M, N), float("nan"), device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.gemm(a, b, c)
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        ops.gemm(a, b, c)
    for rep in range(3):
        case = ex.construct("column", "f32", M, N, K, 100 + rep, "cuda")
        a.copy_(case.a)
        b.copy_(case.b)
        c.fill_(float("nan"))
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        eager = torch.full_like(c, float("nan"))
        ops.gemm(a, b, eager)
        torch.cuda.synchronize()
        assert torch.equal(_bits(c, "f32"), _bits(eager, "f32")), rep
        assert torch.equal(_bits(c, "f32"), _bits(case.want, "f32")), rep


# ------------------------------------------------------------------------------------------------ errors
def _call_ex(path, a_ptr, b_ptr, c, M, N, K, variant=0):
    L = _lib()
    return L.lib.b200k_gemm_ex(a_ptr, b_ptr, c.data_ptr(), M, N, K, path.a_km, path.b_nk, ENUM[path.dt], variant,
                               torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("path", ex.PATHS, ids=str)
def test_unaligned_operand_or_unknown_variant_leaves_c_unchanged(path):
    """A or B one element past a 16-byte boundary returns B200K_EALIGN, variant 5 B200K_EARG; C keeps every bit.  The
    fp32 NN form reads B only through its transpose, so there an unaligned B is accepted and gives the same bits."""
    L = _lib()
    M, N, K = 136, 264, 72 if path.dt != "f32" else 68
    case = ex.construct("column", path.dt, M, N, K, 9, "cuda")
    e = ex.es(path.dt)
    a_st = (case.a.t() if path.a_km else case.a).contiguous().flatten()
    b_st = (case.b.t() if path.b_nk else case.b).contiguous().flatten()
    abuf, bbuf = (torch.cat([st[:1], st]) for st in (a_st, b_st))   # 16-byte aligned, operand from element 1
    aligned_a, aligned_b = a_st.data_ptr(), b_st.data_ptr()
    for what, a_ptr, b_ptr, variant, want_rc in (
            ("A offset by one element", abuf.data_ptr() + e, aligned_b, 0, L.EALIGN),
            ("B offset by one element", aligned_a, bbuf.data_ptr() + e, 0, L.OK if path == F32_NN else L.EALIGN),
            ("variant 5", aligned_a, aligned_b, 5, L.EARG),
            ("variant 5 with high bits", aligned_a, aligned_b, 5 | (0x5A5A << 8), L.EARG)):
        cbuf, c = ex.c_buffer(M, N, path.dt, "cuda")
        before = cbuf.clone()
        rc = _call_ex(path, a_ptr, b_ptr, c, M, N, K, variant)
        torch.cuda.synchronize()
        assert rc == want_rc, (what, rc, L.last_error())
        if rc == L.OK:
            errs = ex.check(case, cbuf, "%s %s" % (path, what))
            assert not errs, "\n".join(errs)
        else:
            assert torch.equal(_bits(cbuf, path.dt), _bits(before, path.dt)), what
