"""CPU: the GEMM's exact-answer helpers (gemm_exact.py).  The grouped rasterisation restated there is a bijection onto
the tile grid; the shape picker reaches every M, N and K edge for every storage path; each construction's closed form
equals an fp64 numpy product of the same inputs; and the checker rejects every kind of kernel error simulated on the
exact answer: an element from the neighbouring k, row or column, a k-block counted twice or left out, two 8-column groups
swapped inside a store slice, a tile written at the wrong (tm, tn), and an overwritten sentinel."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))  # the helpers sit next to this file
import gemm_exact as ex  # noqa: E402

KINDS = ("column", "row", "dense")


@pytest.mark.parametrize("tiles_n", [1, 2, 3, 7])
def test_rasterisation_is_a_bijection(tiles_n):
    for tiles_m in list(range(1, 40)) + [47, 48, 49, 313]:
        seen = [ex.tile_coords(t, tiles_m, tiles_n) for t in range(tiles_m * tiles_n)]
        assert sorted(seen) == [(m, n) for m in range(tiles_m) for n in range(tiles_n)], (tiles_m, tiles_n)


def test_store_boxes_tile_the_column_tile():
    for dt in ex.DTYPES:
        cols = [c for _, _, c in ex.store_boxes(dt, 2)]
        box = 128 // ex.es(dt)
        assert cols == list(range(2 * ex.BN, 3 * ex.BN, box)), dt
        assert ex.locate(dt, 64, 2 * ex.BN + ex.BN - 1) == "tile (0, 2), warpgroup 1, slice %d, box 1" % (ex.slices(dt) - 1)


@pytest.mark.parametrize("path", ex.PATHS, ids=str)
def test_shape_picker_reaches_every_edge(path):
    dt, b, p = path.dt, ex.bk(path.dt), ex.pack(path.dt)
    sh = ex.shapes(dt, path.a_km, path.b_nk)
    Ks = {s.K for s in sh}
    assert {p, b - p, b, b + p, 4 * b, 4 * b + p, 129 * b} <= Ks
    assert {k % b for k in Ks} == set(range(0, b, p))                         # every remainder, and none
    assert set(ex.m_edges(path.a_km)) <= {s.M for s in sh}
    assert set(ex.n_residues(dt)) <= {s.N % ex.BN for s in sh}
    assert set(ex.n_residues(dt)) <= {s.N % ex.BN for s in sh if s.N > ex.BN}   # in a later column tile too
    groups = {ex.geometry(dt, s.M, s.N, s.K)[0] % ex.GROUP_M for s in sh if ex.geometry(dt, s.M, s.N, s.K)[1] >= 3}
    assert {0, 1, 15} <= groups
    assert all(s.K % p == 0 and s.N % p == 0 for s in sh)
    if path.a_km:
        assert all(s.M % 8 == 0 for s in sh)
        assert {72, 200} <= {s.M for s in sh}                                  # 64-wide MN-major boxes cut
    if dt != "f32" and not path.b_nk:
        assert any(s.N % 64 for s in sh)
    assert {1, 63, 64, 65, 127, 128, 129} <= {s.M for s in sh} or path.a_km
    # the selectors reach every k of every K edge, the required ones included
    for _, K in ex.k_edges(dt):
        assert ex.required_ks(dt, K) <= set(range(K))
        assert any(s.K == K and set(ex.affine(K, s.N)) == set(range(K)) for s in sh), K
        assert any(s.K == K and set(ex.affine(K, s.M)) == set(range(K)) for s in sh), K
    assert all(4 * s.K < 2 ** 24 for s in sh)                                  # dense integers stay exact


def test_value_tables_are_distinct_normal_and_tf32_exact():
    for dt in ex.DTYPES:
        t = ex.value_table(dt)
        assert ex._is_prime(t.numel()) and t.numel() > 2 * 129 * ex.bk(dt)
        assert t.view(ex.INT_VIEW[dt]).unique().numel() == t.numel()
        assert torch.isfinite(t.float()).all() and (t.float().abs() >= torch.finfo(ex.TORCH[dt]).tiny).all()
        assert (t.float() < 0).any() and (t.float() > 0).any()
        if dt == "f32":
            assert (t.view(torch.int32) & 0x1FFF == 0).all()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("dt", ex.DTYPES)
def test_closed_form_equals_fp64_product(dt, kind):
    for M, N, K in ((1, 8, 8), (65, 136, 72), (129, 264, 200), (7, 40, 264)):
        K = K // ex.pack(dt) * ex.pack(dt)
        case = ex.construct(kind, dt, M, N, K, ex.salt_of(kind, dt, M, N, K))
        prod = torch.from_numpy(case.a.double().numpy() @ case.b.double().numpy()).to(ex.TORCH[dt])
        assert torch.equal(case.want.view(ex.INT_VIEW[dt]), prod.view(ex.INT_VIEW[dt])), (M, N, K)
        if kind != "dense":
            assert (case.want.float() != 0).all() and torch.isfinite(case.want.float()).all()


# ------------------------------------------------------------------------------------------------ simulated errors
def _rounded(acc, dt):
    return acc.float().to(ex.TORCH[dt])


def _pick(mask):
    m, n = (int(x) for x in mask.nonzero()[0])
    return m, n


def _errors(case):
    """(name, C [M, N] as a broken kernel would leave it, substring the report must contain)."""
    dt, a, b, want = case.dt, case.a, case.b, case.want
    M, N = want.shape
    K = a.size(1)
    acc = a.double() @ b.double()
    out = []
    # one element from the neighbouring k / row / column of the source operand
    if case.kind == "column":
        m, n = 3, 5
        k = case.perm[n]
        for name, i, j in (("neighbouring k", m, (k + 1) % K), ("neighbouring row", m + 1, k)):
            c = want.clone()
            c[m, n] = a[i, j]
            out.append((name, c, "the value of A[%d, %d] arrived" % (i, j)))
    elif case.kind == "row":
        m, n = 3, 5
        k = case.perm[m]
        for name, i, j in (("neighbouring k", (k + 1) % K, n), ("neighbouring column", k, n + 1)):
            c = want.clone()
            c[m, n] = b[i, j]
            out.append((name, c, "the value of B[%d, %d] arrived" % (i, j)))
    else:
        # A[m, k + 1] used in place of A[m, k] in one product
        d = a[:, 1:].double() - a[:, :-1].double()
        delta = d.view(M, K - 1, 1) * b[:-1].double().view(1, K - 1, N)
        mm, kk, nn = (int(x) for x in (delta != 0).nonzero()[0])
        c = want.clone()
        c[mm, nn] = _rounded(acc[mm, nn] + delta[mm, kk, nn], dt)
        out.append(("neighbouring k", c, "(%d, %d)" % (mm, nn)))
        m, n = _pick(want[:-1].view(ex.INT_VIEW[dt]) != want[1:].view(ex.INT_VIEW[dt]))
        c = want.clone()
        c[m, n] = want[m + 1, n]
        out.append(("neighbouring row", c, "(%d, %d)" % (m, n)))
    # one k-block counted twice, or left out
    blk = slice(ex.bk(dt), 2 * ex.bk(dt))
    part = a[:, blk].double() @ b[blk].double()
    for name, sgn in (("k-block 1 counted twice", 1), ("k-block 1 left out", -1)):
        out.append((name, _rounded(acc + sgn * part, dt), "elements differ"))
    # two 8-column groups swapped inside the second slice of column tile 1
    s0 = ex.BN + ex.BN // ex.slices(dt)
    c = want.clone()
    c[:, s0:s0 + 8], c[:, s0 + 8:s0 + 16] = want[:, s0 + 8:s0 + 16], want[:, s0:s0 + 8]
    out.append(("8-column groups swapped", c, "slice 1, box 0"))
    # tile 1 of the grid written at the place of tile 2, and the other way round
    tm, tn, _ = ex.geometry(dt, M, N, K)
    (m1, n1), (m2, n2) = ex.tile_coords(1, tm, tn), ex.tile_coords(2, tm, tn)
    t1 = (slice(m1 * ex.BM, m1 * ex.BM + ex.BM), slice(n1 * ex.BN, n1 * ex.BN + ex.BN))
    t2 = (slice(m2 * ex.BM, m2 * ex.BM + ex.BM), slice(n2 * ex.BN, n2 * ex.BN + ex.BN))
    c = want.clone()
    c[t1], c[t2] = want[t2], want[t1]
    out.append(("tiles (%d, %d) and (%d, %d) swapped" % (m1, n1, m2, n2), c, "elements differ"))
    return out


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("dt", ex.DTYPES)
def test_checker_rejects_simulated_kernel_errors(dt, kind):
    M, N, K = 256, 768, 3 * ex.bk(dt) + ex.pack(dt)          # 2 x 3 tiles (tile 1 is (1, 0), tile 2 is (0, 1)), 4 k-blocks
    case = ex.construct(kind, dt, M, N, K, ex.salt_of("sim", kind, dt))
    cbuf, c = ex.c_buffer(M, N, dt)
    assert ex.check(case, cbuf), "C left as NaN must be rejected"
    c.copy_(case.want)
    assert ex.check(case, cbuf) == []
    for name, broken, expect in _errors(case):
        assert not torch.equal(broken.view(ex.INT_VIEW[dt]), case.want.view(ex.INT_VIEW[dt])), name
        c.copy_(broken)
        errs = ex.check(case, cbuf, name)
        assert errs and expect in errs[0], (name, errs)
    c.copy_(case.want)
    for r, n in ((0, 0), (ex.SENTINEL_ROWS - 1, N - 1), (ex.SENTINEL_ROWS + M, 7), (M + 2 * ex.SENTINEL_ROWS - 1, N - 1)):
        buf = cbuf.clone()
        buf[r, n] = 0
        errs = ex.check(case, buf, "sentinel")
        assert len(errs) == 1 and "sentinel" in errs[0], (r, n, errs)


def test_guarded_operands_sit_in_nan_at_a_16_byte_offset():
    for dt in ex.DTYPES:
        x = ex.coded(5, 24, dt)
        buf, v = ex.guarded(x)
        off = v.data_ptr() - buf.data_ptr()
        assert off == ex.GUARD_BEFORE and off % 16 == 0 and off % 128
        assert v.is_contiguous() and torch.equal(v.view(ex.INT_VIEW[dt]), x.view(ex.INT_VIEW[dt]))
        rest = torch.cat([buf[:off // x.element_size()], buf[off // x.element_size() + x.numel():]])
        assert torch.isnan(rest.float()).all() and rest.numel() * x.element_size() >= ex.GUARD_AFTER


def test_explain_names_the_source():
    case = ex.construct("column", "f16", 4, 16, 16, 0)
    msg = case.explain(1, 2, case.a[1, case.perm[5]])
    assert msg == "should come from A[1, %d]; the value of A[1, %d] arrived" % (case.perm[2], case.perm[5])
    msg = case.explain(1, 2, torch.tensor(float("nan"), dtype=torch.float16))
    assert "no element of A" in msg
