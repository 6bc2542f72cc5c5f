"""The launch rules in tests/support_paths.py against numbers worked out by hand from the launchers, at 132 SMs
(H100 SXM) and 114 SMs (H100 PCIe).  No GPU needed."""
import pytest

import support_paths as P

SXM, PCIE = 132, 114


@pytest.mark.parametrize("sm", [SXM, PCIE])
def test_row_paths_and_rows_per_pass(sm):
    # R = 32 up to H = 1024: 16 CTAs per SM x 8 rows per CTA
    p = P.full_rows("f32", 1024, sm)
    assert (p.vector, p.R, p.cached, p.grid, p.per_pass) == (True, 32, True, 16 * sm, 128 * sm)
    assert P.full_rows("f32", 1028, sm).R == 128 and P.full_rows("f16", 1032, sm).R == 128
    # R = 128 up to 4096: 2 rows per CTA
    p = P.full_rows("f16", 4096, sm)
    assert (p.R, p.cached, p.per_pass) == (128, True, 32 * sm)
    # R = 256 past 4096: one row per CTA; rows cached up to 8192, re-read past it
    p = P.full_rows("f32", 4100, sm)
    assert (p.R, p.cached, p.per_pass) == (256, True, 16 * sm)
    assert P.full_rows("f32", 8192, sm).cached and P.full_rows("f16", 8192, sm).cached
    assert not P.full_rows("f32", 8196, sm).cached and not P.full_rows("f16", 8200, sm).cached
    # H % VN != 0 or unaligned: the scalar kernel, one row per CTA
    for dt, H, aligned in (("f32", 1027, True), ("f16", 4100, True), ("f32", 1024, False)):
        p = P.full_rows(dt, H, sm, aligned)
        assert (p.vector, p.R, p.per_pass) == (False, None, 16 * sm)


def test_row_numbers_at_132_and_114_sms():
    assert [P.full_rows("f32", 1024, s).per_pass for s in (SXM, PCIE)] == [16896, 14592]
    assert [P.full_rows("f32", 4096, s).per_pass for s in (SXM, PCIE)] == [4224, 3648]
    assert [P.full_rows("f32", 8192, s).per_pass for s in (SXM, PCIE)] == [2112, 1824]
    assert P.row("f32", 300, 4096, SXM).grid == 150  # below the cap: ceil(300 / 2) CTAs
    assert P.pass_counts(P.full_rows("f32", 1024, SXM), 8) == {"one": 16896, "one+1": 16897, "two+": 33797}
    assert P.pass_counts(P.full_rows("f32", 8192, PCIE), 1) == {"one": 1824, "one+1": 1825, "two+": 3649}


def test_row_positions_cover_the_register_slots():
    # f32, H = 4096, R = 128: slots of 128 vectors; the row fits the registers exactly
    pos = P.row_positions("f32", 4096, P.full_rows("f32", 4096, SXM))
    assert pos[:4] == [0, 511, 512, 1023] and pos[-2:] == [3584, 4095]
    # f16 past 8192: four 8-value slots of 256 vectors, then the re-read part
    pos = P.row_positions("f16", 8200, P.full_rows("f16", 8200, SXM))
    assert {0, 2047, 2048, 8191, 8192, 8199} <= set(pos)
    # scalar: the 256-thread stride edges and where the vector tail would begin
    assert P.row_positions("f32", 1027, P.full_rows("f32", 1027, SXM)) == [0, 255, 256, 1024, 1026]


def test_reduction_and_dot_grids():
    # 8 CTAs per SM, 1024 vectors per CTA sizing, 256 vectors per CTA per pass
    for sm, grid in ((SXM, 1056), (PCIE, 912)):
        p = P.reduce("f32", 1 << 26, sm)
        assert (p.vector, p.grid, p.per_pass) == (True, grid, 256 * grid)
        assert P.dot("f16", 1 << 26, sm).grid == grid
        p = P.reduce("f16", 1 << 26, sm, aligned=False)
        assert (p.vector, p.grid, p.per_pass, p.unit) == (False, grid, 256 * grid, "elements")
    assert P.reduce("f32", 1 << 26, SXM).per_pass == 270336
    assert P.reduce("fp8", 4096 * 16, SXM).grid == 4 and P.reduce("f32", 3, SXM).grid == 1
    assert P.reduce("f32", 1 << 26, 300).grid == 2048  # capped by the workspace's 2048 partials
    pos = P.reduce_positions("f32", 5 * 270336 * 4 + 7, P.reduce("f32", 5 * 270336 * 4 + 7, SXM))
    assert {0, 3, 4, 1023, 1024, 1081343, 1081344, 3244032, 4325376, 5406720, 5406726} <= set(pos)


def test_elementwise_grids():
    p = P.activation("f32", 1 << 26, SXM)
    assert (p.grid, p.per_pass, p.per_pass * 4) == (1056, 1081344, 4325376)  # 4.3 M fp32 values per pass
    assert P.activation("f32", 1 << 26, PCIE).per_pass * 4 == 3735552
    p = P.activation("f16", 1 << 26, SXM, aligned=False)
    assert (p.vector, p.grid, p.per_pass) == (False, 1056, 270336)
    assert P.add("bf16", 1 << 26, SXM).per_pass == 270336
    p = P.add("f32", 1 << 26, PCIE, aligned=False)
    assert (p.vector, p.grid, p.per_pass) == (False, 1824, 466944)


def test_gemv_transpose_embedding():
    assert [P.gemv("f32", 1 << 20, 128, s).per_pass for s in (SXM, PCIE)] == [8448, 7296]
    assert P.gemv("f16", 100, 264, SXM).grid == 13
    assert not P.gemv("f16", 100, 260, SXM).vector and not P.gemv("f32", 100, 128, SXM, aligned=False).vector
    assert P.gemv_widths("f32")[:4] == [128, 132, 256, 260]
    assert [P.transpose_f32(4096, 4096, s).per_pass for s in (SXM, PCIE)] == [2112, 1824]
    assert P.transpose_f32(4096, 2048, SXM).vector and not P.transpose_f32(4098, 2048, SXM).vector
    M, N = P.tiles_past_passes(SXM, 2, (5, 3))
    assert (M, N) == (6725, 2499) and -(-M // 64) * -(-N // 64) == 4240 > 2 * 2112
    assert P.transpose_u16(3, 1285, 2243, PCIE).grid == 1824
    assert P.embedding(1 << 20, 400, SXM).per_pass == 33792 and not P.embedding(10, 200, SXM).vector
