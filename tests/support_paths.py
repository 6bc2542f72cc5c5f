"""The launch rules of the bandwidth kernels (csrc/support_kernels.cu, csrc/support_kernels2.cu), restated as data.

Each function mirrors one launcher: given the dtype, the shape, whether the pointers are 16-byte aligned and the SM
count, it returns the path the kernel takes, its grid and how much work one pass of the grid-stride loop covers.
The tests use it to pick shapes on both sides of every path switch and across pass boundaries, so the shapes follow
the card the tests run on.  Pure Python: tests/test_support_paths_cpu.py checks it against worked numbers.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

THREADS = 256             # kThreads (support_common.cuh)
REDUCE_MAX_BLOCKS = 2048  # kReduceMaxBlocks: partials in the reduction workspace
TILE = 64                 # kTile of both transposes

# elements per 16-byte vector (RowIO<T>::N, Vec16<T>::N, Loader<DT>::N)
VN = {"f32": 4, "f16": 8, "bf16": 8, "fp8": 16, "i8": 16}


def grid_for(work_items: int, per_block: int, sm_count: int, waves: int) -> int:
    """grid_for() of support_common.cuh: enough CTAs for the work, capped at `waves` per SM, at least one."""
    blocks = (work_items + per_block - 1) // per_block
    return max(1, min(blocks, sm_count * waves))


@dataclass(frozen=True)
class Plan:
    vector: bool              # 16-byte path (False: the scalar fallback)
    grid: int
    per_pass: int             # rows / elements / vectors / tiles one pass of the grid-stride loop covers (see `unit`)
    unit: str                 # what per_pass counts: "rows", "vectors", "elements" or "tiles"
    R: Optional[int] = None   # row kernels: threads per row (None for the scalar row kernel)
    cached: Optional[bool] = None  # row kernels: row held in registers (False: x read again per pass over the row)

    def passes(self, work: int) -> int:
        return -(-work // self.per_pass)


# ------------------------------------------------------------------------------------------------ row kernels
ROW_KERNELS = ("softmax", "rms_norm", "layer_norm")


def row(dtype: str, rows: int, H: int, sm: int, aligned: bool = True) -> Plan:
    """launch_row, the one launcher of the row kernels (softmax modes 1-3 and the normalisation pass of mode 0,
    rms_norm, layer_norm).  R threads own a row, 256 / R rows per CTA, at most 32 values of the row per thread in
    registers."""
    vn = VN[dtype]
    if H % vn == 0 and aligned:
        R = 32 if H <= 32 * 32 else (128 if H <= 32 * 128 else 256)
        rows_per_cta = THREADS // R
        grid = grid_for(rows, rows_per_cta, sm, 16)
        cached = H // vn <= (32 // vn) * R
        return Plan(True, grid, grid * rows_per_cta, "rows", R, cached)
    grid = grid_for(rows, 1, sm, 16)  # row_kernel_scalar: one CTA per row
    return Plan(False, grid, grid, "rows")


def row_positions(dtype: str, H: int, plan: Plan) -> list[int]:
    """Positions in a row where an element is easy to drop or misplace on this path: the first and last element,
    the first and last element of each register slot t + i*R (vector path), the register / re-read boundary, and the
    edges of the 256-thread stride (scalar path)."""
    vn = VN[dtype]
    pos = {0, H - 1}
    if plan.vector:
        nvec = H // vn
        for i in range(32 // vn):
            first, last = i * plan.R, (i + 1) * plan.R - 1
            if first < nvec:
                pos.add(first * vn)
            if last < nvec:
                pos.add(last * vn + vn - 1)
        edge = (32 // vn) * plan.R * vn  # first element past what the registers can hold
        pos.update(p for p in (edge - 1, edge) if p < H)
    else:
        pos.update(p for p in (THREADS - 1, THREADS, H - H % THREADS) if p < H)
        pos.update(p for p in (H - H % vn,) if p < H)  # where the vector path's tail would start
    return sorted(pos)


def row_widths(dtype: str) -> list[int]:
    """Both sides of every row-path switch: R = 32 | 128 at H = 1024, R = 128 | 256 at 4096, cached | re-read at
    8192, plus a width the vector path cannot take (H % VN != 0)."""
    vn = VN[dtype]
    return [1024, 1024 + vn, 4096, 4096 + vn, 8192, 8192 + vn, 1024 + vn - 1]


def pass_counts(plan: Plan, rows_per_cta: int = 1) -> dict[str, int]:
    """Row (or item) counts for this plan at full grid: exactly one pass, one pass plus one row, and two passes and
    more ending on a partially filled CTA (not a multiple of the rows per CTA, where a CTA holds several)."""
    p = plan.per_pass
    return {"one": p, "one+1": p + 1, "two+": 2 * p + (rows_per_cta // 2 + 1 if rows_per_cta > 1 else 1)}


def full_rows(dtype: str, H: int, sm: int, aligned: bool = True) -> Plan:
    """The plan at a row count large enough to fill the capped grid."""
    return row(dtype, 1 << 30, H, sm, aligned)


# ------------------------------------------------------------------------------------------------ reductions
def reduce(dtype: str, n: int, sm: int, aligned: bool = True) -> Plan:
    """launch_reduce (block_all_reduce_sum, and the exp-sum of softmax mode 0) and the dot product launch: the grid
    is sized from the vector count whatever the alignment, capped by the workspace.  One pass of the 16-byte loop is
    grid * 256 vectors; the 4-way unrolled body takes 4 passes at a time and a remainder loop the rest.  Unaligned,
    everything runs through the scalar loop, grid * 256 elements per pass."""
    grid = min(grid_for(n // VN[dtype], THREADS * 4, sm, 8), REDUCE_MAX_BLOCKS)
    if aligned:
        return Plan(True, grid, grid * THREADS, "vectors")
    return Plan(False, grid, grid * THREADS, "elements")


dot = reduce  # b200k_dot_prod: the same sizing (n / VN vectors, 4 per thread per CTA), the same cap


def reduce_positions(dtype: str, n: int, plan: Plan) -> list[int]:
    """Where a needle tells whether every part of the reduction was counted once: first and last element, the pack
    edges, the first and last element of a CTA's share of a pass, the first element of the second, fourth and fifth
    pass (the unrolled body and its remainder loop), the last whole vector and the scalar tail."""
    vn = VN[dtype]
    cand = [0, n - 1]
    if plan.vector:
        nvec, stride = n // vn, plan.per_pass
        cand += [vn - 1, vn, THREADS * vn - 1, THREADS * vn, stride * vn - 1, stride * vn, 3 * stride * vn,
                 4 * stride * vn, (nvec - 1) * vn, nvec * vn]
    else:
        stride = plan.per_pass
        cand += [THREADS - 1, THREADS, stride - 1, stride, 3 * stride, 4 * stride]
    return sorted({p for p in cand if 0 <= p < n})


# ------------------------------------------------------------------------------------------------ elementwise
def add(dtype: str, n: int, sm: int, aligned: bool = True) -> Plan:
    """launch_add: 16-byte vectors (4 per thread in flight, grid * 256 vectors per pass) then the n % VN tail in
    CTA 0; unaligned, the scalar kernel with grid * 256 elements per pass."""
    if aligned:
        grid = grid_for(n // VN[dtype], THREADS * 4, sm, 8)
        return Plan(True, grid, grid * THREADS, "vectors")
    grid = grid_for(n, THREADS, sm, 16)
    return Plan(False, grid, grid * THREADS, "elements")


def activation(dtype: str, n: int, sm: int, aligned: bool = True) -> Plan:
    """launch_act2: chunks of 4 * 256 consecutive vectors per CTA (grid * 1024 vectors per pass), the n % VN tail
    through the scalar loop; unaligned, the scalar loop alone (grid sized as if 1024 per CTA, 256 per pass)."""
    vn = VN[dtype]
    grid = grid_for(n // vn if aligned else n, THREADS * 4, sm, 8)
    if aligned:
        return Plan(True, grid, grid * THREADS * 4, "vectors")
    return Plan(False, grid, grid * THREADS, "elements")


# ------------------------------------------------------------------------------------------------ GEMV
def gemv(dtype: str, M: int, K: int, sm: int, aligned: bool = True) -> Plan:
    """b200k_gemv: one warp per row, 8 rows per CTA.  The 16-byte path (K % VN == 0, aligned A and x) gives each lane
    vector i and, while i + 32 < K / VN, vector i + 32, stepping by 64."""
    grid = grid_for(M, THREADS // 32, sm, 8)
    return Plan(K % VN[dtype] == 0 and aligned, grid, grid * (THREADS // 32), "rows")


def gemv_widths(dtype: str) -> list[int]:
    """K on both sides of the one- / two-vectors-per-lane switch (32 and 64 vectors), past it, and with a tail."""
    vn = VN[dtype]
    return [32 * vn, 33 * vn, 64 * vn, 65 * vn, 129 * vn, 33 * vn + 1]


# ------------------------------------------------------------------------------------------------ transposes
def transpose_f32(M: int, N: int, sm: int, aligned: bool = True) -> Plan:
    """b200k_mat_transpose_f32: 64 x 64 tiles, one per CTA per pass; 16-byte accesses when M and N are multiples of 4."""
    tiles = -(-M // TILE) * -(-N // TILE)
    grid = grid_for(tiles, 1, sm, 16)
    return Plan(M % 4 == 0 and N % 4 == 0 and aligned, grid, grid, "tiles")


def transpose_u16(batch: int, M: int, N: int, sm: int) -> Plan:
    """b200k_transpose_u16_batched: 64 x 64 tiles of every batch entry, one per CTA per pass, 2-byte accesses."""
    tiles = batch * -(-M // TILE) * -(-N // TILE)
    grid = grid_for(tiles, 1, sm, 16)
    return Plan(False, grid, grid, "tiles")


def tiles_past_passes(sm: int, passes: int, extra: tuple[int, int]) -> tuple[int, int]:
    """Ragged (M, N) whose tile count exceeds `passes` full passes of the capped grid: N spans 40 tile columns, M as
    many tile rows as needed; `extra` is added to the whole-tile sizes (values 1..63 make the last tiles ragged)."""
    per_pass = 16 * sm
    tn = 40
    tm = -(-(passes * per_pass + 1) // tn)
    return (tm - 1) * TILE + extra[0], (tn - 1) * TILE + extra[1]


# ------------------------------------------------------------------------------------------------ embedding
def embedding(n: int, row_bytes: int, sm: int, aligned: bool = True) -> Plan:
    """b200k_embedding: one warp per index, 8 per CTA; 16-byte chunks when the row is a multiple of 16 bytes."""
    grid = grid_for(n, THREADS // 32, sm, 32)
    return Plan(row_bytes % 16 == 0 and aligned, grid, grid * (THREADS // 32), "rows")
