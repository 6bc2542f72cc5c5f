"""Exact-answer inputs for the GEMM (csrc/hgemm_wgmma.cu), used by test_gpu_gemm_exact.py and checked on the CPU by
test_gemm_exact_cpu.py.

The kernel's geometry is restated here: 128 x 256 tiles of C, one per CTA, in GROUP_M-row groups; k-blocks of one
128-byte swizzle row (BK = 64 16-bit or 32 fp32 elements) through a 4-stage ring; each consumer warpgroup stores its
64 x 256 block in column slices (two of 128 columns for 16-bit types, four of 64 for fp32), each slice two TMA boxes of
128 bytes.  The shape picker puts M, N and K on each side of those edges.

Three constructions have a closed-form answer that the kernel must match bit for bit:
  column selector  B[k, n] = 1 iff k == pi(n):    C[:, n] = A[:, pi(n)]
  row selector     A[m, k] = 1 iff k == sigma(m): C[m, :] = B[sigma(m), :]
  dense integers   A, B in {-2 .. 2}: every partial sum is an integer of magnitude at most 4 K < 2^24, exact in fp32 in
                   any order, so C is the fp64 product rounded once to the output type (round to nearest even).
pi and sigma are affine permutations (a i + b) mod K.  The selected matrix holds distinct, finite, normal values with
random signs (value (i * cols + j) mod P of a table of P distinct values, P prime, so every row and every column of
fewer than P elements is distinct; TF32 values have a 10-bit mantissa, so the tensor core reads them exactly).  A wrong
element therefore names the k, row or column it came from.  No subnormals and no -0: neither is part of the contract.

Operands are contiguous views at a 16-byte aligned, not 128-byte aligned, offset inside NaN-filled buffers with at least
one full TMA box of NaN after them; any read outside an operand turns into NaN in C through 0 * NaN.  C sits between
sentinel rows that must come back unchanged, and starts as NaN, so an element the kernel does not write shows too.

Pure torch; every function takes the device to build on."""
from __future__ import annotations

import math
import zlib
from dataclasses import dataclass, field

import torch

BM, BN, STAGES, GROUP_M = 128, 256, 4, 16
DTYPES = ("f16", "bf16", "f32")
TORCH = {"f16": torch.float16, "bf16": torch.bfloat16, "f32": torch.float32}
INT_VIEW = {"f16": torch.int16, "bf16": torch.int16, "f32": torch.int32}
GUARD_BEFORE = 48        # bytes of NaN before an operand: 16-byte aligned, not 128-byte aligned
GUARD_AFTER = 256 * 128  # bytes of NaN after an operand: the largest TMA box (256 rows of 128 bytes)
SENTINEL_ROWS = 2        # rows of C's buffer before and after C
SENTINEL = -7.0


def es(dt):
    return 4 if dt == "f32" else 2


def bk(dt):
    return 128 // es(dt)


def pack(dt):
    """The smallest allowed step of K and N (16 bytes)."""
    return 16 // es(dt)


def kstep(dt):
    return 8 if dt == "f32" else 16


def slices(dt):
    return 4 if dt == "f32" else 2


# ------------------------------------------------------------------------------------------------ storage paths
@dataclass(frozen=True)
class Path:
    """One row of the dispatch table: dtype, A stored [K,M], B stored [N,K] (TN)."""
    dt: str
    a_km: int
    b_nk: int

    @property
    def kernel(self):
        if self.dt == "f32":
            return "GemmCfg<2, false, false>" + ("" if self.b_nk else " after b200k_mat_transpose_f32")
        return "GemmCfg<%d, %s, %s>" % ({"f16": 0, "bf16": 1}[self.dt], "true" if self.a_km else "false",
                                         "false" if self.b_nk else "true")

    @property
    def spellings(self):
        """How ops receives B: TN as a strided Bt.t() view and as a contiguous [K,N]-shaped buffer holding B^T."""
        return ("view", "contiguous") if self.b_nk else ("nn",)

    def __str__(self):
        return "%s-%s%s" % (self.dt, "A_km" if self.a_km else "A_mk", "-B_nk" if self.b_nk else "-B_kn")


PATHS = [Path(dt, a, b) for dt in ("f16", "bf16") for a in (0, 1) for b in (0, 1)] + [Path("f32", 0, 1),
                                                                                       Path("f32", 0, 0)]


# ------------------------------------------------------------------------------------------------ geometry
def geometry(dt, M, N, K):
    """(tiles_m, tiles_n, k-blocks) of the launch."""
    return -(-M // BM), -(-N // BN), -(-K // bk(dt))


def tile_coords(tile, tiles_m, tiles_n):
    """(tm, tn) of CTA `tile` in the grouped rasterisation: GROUP_M row tiles walk each column tile together."""
    width = GROUP_M * tiles_n
    g = tile // width
    first_m = g * GROUP_M
    gsz = min(tiles_m - first_m, GROUP_M)
    return first_m + (tile % width) % gsz, (tile % width) // gsz


def store_boxes(dt, tn):
    """(slice, box, first column) of every TMA store box of column tile tn."""
    width, box = BN // slices(dt), 128 // es(dt)
    return [(sl, bx, tn * BN + sl * width + bx * box) for sl in range(slices(dt)) for bx in range(2)]


def locate(dt, m, n):
    """Where element (m, n) of C is computed and stored."""
    sl, bx, _ = [s for s in store_boxes(dt, n // BN) if s[2] <= n][-1]
    return "tile (%d, %d), warpgroup %d, slice %d, box %d" % (m // BM, n // BN, (m % BM) // 64, sl, bx)


# ------------------------------------------------------------------------------------------------ shapes
@dataclass
class Shape:
    M: int
    N: int
    K: int
    tags: list = field(default_factory=list)

    def __str__(self):
        return "(M=%d, N=%d, K=%d: %s)" % (self.M, self.N, self.K, "; ".join(self.tags))


def k_edges(dt):
    b, p = bk(dt), pack(dt)
    named = [("K=PACK", p), ("K=BK-PACK", b - p), ("K=BK", b), ("K=BK+PACK", b + p), ("K=4BK fills the ring", 4 * b),
             ("K=4BK+PACK wraps the ring", 4 * b + p), ("K=129 k-blocks", 129 * b)]
    return named + [("K%%BK=%d" % (r * p), 2 * b + r * p) for r in range(1, b // p)]


def m_edges(a_km):
    return [8, 64, 72, 120, 128, 136] if a_km else [1, 63, 64, 65, 127, 128, 129]


def n_residues(dt):
    """N mod 256 on each side of the epilogue's slice and box boundaries."""
    return [8, 56, 64, 72, 120, 128, 136, 192, 248, 0] if dt != "f32" else [4, 28, 32, 36, 60, 64, 68, 128, 252, 0]


def shapes(dt, a_km=0, b_nk=0):
    """Shapes that put M, N and K on each side of the kernel's edges, each tagged with what it hits.  Every K edge
    appears once with N >= K and once with M >= K, so the column and row selectors reach every k of it."""
    ks, ms, nres = k_edges(dt), m_edges(a_km), n_residues(dt)
    small_k = [k for _, k in ks if k <= 4 * bk(dt) + pack(dt)]
    out = []
    for i, (tag, K) in enumerate(ks):
        r = nres[i % len(nres)]
        out.append(Shape(ms[i % len(ms)], -(-K // BN) * BN + r, K, [tag, "N>=K", "N%%256=%d" % r]))
        out.append(Shape(-(-K // BM) * BM + ms[0], r or BN, K, [tag, "M>=K", "N%%256=%d" % r]))
    for i, M in enumerate(ms):
        out.append(Shape(M, nres[(i + 3) % len(nres)] or BN, small_k[i % len(small_k)], ["M=%d" % M]))
    for i, r in enumerate(nres):
        for base in (0, 2 * BN):
            out.append(Shape(ms[(i + 2) % len(ms)], base + (r or BN), small_k[(i + base) % len(small_k)],
                             ["N%%256=%d" % r]))
    n3 = 2 * BN + 2 * pack(dt)
    for tm, M in ((16, 16 * BM), (17, 16 * BM + ms[0]), (15, 15 * BM - ms[0])):
        out.append(Shape(M, n3, small_k[tm % len(small_k)], ["last group has %d row tiles" % (tm % GROUP_M or GROUP_M),
                                                            "tiles_n=3"]))
    if a_km:
        out.append(Shape(200, 64, bk(dt), ["M=200"]))
    for s in out:
        s.tags.append("tiles %d x %d, %d k-blocks" % geometry(dt, s.M, s.N, s.K))
        if a_km and s.M % 64:
            s.tags.append("A [K,M] 64-column box cut")
        if not b_nk and dt != "f32" and s.N % 64:
            s.tags.append("B [K,N] 64-column box cut")
    return out


# ------------------------------------------------------------------------------------------------ values
def _is_prime(n):
    return n > 1 and all(n % d for d in range(2, int(math.isqrt(n)) + 1))


_TABLES = {}


def value_table(dt):
    """P distinct finite normal values of the dtype (TF32-exact for f32), shuffled, random signs; P prime."""
    if dt not in _TABLES:
        mant, (elo, ehi) = (7, (-70, 70)) if dt == "bf16" else (10, (-10, 10))
        frac = 1.0 + torch.arange(1 << mant, dtype=torch.float64) / (1 << mant)
        mag = torch.cat([frac * 2.0 ** e for e in range(elo, ehi + 1)])
        P = len(mag)
        while not _is_prime(P):
            P -= 1
        g = torch.Generator().manual_seed(1)
        mag = mag[torch.randperm(len(mag), generator=g)[:P]]
        sign = torch.randint(0, 2, (P,), generator=g).double() * 2 - 1
        _TABLES[dt] = (mag * sign).to(TORCH[dt])
    return _TABLES[dt]


def coded(rows, cols, dt, salt=0, device="cpu", row0=0):
    """[rows, cols] (rows row0 .. row0 + rows of a [., cols] matrix): element (i, j) is table[(i * cols + j + salt) % P]."""
    t = value_table(dt).to(device)
    i = torch.arange(row0, row0 + rows, device=device, dtype=torch.int64).view(-1, 1) * cols
    return t[(i + torch.arange(cols, device=device).view(1, -1) + salt) % t.numel()]


def affine(K, count, salt=0):
    """(a i + b) mod K for i < count: gcd(a, K) = 1, a near 0.618 K so neighbours land far apart; b from the salt."""
    a = max(1, int(K * 0.618))
    while math.gcd(a, K) != 1:
        a += 1
    b = salt % K
    return [(a * i + b) % K for i in range(count)]


def required_ks(dt, K):
    """The k a selector must reach: 0, K - 1, both sides of every k-block boundary, every k of one wgmma k-step."""
    req = {0, K - 1} | set(range(min(kstep(dt), K)))
    for j in range(bk(dt), K, bk(dt)):
        req |= {j - 1, j}
    return req


def salt_of(*key):
    return zlib.crc32(repr(key).encode())


@dataclass
class Case:
    """Logical operands a [M, K], b [K, N], the expected C, and how to name the source of a wrong element."""
    kind: str
    dt: str
    a: torch.Tensor
    b: torch.Tensor
    want: torch.Tensor
    perm: list = None

    def explain(self, m, n, got):
        """Which element of the selected operand holds the value that arrived at (m, n)."""
        if self.kind == "dense":
            return "expected the integer product rounded once"
        iv = INT_VIEW[self.dt]
        what, src, (i0, j0) = ("A", self.a, (m, self.perm[n])) if self.kind == "column" else ("B", self.b, (self.perm[m], n))
        head = "should come from %s[%d, %d]" % (what, i0, j0)
        g = torch.tensor([got.item()], dtype=TORCH[self.dt]).view(iv).item()
        # the same row of the source first (a wrong k for A, a wrong column for B), then its column, then anywhere
        for part, at in ((src[i0], lambda h: (i0, h)), (src[:, j0], lambda h: (h, j0)), (src, None)):
            hit = (part.contiguous().view(iv) == g).nonzero()
            if hit.numel():
                i, j = at(int(hit[0, 0])) if at else (int(hit[0, 0]), int(hit[0, 1]))
                return "%s; the value of %s[%d, %d] arrived" % (head, what, i, j)
        return "%s; %r is no element of %s (guard NaN, a zero or garbage)" % (head, got.item(), what)


def construct(kind, dt, M, N, K, salt=0, device="cpu"):
    """A Case of construction `kind` ("column", "row" or "dense") for an M x N x K product."""
    t = TORCH[dt]
    if kind == "column":
        perm = affine(K, N, salt)
        a = coded(M, K, dt, salt, device)
        b = torch.zeros(K, N, dtype=t, device=device)
        idx = torch.tensor(perm, device=device)
        b[idx, torch.arange(N, device=device)] = 1
        return Case(kind, dt, a, b, a[:, idx], perm)
    if kind == "row":
        perm = affine(K, M, salt)
        b = coded(K, N, dt, salt, device)
        a = torch.zeros(M, K, dtype=t, device=device)
        idx = torch.tensor(perm, device=device)
        a[torch.arange(M, device=device), idx] = 1
        return Case(kind, dt, a, b, b[idx], perm)
    assert kind == "dense"
    assert 4 * K < 2 ** 24, "K = %d: integer partial sums would no longer be exact in fp32" % K
    g = torch.Generator(device=device).manual_seed(salt)
    a = torch.randint(-2, 3, (M, K), generator=g, device=device).to(t)
    b = torch.randint(-2, 3, (K, N), generator=g, device=device).to(t)
    return Case(kind, dt, a, b, dense_expected(a, b, dt))


def dense_expected(a, b, dt):
    """The fp64 product rounded once to dt.  The integer sums are exact in fp32, so the float step rounds nothing."""
    return (a.double() @ b.double()).float().to(TORCH[dt])


# ------------------------------------------------------------------------------------------------ guards and checks
def guarded(storage):
    """(buffer, view): a contiguous copy of `storage` inside a NaN buffer, GUARD_BEFORE bytes from its start and with
    GUARD_AFTER bytes of NaN after it."""
    e = storage.element_size()
    pre, post = GUARD_BEFORE // e, GUARD_AFTER // e
    buf = torch.full((pre + storage.numel() + post,), float("nan"), dtype=storage.dtype, device=storage.device)
    view = buf[pre:pre + storage.numel()].view(storage.shape)
    view.copy_(storage)
    return buf, view


def c_buffer(M, N, dt, device="cpu"):
    """(buffer, C): C [M, N] is NaN, with SENTINEL_ROWS rows of SENTINEL before and after it.  There are no sentinel
    columns: the C ABI takes no leading dimension, so C's rows are N wide and back to back, and a store past column N
    of row m lands on row m + 1, which the tile owning it may overwrite later.  Such a store needs a wrong C tensor map
    (TMA clips to its [M, N]); a later write over it would hide it, and only the sentinel rows catch the ends of C."""
    buf = torch.full((M + 2 * SENTINEL_ROWS, N), SENTINEL, dtype=TORCH[dt], device=device)
    c = buf[SENTINEL_ROWS:SENTINEL_ROWS + M]
    c.fill_(float("nan"))
    return buf, c


def check(case, cbuf, what=""):
    """Error messages (empty when C equals the closed form bit for bit and the sentinel rows are intact)."""
    iv, S = INT_VIEW[case.dt], SENTINEL_ROWS
    M, N = case.want.shape
    errs = []
    guard = torch.cat([cbuf[:S], cbuf[S + M:]])
    bad = (guard.float() != SENTINEL).nonzero()
    if bad.numel():
        r, n = (int(x) for x in bad[0])
        errs.append("%s: %d sentinel elements of C's buffer overwritten, first at row %d, column %d (row %d of C)"
                    % (what, bad.size(0), r if r < S else r + M, n, (r - S) if r < S else M + r - S))
    c = cbuf[S:S + M]
    diff = (c.contiguous().view(iv) != case.want.contiguous().view(iv)).nonzero()
    if diff.numel():
        m, n = (int(x) for x in diff[0])
        errs.append("%s: %d of %d elements differ; first at (m, n) = (%d, %d) [%s]: got %r, want %r; %s"
                    % (what, diff.size(0), M * N, m, n, locate(case.dt, m, n), c[m, n].item(), case.want[m, n].item(),
                       case.explain(m, n, c[m, n].cpu())))
    return errs
