"""Exact-answer inputs for attention, shared by every mode (dense, FFPA, packed, KV-cache decode, append), used by
test_gpu_attention_exact.py and checked against attention_ref in test_attention_exact_cpu.py.

Row r of Q is A * e_c: one non-zero column c, chosen per row.  Within one block of keys (one (sequence, K/V head)),
column c of K is A at one key, the column's needle, and 0 everywhere else.  The score of row r is then A^2 at its needle
and exactly 0 at every other key.  V holds integers in [-8, 8], so every sum the tensor core forms is exact in fp32.
A row sees a prefix [0, n) of its block (length, causal diagonal, cache capacity), and the kernel must produce:
  - its needle is visible (needle key < n):  O = V[needle], bit for bit;
  - it is not:                               O = dtype(fp32(sum_{j<n} V[j]) * fp32(1 / n)), the kernel's o * (1 / l)
                                             with every P = 1;
  - n = 0:                                   O = 0.
This needs M = A^2 * scale * log2(e) between about 150 and 4096: above 126, ex2.approx.ftz flushes every non-needle
weight (and, for split decode, the combine weight of every split without the needle) to exactly 0; below 4096 the
rounding residual of the running max leaves the needle's P within half an ulp of 1, so it rounds to 1.0 in fp16 and
bf16.  At the default scale 1 / sqrt(D), A = 64 gives M = 185 (D = 1024) to 1044 (D = 32).

Keys are addressed flat: every block's keys are consecutive rows of one [T, D] array, so the expected value of a row is
two gathers and one prefix sum, whatever the layout of the tensors the kernel reads."""
from __future__ import annotations

import torch

A = 64.0


def values(T: int, D: int, dtype, generator: torch.Generator, device="cpu") -> torch.Tensor:
    """V [T, D]: integers uniform in [-8, 8]."""
    return torch.randint(-8, 9, (T, D), generator=generator, device=device).to(dtype)


def keys(T: int, D: int, key: torch.Tensor, col: torch.Tensor, dtype, device="cpu") -> torch.Tensor:
    """K [T, D]: A at (key[i], col[i]) for each needle i, 0 elsewhere.  The caller places at most one needle per
    (block, column)."""
    k = torch.zeros(T, D, dtype=dtype, device=device)
    k[key.to(device).long(), col.to(device).long()] = A
    return k


def queries(col: torch.Tensor, D: int, dtype) -> torch.Tensor:
    """Q [R, D]: row r is A * e_col[r]."""
    q = torch.zeros(col.numel(), D, dtype=dtype, device=col.device)
    q[torch.arange(col.numel(), device=col.device), col.long().view(-1)] = A
    return q


def expected(v: torch.Tensor, first: torch.Tensor, n: torch.Tensor, needle: torch.Tensor, dtype):
    """(O [R, D] in dtype, mean [R] bool) for rows that see keys [first, first + n) of the flat V [T, D] and whose needle
    is flat key `needle` (negative: the row's block has no needle in the row's column).  `mean` marks the rows whose
    needle is not visible; their value goes through 1 / n."""
    dev = v.device
    first, n, needle = (t.to(dev).long().view(-1) for t in (first, n, needle))
    pre = torch.cat([torch.zeros(1, v.size(1), dtype=torch.float64, device=dev), v.double().cumsum(0)])
    vis = (needle >= first) & (needle < first + n)
    total = (pre[first + n] - pre[first]).float()                        # an exact integer sum, held exactly in fp32
    inv = torch.ones_like(n, dtype=torch.float32) / n.clamp(min=1).float()
    mean = total * inv.view(-1, 1)
    out = torch.where(vis.view(-1, 1), v[needle.clamp(min=0)].float(), mean)
    out = torch.where((n > 0).view(-1, 1), out, torch.zeros_like(out))
    return out.to(dtype), (~vis) & (n > 0)


def ulp(x: torch.Tensor, dtype) -> torch.Tensor:
    """One ulp of dtype at |x| (the subnormal spacing below the smallest normal)."""
    mant, emin = (10, -14) if dtype == torch.float16 else (7, -126)
    e = torch.floor(torch.log2(x.float().abs().clamp(min=2.0 ** emin)))
    return torch.pow(2.0, e - mant)
