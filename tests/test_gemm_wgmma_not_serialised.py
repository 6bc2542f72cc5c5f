"""Static check on the machine code of the GEMM (cuobjdump -sass; no GPU needed): its wgmma main loop is pipelined.

ptxas serialises every wgmma of a kernel that contains a function call, a printf for instance: each HGMMA then carries
the `gsb0` scoreboard and is followed by `WARPGROUP.DEPBAR.LE gsb0, 0x0`, so a warpgroup waits for every MMA before it
issues the next one.  The source still reads `wgmma.wait_group 1`; only the SASS shows the difference."""
import collections
import functools
import os
import re
import shutil
import subprocess

import pytest

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cuda-learn-notes_b200", "b200k", "libb200k.so")


@functools.lru_cache(maxsize=1)
def _gemm_kernels():
    if shutil.which("cuobjdump") is None or shutil.which("c++filt") is None:
        pytest.skip("cuobjdump / c++filt not on PATH")
    if not os.path.exists(LIB):
        pytest.skip("libb200k.so not built")
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    counts, cur = collections.defaultdict(collections.Counter), None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts[cur]["_"] += 0
            continue
        if cur is None:
            continue
        if re.search(r"\bHGMMA\.", line):
            counts[cur]["hgmma"] += 1
            if re.search(r"\bgsb0\b", line):
                counts[cur]["hgmma_gsb0"] += 1
        if re.search(r"WARPGROUP\.DEPBAR\.LE\s+gsb0,\s*0x1\b", line):
            counts[cur]["depbar_1"] += 1
        if re.search(r"\bCALL\.", line):
            counts[cur]["call"] += 1
    names = subprocess.run(["c++filt"], input="\n".join(counts), capture_output=True, text=True, check=True).stdout.splitlines()
    ks = {n: counts[m] for n, m in zip(names, counts) if "b200k::hgemm_wgmma_kernel" in n}
    assert len(ks) == 9, sorted(ks)  # f16 and bf16 x (A, B each K- or MN-major), and tf32
    return ks


def test_gemm_kernels_contain_no_call():
    for name, c in _gemm_kernels().items():
        assert c["call"] == 0, name


def test_gemm_wgmma_is_not_serialised():
    for name, c in _gemm_kernels().items():
        assert c["hgmma"] > 0, name
        assert c["hgmma_gsb0"] < c["hgmma"], (name, dict(c))
        assert c["depbar_1"] >= 1, (name, dict(c))
