"""Static check on the machine code of the attention backward (cuobjdump -sass; no GPU needed): each kernel is one body
instantiated once per layout mode (dense, packed), dtype and padded head dim, and every instantiation contains no
function call and has wgmmas that are not serialised.

ptxas serialises every wgmma of a kernel that contains a call (a printf behind an mbarrier wait, for instance): each
HGMMA then carries the `gsb0` scoreboard.  In a kernel that is not serialised only the last HGMMA of a group does."""
import collections
import functools
import os
import re
import shutil
import subprocess

import pytest

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cuda-learn-notes_b200", "b200k", "libb200k.so")


@functools.lru_cache(maxsize=1)
def _bwd_kernels():
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
        if re.search(r"\bCALL\.", line):
            counts[cur]["call"] += 1
    names = subprocess.run(["c++filt"], input="\n".join(counts), capture_output=True, text=True, check=True).stdout.splitlines()
    ks = {n: counts[m] for n, m in zip(names, counts) if "b200k::attn_bwd_" in n}
    # f16 and bf16 x (head dims padded to 64, 128) x (dense, packed) for the dK/dV and the dQ kernel, and the prep kernel
    # per dtype and layout: each one body instantiated per mode
    expected = set()
    for dt in (0, 1):
        for dp in (64, 128):
            kv, q = "b200k::AttnCfg<%d, %d, 1, 64, false>" % (dt, dp), "b200k::AttnCfg<%d, %d, 2, 64, false>" % (dt, dp)
            for mode in ("BwdKeysDense", "BwdKeysPacked"):
                expected.add("b200k::attn_bwd_dkdv_kernel<%s, b200k::%s<%s > >" % (kv, mode, kv))
            for mode in ("AttnDense", "AttnPacked"):
                expected.add("b200k::attn_bwd_dq_kernel<%s, b200k::%s<%s > >" % (q, mode, q))
        for packed in ("false", "true"):
            expected.add("b200k::attn_bwd_prep_kernel<%d, %s>" % (dt, packed))
    kernels = [re.sub(r"^void ", "", n.split("(")[0]) for n in ks]
    assert len(kernels) == len(set(kernels)) == 20, sorted(kernels)
    assert set(kernels) == expected, (sorted(set(kernels) - expected), sorted(expected - set(kernels)))
    return ks


def test_backward_kernels_of_every_mode_contain_no_call():
    for name, c in _bwd_kernels().items():
        assert c["call"] == 0, name


def test_backward_wgmma_of_every_mode_is_not_serialised():
    for name, c in _bwd_kernels().items():
        if "prep_kernel" in name:
            assert c["hgmma"] == 0, name  # a bandwidth kernel
            continue
        assert c["hgmma"] > 0, name
        assert c["hgmma_gsb0"] < c["hgmma"], (name, dict(c))
