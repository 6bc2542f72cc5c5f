"""CPU: the coverage table of kernel_inventory.py against the built library (cuobjdump -sass; no GPU needed).  Every
function of libb200k.so has a row naming the GPU case of test_gpu_kernel_coverage.py that launches it, every row names
a function the library has, and each row's case launches that row's kernel."""
import collections
import functools
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kernel_inventory as ki  # noqa: E402


@functools.lru_cache(maxsize=1)
def _names():
    return ki.library_kernels()


def _library():
    names = _names()
    if names is None:
        pytest.skip("libb200k.so not built, or cuobjdump / c++filt not on PATH")
    return names


def test_every_library_kernel_has_a_row_and_every_row_a_kernel():
    names = _library()
    dup = [n for n, c in collections.Counter(names).items() if c > 1]
    assert not dup, "two functions normalise to one name: %s" % dup
    lib, table = set(names), set(ki.COVERAGE)
    unmapped, gone = sorted(lib - table), sorted(table - lib)
    assert not unmapped, "%d kernels of the library have no row in kernel_inventory.COVERAGE:\n  %s" % (
        len(unmapped), "\n  ".join(unmapped))
    assert not gone, "%d rows of kernel_inventory.COVERAGE name no kernel of the library:\n  %s" % (
        len(gone), "\n  ".join(gone))
    print("\n%d kernels in libb200k.so, all mapped to %d GPU cases" % (len(lib), len(set(ki.COVERAGE.values()))))


@pytest.mark.parametrize("kernel", sorted(ki.COVERAGE))
def test_each_row_is_launched_by_its_case(kernel):
    assert kernel in ki.launched(ki.COVERAGE[kernel]), (kernel, ki.COVERAGE[kernel])


def test_launched_sets_name_only_library_kernels():
    names = set(_library())
    for case in set(ki.COVERAGE.values()):
        assert ki.launched(case) <= names, (case, sorted(ki.launched(case) - names))


@pytest.mark.parametrize("raw,want", [
    ("void b200k::attn_combine_kernel<1, float, true>(float const*, float const*, void*, long long, int, int, float*)",
     "b200k::attn_combine_kernel<1,float,true>"),
    ("void b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0, 64, 1, 128, false>, b200k::WithLse<b200k::Fp8Kv<b200k::"
     "AttnDecode<b200k::AttnCfg<0, 64, 1, 128, false> >, 4> > >(CUtensorMap_st, CUtensorMap_st, CUtensorMap_st, void*, "
     "int, int, float, b200k::WithLse<b200k::Fp8Kv<b200k::AttnDecode<b200k::AttnCfg<0, 64, 1, 128, false> >, 4> >)",
     "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,64,1,128,false>,b200k::WithLse<b200k::Fp8Kv<b200k::AttnDecode<"
     "b200k::AttnCfg<0,64,1,128,false>>,4>>>"),
    ("b200k::embedding_kernel(int const*, unsigned char const*, unsigned char*, long, long, long, bool)",
     "b200k::embedding_kernel"),
    ("void b200k::attn_combine_kernel<0, unsigned short, false>(unsigned short const*, float const*, void*, long long, "
     "int, int, float*)", "b200k::attn_combine_kernel<0,unsigned short,false>"),
])
def test_normalize(raw, want):
    assert ki.normalize(raw) == want
    assert ki.normalize(want) == want
