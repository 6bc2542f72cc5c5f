"""CPU: the C-ABI library loads without a GPU, exports every symbol include/b200k.h declares, and validates
arguments before touching the device.  No compute is attempted here."""
import ctypes

import pytest

from b200k import _loader as L


def test_header_symbols_are_all_exported_and_bound():
    declared = L.declared_symbols()
    assert len(declared) >= 15
    raw = ctypes.CDLL(L.LIB_PATH)
    for name in declared:
        assert hasattr(raw, name), "libb200k.so does not export %s" % name
    assert sorted(L._SIGS) == declared, "ctypes signature table and include/b200k.h disagree"


def test_abi_version_and_workspace():
    assert L.lib.b200k_abi_version() == 1
    assert L.lib.b200k_reduce_workspace_bytes() >= 2048 * 4


def test_argument_validation_happens_before_cuda():
    lib = L.lib
    one = ctypes.c_void_p(16)  # never dereferenced: validation fails first
    assert lib.b200k_hgemm_f16(None, one, one, 8, 8, 8, 0, 0, None) == L.EARG
    assert lib.b200k_hgemm_f16(one, one, one, 8, 8, 7, 0, 0, None) == L.ESHAPE
    assert b"multiples of 8" in lib.b200k_last_error()
    assert lib.b200k_hgemm_f16(one, one, one, 0, 8, 8, 0, 0, None) == L.ESHAPE
    assert lib.b200k_fa2_fwd_f16(None, one, one, one, 1, 1, 8, 64, 0.0, 0, 0, None) == L.EARG
    assert lib.b200k_fa2_fwd_f16(one, one, one, one, 1, 0, 8, 64, 0.0, 0, 0, None) == L.ESHAPE
    assert lib.b200k_ffpa_fwd_f16(one, one, one, one, 1, 1, 8, 200, 0.0, 0, None) == L.EHEADDIM
    assert b"headdim not support" in lib.b200k_last_error()
    assert lib.b200k_elementwise_add(one, one, one, 4, 99, None) in (L.EDTYPE, L.ECUDA, L.EARCH)
    assert lib.b200k_rope_f32(one, one, 4, 7, 1, None) == L.ESHAPE
    assert lib.b200k_softmax(one, one, 4, 8, L.F32, 9, None, None) == L.EARG
    assert lib.b200k_embedding(one, one, one, 4, 4, 4, L.I8, None) == L.EDTYPE
    # generic GEMM entry: fp32 rows must be 16-byte multiples too (4 elements), unknown dtypes are refused
    assert lib.b200k_gemm(one, one, one, 8, 8, 6, 0, L.F32, 0, None) == L.ESHAPE
    assert b"multiples of 4" in lib.b200k_last_error()
    assert lib.b200k_gemm(one, one, one, 8, 8, 4, 0, L.BF16, 0, None) == L.ESHAPE
    assert lib.b200k_gemm(one, one, one, 8, 8, 8, 0, L.I8, 0, None) == L.EDTYPE
    assert lib.b200k_gemm(None, one, one, 8, 8, 8, 1, L.F32, 0, None) == L.EARG
    # variant: 0 .. 4 in the low 8 bits, higher bits ignored; 5 is unknown whatever the high bits hold
    for v in (5, 5 | (0x5A5A << 8)):
        assert lib.b200k_hgemm_f16(one, one, one, 8, 8, 8, 0, v, None) == L.EARG
        assert b"variant 5 unknown" in lib.b200k_last_error()
        for dt in (L.F16, L.BF16, L.F32):
            assert lib.b200k_gemm(one, one, one, 8, 8, 8, 1, dt, v, None) == L.EARG
        assert lib.b200k_gemm_ex(one, one, one, 8, 8, 8, 1, 0, L.BF16, v, None) == L.EARG
    # second set of support kernels
    assert lib.b200k_layer_norm(one, one, 0, 8, 1.0, 0.0, 1e-5, L.F32, 1, None) == L.ESHAPE
    assert lib.b200k_mat_transpose_f32(one, None, 4, 4, None) == L.EARG
    assert lib.b200k_gemv(one, one, one, 4, 0, L.F32, None) == L.ESHAPE
    assert lib.b200k_dot_prod(one, one, None, 4, L.F32, one, None) == L.EARG
    # round-2 entry points
    assert lib.b200k_fa2_fwd(one, one, one, one, 1, 1, 8, 64, 0.0, 0, L.F32, 0, None, 0, None) == L.EDTYPE
    assert lib.b200k_fa2_fwd(one, one, one, one, 1, 1, 8, 64, 0.0, 1, L.BF16, 0, None, 0, None) == L.EARG   # bf16 + [B,H,D,N] V
    assert lib.b200k_fa2_fwd(one, one, one, one, 1, 1, 8, 48, 0.0, 0, L.F16, 1, None, 0, None) == L.EHEADDIM
    assert lib.b200k_gemm_ex(one, one, one, 12, 8, 8, 1, 0, L.F16, 0, None) == L.ESHAPE     # A^T storage: M % 8
    assert lib.b200k_gemm_ex(one, one, one, 8, 8, 8, 1, 0, L.F32, 0, None) == L.EDTYPE
    assert lib.b200k_transpose_u16_batched(one, None, 1, 4, 4, None) == L.EARG
    assert lib.b200k_transpose_u16_batched(one, one, 0, 4, 4, None) == L.ESHAPE


def test_no_gpu_means_loud_failure_not_fallback():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    one = ctypes.c_void_p(16)
    rc = L.lib.b200k_hgemm_f16(one, one, one, 128, 128, 128, 0, 0, None)
    assert rc in (L.ECUDA, L.EARCH) and L.last_error()
    with pytest.raises(L.B200KError):
        L.device_info()
