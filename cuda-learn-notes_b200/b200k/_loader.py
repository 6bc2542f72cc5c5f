"""ctypes binding of libb200k.so — the C ABI declared in include/b200k.h.

The library is built in-tree by ``make -C cuda-learn-notes_b200/csrc`` (plain nvcc, sm_90a; see
``__graft_entry__.build``).  There is NO fallback: if the shared object is missing or a symbol cannot be
resolved, importing this module raises, and every op raises ``RuntimeError`` when the C side reports an error.

Replaces the reference's JIT loaders: kernels/hgemm/tools/utils.py:L116-132 (try_load_hgemm_library),
ffpa-attn-mma/env.py:L386-410 (try_load_ffpa_library), flash_attn_mma.py:L177-181 (cpp_extension.load).
"""
from __future__ import annotations

import ctypes
import os
import re
import subprocess
from ctypes import c_char_p, c_float, c_int, c_int64, c_size_t, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC_DIR = os.path.normpath(os.path.join(_HERE, "..", "csrc"))
REPO_ROOT = os.path.normpath(os.path.join(_HERE, "..", ".."))
HEADER = os.path.join(REPO_ROOT, "include", "b200k.h")
LIB_PATH = os.path.join(_HERE, "libb200k.so")

# error codes (include/b200k.h)
OK, EDTYPE, ESHAPE, EALIGN, EHEADDIM, ECUDA, EARCH, EARG = 0, -1, -2, -3, -4, -5, -6, -7

# dtype enums (include/b200k.h)
F32, F16, BF16, I8, FP8_E4M3, FP8_E5M2, I32 = 0, 1, 2, 3, 4, 5, 6

HGEMM_AUTO, HGEMM_1CTA_128x256, HGEMM_2CTA_256x256, HGEMM_2CTA_256x128, HGEMM_2CTA_512x256 = 0, 1, 2, 3, 4

# activation ops (include/b200k.h)
ACT_RELU, ACT_SIGMOID, ACT_GELU, ACT_SWISH, ACT_ELU, ACT_HARDSWISH, ACT_HARDSHRINK = range(7)


def build(verbose: bool = False) -> str:
    """Compile libb200k.so in-tree with nvcc (seconds; no torch headers involved)."""
    cmd = ["make", "-C", CSRC_DIR, "-j", str(os.cpu_count() or 4)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        print(res.stdout)
        print(res.stderr)
    if res.returncode != 0:
        raise RuntimeError("building libb200k.so failed (make -C %s)" % CSRC_DIR)
    return LIB_PATH


def declared_symbols() -> list[str]:
    """Every function name include/b200k.h declares (used by the export test)."""
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200k_[a-z0-9_]+)\s*\(", text)))


_SIGS = {
    "b200k_abi_version": (c_int, []),
    "b200k_last_error": (c_char_p, []),
    "b200k_device_info": (c_int, [ctypes.POINTER(c_int)] * 3),
    "b200k_hgemm_f16": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int, c_int, c_void_p]),
    "b200k_gemm": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int, c_int, c_int, c_void_p]),
    "b200k_gemm_ex": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int, c_int, c_int, c_int, c_void_p]),
    "b200k_fa2_fwd_f16": (c_int, [c_void_p] * 4 + [c_int64] * 4 + [c_float, c_int, c_int, c_void_p]),
    "b200k_ffpa_fwd_f16": (c_int, [c_void_p] * 4 + [c_int64] * 4 + [c_float, c_int, c_void_p]),
    "b200k_fa2_fwd": (c_int, [c_void_p] * 4 + [c_int64] * 4 + [c_float, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    "b200k_fa2_fwd_varlen": (c_int, [c_void_p] * 6 + [c_int64] * 7 + [c_float, c_int, c_int, c_void_p]),
    "b200k_fa2_fwd_kvcache": (c_int, [c_void_p] * 6 + [c_int64] * 8 + [c_float, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "b200k_fa2_fwd_kvcache_workspace_bytes": (c_int, [c_int64] * 6 + [ctypes.POINTER(c_size_t)]),
    "b200k_fa2_fwd_kvcache_append": (c_int, [c_void_p] * 8 + [c_int64] + [c_void_p] * 2 + [c_int64] * 2 + [c_int]
                                     + [c_int64] * 8 + [c_float, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "b200k_fa2_fwd_kvcache_append_workspace_bytes": (c_int, [c_int64] * 6 + [c_int, ctypes.POINTER(c_size_t)]),
    "b200k_fa2_fwd_lse": (c_int, [c_void_p] * 5 + [c_int64] * 4 + [c_float, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    "b200k_fa2_fwd_varlen_lse": (c_int, [c_void_p] * 7 + [c_int64] * 7 + [c_float, c_int, c_int, c_void_p]),
    "b200k_fa2_fwd_kvcache_lse": (c_int, [c_void_p] * 7 + [c_int64] * 8
                                  + [c_float, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "b200k_fa2_fwd_kvcache_append_lse": (c_int, [c_void_p] * 9 + [c_int64] + [c_void_p] * 2 + [c_int64] * 2 + [c_int]
                                         + [c_int64] * 8 + [c_float, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "b200k_fa2_varlen_paged": (c_int, [c_void_p] * 8 + [c_int64] * 9 + [c_float, c_int, c_int, c_void_p]),
    "b200k_fa2_kvcache_fp8": (c_int, [c_void_p] * 9 + [c_int] + [c_void_p] * 2 + [c_int64] + [c_void_p] * 2
                              + [c_int64] * 2 + [c_int] + [c_int64] * 8 + [c_float, c_int, c_int, c_void_p, c_size_t,
                                                                         c_void_p]),
    "b200k_fa2_kvcache_fp8_workspace_bytes": (c_int, [c_int64] * 6 + [c_int, c_int, ctypes.POINTER(c_size_t)]),
    "b200k_fa2_varlen_paged_fp8": (c_int, [c_void_p] * 10 + [c_int] + [c_int64] * 9 + [c_float, c_int, c_int, c_void_p]),
    "b200k_attn_merge": (c_int, [c_void_p] * 4 + [c_int64] * 3 + [c_int, c_void_p]),
    "b200k_fa2_bwd": (c_int, [c_void_p] * 9 + [c_int64] * 4 + [c_float, c_int, c_int, c_void_p, c_void_p, c_size_t,
                                                               c_void_p]),
    "b200k_fa2_bwd_workspace_bytes": (c_int, [c_int64] * 3 + [ctypes.POINTER(c_size_t)]),
    "b200k_fa2_bwd_varlen": (c_int, [c_void_p] * 11 + [c_int64] * 8 + [c_float, c_int, c_int, c_void_p, c_size_t,
                                                                     c_void_p]),
    "b200k_fa2_bwd_varlen_workspace_bytes": (c_int, [c_int64] * 2 + [ctypes.POINTER(c_size_t)]),
    "b200k_elementwise_add": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p]),
    "b200k_reduce_workspace_bytes": (c_size_t, []),
    "b200k_block_all_reduce_sum": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p]),
    "b200k_softmax": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_void_p, c_void_p]),
    "b200k_rms_norm": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_float, c_float, c_int, c_int, c_int, c_void_p]),
    "b200k_rope_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_void_p]),
    "b200k_max_i32": (c_int, [c_void_p, c_int64, c_void_p, c_void_p]),
    "b200k_histogram_i32": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p]),
    "b200k_embedding": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int, c_void_p]),
    "b200k_transpose_u16_batched": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p]),
    "b200k_activation": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p]),
    "b200k_layer_norm": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_float, c_float, c_float, c_int, c_int, c_void_p]),
    "b200k_dot_prod": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p]),
    "b200k_mat_transpose_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p]),
    "b200k_gemv": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int, c_void_p]),
}


def _load() -> ctypes.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "libb200k.so is not built (%s). Run `python -c 'import __graft_entry__ as g; g.build()'` or "
            "`make -C cuda-learn-notes_b200/csrc`. There is no CPU or PyTorch fallback." % LIB_PATH
        )
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in _SIGS.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export it: fail loudly
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


class B200KError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(msg)
        self.code = code


def last_error() -> str:
    return (lib.b200k_last_error() or b"").decode("utf-8", "replace")


def check(rc: int) -> None:
    if rc != OK:
        raise B200KError(rc, last_error() or ("libb200k error %d" % rc))


def device_info() -> dict:
    sm, maj, mnr = c_int(0), c_int(0), c_int(0)
    check(lib.b200k_device_info(ctypes.byref(sm), ctypes.byref(maj), ctypes.byref(mnr)))
    return {"sm_count": sm.value, "cc": (maj.value, mnr.value)}
