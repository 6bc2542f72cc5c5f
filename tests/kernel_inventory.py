"""Every kernel libb200k.so ships, and the GPU case that launches it.

COVERAGE has one row per `__global__` function in the library: its demangled name without the parameter list, and the
id of the case in test_gpu_kernel_coverage.py that launches it.  test_kernel_inventory_cpu.py holds the table to the
built library both ways (a new instantiation with no row fails, and so does a row whose kernel is gone), and
`launched(case)` gives the exact set of library kernels a case launches, which the GPU test compares with what
torch.profiler records.

Names are normalised (`normalize`): no return type, no parameter list, no blanks next to `<`, `>` or `,`.  So
`void b200k::attn_combine_kernel<1, float, true>(float const*, ...)` is `b200k::attn_combine_kernel<1,float,true>`,
whichever demangler produced it.

Case ids are `-`-separated tokens: the family first, then its options.  Head dims are `d<D>`, row widths `h<H>`.
"""
from __future__ import annotations

import os
import re
import shutil
import subprocess

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cuda-learn-notes_b200", "b200k",
                   "libb200k.so")


def strip_params(name: str) -> str:
    """`name` without its trailing parenthesised parameter list (if it has one)."""
    name = name.strip()
    if not name.endswith(")"):
        return name
    depth = 0
    for i in range(len(name) - 1, -1, -1):
        if name[i] == ")":
            depth += 1
        elif name[i] == "(":
            depth -= 1
            if depth == 0:
                return name[:i]
    return name


def normalize(demangled: str) -> str:
    n = strip_params(demangled)
    n = re.sub(r"\s+", " ", n).strip()
    n = re.sub(r"^void ", "", n)
    return re.sub(r"\s*([<>,])\s*", r"\1", n)


def library_kernels(lib: str = LIB) -> list[str] | None:
    """The normalised names of every function in `lib` (cuobjdump -sass, then c++filt), or None when the library or
    the tools are missing."""
    if shutil.which("cuobjdump") is None or shutil.which("c++filt") is None or not os.path.exists(lib):
        return None
    sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    mangled = re.findall(r"Function : (\S+)", sass)
    names = subprocess.run(["c++filt"], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout
    return [normalize(n) for n in names.splitlines()]


# ------------------------------------------------------------------------------------------------ kernel names
DT = {"f16": 0, "bf16": 1}
FMT = {"e4m3": 4, "e5m2": 5}
TYPE = {"f32": "float", "f16": "__half", "bf16": "__nv_bfloat16"}
DTYPE_ENUM = {"f32": 0, "f16": 1, "bf16": 2, "i8": 3, "e4m3": 4, "e5m2": 5}
ACT = {"relu": 0, "sigmoid": 1, "gelu": 2, "swish": 3, "elu": 4, "hardswish": 5, "hardshrink": 6}


def _b(x: bool) -> str:
    return "true" if x else "false"


def attn_cfg(dt: str, dv: int, nwg: int, bn: int, vdn: bool = False) -> str:
    return "b200k::AttnCfg<%d,%d,%d,%d,%s>" % (DT[dt], dv, nwg, bn, _b(vdn))


def attn_fwd(cfg: str, mode: str, fmt: str | None = None, lse: bool = False) -> str:
    m = "b200k::%s<%s>" % (mode, cfg)
    if fmt:
        m = "b200k::Fp8Kv<%s,%d>" % (m, FMT[fmt])
    if lse:
        m = "b200k::WithLse<%s>" % m
    return "b200k::attn_fwd_wgmma_kernel<%s,%s>" % (cfg, m)


def combine(dt: str, part: str, lse: bool) -> str:
    return "b200k::attn_combine_kernel<%d,%s,%s>" % (DT[dt], part, _b(lse))


def dv_of(D: int) -> int:
    """O columns of one CTA for D <= 128 (forward) and the padded head dim of the backward."""
    return 64 if D <= 64 else 128


def ffpa_cfg(D: int) -> tuple[int, int]:
    """(DV, consumer warpgroups) of b200k_ffpa_fwd_f16 for D > 128."""
    nqc = (D + 63) // 64
    slices = (nqc + 3) // 4
    chunks = (nqc + slices - 1) // slices
    return (192, 2) if chunks == 3 else (256, 1)


def row_threads(t: str, H: int) -> int | None:
    """Threads per row of launch_row (support_paths.row), None for the scalar kernel."""
    vn = 4 if t == "f32" else 8
    if H % vn:
        return None
    return 32 if H <= 1024 else (128 if H <= 4096 else 256)


def row_kernel(t: str, op: int, H: int) -> str:
    r = row_threads(t, H)
    if r is None:
        return "b200k::row_kernel_scalar<%s,%d>" % (TYPE[t], op)
    return "b200k::row_kernel<%s,%d,%d>" % (TYPE[t], r, op)


def _opt(toks: list[str], prefix: str) -> int:
    return next(int(t[len(prefix):]) for t in toks if re.fullmatch(prefix + r"\d+", t))


def launched(case: str) -> frozenset[str]:
    """The library kernels case `case` launches, each exactly once or more, and nothing else of the library."""
    toks = case.split("-")
    fam, opts = toks[0], set(toks[1:])
    dt = next((t for t in toks[1:] if t in ("f16", "bf16", "f32", "tf32", "i8") + tuple(FMT)), None)
    fmt = next((t for t in toks[2:] if t in FMT), None) if fam in ("paged", "decode", "append") else None
    lse = "lse" in opts
    if fam == "gemm":
        layout = toks[2]
        if dt == "tf32":
            out = {"b200k::hgemm_wgmma_kernel<b200k::GemmCfg<2,false,false>>"}
            return frozenset(out | ({"b200k::transpose_f32x4_kernel"} if layout == "nn" else set()))
        km, nn = layout.startswith("km"), layout.endswith("nn")
        return frozenset({"b200k::hgemm_wgmma_kernel<b200k::GemmCfg<%d,%s,%s>>" % (DT[dt], _b(km), _b(nn))})
    if fam == "dense":
        D = _opt(toks, "d")
        return frozenset({attn_fwd(attn_cfg(dt, dv_of(D), 2, 128, "vdn" in opts), "AttnDense", lse=lse)})
    if fam == "ffpa":
        dv, nwg = ffpa_cfg(_opt(toks, "d"))
        return frozenset({attn_fwd(attn_cfg("f16", dv, nwg, 64), "AttnDense")})
    if fam in ("packed", "paged"):
        D = _opt(toks, "d")
        mode = "AttnPacked" if fam == "packed" else "AttnPackedPaged"
        return frozenset({attn_fwd(attn_cfg(dt, dv_of(D), 2, 128), mode, fmt, lse)})
    if fam in ("decode", "append"):
        D = _opt(toks, "d") if fam == "decode" else 128
        split = "split" in opts  # the append cases' caches hold 256 keys: too few to split
        cfg = attn_cfg(dt, dv_of(D), 1, 128)
        out = {attn_fwd(cfg, "AttnDecode", fmt, lse and not split)}
        if split:
            out.add(combine(dt, "float", lse))
        if fam == "append":
            rot, inter = toks[-1] != "plain", toks[-1] == "inter"
            out.add("b200k::kvcache_append_kernel<%d,%s,%s,%d>" % (DT[dt], _b(rot), _b(inter), FMT[fmt] if fmt else 0))
        return frozenset(out)
    if fam == "merge":
        return frozenset({combine(dt, "unsigned short", lse)})
    if fam == "bwd":
        packed, D = toks[1] == "packed", _opt(toks, "d")
        kv, q = attn_cfg(dt, dv_of(D), 1, 64), attn_cfg(dt, dv_of(D), 2, 64)
        return frozenset({"b200k::attn_bwd_prep_kernel<%d,%s>" % (DT[dt], _b(packed)),
                          "b200k::attn_bwd_dkdv_kernel<%s,b200k::BwdKeys%s<%s>>" % (kv, "Packed" if packed else "Dense", kv),
                          "b200k::attn_bwd_dq_kernel<%s,b200k::Attn%s<%s>>" % (q, "Packed" if packed else "Dense", q)})
    if fam in ("softmax", "rmsnorm", "layernorm"):
        H = _opt(toks, "h")
        if fam == "softmax":
            op = 1 if "m2" in opts else 0
        else:
            op = 4 if fam == "layernorm" else (3 if "acc16" in opts else 2)
        out = {row_kernel(dt, op, H)}
        if "m0" in opts:
            out.add("b200k::reduce_sum_kernel<0,false,true>")
        return frozenset(out)
    if fam == "reduce":
        return frozenset({"b200k::reduce_sum_kernel<%d,%s,false>" % (DTYPE_ENUM[toks[1]], _b("acc16" in opts))})
    if fam == "add":
        return frozenset({"b200k::elementwise_add_%s_kernel<%s>" % (toks[2], TYPE[dt])})
    if fam == "hist":
        if toks[1] == "auto":
            return frozenset({"b200k::init_i32_kernel", "b200k::max_i32_kernel", "b200k::histogram_i32_kernel<true>"})
        return frozenset({"b200k::histogram_i32_kernel<%s>" % _b(toks[1] == "smem")})
    if fam == "act":
        return frozenset({"b200k::activation_kernel<%s,%d,%s>" % (TYPE[dt], ACT[toks[2]], _b("clamp" in opts))})
    if fam in ("dot", "gemv"):
        return frozenset({"b200k::%s_kernel<%s>" % (fam, TYPE[dt])})
    if fam == "transpose":
        return frozenset({{"f32x4": "b200k::transpose_f32x4_kernel", "f32": "b200k::transpose_kernel<float>",
                           "u16": "b200k::transpose_kernel<unsigned short>"}[toks[1]]})
    if fam in ("embedding", "rope"):
        return frozenset({"b200k::%s_kernel" % ("rope_f32" if fam == "rope" else fam)})
    raise KeyError(case)


# ------------------------------------------------------------------------------------------------ the table
# kernel (normalised name) -> the case of test_gpu_kernel_coverage.py that launches it
COVERAGE: dict[str, str] = {
    "b200k::hgemm_wgmma_kernel<b200k::GemmCfg<2,false,false>>": "gemm-tf32-nn",
    "b200k::hgemm_wgmma_kernel<b200k::GemmCfg<1,false,false>>": "gemm-bf16-tn",
    "b200k::hgemm_wgmma_kernel<b200k::GemmCfg<1,false,true>>": "gemm-bf16-nn",
    "b200k::hgemm_wgmma_kernel<b200k::GemmCfg<1,true,false>>": "gemm-bf16-kmtn",
    "b200k::hgemm_wgmma_kernel<b200k::GemmCfg<1,true,true>>": "gemm-bf16-kmnn",
    "b200k::hgemm_wgmma_kernel<b200k::GemmCfg<0,false,false>>": "gemm-f16-tn",
    "b200k::hgemm_wgmma_kernel<b200k::GemmCfg<0,false,true>>": "gemm-f16-nn",
    "b200k::hgemm_wgmma_kernel<b200k::GemmCfg<0,true,false>>": "gemm-f16-kmtn",
    "b200k::hgemm_wgmma_kernel<b200k::GemmCfg<0,true,true>>": "gemm-f16-kmnn",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,256,1,64,false>,b200k::AttnDense<b200k::AttnCfg<0,256,1,64,false>>>": "ffpa-d256",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,192,2,64,false>,b200k::AttnDense<b200k::AttnCfg<0,192,2,64,false>>>": "ffpa-d192",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,128,2,128,false>,b200k::AttnPackedPaged<b200k::AttnCfg<1,128,2,128,false>>>": "paged-bf16-d128",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,128,2,128,false>,b200k::WithLse<b200k::AttnPackedPaged<b200k::AttnCfg<1,128,2,128,false>>>>": "paged-bf16-d96-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,128,2,128,false>,b200k::Fp8Kv<b200k::AttnPackedPaged<b200k::AttnCfg<1,128,2,128,false>>,5>>": "paged-bf16-e5m2-d96",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,128,2,128,false>,b200k::WithLse<b200k::Fp8Kv<b200k::AttnPackedPaged<b200k::AttnCfg<1,128,2,128,false>>,5>>>": "paged-bf16-e5m2-d128-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,128,2,128,false>,b200k::Fp8Kv<b200k::AttnPackedPaged<b200k::AttnCfg<1,128,2,128,false>>,4>>": "paged-bf16-e4m3-d96",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,128,2,128,false>,b200k::WithLse<b200k::Fp8Kv<b200k::AttnPackedPaged<b200k::AttnCfg<1,128,2,128,false>>,4>>>": "paged-bf16-e4m3-d128-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,64,2,128,false>,b200k::AttnPackedPaged<b200k::AttnCfg<1,64,2,128,false>>>": "paged-bf16-d64",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,64,2,128,false>,b200k::WithLse<b200k::AttnPackedPaged<b200k::AttnCfg<1,64,2,128,false>>>>": "paged-bf16-d32-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,64,2,128,false>,b200k::Fp8Kv<b200k::AttnPackedPaged<b200k::AttnCfg<1,64,2,128,false>>,5>>": "paged-bf16-e5m2-d32",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,64,2,128,false>,b200k::WithLse<b200k::Fp8Kv<b200k::AttnPackedPaged<b200k::AttnCfg<1,64,2,128,false>>,5>>>": "paged-bf16-e5m2-d64-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,64,2,128,false>,b200k::Fp8Kv<b200k::AttnPackedPaged<b200k::AttnCfg<1,64,2,128,false>>,4>>": "paged-bf16-e4m3-d32",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,64,2,128,false>,b200k::WithLse<b200k::Fp8Kv<b200k::AttnPackedPaged<b200k::AttnCfg<1,64,2,128,false>>,4>>>": "paged-bf16-e4m3-d64-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,128,2,128,false>,b200k::AttnPackedPaged<b200k::AttnCfg<0,128,2,128,false>>>": "paged-f16-d128",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,128,2,128,false>,b200k::WithLse<b200k::AttnPackedPaged<b200k::AttnCfg<0,128,2,128,false>>>>": "paged-f16-d96-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,128,2,128,false>,b200k::Fp8Kv<b200k::AttnPackedPaged<b200k::AttnCfg<0,128,2,128,false>>,5>>": "paged-f16-e5m2-d96",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,128,2,128,false>,b200k::WithLse<b200k::Fp8Kv<b200k::AttnPackedPaged<b200k::AttnCfg<0,128,2,128,false>>,5>>>": "paged-f16-e5m2-d128-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,128,2,128,false>,b200k::Fp8Kv<b200k::AttnPackedPaged<b200k::AttnCfg<0,128,2,128,false>>,4>>": "paged-f16-e4m3-d96",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,128,2,128,false>,b200k::WithLse<b200k::Fp8Kv<b200k::AttnPackedPaged<b200k::AttnCfg<0,128,2,128,false>>,4>>>": "paged-f16-e4m3-d128-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,64,2,128,false>,b200k::AttnPackedPaged<b200k::AttnCfg<0,64,2,128,false>>>": "paged-f16-d64",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,64,2,128,false>,b200k::WithLse<b200k::AttnPackedPaged<b200k::AttnCfg<0,64,2,128,false>>>>": "paged-f16-d32-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,64,2,128,false>,b200k::Fp8Kv<b200k::AttnPackedPaged<b200k::AttnCfg<0,64,2,128,false>>,5>>": "paged-f16-e5m2-d32",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,64,2,128,false>,b200k::WithLse<b200k::Fp8Kv<b200k::AttnPackedPaged<b200k::AttnCfg<0,64,2,128,false>>,5>>>": "paged-f16-e5m2-d64-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,64,2,128,false>,b200k::Fp8Kv<b200k::AttnPackedPaged<b200k::AttnCfg<0,64,2,128,false>>,4>>": "paged-f16-e4m3-d32",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,64,2,128,false>,b200k::WithLse<b200k::Fp8Kv<b200k::AttnPackedPaged<b200k::AttnCfg<0,64,2,128,false>>,4>>>": "paged-f16-e4m3-d64-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,128,2,128,false>,b200k::AttnPacked<b200k::AttnCfg<1,128,2,128,false>>>": "packed-bf16-d96",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,128,2,128,false>,b200k::WithLse<b200k::AttnPacked<b200k::AttnCfg<1,128,2,128,false>>>>": "packed-bf16-d128-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,64,2,128,false>,b200k::AttnPacked<b200k::AttnCfg<1,64,2,128,false>>>": "packed-bf16-d32",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,64,2,128,false>,b200k::WithLse<b200k::AttnPacked<b200k::AttnCfg<1,64,2,128,false>>>>": "packed-bf16-d64-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,128,2,128,false>,b200k::AttnPacked<b200k::AttnCfg<0,128,2,128,false>>>": "packed-f16-d96",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,128,2,128,false>,b200k::WithLse<b200k::AttnPacked<b200k::AttnCfg<0,128,2,128,false>>>>": "packed-f16-d128-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,64,2,128,false>,b200k::AttnPacked<b200k::AttnCfg<0,64,2,128,false>>>": "packed-f16-d32",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,64,2,128,false>,b200k::WithLse<b200k::AttnPacked<b200k::AttnCfg<0,64,2,128,false>>>>": "packed-f16-d64-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,128,2,128,false>,b200k::AttnDense<b200k::AttnCfg<1,128,2,128,false>>>": "dense-bf16-d96",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,128,2,128,false>,b200k::WithLse<b200k::AttnDense<b200k::AttnCfg<1,128,2,128,false>>>>": "dense-bf16-d128-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,64,2,128,false>,b200k::AttnDense<b200k::AttnCfg<1,64,2,128,false>>>": "dense-bf16-d32",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,64,2,128,false>,b200k::WithLse<b200k::AttnDense<b200k::AttnCfg<1,64,2,128,false>>>>": "dense-bf16-d64-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,128,2,128,false>,b200k::AttnDense<b200k::AttnCfg<0,128,2,128,false>>>": "dense-f16-d96",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,128,2,128,false>,b200k::WithLse<b200k::AttnDense<b200k::AttnCfg<0,128,2,128,false>>>>": "dense-f16-d128-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,64,2,128,false>,b200k::AttnDense<b200k::AttnCfg<0,64,2,128,false>>>": "dense-f16-d32",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,64,2,128,false>,b200k::WithLse<b200k::AttnDense<b200k::AttnCfg<0,64,2,128,false>>>>": "dense-f16-d64-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,128,2,128,true>,b200k::AttnDense<b200k::AttnCfg<0,128,2,128,true>>>": "dense-f16-d128-vdn",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,128,2,128,true>,b200k::WithLse<b200k::AttnDense<b200k::AttnCfg<0,128,2,128,true>>>>": "dense-f16-d96-vdn-lse",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,64,2,128,true>,b200k::AttnDense<b200k::AttnCfg<0,64,2,128,true>>>": "dense-f16-d64-vdn",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,64,2,128,true>,b200k::WithLse<b200k::AttnDense<b200k::AttnCfg<0,64,2,128,true>>>>": "dense-f16-d32-vdn-lse",
    "b200k::kvcache_append_kernel<0,true,false,0>": "append-f16-neox",
    "b200k::kvcache_append_kernel<0,true,true,0>": "append-f16-inter",
    "b200k::kvcache_append_kernel<0,false,false,0>": "append-f16-plain",
    "b200k::kvcache_append_kernel<1,true,false,0>": "append-bf16-neox",
    "b200k::kvcache_append_kernel<1,true,true,0>": "append-bf16-inter",
    "b200k::kvcache_append_kernel<1,false,false,0>": "append-bf16-plain",
    "b200k::kvcache_append_kernel<0,true,false,5>": "append-f16-e5m2-neox",
    "b200k::kvcache_append_kernel<0,true,true,5>": "append-f16-e5m2-inter",
    "b200k::kvcache_append_kernel<0,false,false,5>": "append-f16-e5m2-plain",
    "b200k::kvcache_append_kernel<1,true,false,5>": "append-bf16-e5m2-neox",
    "b200k::kvcache_append_kernel<1,true,true,5>": "append-bf16-e5m2-inter",
    "b200k::kvcache_append_kernel<1,false,false,5>": "append-bf16-e5m2-plain",
    "b200k::kvcache_append_kernel<0,true,false,4>": "append-f16-e4m3-neox",
    "b200k::kvcache_append_kernel<0,true,true,4>": "append-f16-e4m3-inter",
    "b200k::kvcache_append_kernel<0,false,false,4>": "append-f16-e4m3-plain",
    "b200k::kvcache_append_kernel<1,true,false,4>": "append-bf16-e4m3-neox",
    "b200k::kvcache_append_kernel<1,true,true,4>": "append-bf16-e4m3-inter",
    "b200k::kvcache_append_kernel<1,false,false,4>": "append-bf16-e4m3-plain",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,128,1,128,false>,b200k::AttnDecode<b200k::AttnCfg<1,128,1,128,false>>>": "decode-bf16-d128-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,128,1,128,false>,b200k::WithLse<b200k::AttnDecode<b200k::AttnCfg<1,128,1,128,false>>>>": "decode-bf16-d96-lse-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,128,1,128,false>,b200k::Fp8Kv<b200k::AttnDecode<b200k::AttnCfg<1,128,1,128,false>>,5>>": "decode-bf16-e5m2-d128-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,128,1,128,false>,b200k::WithLse<b200k::Fp8Kv<b200k::AttnDecode<b200k::AttnCfg<1,128,1,128,false>>,5>>>": "decode-bf16-e5m2-d96-lse-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,128,1,128,false>,b200k::Fp8Kv<b200k::AttnDecode<b200k::AttnCfg<1,128,1,128,false>>,4>>": "decode-bf16-e4m3-d128-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,128,1,128,false>,b200k::WithLse<b200k::Fp8Kv<b200k::AttnDecode<b200k::AttnCfg<1,128,1,128,false>>,4>>>": "decode-bf16-e4m3-d96-lse-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,64,1,128,false>,b200k::AttnDecode<b200k::AttnCfg<1,64,1,128,false>>>": "decode-bf16-d32-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,64,1,128,false>,b200k::WithLse<b200k::AttnDecode<b200k::AttnCfg<1,64,1,128,false>>>>": "decode-bf16-d64-lse-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,64,1,128,false>,b200k::Fp8Kv<b200k::AttnDecode<b200k::AttnCfg<1,64,1,128,false>>,5>>": "decode-bf16-e5m2-d32-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,64,1,128,false>,b200k::WithLse<b200k::Fp8Kv<b200k::AttnDecode<b200k::AttnCfg<1,64,1,128,false>>,5>>>": "decode-bf16-e5m2-d64-lse-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,64,1,128,false>,b200k::Fp8Kv<b200k::AttnDecode<b200k::AttnCfg<1,64,1,128,false>>,4>>": "decode-bf16-e4m3-d32-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<1,64,1,128,false>,b200k::WithLse<b200k::Fp8Kv<b200k::AttnDecode<b200k::AttnCfg<1,64,1,128,false>>,4>>>": "decode-bf16-e4m3-d64-lse-unsplit",
    "b200k::attn_combine_kernel<1,float,false>": "decode-bf16-d128-split",
    "b200k::attn_combine_kernel<1,float,true>": "decode-bf16-d64-lse-split",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,128,1,128,false>,b200k::AttnDecode<b200k::AttnCfg<0,128,1,128,false>>>": "decode-f16-d128-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,128,1,128,false>,b200k::WithLse<b200k::AttnDecode<b200k::AttnCfg<0,128,1,128,false>>>>": "decode-f16-d96-lse-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,128,1,128,false>,b200k::Fp8Kv<b200k::AttnDecode<b200k::AttnCfg<0,128,1,128,false>>,5>>": "decode-f16-e5m2-d128-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,128,1,128,false>,b200k::WithLse<b200k::Fp8Kv<b200k::AttnDecode<b200k::AttnCfg<0,128,1,128,false>>,5>>>": "decode-f16-e5m2-d96-lse-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,128,1,128,false>,b200k::Fp8Kv<b200k::AttnDecode<b200k::AttnCfg<0,128,1,128,false>>,4>>": "decode-f16-e4m3-d128-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,128,1,128,false>,b200k::WithLse<b200k::Fp8Kv<b200k::AttnDecode<b200k::AttnCfg<0,128,1,128,false>>,4>>>": "decode-f16-e4m3-d96-lse-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,64,1,128,false>,b200k::AttnDecode<b200k::AttnCfg<0,64,1,128,false>>>": "decode-f16-d32-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,64,1,128,false>,b200k::WithLse<b200k::AttnDecode<b200k::AttnCfg<0,64,1,128,false>>>>": "decode-f16-d64-lse-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,64,1,128,false>,b200k::Fp8Kv<b200k::AttnDecode<b200k::AttnCfg<0,64,1,128,false>>,5>>": "decode-f16-e5m2-d32-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,64,1,128,false>,b200k::WithLse<b200k::Fp8Kv<b200k::AttnDecode<b200k::AttnCfg<0,64,1,128,false>>,5>>>": "decode-f16-e5m2-d64-lse-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,64,1,128,false>,b200k::Fp8Kv<b200k::AttnDecode<b200k::AttnCfg<0,64,1,128,false>>,4>>": "decode-f16-e4m3-d32-unsplit",
    "b200k::attn_fwd_wgmma_kernel<b200k::AttnCfg<0,64,1,128,false>,b200k::WithLse<b200k::Fp8Kv<b200k::AttnDecode<b200k::AttnCfg<0,64,1,128,false>>,4>>>": "decode-f16-e4m3-d64-lse-unsplit",
    "b200k::attn_combine_kernel<0,float,false>": "decode-f16-d128-split",
    "b200k::attn_combine_kernel<0,float,true>": "decode-f16-d64-lse-split",
    "b200k::attn_combine_kernel<0,unsigned short,false>": "merge-f16",
    "b200k::attn_combine_kernel<0,unsigned short,true>": "merge-f16-lse",
    "b200k::attn_combine_kernel<1,unsigned short,false>": "merge-bf16",
    "b200k::attn_combine_kernel<1,unsigned short,true>": "merge-bf16-lse",
    "b200k::attn_bwd_dq_kernel<b200k::AttnCfg<0,128,2,64,false>,b200k::AttnPacked<b200k::AttnCfg<0,128,2,64,false>>>": "bwd-packed-f16-d96",
    "b200k::attn_bwd_dkdv_kernel<b200k::AttnCfg<0,128,1,64,false>,b200k::BwdKeysPacked<b200k::AttnCfg<0,128,1,64,false>>>": "bwd-packed-f16-d96",
    "b200k::attn_bwd_dq_kernel<b200k::AttnCfg<0,64,2,64,false>,b200k::AttnPacked<b200k::AttnCfg<0,64,2,64,false>>>": "bwd-packed-f16-d64",
    "b200k::attn_bwd_dkdv_kernel<b200k::AttnCfg<0,64,1,64,false>,b200k::BwdKeysPacked<b200k::AttnCfg<0,64,1,64,false>>>": "bwd-packed-f16-d64",
    "b200k::attn_bwd_prep_kernel<0,true>": "bwd-packed-f16-d64",
    "b200k::attn_bwd_dq_kernel<b200k::AttnCfg<1,128,2,64,false>,b200k::AttnPacked<b200k::AttnCfg<1,128,2,64,false>>>": "bwd-packed-bf16-d96",
    "b200k::attn_bwd_dkdv_kernel<b200k::AttnCfg<1,128,1,64,false>,b200k::BwdKeysPacked<b200k::AttnCfg<1,128,1,64,false>>>": "bwd-packed-bf16-d96",
    "b200k::attn_bwd_dq_kernel<b200k::AttnCfg<1,64,2,64,false>,b200k::AttnPacked<b200k::AttnCfg<1,64,2,64,false>>>": "bwd-packed-bf16-d64",
    "b200k::attn_bwd_dkdv_kernel<b200k::AttnCfg<1,64,1,64,false>,b200k::BwdKeysPacked<b200k::AttnCfg<1,64,1,64,false>>>": "bwd-packed-bf16-d64",
    "b200k::attn_bwd_prep_kernel<1,true>": "bwd-packed-bf16-d64",
    "b200k::attn_bwd_dq_kernel<b200k::AttnCfg<0,128,2,64,false>,b200k::AttnDense<b200k::AttnCfg<0,128,2,64,false>>>": "bwd-dense-f16-d96",
    "b200k::attn_bwd_dkdv_kernel<b200k::AttnCfg<0,128,1,64,false>,b200k::BwdKeysDense<b200k::AttnCfg<0,128,1,64,false>>>": "bwd-dense-f16-d96",
    "b200k::attn_bwd_dq_kernel<b200k::AttnCfg<0,64,2,64,false>,b200k::AttnDense<b200k::AttnCfg<0,64,2,64,false>>>": "bwd-dense-f16-d64",
    "b200k::attn_bwd_dkdv_kernel<b200k::AttnCfg<0,64,1,64,false>,b200k::BwdKeysDense<b200k::AttnCfg<0,64,1,64,false>>>": "bwd-dense-f16-d64",
    "b200k::attn_bwd_prep_kernel<0,false>": "bwd-dense-f16-d64",
    "b200k::attn_bwd_dq_kernel<b200k::AttnCfg<1,128,2,64,false>,b200k::AttnDense<b200k::AttnCfg<1,128,2,64,false>>>": "bwd-dense-bf16-d96",
    "b200k::attn_bwd_dkdv_kernel<b200k::AttnCfg<1,128,1,64,false>,b200k::BwdKeysDense<b200k::AttnCfg<1,128,1,64,false>>>": "bwd-dense-bf16-d96",
    "b200k::attn_bwd_dq_kernel<b200k::AttnCfg<1,64,2,64,false>,b200k::AttnDense<b200k::AttnCfg<1,64,2,64,false>>>": "bwd-dense-bf16-d64",
    "b200k::attn_bwd_dkdv_kernel<b200k::AttnCfg<1,64,1,64,false>,b200k::BwdKeysDense<b200k::AttnCfg<1,64,1,64,false>>>": "bwd-dense-bf16-d64",
    "b200k::attn_bwd_prep_kernel<1,false>": "bwd-dense-bf16-d64",
    "b200k::row_kernel_scalar<__half,4>": "layernorm-f16-h1001",
    "b200k::row_kernel<__half,256,4>": "layernorm-f16-h6144",
    "b200k::row_kernel<__half,128,4>": "layernorm-f16-h4096",
    "b200k::row_kernel<__half,32,4>": "layernorm-f16-h1000",
    "b200k::row_kernel_scalar<float,4>": "layernorm-f32-h1001",
    "b200k::row_kernel<float,256,4>": "layernorm-f32-h6144",
    "b200k::row_kernel<float,128,4>": "layernorm-f32-h4096",
    "b200k::row_kernel<float,32,4>": "layernorm-f32-h1000",
    "b200k::row_kernel_scalar<__half,2>": "rmsnorm-f16-h1001",
    "b200k::row_kernel<__half,256,2>": "rmsnorm-f16-h6144",
    "b200k::row_kernel<__half,128,2>": "rmsnorm-f16-h4096",
    "b200k::row_kernel<__half,32,2>": "rmsnorm-f16-h1000",
    "b200k::row_kernel_scalar<__half,3>": "rmsnorm-f16-acc16-h1001",
    "b200k::row_kernel<__half,256,3>": "rmsnorm-f16-acc16-h6144",
    "b200k::row_kernel<__half,128,3>": "rmsnorm-f16-acc16-h4096",
    "b200k::row_kernel<__half,32,3>": "rmsnorm-f16-acc16-h1000",
    "b200k::row_kernel_scalar<float,2>": "rmsnorm-f32-h1001",
    "b200k::row_kernel<float,256,2>": "rmsnorm-f32-h6144",
    "b200k::row_kernel<float,128,2>": "rmsnorm-f32-h4096",
    "b200k::row_kernel<float,32,2>": "rmsnorm-f32-h1000",
    "b200k::row_kernel_scalar<__half,1>": "softmax-f16-m2-h1001",
    "b200k::row_kernel<__half,256,1>": "softmax-f16-m2-h6144",
    "b200k::row_kernel<__half,128,1>": "softmax-f16-m2-h4096",
    "b200k::row_kernel<__half,32,1>": "softmax-f16-m2-h1000",
    "b200k::row_kernel_scalar<__half,0>": "softmax-f16-m1-h1001",
    "b200k::row_kernel<__half,256,0>": "softmax-f16-m1-h6144",
    "b200k::row_kernel<__half,128,0>": "softmax-f16-m1-h4096",
    "b200k::row_kernel<__half,32,0>": "softmax-f16-m1-h1000",
    "b200k::row_kernel_scalar<float,1>": "softmax-f32-m2-h1001",
    "b200k::row_kernel<float,256,1>": "softmax-f32-m2-h6144",
    "b200k::row_kernel<float,128,1>": "softmax-f32-m2-h4096",
    "b200k::row_kernel<float,32,1>": "softmax-f32-m2-h1000",
    "b200k::row_kernel_scalar<float,0>": "softmax-f32-m1-h1001",
    "b200k::row_kernel<float,256,0>": "softmax-f32-m1-h6144",
    "b200k::row_kernel<float,128,0>": "softmax-f32-m1-h4096",
    "b200k::row_kernel<float,32,0>": "softmax-f32-m0-h1000",
    "b200k::reduce_sum_kernel<0,false,true>": "softmax-f32-m0-h1000",
    "b200k::reduce_sum_kernel<3,false,false>": "reduce-i8",
    "b200k::reduce_sum_kernel<5,false,false>": "reduce-e5m2",
    "b200k::reduce_sum_kernel<5,true,false>": "reduce-e5m2-acc16",
    "b200k::reduce_sum_kernel<4,false,false>": "reduce-e4m3",
    "b200k::reduce_sum_kernel<4,true,false>": "reduce-e4m3-acc16",
    "b200k::reduce_sum_kernel<2,false,false>": "reduce-bf16",
    "b200k::reduce_sum_kernel<2,true,false>": "reduce-bf16-acc16",
    "b200k::reduce_sum_kernel<1,false,false>": "reduce-f16",
    "b200k::reduce_sum_kernel<1,true,false>": "reduce-f16-acc16",
    "b200k::reduce_sum_kernel<0,false,false>": "reduce-f32",
    "b200k::elementwise_add_scalar_kernel<__nv_bfloat16>": "add-bf16-scalar",
    "b200k::elementwise_add_vec_kernel<__nv_bfloat16>": "add-bf16-vec",
    "b200k::elementwise_add_scalar_kernel<__half>": "add-f16-scalar",
    "b200k::elementwise_add_vec_kernel<__half>": "add-f16-vec",
    "b200k::elementwise_add_scalar_kernel<float>": "add-f32-scalar",
    "b200k::elementwise_add_vec_kernel<float>": "add-f32-vec",
    "b200k::histogram_i32_kernel<false>": "hist-global",
    "b200k::histogram_i32_kernel<true>": "hist-auto",
    "b200k::embedding_kernel": "embedding",
    "b200k::max_i32_kernel": "hist-auto",
    "b200k::init_i32_kernel": "hist-auto",
    "b200k::rope_f32_kernel": "rope",
    "b200k::dot_kernel<__half>": "dot-f16",
    "b200k::dot_kernel<float>": "dot-f32",
    "b200k::activation_kernel<__half,6,false>": "act-f16-hardshrink",
    "b200k::activation_kernel<__half,5,false>": "act-f16-hardswish",
    "b200k::activation_kernel<__half,4,false>": "act-f16-elu",
    "b200k::activation_kernel<__half,3,false>": "act-f16-swish",
    "b200k::activation_kernel<__half,2,true>": "act-f16-gelu-clamp",
    "b200k::activation_kernel<__half,2,false>": "act-f16-gelu",
    "b200k::activation_kernel<__half,1,true>": "act-f16-sigmoid-clamp",
    "b200k::activation_kernel<__half,1,false>": "act-f16-sigmoid",
    "b200k::activation_kernel<__half,0,false>": "act-f16-relu",
    "b200k::activation_kernel<float,6,false>": "act-f32-hardshrink",
    "b200k::activation_kernel<float,5,false>": "act-f32-hardswish",
    "b200k::activation_kernel<float,4,false>": "act-f32-elu",
    "b200k::activation_kernel<float,3,false>": "act-f32-swish",
    "b200k::activation_kernel<float,2,true>": "act-f32-gelu-clamp",
    "b200k::activation_kernel<float,2,false>": "act-f32-gelu",
    "b200k::activation_kernel<float,1,false>": "act-f32-sigmoid",
    "b200k::activation_kernel<float,0,false>": "act-f32-relu",
    "b200k::gemv_kernel<__half>": "gemv-f16",
    "b200k::gemv_kernel<float>": "gemv-f32",
    "b200k::transpose_kernel<unsigned short>": "transpose-u16",
    "b200k::transpose_kernel<float>": "transpose-f32",
    "b200k::transpose_f32x4_kernel": "transpose-f32x4",
}
