"""CPU: the alignment rule of every pointer of every attention entry point, checked before any CUDA call.

Each entry point is called with valid shapes and fake device addresses, 256-byte aligned and never dereferenced, then
one pointer at a time is moved 2, 4, 8 and 12 bytes.  Below its rule (Q, K, V, the caches, K_new, V_new, cos, sin, the
workspaces, O_parts and the merge's O: 16 bytes; a forward's O, lse and the int32 arrays: 4 bytes) the call must return
B200K_EALIGN and name the pointer; at or above it the call must get past validation, which on a machine without a GPU
means B200K_ECUDA or B200K_EARCH from the device query.  A null pointer the call cannot take is B200K_EARG.

On a machine with a GPU the accepted calls would launch kernels on the fake addresses, so this module runs only without
one; test_gpu_attention_align.py checks the same rules with real buffers."""
import ctypes

import pytest
import torch

from b200k import _loader as L

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="fake device addresses; needs a machine without a GPU")

PAST_VALIDATION = (L.ECUDA, L.EARCH)
OFFSETS = (2, 4, 8, 12)

DENSE = dict(Q=16, K=16, V=16, O=4)
DECODE = dict(Q=16, K_cache=16, V_cache=16, O=4, cache_seqlens=4, block_table=4)
APPEND = dict(DECODE, K_new=16, V_new=16, rotary_cos=16, rotary_sin=16, workspace=16)
SHAPE = [1, 1, 8]                                   # B, H, N of the dense calls
DEC = [1, 1, 2, 1, 64, 1, 128, 1, 0.0, L.F16, 0]    # B, Lq, H, H_kv, D, num_pages, page_size, pages_per_seq, scale,
#                                                     dtype, causal: a contiguous cache of 128 keys, or one page of 128


def _lse(spec):
    """The *_lse form of a call: lse right after O."""
    i = spec.index("O") + 1
    return spec[:i] + ["lse"] + spec[i:]


def _decode(workspace):
    return ["Q", "K_cache", "V_cache", "O", "cache_seqlens", "block_table"] + DEC + workspace


_APPEND = (["Q", "K_cache", "V_cache", "O", "cache_seqlens", "block_table", "K_new", "V_new", 1, "rotary_cos",
            "rotary_sin", 128, 64, 1] + DEC + ["workspace", 1 << 20, None])
_VARLEN = ["Q", "K", "V", "O", "cu_seqlens_q", "cu_seqlens_k", 1, 8, 8, 8, 2, 1, 64, 0.0, L.F16, 0, None]
_FA2 = ["Q", "K", "V", "O"] + SHAPE + [64, 0.0, 0, L.F16, 0, "seqlens_k", 0, None]

# (test id, symbol, arguments: a string names a pointer, anything else is passed as it is, {pointer: alignment},
#  pointers whose NULL gets past validation)
ENTRIES = [
    ("fa2_fwd_f16", "b200k_fa2_fwd_f16", ["Q", "K", "V", "O"] + SHAPE + [64, 0.0, 0, 0, None], DENSE, set()),
    ("fa2_fwd", "b200k_fa2_fwd", _FA2, dict(DENSE, seqlens_k=4), {"seqlens_k"}),
    ("fa2_fwd_lse", "b200k_fa2_fwd_lse", _lse(_FA2), dict(DENSE, seqlens_k=4, lse=4), {"seqlens_k", "lse"}),
    ("ffpa_fwd_f16_d256", "b200k_ffpa_fwd_f16", ["Q", "K", "V", "O"] + SHAPE + [256, 0.0, 0, None], DENSE, set()),
    ("ffpa_fwd_f16_d64", "b200k_ffpa_fwd_f16", ["Q", "K", "V", "O"] + SHAPE + [64, 0.0, 0, None], DENSE, set()),
    ("fa2_fwd_varlen", "b200k_fa2_fwd_varlen", _VARLEN, dict(DENSE, cu_seqlens_q=4, cu_seqlens_k=4), set()),
    ("fa2_fwd_varlen_lse", "b200k_fa2_fwd_varlen_lse", _lse(_VARLEN), dict(DENSE, cu_seqlens_q=4, cu_seqlens_k=4, lse=4),
     {"lse"}),
    # the workspace may be NULL when the call runs unsplit, which only the device query tells
    ("fa2_fwd_kvcache", "b200k_fa2_fwd_kvcache", _decode(["workspace", 1 << 20, None]), dict(DECODE, workspace=16),
     {"block_table", "workspace"}),
    ("fa2_fwd_kvcache_lse", "b200k_fa2_fwd_kvcache_lse", _lse(_decode(["workspace", 1 << 20, None])),
     dict(DECODE, workspace=16, lse=4), {"block_table", "workspace", "lse"}),
    # a NULL workspace is refused after the device query, with its size; cos and sin are NULL only together
    ("fa2_fwd_kvcache_append", "b200k_fa2_fwd_kvcache_append", _APPEND, APPEND, {"block_table", "workspace"}),
    ("fa2_fwd_kvcache_append_lse", "b200k_fa2_fwd_kvcache_append_lse", _lse(_APPEND), dict(APPEND, lse=4),
     {"block_table", "workspace", "lse"}),
    ("attn_merge", "b200k_attn_merge", ["O_parts", "lse_parts", "O", "lse", 2, 4, 64, L.F16, None],
     dict(O_parts=16, lse_parts=4, O=16, lse=4), {"lse"}),
]
BY_ID = {e[0]: e for e in ENTRIES}


def _call(entry, **moved):
    """Calls the entry point with pointer i at (i + 1) MiB, or at the address `moved` gives (None: NULL)."""
    _, sym, spec, rules, _ = entry
    names = [a for a in spec if isinstance(a, str)]
    assert sorted(names) == sorted(rules), entry[0]
    addr = {n: (i + 1) << 20 for i, n in enumerate(names)}
    for n, off in moved.items():
        addr[n] = None if off is None else addr[n] + off
    args = [ctypes.c_void_p(addr[a]) if isinstance(a, str) and addr[a] is not None else (None if isinstance(a, str) else a)
            for a in spec]
    return getattr(L.lib, sym)(*args)


def test_every_pointer_of_every_entry_point_is_in_the_table():
    """The table covers the 10 forward entry points and the merge, with every pointer argument of each."""
    syms = {e[1] for e in ENTRIES}
    assert syms == {s for s in L.declared_symbols() if s.startswith(("b200k_fa2_fwd", "b200k_ffpa_fwd", "b200k_attn_merge"))
                    and not s.endswith("_workspace_bytes")}
    for e in ENTRIES:
        assert len(e[2]) == len(L._SIGS[e[1]][1]), e[0]
        assert sum(t is ctypes.c_void_p for t in L._SIGS[e[1]][1]) == len(e[3]) + 1, e[0]   # + the stream


@pytest.mark.parametrize("eid", [e[0] for e in ENTRIES])
def test_aligned_call_gets_past_validation(eid):
    assert _call(BY_ID[eid]) in PAST_VALIDATION, L.last_error()


ROWS = [(e[0], name, off) for e in ENTRIES for name in e[3] for off in OFFSETS]


@pytest.mark.parametrize("eid,name,offset", ROWS, ids=["%s-%s-%d" % r for r in ROWS])
def test_pointer_below_its_alignment_is_refused_before_cuda(eid, name, offset):
    entry = BY_ID[eid]
    need = entry[3][name]
    rc = _call(entry, **{name: offset})
    if offset % need:
        assert rc == L.EALIGN, (rc, L.last_error())
        assert ": %s must be %d-byte aligned" % (name, need) in L.last_error()
    else:
        assert rc in PAST_VALIDATION, (rc, L.last_error())


NULLS = [(e[0], name) for e in ENTRIES for name in e[3]]


@pytest.mark.parametrize("eid,name", NULLS, ids=["%s-%s" % r for r in NULLS])
def test_null_pointer(eid, name):
    entry = BY_ID[eid]
    rc = _call(entry, **{name: None})
    if name in entry[4]:
        assert rc in PAST_VALIDATION, (rc, L.last_error())
    else:
        assert rc == L.EARG, (rc, L.last_error())
