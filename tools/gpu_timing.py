"""What every GPU script under tools/ measures with: the card's description, CUDA-event timing of calls that take turns
(eagerly or as CUDA graphs), the attention work count, and the A/B of two builds of the library in one process.

Times are seconds per call; each script converts them to its own unit.  Importing this module puts the package
directory on sys.path, so a script imports b200k next.
"""
import contextlib
import ctypes
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cuda-learn-notes_b200"))
BASE_DIR = os.path.join(ROOT, "build_ab", "base")
BASE_LIB = os.path.join(BASE_DIR, "cuda-learn-notes_b200", "b200k", "libb200k.so")


def gpu_info(torch):
    """Name, power limit and maximum SM clock of the current GPU (read-only nvidia-smi query).  Exits when there is
    no CUDA device: a timing taken without one says nothing about the GPU."""
    if not torch.cuda.is_available():
        sys.exit("%s needs a CUDA device" % os.path.basename(sys.argv[0]))
    info = {"gpu": torch.cuda.get_device_name(), "power_limit_w": None, "max_sm_mhz": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, power, mhz = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        info.update(gpu=name, power_limit_w=float(power), max_sm_mhz=float(mhz))
    except Exception as e:  # the name from torch stays; the missing fields are reported as such
        info["nvidia_smi_error"] = str(e)[:200]
    return info


def capture(fn, iters):
    """A CUDA graph of `iters` calls of fn, after one warm-up call on the current stream and one on a side stream
    (tensor maps, shared-memory attributes and backend choices are set up outside the capture)."""
    import torch

    fn()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    return g


def time_rounds(fns, iters, rounds, graph=False, swap=False):
    """{name: [seconds per call, one per round]} for the functions of `fns`.  Each function (or its graph) runs once to
    warm up; then in every round the functions take turns, each timed with CUDA events over `iters` calls, or over one
    replay of a graph of `iters` calls when `graph`.  `swap` reverses the order every other round."""
    import torch

    if graph:
        fns = {name: capture(fn, iters).replay for name, fn in fns.items()}
    calls = 1 if graph else iters
    for fn in fns.values():
        fn()
    torch.cuda.synchronize()
    names = list(fns)
    times = {name: [] for name in names}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for r in range(rounds):
        for name in (names[::-1] if swap and r % 2 else names):
            e0.record()
            for _ in range(calls):
                fns[name]()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) * 1e-3 / iters)
    return times


def stats(samples):
    """(median, min, max) of a list of samples."""
    return statistics.median(samples), min(samples), max(samples)


def visible_pairs(lq, lk, causal):
    """(query row, key) pairs the attention computes: Lq * Lk, or with the bottom-right causal mask
    sum over rows r of clamp(r + Lk - Lq + 1, 0, Lk)."""
    if not causal:
        return int(lq) * int(lk)
    r = np.arange(int(lq), dtype=np.int64)
    return int(np.clip(r + int(lk) - int(lq) + 1, 0, int(lk)).sum())


def build_base(rev):
    """The whole tree at `rev` into build_ab/base (git-ignored), then its library with its own Makefile."""
    if os.path.isdir(BASE_DIR):
        subprocess.run(["rm", "-rf", BASE_DIR], check=True)
    os.makedirs(BASE_DIR)
    archive = subprocess.run(["git", "-C", ROOT, "archive", rev], capture_output=True, check=True).stdout
    subprocess.run(["tar", "-x", "-C", BASE_DIR], input=archive, check=True)
    subprocess.run(["make", "-C", os.path.join(BASE_DIR, "cuda-learn-notes_b200", "csrc"), "-j", str(os.cpu_count() or 4)],
                   check=True, stdout=subprocess.DEVNULL)
    print("built %s at %s" % (BASE_LIB, subprocess.run(["git", "-C", ROOT, "rev-parse", rev], capture_output=True,
                                                      text=True, check=True).stdout.strip()))


def load_lib(path):
    """Another build's libb200k.so through ctypes, with the signatures of b200k._loader."""
    from b200k import _loader

    lib = ctypes.CDLL(os.path.abspath(path))
    for name, (res, argtypes) in _loader._SIGS.items():
        if not hasattr(lib, name):  # an entry point the other build predates; no case here calls it
            continue
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = argtypes
    return lib


@contextlib.contextmanager
def using(lib):
    """b200k.ops calls `lib` inside the block."""
    from b200k import ops

    saved = ops._lib
    ops._lib = lib
    try:
        yield
    finally:
        ops._lib = saved


def same_bits(a, b):
    """Same dtype, shape and bytes: a NaN or a -0 counts like any other value."""
    import torch

    raw = [t.contiguous().reshape(-1).view(torch.uint8) for t in (a, b)]
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(*raw)


def compare_and_time(torch, libs, cases, timed, rounds, unit=("tflops", 1e-12), graph=True):
    """Runs each (name, run) of `cases` through libs["base"] and libs["new"] and prints the ones whose outputs differ
    in any bit, then times each (name, work, fn) of `timed` (a rate in `unit` = (name, scale) is work / time * scale):
    one CUDA graph per build (or, with graph=False, eager calls, host cost included), sized to about 100 ms, the
    builds alternating and swapping order every other round.
    Returns (differing cases, timed cases whose new median lies above the base's maximum)."""
    bad = 0
    for name, run in cases:
        outs = {}
        for key, lib in libs.items():
            with using(lib):
                outs[key] = run()
        same = len(outs["base"]) == len(outs["new"]) and all(same_bits(a, b) for a, b in zip(outs["base"], outs["new"]))
        bad += not same
        if not same:
            print(json.dumps({"case": name, "bit_equal": False}), flush=True)
    if cases:
        print(json.dumps({"equal_cases": len(cases), "differing": bad}), flush=True)

    def on(lib, fn):
        def run():
            with using(lib):
                fn()
        return run

    slow = 0
    for name, work, fn in timed:
        with using(libs["base"]):  # about 100 ms of work per build per round
            per_call = time_rounds({"base": fn}, 3, 1)["base"][0]
        iters = max(3, min(2000, int(0.1 / per_call)))
        times = time_rounds({key: on(lib, fn) for key, lib in libs.items()}, iters, rounds, graph=graph, swap=True)
        us = {k: [s * 1e6 for s in stats(v)] for k, v in times.items()}  # median, min, max
        line = {"case": name, "iters_per_round": iters}
        for k, (med, lo, hi) in us.items():
            line[k + "_us"] = round(med, 2)
            line[k + "_min_max_us"] = [round(lo, 2), round(hi, 2)]
            line[k + "_" + unit[0]] = round(work / (med * 1e-6) * unit[1], 1)
        slow += us["new"][0] > us["base"][2]
        line["new_over_base"] = round(us["new"][0] / us["base"][0], 4)
        line["new_median_inside_base_range"] = us["base"][1] <= us["new"][0] <= us["base"][2]
        print(json.dumps(line), flush=True)
        torch.cuda.empty_cache()
    return bad, slow
