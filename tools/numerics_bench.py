"""Time the two kernels whose arithmetic tests/test_gpu_numerics.py pins down — the GEGLU GEMM (erfc-based gelu epilogue) and
the persistent GroupNorm (shifted statistics) — against another build of the library, alternated in one process.

    python tools/numerics_bench.py --other path/to/libanyv2v_b200.so [--iters 50] [--rounds 5]

Both libraries are loaded with ctypes and driven through the same ``ops`` wrappers (the wrapper's library handle is swapped
between calls).  Each round times every shape with CUDA events, first on one build and then on the other; the report gives the
median over rounds of the mean time per call.  The card name and power limit are printed with the numbers."""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from anyv2v_b200 import _lib, ops  # noqa: E402


def _load(path):
    lib = ctypes.CDLL(path)
    for name, (res, args) in _lib.EXPORTS.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def _cases(dev):
    torch.manual_seed(0)
    M, N, K = 196608, 2560, 320  # GEGLU of an edit step: 3 clips x 16 frames x 64 x 64 tokens, FF 320 -> 2 x 1280
    a = torch.randn(M, K, device=dev).half()
    wp, bp = ops.geglu_pack((torch.randn(N, K, device=dev) * K ** -0.5).half(), (torch.randn(N, device=dev) * 0.1).half())
    geglu_out = torch.empty(M, N // 2, device=dev, dtype=torch.float16)
    cases = {f"geglu {M}x{N}x{K}": lambda: ops.linear(a, wp, bias=bp, out=geglu_out, geglu=True)}
    # GroupNorm(+SiLU) of an edit step: per-frame norms of the resnets at each level, the per-clip norm of the temporal blocks
    for n, rows, C, silu in ((48, 4096, 320, True), (48, 1024, 640, True), (48, 256, 1280, True), (48, 64, 1280, True),
                             (3, 65536, 320, False)):
        x = (torch.randn(n, rows, C, device=dev) + 3).half()
        gm, bt = torch.ones(C, device=dev).half(), torch.zeros(C, device=dev).half()
        y = torch.empty_like(x)
        cases[f"groupnorm {n}x{rows}x{C} silu={int(silu)}"] = (lambda x=x, gm=gm, bt=bt, y=y, silu=silu:
                                                                ops.groupnorm(x, gm, bt, 32, 1e-5, silu, out=y))
    return cases


def _time(fn, iters):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) * 1e3 / iters  # us per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", required=True, help="the other build of libanyv2v_b200.so")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("numerics_bench: no CUDA device")
    dev = "cuda"
    libs = {"this": _lib.lib(), "other": _load(os.path.abspath(args.other))}
    cases = _cases(dev)
    times = {(lib, c): [] for lib in libs for c in cases}
    for name, lib in libs.items():  # warm-up: module load, first launches
        _lib._lib = lib
        for fn in cases.values():
            fn()
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for c, fn in cases.items():
            for name, lib in libs.items():
                _lib._lib = lib
                times[(name, c)].append(_time(fn, args.iters))
    _lib._lib = libs["this"]
    print("card:", _card())
    rows = []
    for c in cases:
        t_this, t_other = statistics.median(times[("this", c)]), statistics.median(times[("other", c)])
        rows.append(dict(case=c, this_us=round(t_this, 2), other_us=round(t_other, 2), ratio=round(t_this / t_other, 4)))
        print(f"{c:40s} this {t_this:9.2f} us   other {t_other:9.2f} us   this/other {t_this / t_other:.4f}")
    print(json.dumps(rows))


if __name__ == "__main__":
    main()
