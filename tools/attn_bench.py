"""Time every rows-mode attention shape of one inversion step (batch 16: one clip of 16 frames) and one PnP edit step (batch
48; the injected sites at n_v = 3 over the 16 source sequences) of the bench workload against other builds of the library,
alternated in one process.

    python tools/attn_bench.py --other path/to/libanyv2v_b200.so [--other ...] [--iters 20] [--rounds 5]

Each round times every shape with CUDA events on this build and then on each other build; the report gives, per shape, the
median over rounds of the mean time per call and the achieved TFLOP/s over the FLOPs the kernel needs: 4 * rows * keys * 64
per head for QK^T and PV, with PV counted once per V branch at n_v = 3 (as bench.attention_roofline counts it), and the share
of the H100 SXM data-sheet 989 TFLOP/s.  The card name, power limit and SM clock are printed with the numbers."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from anyv2v_b200 import _lib, ops  # noqa: E402
from tools.numerics_bench import _card, _load, _time  # noqa: E402

PEAK_TFLOPS = 989.0
LEVELS = ((4096, 5), (1024, 10), (256, 20), (64, 20))  # (tokens per frame, heads) of the UNet's spatial transformers
N_CTX = 145  # text + image context tokens of the cross-attention


def _cases(dev):
    """name -> (fn, flops)"""
    torch.manual_seed(0)
    cases = {}
    for step, B in (("inv", 16), ("edit", 48)):
        for seq, heads in LEVELS:
            C = heads * 64
            q = torch.randn(B * seq, C, device=dev).half()
            kv = torch.randn(B * seq, 2 * C, device=dev).half()
            o = torch.empty(3 * B * seq, C, device=dev).half()
            cases[f"{step} self   {seq:4d}x{heads:2d} b{B} nv1"] = (
                lambda q=q, kv=kv, o=o, h=heads, s=seq, b=B, C=C: ops.attention(q, kv[:, :C], kv[:, C:], h, s, b, o[:b * s]),
                4 * B * heads * seq * seq * 64)
            if step == "edit":  # injected: Q / K of the 16 source sequences, V of all three branches
                S = B // 3
                cases[f"{step} inject {seq:4d}x{heads:2d} b{S} nv3"] = (
                    lambda q=q, kv=kv, o=o, h=heads, s=seq, S=S, C=C: ops.attention(
                        q[:S * s], kv[:S * s, :C], kv[:, C:], h, s, S, o, n_v=3, v_branch_stride=S * s * 2 * C,
                        o_branch_stride=S * s * C),
                    2 * (1 + 3) * S * heads * seq * seq * 64)
            ctx = torch.randn(B // 16 * N_CTX, 2 * C, device=dev).half()
            cases[f"{step} cross  {seq:4d}x{heads:2d} b{B} kv{N_CTX}"] = (
                lambda q=q, ctx=ctx, o=o, h=heads, s=seq, b=B, C=C: ops.attention(
                    q, ctx[:, :C], ctx[:, C:], h, s, b, o[:b * s], seq_kv=N_CTX, kv_batch_div=16),
                4 * B * heads * seq * N_CTX * 64)
    return cases


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", action="append", required=True, help="another build of libanyv2v_b200.so (repeatable)")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attn_bench: no CUDA device")
    libs = {"this": _lib.lib()}
    for path in args.other:
        libs[path] = _load(os.path.abspath(path))
    cases = _cases("cuda")
    times = {(lib, c): [] for lib in libs for c in cases}
    for lib in libs.values():  # warm-up: module load, first launches
        _lib._lib = lib
        for fn, _ in cases.values():
            fn()
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for c, (fn, _) in cases.items():
            for name, lib in libs.items():
                _lib._lib = lib
                times[(name, c)].append(_time(fn, args.iters))
    _lib._lib = libs["this"]
    print("card (name, power limit, max SM clock):", _card())
    tag = lambda n: n if n == "this" else os.path.basename(os.path.dirname(os.path.abspath(n))) or n
    rows = []
    total = {name: 0.0 for name in libs}
    for c, (_, flops) in cases.items():
        row = dict(case=c, gflop=round(flops / 1e9, 2))
        line = f"{c:34s}"
        for name in libs:
            t = statistics.median(times[(name, c)])
            total[name] += t
            row[tag(name)] = dict(us=round(t, 2), tflops=round(flops / t / 1e6, 1))
            line += f" | {tag(name)} {t:9.2f} us {flops / t / 1e6:6.1f} TF/s {flops / t / 1e6 / PEAK_TFLOPS:6.1%} of peak"
        rows.append(row)
        print(line)
    print("sum over shapes (one call each):", ", ".join(f"{tag(n)} {t:.1f} us" for n, t in total.items()))
    print(json.dumps(rows))


if __name__ == "__main__":
    main()
