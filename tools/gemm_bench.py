"""Time every distinct GEMM shape of one inversion step (UNet batch 1) and one PnP edit step (batch 3) of the bench workload
(16 frames of 64 x 64 latents) against other builds of the library, alternated in one process.

    python tools/gemm_bench.py --other path/to/libanyv2v_b200.so [--other ...] [--iters 20] [--rounds 5]

Each round times every shape with CUDA events on this build and then on each other build; the report gives, per shape, the
median over rounds of the mean time per call, the achieved TFLOP/s and GB/s (operations and the least HBM bytes of the
GEMM: A, W, the output and the residual once each), and the share of the shape's bound: max(FLOPs / 989 TFLOP/s,
bytes / 3.35 TB/s), the H100 SXM data-sheet rates, with the bound named.  The card name, power limit and SM clock are
printed with the numbers.  Before timing, every shape's output is compared with torch.equal against each other build's on
the same inputs: a change of kernel that keeps the arithmetic must keep every bit."""
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

PEAK_TFLOPS, PEAK_GBS = 989.0, 3350.0
F = 16


def _w(n, k, dev):
    return (torch.randn(n, k, device=dev) * k ** -0.5).half()


def _cases(dev):
    """name -> (fn, flops, bytes)"""
    torch.manual_seed(0)
    cases = {}
    for B in (1, 3):  # inversion step, edit step
        for lvl, (hw, C) in enumerate(((64, 320), (32, 640), (16, 1280))):
            M = B * F * hw * hw
            x = torch.randn(M, C, device=dev).half()
            res = torch.randn(M, C, device=dev).half()
            out = torch.empty(M, C, device=dev).half()
            bias = (torch.randn(C, device=dev) * 0.1).half()
            # GEGLU feed-forward (C -> 2 x 4C, h * gelu(gate))
            wp, bp = ops.geglu_pack(_w(8 * C, C, dev), (torch.randn(8 * C, device=dev) * 0.1).half())
            gout = torch.empty(M, 4 * C, device=dev).half()
            cases[f"geglu {M}x{8 * C}x{C}"] = (lambda x=x, wp=wp, bp=bp, o=gout: ops.linear(x, wp, bias=bp, out=o, geglu=True),
                                              2 * M * 8 * C * C, 2 * (M * C + 8 * C * C + M * 4 * C))
            # linear + residual (attention out-projection, proj_out) and the FF down-projection (K = 4C)
            for K in (C, 4 * C):
                a = x if K == C else gout
                w = _w(C, K, dev)
                cases[f"linear+res {M}x{C}x{K}"] = (lambda a=a, w=w, b=bias, r=res, o=out: ops.linear(a, w, bias=b, residual=r, out=o),
                                                   2 * M * C * K, 2 * (M * K + C * K + 2 * M * C))
            # q | k | v projection
            wq = _w(3 * C, C, dev)
            qkv = torch.empty(M, 3 * C, device=dev).half()
            cases[f"linear {M}x{3 * C}x{C}"] = (lambda x=x, w=wq, o=qkv: ops.linear(x, w, out=o),
                                              2 * M * 3 * C * C, 2 * (M * C + 3 * C * C + M * 3 * C))
            # temporal conv (3, 1, 1)
            wt = _w(C, 3 * C, dev)
            x3 = x.view(B, F * hw * hw, C)
            cases[f"tconv3 {M}x{C}x{3 * C}"] = (lambda x3=x3, w=wt, b=bias, o=out, hw=hw: ops.tconv3(x3, w, F, hw * hw, bias=b, out=o.view(x3.shape)),
                                               2 * M * C * 3 * C, 2 * (M * C + 3 * C * C + M * C))
            # 3 x 3 conv + residual (resnet conv2) and 3 x 3 conv of the concatenated skip (2C in)
            xi = x.view(B * F, hw, hw, C)
            wc = _w(C, 9 * C, dev)
            cases[f"conv3x3+res {M}x{C}x{9 * C}"] = (lambda xi=xi, w=wc, b=bias, r=res, o=out: ops.conv3x3(xi, w, bias=b, residual=r, out=o),
                                                    2 * M * C * 9 * C, 2 * (M * C + 9 * C * C + 2 * M * C))
            # linear + bias + a per-frame rowbias (the time-embedding epilogue of a resnet's conv1, on a short K loop)
            tproj = (torch.randn(B * F, C, device=dev) * 0.5).half()
            wl = _w(C, C, dev)
            cases[f"linear+rowbias {M}x{C}x{C}"] = (lambda x=x, w=wl, b=bias, t=tproj, o=out, r=hw * hw: ops.linear(x, w, bias=b, rowbias=t, rows_per_rowbias=r, out=o),
                                                   2 * M * C * C, 2 * (M * C + C * C + B * F * C + M * C))
            if B == 3 and lvl == 2:
                # conv injection of the edit step: conv2 of the source clip, its tile stored to the 3 branch slots, each + its shortcut
                Ms = F * hw * hw
                cases[f"conv3x3+res 3 slots {Ms}x{C}x{9 * C}"] = (
                    lambda xi=xi[:F], w=wc, b=bias, r=res, o=out, s=Ms * C: ops.conv3x3(xi, w, bias=b, residual=r.view(3, -1, r.shape[1]), out=o.view(3, -1, o.shape[1]), n_slots=3, slot_stride=s),
                    2 * Ms * C * 9 * C, 2 * (Ms * C + 9 * C * C + 2 * 3 * Ms * C))
            # resnet conv1: 3 x 3 conv + bias + the per-frame time embedding (rowbias), no residual
            cases[f"conv3x3+rowbias {M}x{C}x{9 * C}"] = (lambda xi=xi, w=wc, b=bias, t=tproj, o=out, r=hw * hw: ops.conv3x3(xi, w, bias=b, rowbias=t, rows_per_rowbias=r, out=o),
                                                        2 * M * C * 9 * C, 2 * (M * C + 9 * C * C + B * F * C + M * C))
            if lvl == 0:
                x2 =torch.randn(B * F, hw, hw, 2 * C, device=dev).half()
                wc2 = _w(C, 18 * C, dev)
                cases[f"conv3x3 {M}x{C}x{18 * C}"] = (lambda xi=x2, w=wc2, b=bias, o=out: ops.conv3x3(xi, w, bias=b, out=o),
                                                     2 * M * C * 18 * C, 2 * (M * 2 * C + 18 * C * C + M * C))
        # the 8 x 8 level (mid block and down block 3): two frames per 128-row tile
        hw, C = 8, 1280
        M = B * F * hw * hw
        x8 = torch.randn(B * F, hw, hw, C, device=dev).half()
        r8 = torch.randn(M, C, device=dev).half()
        o8 = torch.empty(M, C, device=dev).half()
        b8 = (torch.randn(C, device=dev) * 0.1).half()
        wc8, wt8 = _w(C, 9 * C, dev), _w(C, 3 * C, dev)
        cases[f"conv3x3+res {M}x{C}x{9 * C}"] = (lambda xi=x8, w=wc8, b=b8, r=r8, o=o8: ops.conv3x3(xi, w, bias=b, residual=r, out=o),
                                                2 * M * C * 9 * C, 2 * (M * C + 9 * C * C + 2 * M * C))
        cases[f"tconv3 {M}x{C}x{3 * C}"] = (lambda x3=x8.view(B, F * hw * hw, C), w=wt8, b=b8, o=o8, hw=hw: ops.tconv3(x3, w, F, hw * hw, bias=b, out=o.view(x3.shape)),
                                           2 * M * C * 3 * C, 2 * (M * C + 3 * C * C + M * C))
        # up-sampling (nearest x 2 + 3 x 3 conv as four phase GEMMs, K = 4 Cin) into levels 1 and 0's resolutions
        for hw, C in ((8, 1280), (16, 1280), (32, 640)):
            Ml = B * F * hw * hw
            xl = torch.randn(B * F, hw, hw, C, device=dev).half()
            wph = torch.stack([_w(C, 4 * C, dev) for _ in range(4)])
            ob = torch.empty(B * F, 2 * hw, 2 * hw, C, device=dev).half()
            cases[f"upsample 4x{Ml}x{C}x{4 * C}"] = (lambda xl=xl, w=wph, o=ob: ops.upsample2x_conv3x3(xl, w, out=o),
                                                    4 * 2 * Ml * C * 4 * C, 2 * (Ml * C + 16 * C * C + 4 * Ml * C))
    return cases


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", action="append", required=True, help="another build of libanyv2v_b200.so (repeatable)")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gemm_bench: no CUDA device")
    libs = {"this": _lib.lib()}
    for path in args.other:
        libs[path] = _load(os.path.abspath(path))
    cases = _cases("cuda")
    times = {(lib, c): [] for lib in libs for c in cases}
    for lib in libs.values():  # warm-up: module load, first launches
        _lib._lib = lib
        for fn, _, _ in cases.values():
            fn()
    torch.cuda.synchronize()
    equal = {}
    for c, (fn, _, _) in cases.items():
        outs = {}
        for name, lib in libs.items():
            _lib._lib = lib
            outs[name] = fn().clone()
        equal[c] = all(torch.equal(outs["this"], o) for o in outs.values())
    for _ in range(args.rounds):
        for c, (fn, _, _) in cases.items():
            for name, lib in libs.items():
                _lib._lib = lib
                times[(name, c)].append(_time(fn, args.iters))
    _lib._lib = libs["this"]
    print("card (name, power limit, max SM clock):", _card())
    rows = []
    total = {name: 0.0 for name in libs}
    for c, (_, flops, nbytes) in cases.items():
        bound_us = max(flops / (PEAK_TFLOPS * 1e6), nbytes / (PEAK_GBS * 1e3))
        which = "tensor" if flops / (PEAK_TFLOPS * 1e6) >= nbytes / (PEAK_GBS * 1e3) else "HBM"
        row = dict(case=c, gflop=round(flops / 1e9, 1), bound=which, equal=equal[c])
        line = f"{c:32s}"
        for name in libs:
            t = statistics.median(times[(name, c)])
            total[name] += t
            tag = "this" if name == "this" else os.path.basename(os.path.dirname(os.path.abspath(name))) or name
            row[tag] = dict(us=round(t, 2), tflops=round(flops / t / 1e6, 1), gbs=round(nbytes / t / 1e3, 1),
                            of_bound=round(bound_us / t, 3))
            line += f" | {tag} {t:9.2f} us {flops / t / 1e6:6.1f} TF/s {nbytes / t / 1e3:7.1f} GB/s {bound_us / t:6.1%} of {which}"
        rows.append(row)
        print(line + ("" if equal[c] else " | OUTPUT DIFFERS"))
    print("sum over shapes (one call each):", ", ".join(f"{n if n == 'this' else os.path.basename(os.path.dirname(os.path.abspath(n)))} {t:.1f} us"
                                                   for n, t in total.items()))
    linear = [c for c in cases if c.split()[0] in ("linear", "linear+res", "linear+rowbias", "geglu")]
    print("sum over the linear-mode shapes:", ", ".join(f"{n if n == 'this' else os.path.basename(os.path.dirname(os.path.abspath(n)))} "
                                                        f"{sum(statistics.median(times[(n, c)]) for c in linear):.1f} us" for n in libs))
    conv = [c for c in cases if c not in linear]
    print("sum over the conv-mode shapes:", ", ".join(f"{n if n == 'this' else os.path.basename(os.path.dirname(os.path.abspath(n)))} "
                                                      f"{sum(statistics.median(times[(n, c)]) for c in conv):.1f} us" for n in libs))
    differ = [c for c in cases if not equal[c]]
    print("outputs torch.equal across builds:", "every shape" if not differ else f"NO, differ on {differ}")
    print(json.dumps(rows))


if __name__ == "__main__":
    main()
