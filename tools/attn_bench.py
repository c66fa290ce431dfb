"""Time every rows-mode attention shape of one inversion step (batch 16: one clip of 16 frames) and one PnP edit step (batch
48; the injected sites at n_v = 3 over the 16 source sequences) of the bench workload against other builds of the library,
alternated in one process.

    python tools/attn_bench.py [--other path/to/libanyv2v_b200.so ...] [--frames F ...] [--iters 20] [--rounds 5]

Each round times every shape with CUDA events on this build and then on each other build; the report gives, per shape, the
median over rounds of the mean time per call and the achieved TFLOP/s over the FLOPs the kernel needs: 4 * rows * keys * 64
per head for QK^T and PV, with PV counted once per V branch at n_v = 3 (as bench.attention_roofline counts it), and the share
of the H100 SXM data-sheet 989 TFLOP/s.  The card name, power limit and SM clock are printed with the numbers.

--frames adds the fused temporal self-attention (av2v_tattn_fused_f16) for each frame count F at every shape the UNet runs it
at: the 64 x 64, 32 x 32, 16 x 16 and 8 x 8 levels (HW 4096 / 1024 / 256 / 64, Cx 320 / 640 / 1280 / 1280, 5 / 10 / 20 / 20
heads) and transformer_in (HW 4096, Cx 320, 8 heads), at n_v = 1 (one clip) and n_v = 3 (three clips, Q / K from the source).
Beside each, the unfused control times the same computation as the UNet's other path does it: ops.linear for Q|K|V (Q|K of
the source clip and V of all three at n_v = 3) and the frames-mode ops.attention.  Their FLOPs count only the slots that
hold a frame, not the empty tail of a CTA's 128 slots: the projections (2 * Cx * 64 per head and row, for Q and K of the
source rows and V of every row) plus QK^T and PV over the F frames of each pixel.  The fused kernel's x-read rate (bytes of x
over the call time) is printed: a kernel that reads x from HBM once per call is bounded by it at 3.35 TB/s.

The outputs of every build are compared with this build's (torch.equal) for the rows-mode cases (attn_rows_kernel at 512 keys
or more, attn_kernel below) and the fused ones.  A build that rejects a case is reported as "unsupported"."""
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


FUSED_SHAPES = ((4096, 320, 5), (1024, 640, 10), (256, 1280, 20), (64, 1280, 20), (4096, 320, 8))  # (HW, Cx, heads)


def _fused_cases(dev, frames):
    """name -> (fn, flops, out, x bytes) of the fused temporal attention (out: its output) and of the unfused control"""
    cases = {}
    for F in frames:
        for HW, Cx, heads in FUSED_SHAPES:
            C = heads * 64
            for nv in (1, 3):
                g = torch.Generator(device=dev).manual_seed(F * 1000 + HW + heads + nv)
                rows = nv * F * HW
                x = torch.randn(rows, Cx, device=dev, generator=g).half()
                w = (torch.randn(3 * C, Cx, device=dev, generator=g) * Cx ** -0.5).half()
                o = torch.empty(rows, C, device=dev).half()
                src = F * HW  # rows of the source clip (the only clip at n_v = 1)
                flops = 2 * Cx * C * (2 * src + rows) + 2 * (1 + nv) * HW * heads * F * F * 64
                tag = f"F={F:3d} {HW}x{Cx}x{heads} nv{nv}"
                cases[f"fused   {tag}"] = (
                    lambda x=x, w=w, o=o, F=F, HW=HW, nv=nv, h=heads: ops.temporal_attention_fused(x, w, h, F, HW, nv, o, n_v=nv),
                    flops, o, x.numel() * 2)
                if nv == 1:
                    qkv = torch.empty(rows, 3 * C, device=dev).half()
                    fn = lambda x=x, w=w, o=o, qkv=qkv, F=F, HW=HW, h=heads, C=C: ops.attention(
                        *ops.linear(x, w, out=qkv).split(C, 1), h, F, HW, o, frames_mode=True, HW=HW)
                else:
                    qk, v = torch.empty(src, 2 * C, device=dev).half(), torch.empty(rows, C, device=dev).half()

                    def fn(x=x, w=w, o=o, qk=qk, v=v, F=F, HW=HW, h=heads, C=C, src=src):
                        ops.linear(x[:src], w[:2 * C], out=qk)
                        ops.linear(x, w[2 * C:], out=v)
                        ops.attention(qk[:, :C], qk[:, C:], v, h, F, HW, o, n_v=3, v_branch_stride=src * C,
                                      o_branch_stride=src * C, frames_mode=True, HW=HW)
                cases[f"unfused {tag}"] = (fn, flops, None, x.numel() * 2)
    return cases


def _cases(dev):
    """name -> (fn, flops, out, 0); out: the rows every case of a level writes, o[:B * seq] (n_v = 3: 3 branches of B / 3)"""
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
                4 * B * heads * seq * seq * 64, o[:B * seq], 0)
            if step == "edit":  # injected: Q / K of the 16 source sequences, V of all three branches
                S = B // 3
                cases[f"{step} inject {seq:4d}x{heads:2d} b{S} nv3"] = (
                    lambda q=q, kv=kv, o=o, h=heads, s=seq, S=S, C=C: ops.attention(
                        q[:S * s], kv[:S * s, :C], kv[:, C:], h, s, S, o, n_v=3, v_branch_stride=S * s * 2 * C,
                        o_branch_stride=S * s * C),
                    2 * (1 + 3) * S * heads * seq * seq * 64, o[:B * seq], 0)
            ctx = torch.randn(B // 16 * N_CTX, 2 * C, device=dev).half()
            cases[f"{step} cross  {seq:4d}x{heads:2d} b{B} kv{N_CTX}"] = (
                lambda q=q, ctx=ctx, o=o, h=heads, s=seq, b=B, C=C: ops.attention(
                    q, ctx[:, :C], ctx[:, C:], h, s, b, o[:b * s], seq_kv=N_CTX, kv_batch_div=16),
                4 * B * heads * seq * N_CTX * 64, o[:B * seq], 0)
    return cases


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", action="append", default=[], help="another build of libanyv2v_b200.so (repeatable)")
    ap.add_argument("--frames", type=int, nargs="*", default=[], help="frame counts of the fused temporal attention cases")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attn_bench: no CUDA device")
    libs = {"this": _lib.lib()}
    for path in args.other:
        libs[path] = _load(os.path.abspath(path))
    cases = {**_cases("cuda"), **_fused_cases("cuda", args.frames)}
    times = {(lib, c): [] for lib in libs for c in cases}
    unsupported = set()
    outs = {}
    for name, lib in libs.items():  # warm-up: module load, first launches; the outputs of each build
        _lib._lib = lib
        for c, (fn, _, out, _) in cases.items():
            try:
                if out is not None:
                    out.fill_(float("nan"))
                fn()
                if out is not None:
                    outs[(name, c)] = out.clone()
            except _lib.Av2vError:
                unsupported.add((name, c))
        torch.cuda.synchronize()
    for (name, c), out in outs.items():
        if name != "this" and ("this", c) in outs:
            ref = outs[("this", c)]
            same = torch.equal(out, ref)
            print(f"output {c}: {name} {'torch.equal to this build' if same else 'DIFFERS from this build'}"
                  + ("" if same else f" (max |diff| {(out.float() - ref.float()).abs().max().item():.3e})"))
    outs.clear()
    for _ in range(args.rounds):
        for c, (fn, *_) in cases.items():
            for name, lib in libs.items():
                if (name, c) in unsupported:
                    continue
                _lib._lib = lib
                times[(name, c)].append(_time(fn, args.iters))
    _lib._lib = libs["this"]
    print("card (name, power limit, max SM clock):", _card())
    tag = lambda n: n if n == "this" else os.path.basename(os.path.dirname(os.path.abspath(n))) or n
    rows = []
    total = {name: 0.0 for name in libs}
    for c, (_, flops, _, xbytes) in cases.items():
        row = dict(case=c, gflop=round(flops / 1e9, 2))
        line = f"{c:40s}"
        for name in libs:
            if (name, c) in unsupported:
                row[tag(name)] = "unsupported"
                line += f" | {tag(name)} unsupported"
                continue
            t = statistics.median(times[(name, c)])
            total[name] += t
            row[tag(name)] = dict(us=round(t, 2), tflops=round(flops / t / 1e6, 1))
            line += f" | {tag(name)} {t:9.2f} us {flops / t / 1e6:6.1f} TF/s {flops / t / 1e6 / PEAK_TFLOPS:6.1%} of peak"
            if xbytes:
                row[tag(name)]["x_tb_s"] = round(xbytes / t / 1e6, 2)
                line += f" x {xbytes / t / 1e6:5.2f} TB/s"
        rows.append(row)
        print(line)
    print("sum over shapes (one call each):", ", ".join(f"{tag(n)} {t:.1f} us" for n, t in total.items()))
    print(json.dumps(rows))


if __name__ == "__main__":
    main()
