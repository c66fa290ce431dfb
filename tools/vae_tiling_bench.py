"""VAE tiling / slicing at the reference's default frame size, full-size KL-f8 VAE (random init), one GPU.

  decode 16 x 704 x 1280: tiled (ours: tiles batched by shape + one stitch kernel) against diffusers' sequential tiled loop
  in torch fp16 over the oracle modules; the stitch kernel alone against the loop's blend alone; untiled decode (ours)
  encode with slicing at 16 and 128 frames (ours, `encode_vae_video`), with and without tiling

Times are CUDA-event medians over --iters runs after one warm-up; peak memory is torch.cuda.max_memory_allocated over one
run, minus what was allocated before it.  Prints one line per number and, with --out, writes them as JSON.
Usage: python tools/vae_tiling_bench.py [--frames 16] [--long-frames 128] [--iters 3] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
from anyv2v_b200 import ops  # noqa: E402
from anyv2v_b200 import vae as product  # noqa: E402
from oracle import vae_ref  # noqa: E402  (timing comparison only: development tool, not the product path)
import vae_tiling_ref as vt  # noqa: E402

dev = "cuda"


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        out = torch.cuda.get_device_name()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def measure(fn, iters):
    """-> (median ms, peak bytes above the allocation before the call)"""
    fn()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    times = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return sorted(times)[len(times) // 2], torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--long-frames", type=int, default=128)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    res = dict(gpu=gpu_info(), frames=args.frames, size="704x1280")
    print(res["gpu"], flush=True)

    ref = vae_ref.seeded_vae(vae_ref.SD_VAE_CONFIG, seed=8888, dtype=torch.float16).to(dev)
    ours = product.AutoencoderKL(**product.SD_VAE_CONFIG)
    ours.load_state_dict(ref.state_dict())
    ours = ours.to(device=dev, dtype=torch.float16).eval()
    loop = vt.DiffusersTiling(ref, ours.tile_sample_min_size)
    g = torch.Generator().manual_seed(0)
    z = torch.randn(args.frames, 4, 88, 160, generator=g).to(dev).half()

    def rec(key, ms, peak):
        res[key] = dict(ms=round(ms, 3), peak_gib=round(peak / 2**30, 3))
        print(f"{key:40s} {ms:10.2f} ms   peak {peak / 2**30:7.2f} GiB", flush=True)

    rec("decode_untiled_ours", *measure(lambda: ours.decode(z), args.iters))
    ours.enable_tiling()
    loop.enable_tiling()
    rec("decode_tiled_ours", *measure(lambda: ours.decode(z), args.iters))
    rec("decode_tiled_torch_fp16_loop", *measure(lambda: loop.decode(z), args.iters))
    a, b = ours.decode(z).sample, loop.decode(z).sample
    res["decode_tiled_rms_rel_ours_vs_loop"] = float((a.double() - b.double()).pow(2).mean().sqrt() / b.double().pow(2).mean().sqrt())
    print(f"decode tiled: rms rel difference ours vs torch fp16 loop {res['decode_tiled_rms_rel_ours_vs_loop']:.3e}", flush=True)

    # the seams alone: the stitch kernel on the raw tiles of one tiled decode, and the loop's blends on the same tiles
    captured = []
    real = ops.tile_stitch

    def capture(*a_):
        captured.append(a_)
        return real(*a_)
    ops.tile_stitch = capture
    ours.decode(z)
    ops.tile_stitch = real
    tiles, H, W, tile, step, blend, row_limit = captured[0]
    rec("stitch_kernel", *measure(lambda: ops.tile_stitch(tiles, H, W, tile, step, blend, row_limit), max(args.iters, 20)))
    rows = [[torch.stack([img[i][j] for img in tiles]) for j in range(len(tiles[0][0]))] for i in range(len(tiles[0]))]

    def blend_only():
        vt.blend_loop([[t.clone() for t in r] for r in rows], blend, row_limit)
    rec("stitch_torch_fp16_loop_incl_tile_copies", *measure(blend_only, args.iters))
    del tiles, rows, captured, a, b
    ours.disable_tiling()

    # encode with slicing (one frame per encoder pass, as the reference does)
    for f in (args.frames, args.long_frames):
        x = torch.randn(f, 3, 704, 1280, generator=g).clamp(-1, 1).to(dev).half()
        ours.enable_slicing()
        rec(f"encode_sliced_{f}f", *measure(lambda: product.encode_vae_video(ours, x), args.iters))
        ours.enable_tiling()
        rec(f"encode_sliced_tiled_{f}f", *measure(lambda: product.encode_vae_video(ours, x), args.iters))
        ours.disable_tiling()
        ours.disable_slicing()
        if f == args.frames:  # one batch of 128 full-resolution frames does not fit the GPU: only the smaller clip
            rec(f"encode_unsliced_{f}f", *measure(lambda: product.encode_vae_video(ours, x), args.iters))
        del x
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
