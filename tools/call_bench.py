"""Cost of the image-to-video call `pipe(...)` and of stochastic DDIM (eta > 0) on one GPU.

1. `call_step` time (CUDA-graph replay, as `pipe(...)` runs it; UNet batch 2 = CFG) of the full-size UNet at 16 x 512^2 and at
   the reference default 704 x 1280 (latent 88 x 160), eta = 0 and eta = 1 alternated in one process: medians over the timed
   windows, after a warm-up that runs, captures and replays every graph.  Peak memory per size.
2. Kernel time of the eta > 0 step (ops.ddim_step_eta) against the eta = 0 step (ops.ddim_step) at n = 4 * 16 * 64 * 64, from
   CUDA events around many launches.
Prints the card's name and power limit first: the numbers belong to them.

    python tools/call_bench.py [--reps 5] [--steps 4] [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from freeu_bench import card  # noqa: E402

SIZES = {"512x512": (64, 64), "704x1280": (88, 160)}


def kernel_times(launches: int):
    from anyv2v_b200 import ops
    from anyv2v_b200.schedulers import DDIMScheduler
    n = 4 * 16 * 64 * 64
    g = torch.Generator(device="cuda").manual_seed(0)
    x, vn, ve, z = (torch.randn(n, device="cuda", generator=g).half() for _ in range(4))
    out = torch.empty_like(x)
    s = DDIMScheduler()
    s.set_timesteps(50)
    ca, cb, cc, cd, cs = s.coefficients(501, 1.0)
    calls = {"eta0": lambda: ops.ddim_step(x, vn, ve, 9.0, ca, cb, cc, cd, out=out),
             "eta1": lambda: ops.ddim_step_eta(x, vn, ve, z, 9.0, ca, cb, cc, cd, cs, out=out)}
    res = {}
    for name, fn in calls.items():
        for _ in range(20):
            fn()
    for name, fn in list(calls.items()) * 3:  # alternated; the last window of each is kept
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            fn()
        e1.record()
        torch.cuda.synchronize()
        res.setdefault(name, []).append(e0.elapsed_time(e1) * 1e3 / launches)
    return {f"ddim_step_{k}_us": dict(median=round(sorted(v)[len(v) // 2], 2), min=round(min(v), 2), n=n) for k, v in res.items()}


def step_times(reps: int, steps: int):
    from anyv2v_b200 import distributed
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import synthetic_conditioning
    from anyv2v_b200.schedulers import DDIMScheduler
    from anyv2v_b200.unet_i2vgen_xl import I2VGEN_XL_CONFIG, I2VGenXLUNet
    dev = torch.device("cuda")
    unet = distributed.build_unet_replicated(I2VGenXLUNet, I2VGEN_XL_CONFIG, 8888, dev)
    pipe = I2VGenXLPipeline(unet, DDIMScheduler())
    out = {}
    for size, (h, w) in SIZES.items():
        c = {k: v.to(dev) for k, v in synthetic_conditioning(16, h, w, 1024, 8888, "cpu").items()}
        torch.cuda.reset_peak_memory_stats()
        states = {eta: pipe.prepare_call(c["video_latents"], c["edit_prompt"], c["edit_image_latents"], c["edit_image_emb"], 8,
                                         50, 9.0, c["neg_prompt"], eta, torch.Generator(device=dev).manual_seed(1))
                  for eta in (0.0, 1.0)}

        def window(eta, n):
            st = states[eta]
            st.latents.copy_(c["video_latents"])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(n):
                pipe.call_step(st, i)
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3 / n

        for eta in states:  # warm-up: eager pass, capture, replays
            window(eta, 3)
        times = {eta: [] for eta in states}
        for _ in range(reps):
            for eta in states:
                times[eta].append(window(eta, steps))
        med = lambda v: sorted(v)[len(v) // 2]
        for eta, v in times.items():
            out[f"call_step_ms_{size}_eta{int(eta)}"] = dict(median=round(med(v), 2), min=round(min(v), 2), max=round(max(v), 2))
        out[f"peak_memory_gib_{size}"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
        del states
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="alternations of eta = 0 / eta = 1 (timed windows per setting)")
    ap.add_argument("--steps", type=int, default=4, help="steps per timed window")
    ap.add_argument("--launches", type=int, default=500, help="kernel launches per timed window")
    ap.add_argument("--out", type=str, default=None, help="also write the result as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("call_bench needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    torch.set_grad_enabled(False)
    res = {"card": card()}
    print("card (name, power limit, max SM clock):", res["card"], flush=True)
    res["kernel"] = kernel_times(args.launches)
    for k, v in res["kernel"].items():
        print(k, v, flush=True)
    res["steps"] = step_times(args.reps, args.steps)
    for k, v in res["steps"].items():
        print(k, v, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
