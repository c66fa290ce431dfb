"""FreeU cost on the 16-frame 512 x 512 workload of bench.py (needs one GPU).

1. Kernel time of ops.freeu at the six skip connections of a PnP edit step (B = 3 branches x 16 frames; up_blocks[0] at
   8 x 8, up_blocks[1] at 16 x 16), from CUDA events around many launches, and the rate over the bytes the op needs (skip read
   once, filtered skip written once, half of hidden read and written) against the H100 SXM data-sheet 3.35 TB/s.
2. Inversion and edit step times (CUDA-graph replay, as bench.py runs them) with FreeU off and on, alternated in one process.
Prints the card's name and power limit first: the numbers belong to them.

    python tools/freeu_bench.py [--reps 5] [--steps 4] [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FREEU = dict(s1=0.9, s2=0.2, b1=1.5, b2=1.6)
HBM_BYTES_PER_S = 3.35e12
F, H, W = 16, 64, 64  # bench.py's workload: 16 frames of 64 x 64 latents
#: (NF, h, w, hidden channels, skip channels) of the six FreeU calls of an edit step (I2VGEN_XL_CONFIG, 3 branches x 16 frames)
SHAPES = [(48, 8, 8, 1280, 1280)] * 3 + [(48, 16, 16, 1280, 1280)] * 2 + [(48, 16, 16, 1280, 640)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def kernel_times(launches: int):
    from anyv2v_b200 import ops
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for nf, h, w, ch, cs in SHAPES:
        hidden = torch.randn(nf, h, w, ch, device="cuda", generator=g).half()
        skip = torch.randn(nf, h, w, cs, device="cuda", generator=g).half()
        out = torch.empty_like(skip)
        for _ in range(10):
            ops.freeu(hidden, skip, 1.0, 0.9, out=out)  # b = 1: hidden keeps its values over the launches
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            ops.freeu(hidden, skip, 1.0, 0.9, out=out)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / launches
        nbytes = 2 * skip.numel() * 2 + hidden.numel() * 2
        rate = nbytes / (us * 1e-6)
        rows.append(dict(shape=[nf, h, w], hidden_channels=ch, skip_channels=cs, us=round(us, 2), bytes=nbytes,
                         gb_per_s=round(rate / 1e9, 1), share_of_3_35_tb_s=round(rate / HBM_BYTES_PER_S, 3)))
    return rows


def step_times(reps: int, steps: int):
    from anyv2v_b200 import distributed
    from anyv2v_b200.latent_store import LatentStore
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp, synthetic_conditioning
    from anyv2v_b200.schedulers import DDIMInverseScheduler, DDIMScheduler
    from anyv2v_b200.unet_i2vgen_xl import I2VGEN_XL_CONFIG, I2VGenXLUNet
    dev = torch.device("cuda")
    unet = distributed.build_unet_replicated(I2VGenXLUNet, I2VGEN_XL_CONFIG, 8888, dev)
    c = {k: v.to(dev) for k, v in synthetic_conditioning(F, H, W, 1024, 8888, "cpu").items()}
    pipe = I2VGenXLPipeline(unet, DDIMInverseScheduler())
    inv_sched = pipe.scheduler
    st_inv = pipe.prepare_invert(c["video_latents"], c["inv_prompt"], c["src_image_latents"], c["src_image_emb"], 8, 50, 1.0,
                                 None, False)
    edit_sched = DDIMScheduler()
    edit_sched.set_timesteps(50)
    pipe.scheduler = edit_sched
    init_pnp(pipe, edit_sched, SimpleNamespace(n_steps=50, pnp_f_t=1.0, pnp_spatial_attn_t=1.0, pnp_temp_attn_t=0.0))  # bench.py's PNP
    store = LatentStore(None, write_files=False)
    g = torch.Generator().manual_seed(4242)
    for t in edit_sched.timesteps.tolist()[:steps + 2]:
        store.put(int(t), torch.randn(1, 4, F, H, W, generator=g).half().to(dev))
    st_edit = pipe.prepare_edit(c["video_latents"].clone(), c["edit_prompt"], c["neg_prompt"], c["inv_prompt"], c["edit_image_emb"],
                                c["edit_image_latents"], c["src_image_emb"], c["src_image_latents"], 8, 50, 9.0, 0, None, store, True)
    st_inv.store = store

    def window(loop, n):
        """n steps of one loop from the same start; ms per step (host clock around work that ends in a synchronise)"""
        st_inv.latents.copy_(c["video_latents"])
        st_edit.latents.copy_(c["video_latents"])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(n):
            if loop == "inv":
                pipe.scheduler = inv_sched
                pipe.invert_step(st_inv, i)
            else:
                pipe.scheduler = edit_sched
                pipe.edit_step(st_edit, i)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / n

    settings = {"off": None, "on": FREEU}

    def apply(name):
        if settings[name] is None:
            pipe.disable_freeu()
        else:
            pipe.enable_freeu(**settings[name])

    for name in settings:  # warm-up: eager pass, then capture, of every (loop, setting) graph
        apply(name)
        window("inv", 3)
        window("edit", 3)
    times = {(loop, name): [] for loop in ("inv", "edit") for name in settings}
    for _ in range(reps):
        for name in settings:
            apply(name)
            for loop in ("inv", "edit"):
                times[(loop, name)].append(window(loop, steps))
    pipe.disable_freeu()
    med = lambda v: sorted(v)[len(v) // 2]
    return {f"{loop}_ms_freeu_{name}": dict(median=round(med(v), 2), min=round(min(v), 2), max=round(max(v), 2))
            for (loop, name), v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="alternations of FreeU off / on")
    ap.add_argument("--steps", type=int, default=4, help="steps per timed window")
    ap.add_argument("--launches", type=int, default=200, help="kernel launches per timed shape")
    ap.add_argument("--out", type=str, default=None, help="also write the result as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("freeu_bench needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    torch.set_grad_enabled(False)
    res = {"card": card()}
    print("card (name, power limit, max SM clock):", res["card"], flush=True)
    res["kernel"] = kernel_times(args.launches)
    for r in res["kernel"]:
        print("freeu kernel", r, flush=True)
    res["steps"] = step_times(args.reps, args.steps)
    for k, v in res["steps"].items():
        print(k, v, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
