"""Cost of an injected PnP edit step with the source branch's features taken from a SourceFeatureCache, on one GPU.

`edit_step` time (CUDA-graph replay, as `sample_with_pnp` runs it) of the full-size UNet at 16 x 512^2 on the BASELINE config-3
injection schedule, without the cache (three branches) against with a cache filled by the same steps (two branches, source
features copied into the step's static buffers), alternated in one process: for each kind of injected step (all three
injections: steps 0-24, conv injection only: 25-39) the medians over the timed windows, after a warm-up that fills the cache
and runs, captures and replays every graph.  Also reports the cache's size per step kind and the peak device memory.
Prints the card's name, power limit and clocks first: the numbers belong to them.

    python tools/source_cache_bench.py [--reps 7] [--steps 4] [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from freeu_bench import card  # noqa: E402

N_STEPS = 50
CONFIG3 = SimpleNamespace(n_steps=N_STEPS, pnp_f_t=0.8, pnp_spatial_attn_t=0.5, pnp_temp_attn_t=0.5)
CLASSES = {"conv+spatial+temporal": 0, "conv only": 25}  # first step of each injected kind under config 3


def step_times(reps: int, steps: int):
    from anyv2v_b200 import distributed
    from anyv2v_b200.latent_store import LatentStore
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp, synthetic_conditioning
    from anyv2v_b200.schedulers import DDIMScheduler
    from anyv2v_b200.unet_i2vgen_xl import I2VGEN_XL_CONFIG, I2VGenXLUNet
    dev = torch.device("cuda")
    unet = distributed.build_unet_replicated(I2VGenXLUNet, I2VGEN_XL_CONFIG, 8888, dev)
    sched = DDIMScheduler()
    sched.set_timesteps(N_STEPS)
    pipe = I2VGenXLPipeline(unet, sched)
    init_pnp(pipe, sched, CONFIG3)
    c = {k: v.to(dev) for k, v in synthetic_conditioning(16, 64, 64, 1024, 8888, "cpu").items()}
    store = LatentStore(None, write_files=False)
    g = torch.Generator().manual_seed(3)
    for t in sched.timesteps.tolist():
        store.put(int(t), torch.randn(1, 4, 16, 64, 64, generator=g).half().to(dev))
    cache = pipe.source_feature_cache(max_bytes=40 << 30)
    states = {name: pipe.prepare_edit(c["video_latents"].clone(), c["edit_prompt"], c["neg_prompt"], c["inv_prompt"],
                                      c["edit_image_emb"], c["edit_image_latents"], c["src_image_emb"], c["src_image_latents"],
                                      8, N_STEPS, 9.0, 0, None, store, True, 0.0, None, cache if name == "cached" else None)
              for name in ("uncached", "cached")}

    def window(name, i0, n):
        st = states[name]
        st.latents.copy_(c["video_latents"])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(i0, i0 + n):
            pipe.edit_step(st, i)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / n

    sizes = {}
    for cls, i0 in CLASSES.items():  # warm-up: the cached state's first window fills the cache, the later ones replay it
        before = cache.nbytes
        for _ in range(3):
            for name in states:
                window(name, i0, steps)
        sizes[cls] = round((cache.nbytes - before) / steps / 2**20, 1)
    out = {"cache_MiB_per_step": sizes, "cache_GiB_total": round(cache.nbytes / 2**30, 2)}
    med = lambda v: sorted(v)[len(v) // 2]
    for cls, i0 in CLASSES.items():
        times = {name: [] for name in states}
        for _ in range(reps):
            for name in states:
                times[name].append(window(name, i0, steps))
        row = {name: dict(median=round(med(v), 2), min=round(min(v), 2), max=round(max(v), 2)) for name, v in times.items()}
        row["saving_pct"] = round(100 * (1 - med(times["cached"]) / med(times["uncached"])), 2)
        out[f"edit_step_ms {cls}"] = row
    out["peak_allocated_GiB"] = round(torch.cuda.max_memory_allocated() / 2**30, 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7, help="alternations of uncached / cached (timed windows per setting)")
    ap.add_argument("--steps", type=int, default=4, help="steps per timed window")
    ap.add_argument("--out", type=str, default=None, help="also write the result as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("source_cache_bench needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    torch.set_grad_enabled(False)
    res = {"card": card()}
    print("card (name, power limit, max SM clock):", res["card"], flush=True)
    res["steps"] = step_times(args.reps, args.steps)
    res["card_after"] = card()
    for k, v in res["steps"].items():
        print(k, v, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
