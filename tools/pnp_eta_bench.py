"""Cost of stochastic DDIM (eta > 0) in the PnP edit on one GPU.

`edit_step` time (CUDA-graph replay, as `sample_with_pnp` runs it) of the full-size UNet at 16 x 512^2 on the BASELINE config-3
injection schedule, eta = 0 against eta = 1 with a CPU generator (what the reference's runner passes), alternated in one
process: for each kind of step (all three injections: steps 0-24, conv injection only: 25-39, dead source branch: 40-49) the
medians over the timed windows, after a warm-up that runs, captures and replays every graph.  The eta = 1 step adds a host
draw of 4 x 16 x 64 x 64 values, one host-to-device copy, the copy into the captured graph's noise buffer and the eta
variant of the step kernel.  Prints the card's name and power limit first: the numbers belong to them.

    python tools/pnp_eta_bench.py [--reps 7] [--steps 4] [--out result.json]
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
CLASSES = {"conv+spatial+temporal": 0, "conv only": 25, "dead source": 40}  # first step of each kind under config 3


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
    states = {eta: pipe.prepare_edit(c["video_latents"].clone(), c["edit_prompt"], c["neg_prompt"], c["inv_prompt"],
                                     c["edit_image_emb"], c["edit_image_latents"], c["src_image_emb"], c["src_image_latents"],
                                     8, N_STEPS, 9.0, 0, None, store, True, eta, torch.Generator().manual_seed(8888))
              for eta in (0.0, 1.0)}

    def window(eta, i0, n):
        st = states[eta]
        st.latents.copy_(c["video_latents"])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(i0, i0 + n):
            pipe.edit_step(st, i)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / n

    for i0 in CLASSES.values():  # warm-up: eager pass, capture, replays of every graph
        for eta in states:
            window(eta, i0, 3)
    out = {}
    med = lambda v: sorted(v)[len(v) // 2]
    for name, i0 in CLASSES.items():
        times = {eta: [] for eta in states}
        for _ in range(reps):
            for eta in states:
                times[eta].append(window(eta, i0, steps))
        row = {f"eta{int(eta)}": dict(median=round(med(v), 2), min=round(min(v), 2), max=round(max(v), 2))
               for eta, v in times.items()}
        row["overhead_pct"] = round(100 * (med(times[1.0]) / med(times[0.0]) - 1), 2)
        out[f"edit_step_ms {name}"] = row
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7, help="alternations of eta = 0 / eta = 1 (timed windows per setting)")
    ap.add_argument("--steps", type=int, default=4, help="steps per timed window")
    ap.add_argument("--out", type=str, default=None, help="also write the result as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pnp_eta_bench needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    torch.set_grad_enabled(False)
    res = {"card": card()}
    print("card (name, power limit, max SM clock):", res["card"], flush=True)
    res["steps"] = step_times(args.reps, args.steps)
    for k, v in res["steps"].items():
        print(k, v, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
