"""DPM-Solver++(2M) against DDIM on one GPU, at 16 x 512^2 on the full-size UNet.

1. The step kernel alone: ``ops.dpmpp2m_step`` (second-order row, CFG) against ``ops.ddim_step`` (CFG) on one video's
   latents (4 x 16 x 64 x 64), out of place, CUDA events around 200 launches per window.
2. One loop iteration under CUDA-graph replay (UNet on [uncond, cond] + the step): `call_step` of a 25-step DPM-Solver++
   `__call__` state against a 50-step DDIM one.
3. Whole runs: a 25-step DPM-Solver++ `__call__` against a 50-step DDIM `__call__`, and a 25-step DPM-Solver++ PnP edit
   against a 50-step DDIM edit (BASELINE config-3 injections, source latents at every timestep of a 50-step inversion),
   each with ``ddim_init_latents_t_idx=1`` (24 against 49 UNet passes): the steps of one loop state per setting, replayed
   from the same initial latents after one warm-up run that captures the graphs (conditioning, done once per clip, is not
   in the time).
The two settings of each comparison alternate window by window in one process; medians are reported.  Prints the card's
name, power limit and max SM clock first: the numbers belong to them.

    python tools/dpm_solver_bench.py [--reps 5] [--runs 2] [--parts kernel,call,edit] [--out result.json]
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

F_, H_, W_ = 16, 64, 64
DPM_STEPS, DDIM_STEPS = 25, 50
CONFIG3 = dict(pnp_f_t=0.8, pnp_spatial_attn_t=0.5, pnp_temp_attn_t=0.5)
med = lambda v: sorted(v)[len(v) // 2]


def _stats(v, nd=2):
    return dict(median=round(med(v), nd), min=round(min(v), nd), max=round(max(v), nd))


def _schedulers():
    from anyv2v_b200.schedulers import DDIMScheduler, DPMSolverMultistepScheduler
    ddim = DDIMScheduler()
    return {"ddim": (ddim, DDIM_STEPS), "dpm": (DPMSolverMultistepScheduler.from_config(ddim.config), DPM_STEPS)}


def kernel_times(reps: int, launches: int = 200):
    from anyv2v_b200 import ops
    n = 4 * F_ * H_ * W_
    g = torch.Generator(device="cuda").manual_seed(1)
    x, vn, ve, p = (torch.randn(n, device="cuda", generator=g).half() for _ in range(4))
    out = torch.empty_like(x)
    (ddim, _), (dpm, _) = _schedulers().values()
    ddim.set_timesteps(DDIM_STEPS)
    dpm.set_timesteps(DPM_STEPS)
    c_ddim = ddim.coefficient_table(ddim.timesteps.tolist()[20:21], 9.0, "cuda")[0]
    c_dpm = dpm.coefficient_table(dpm.timesteps.tolist()[1:], 9.0, "cuda")[10]
    assert float(c_dpm[4]) != 0.0   # a second-order row: the kernel reads x0_prev
    run = {"ddim": lambda: ops.ddim_step(x, vn, ve, 0.0, 0.0, 0.0, 0.0, 0.0, out=out, coef_dev=c_ddim),
           "dpm": lambda: ops.dpmpp2m_step(x, vn, ve, p, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, out=out, coef_dev=c_dpm)}

    def window(name):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            run[name]()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) * 1e3 / launches

    for name in run:
        window(name)
    times = {name: [] for name in run}
    for _ in range(reps):
        for name in run:
            times[name].append(window(name))
    # bytes the algorithm moves: DDIM reads x, v_neg, v_edit and writes out; DPM also reads and writes x0_prev
    res = {f"{name}_step_kernel_us": _stats(v) for name, v in times.items()}
    for name, moved in (("ddim", 4), ("dpm", 6)):
        res[f"{name}_step_kernel_GBps"] = round(moved * 2 * n / (med(times[name]) * 1e-6) / 1e9, 1)
    return res


def loop_times(reps: int, runs: int, parts):
    from anyv2v_b200 import distributed
    from anyv2v_b200.latent_store import LatentStore
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp, synthetic_conditioning
    from anyv2v_b200.unet_i2vgen_xl import I2VGEN_XL_CONFIG, I2VGenXLUNet
    dev = torch.device("cuda")
    unet = distributed.build_unet_replicated(I2VGenXLUNet, I2VGEN_XL_CONFIG, 8888, dev)
    c = {k: v.to(dev) for k, v in synthetic_conditioning(F_, H_, W_, 1024, 8888, "cpu").items()}
    scheds = _schedulers()
    pipes = {name: I2VGenXLPipeline(unet, s) for name, (s, _) in scheds.items()}
    res = {}

    # 2. one __call__ loop iteration under graph replay (the states are kept: a graph is never destroyed during a run)
    states = {name: pipes[name].prepare_call(c["video_latents"], c["edit_prompt"], c["edit_image_latents"], c["edit_image_emb"],
                                             8, n, 9.0, c["neg_prompt"]) for name, (_, n) in scheds.items()}

    def window(name, i0, k):
        st = states[name]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(i0, i0 + k):
            pipes[name].call_step(st, i)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / k

    if "call" in parts:
        for name in states:
            window(name, 0, 3)   # eager, capture, replay
        times = {name: [] for name in states}
        for _ in range(reps):
            for name in states:
                times[name].append(window(name, 3, 4))
        res["call_step_ms_graph_replay"] = {name: _stats(v) for name, v in times.items()}

    # 3. whole __call__: the 24 (DPM) / 49 (DDIM) steps of the state above, replayed from the initial latents
    def whole(name, sts, step, before=None):
        st = sts[name]
        if before is not None:
            before(name)
        st.latents.copy_(c["video_latents"])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(len(st.timesteps)):
            step(pipes[name], st, i)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    def compare(what, sts, step, before=None):
        for name in sts:
            whole(name, sts, step, before)  # warm-up: every graph of the run is captured
        t = {name: [] for name in sts}
        for _ in range(runs):
            for name in sts:
                t[name].append(whole(name, sts, step, before))
        res[f"{what}_s"] = {f"{name} {scheds[name][1]} steps": _stats(v, 3) for name, v in t.items()}
        res[f"{what}_speedup"] = round(med(t["ddim"]) / med(t["dpm"]), 3)

    if "call" in parts:
        compare("call", states, lambda pipe, st, i: pipe.call_step(st, i))
    if "edit" in parts:
        # 4. whole PnP edit (config 3), source latents at every timestep of a 50-step inversion
        store = LatentStore(None, write_files=False)
        g = torch.Generator().manual_seed(3)
        scheds["ddim"][0].set_timesteps(DDIM_STEPS)
        for t in scheds["ddim"][0].timesteps.tolist():
            store.put(int(t), torch.randn(1, 4, F_, H_, W_, generator=g).half().to(dev))
        edits = {}

        def hooks(name):  # the two edits share the UNet: each registers its own injection timesteps before it runs
            sched, n = scheds[name]
            init_pnp(pipes[name], sched, SimpleNamespace(n_steps=n, **CONFIG3))
        for name, (sched, n) in scheds.items():
            sched.set_timesteps(n)
            pipes[name] = I2VGenXLPipeline(unet, sched)
            hooks(name)
            edits[name] = pipes[name].prepare_edit(c["video_latents"], c["edit_prompt"], c["neg_prompt"], c["inv_prompt"],
                                                   c["edit_image_emb"], c["edit_image_latents"], c["src_image_emb"],
                                                   c["src_image_latents"], 8, n, 9.0, 1, None, store, True)
        compare("pnp_edit", edits, lambda pipe, st, i: pipe.edit_step(st, i), hooks)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="alternated timed windows of the kernel and loop-iteration timings")
    ap.add_argument("--runs", type=int, default=2, help="alternated timed whole runs per setting")
    ap.add_argument("--parts", type=str, default="kernel,call,edit", help="which of kernel, call, edit to time")
    ap.add_argument("--out", type=str, default=None, help="also write the result as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dpm_solver_bench needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    torch.set_grad_enabled(False)
    res = {"card": card()}
    print("card (name, power limit, max SM clock):", res["card"], flush=True)
    parts = args.parts.split(",")
    if "kernel" in parts:
        res.update(kernel_times(args.reps))
    if "call" in parts or "edit" in parts:
        res.update(loop_times(args.reps, args.runs, parts))
    for k, v in res.items():
        print(k, v, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
