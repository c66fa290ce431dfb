"""Step time against the frame count at 512x512: one inversion step (B = 1) and one PnP edit step with conv, spatial and
temporal injection (B = 3) of the full-size UNet, for each frame count given (default 128, BASELINE config 5).

    python tools/run_long_video_step.py [F ...] [--steps N]

Per F it prints ms per step of each kind (CUDA events over N steps after two warm-up steps), ms per step per frame and the
peak memory of that F; the card name, power limit and max SM clock are read in the same run.  The last line is JSON."""
import argparse
import gc
import json
import os
import sys
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from anyv2v_b200 import distributed  # noqa: E402
from anyv2v_b200.pipeline import I2VGenXLPipeline  # noqa: E402
from anyv2v_b200.run_group_pnp_edit import init_pnp, synthetic_conditioning  # noqa: E402
from anyv2v_b200.schedulers import DDIMInverseScheduler, DDIMScheduler  # noqa: E402
from anyv2v_b200.unet_i2vgen_xl import I2VGEN_XL_CONFIG, I2VGenXLUNet  # noqa: E402
from tools.numerics_bench import _card  # noqa: E402


def timed(fn, n):
    fn()
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def measure(unet, F, n):
    dev = torch.device("cuda", 0)
    gc.collect()  # the previous frame count's pipeline, states and CUDA graphs
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    pipe = I2VGenXLPipeline(unet, DDIMInverseScheduler())
    c = synthetic_conditioning(F, 64, 64, 1024, 8888, dev)
    st_inv = pipe.prepare_invert(c["video_latents"], c["inv_prompt"], c["src_image_latents"], c["src_image_emb"], 8, 50, 1.0, None,
                                 False)
    inv_sched = pipe.scheduler
    es = DDIMScheduler()
    es.set_timesteps(50)
    pipe.scheduler = es
    init_pnp(pipe, es, SimpleNamespace(n_steps=50, pnp_f_t=1.0, pnp_spatial_attn_t=1.0, pnp_temp_attn_t=1.0))
    for t in es.timesteps.tolist()[:n + 2]:
        st_inv.store._mem[int(t)] = torch.randn(1, 4, F, 64, 64, device=dev).half()
    st_edit = pipe.prepare_edit(c["video_latents"].clone(), c["edit_prompt"], c["neg_prompt"], c["inv_prompt"], c["edit_image_emb"],
                                c["edit_image_latents"], c["src_image_emb"], c["src_image_latents"], 8, 50, 9.0, 0, None,
                                st_inv.store, True)
    i = [0, 0]

    def inv():
        pipe.scheduler = inv_sched
        pipe.invert_step(st_inv, i[0])
        i[0] += 1

    def edit():
        pipe.scheduler = es
        pipe.edit_step(st_edit, i[1])
        i[1] += 1

    inv_ms = timed(inv, n)
    edit_ms = timed(edit, n)
    finite = bool(torch.isfinite(st_inv.latents).all() and torch.isfinite(st_edit.latents).all())
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    init_pnp(pipe, es, SimpleNamespace(n_steps=50, pnp_f_t=0.0, pnp_spatial_attn_t=0.0, pnp_temp_attn_t=0.0))
    return dict(F=F, inversion_ms=round(inv_ms, 2), edit_ms=round(edit_ms, 2), inversion_ms_per_frame=round(inv_ms / F, 3),
                edit_ms_per_frame=round(edit_ms / F, 3), peak_gib=round(peak, 2), finite=finite)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("frames", type=int, nargs="*", default=[128])
    ap.add_argument("--steps", type=int, default=2, help="timed steps of each kind per frame count")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("run_long_video_step: no CUDA device")
    torch.set_grad_enabled(False)
    card = _card()
    print("card (name, power limit, max SM clock):", card, flush=True)
    unet = distributed.build_unet_replicated(I2VGenXLUNet, I2VGEN_XL_CONFIG, 8888, torch.device("cuda", 0))
    rows = []
    for F in args.frames:
        r = measure(unet, F, args.steps)
        rows.append(r)
        print(f"F={F:4d}: inversion {r['inversion_ms']:8.1f} ms/step ({r['inversion_ms_per_frame']:6.2f} per frame)  "
              f"edit (conv+spatial+temporal injection) {r['edit_ms']:8.1f} ms/step ({r['edit_ms_per_frame']:6.2f} per frame)  "
              f"peak {r['peak_gib']:.1f} GiB  finite {r['finite']}", flush=True)
    print(json.dumps(dict(card=card, rows=rows)))


if __name__ == "__main__":
    main()
