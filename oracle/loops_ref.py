"""ORACLE (test infrastructure): the two sampling loops of the reference over pre-encoded (synthetic) conditioning.

Follows /root/reference/i2vgen-xl/pipelines/pipeline_i2vgen_xl.py:
  invert loop            :1385-1433  (cfg = 1 -> single branch; latent saved per timestep)
  sample_with_pnp loop   :1131-1179  (3 branches [source, uncond, cond]; register_time; CFG :1162; DDIM step :1173)
  image-latent + frame-position mask assembly :532-562
CLIP / VAE encoders are outside the metric (SURVEY 8d) — the loops take their outputs as tensors.
The scheduler update is elementwise, so the [B,C,F,h,w] <-> [B*F,C,h,w] permutes at :1168-1176 are identities
for the arithmetic and are not restated.
"""
from __future__ import annotations

from types import SimpleNamespace

import torch

from .schedulers_ref import DDIMInverseScheduler, DDIMScheduler, cfg_combine


def frame_position_latents(first_frame_latent: torch.Tensor, num_frames: int) -> torch.Tensor:
    """[b,4,h,w] -> [b,4,F,h,w]: frame 0 = the latent, frame k = constant k/(F-1) (pipeline :548-554)."""
    x = first_frame_latent.unsqueeze(2)
    masks = [torch.ones_like(x) * ((k + 1) / (num_frames - 1)) for k in range(num_frames - 1)]
    return torch.cat([x] + masks, dim=2) if masks else x


def synthetic_inputs(F: int, h: int, w: int, cross_dim: int = 1024, seed: int = 8888, dtype=torch.float32,
                     device="cpu") -> SimpleNamespace:
    """Seeded synthetic conditioning of SURVEY 8d (reference default seed, template.yaml:4)."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)
    ns = SimpleNamespace()
    ns.video_latents = rn(1, 4, F, h, w)
    ns.src_image_latents = frame_position_latents(rn(1, 4, h, w), F)
    ns.edit_image_latents = frame_position_latents(rn(1, 4, h, w), F)
    ns.inv_prompt = rn(1, 77, cross_dim)
    ns.neg_prompt = rn(1, 77, cross_dim)
    ns.edit_prompt = rn(1, 77, cross_dim)
    ns.src_image_emb = rn(1, 1, cross_dim)
    ns.edit_image_emb = rn(1, 1, cross_dim)
    ns.fps = torch.tensor([8])
    for k, v in vars(ns).items():
        if v.is_floating_point():
            setattr(ns, k, v.to(device=device, dtype=dtype))
        else:
            setattr(ns, k, v.to(device))
    return ns


@torch.no_grad()
def invert_loop(unet, latents, prompt_embeds, image_latents, image_embeddings, fps, n_steps: int):
    """-> {t: latents_at_t}, exactly what the reference writes to ddim_latents_{t}.pt (:1422-1428)."""
    sched = DDIMInverseScheduler()
    sched.set_timesteps(n_steps)
    saved = {}
    for t in sched.timesteps:
        v = unet(latents, t, fps, image_latents, image_embeddings, prompt_embeds)[0]
        latents, _ = sched.step(v, int(t), latents)
        saved[int(t)] = latents.clone()
    return saved


@torch.no_grad()
def pnp_edit_loop(pipe, register_time, inv_latents: dict, latents, prompt_embeds_all, image_latents_all,
                  image_embeddings_all, fps_all, n_steps: int, guidance: float, t_idx: int = 0,
                  scheduler: DDIMScheduler | None = None, callback=None):
    """pipe: object with .unet whose hooks were registered by init_pnp. Returns final latents [1,4,F,h,w].
    ``callback(i, t, latents)`` (optional) sees the latents after every step, as the pipeline's callback does."""
    sched = scheduler or DDIMScheduler()
    sched.set_timesteps(n_steps)
    for i, t in enumerate(sched.timesteps[t_idx:]):
        x_in = torch.cat([inv_latents[int(t)], latents, latents])
        register_time(pipe, int(t))
        v = pipe.unet(x_in, t, fps_all, image_latents_all, image_embeddings_all, prompt_embeds_all)[0]
        _, v_neg, v_edit = v.chunk(3)
        latents, _ = sched.step(cfg_combine(v_neg, v_edit, guidance), int(t), latents)
        if callback is not None:
            callback(i, int(t), latents)
    return latents


def edit_conditioning(ns):
    """[source, uncond, cond] stacks (pipeline :1043-1046, :1093-1101); the uncond image embedding is zeros (:438)."""
    prompts = torch.cat([ns.inv_prompt, ns.neg_prompt, ns.edit_prompt])
    img_lat = torch.cat([ns.src_image_latents, ns.edit_image_latents, ns.edit_image_latents])
    img_emb = torch.cat([ns.src_image_emb, torch.zeros_like(ns.edit_image_emb), ns.edit_image_emb])
    fps = ns.fps.repeat(3)
    return prompts, img_lat, img_emb, fps
