"""TEST INFRASTRUCTURE — the PnP edit loop of the reference's `sample_with_pnp` with stochastic DDIM (eta > 0), for the tests of
`I2VGenXLPipeline.sample_with_pnp(eta=...)`; nothing outside tests/ imports it.  The scheduler step and `randn_tensor` are those
of tests/sampling_ref.py (diffusers' `DDIMScheduler.step` with eta, with the fp16 rounding model of oracle/schedulers_ref.py)."""
from __future__ import annotations

import torch

from oracle import schedulers_ref
from oracle.schedulers_ref import cfg_combine
from sampling_ref import randn_tensor, step


@torch.no_grad()
def pnp_edit_loop_eta(pipe, register_time, inv_latents: dict, latents, prompt_embeds_all, image_latents_all,
                      image_embeddings_all, fps_all, n_steps: int, guidance: float, eta: float, generator=None, t_idx: int = 0,
                      max_steps=None, noise_dtype=torch.float16, callback=None):
    """The PnP edit loop of the reference's `sample_with_pnp` (pipeline_i2vgen_xl.py:1131-1179) with stochastic DDIM: the
    loop of oracle/loops_ref.pnp_edit_loop, with the [B, C, F, h, w] -> [B*F, C, h, w] reshape around the step (:1168-1176)
    and ``DDIMScheduler.step(..., eta, generator)`` (extra_step_kwargs, :1126) drawing the variance noise inside the step.
    ``pipe.unet`` carries the reference's hooks; ``inv_latents`` {t: source latent}.  The noise is drawn in ``noise_dtype``:
    the reference's model output is fp16, so are its draws, whatever precision this loop computes in.  ``t_idx`` /
    ``max_steps``: the steps ``timesteps[t_idx:][:max_steps]`` of the ``n_steps`` schedule.  Returns the final latents."""
    sched = schedulers_ref.DDIMScheduler()
    sched.set_timesteps(n_steps)
    timesteps = sched.timesteps[t_idx:]
    if max_steps is not None:
        timesteps = timesteps[:max_steps]
    for i, t in enumerate(timesteps):
        x_in = torch.cat([inv_latents[int(t)], latents, latents])
        register_time(pipe, int(t))
        v = pipe.unet(x_in, torch.tensor([int(t)], device=latents.device), fps_all, image_latents_all, image_embeddings_all,
                      prompt_embeds_all)[0]
        _, v_neg, v_edit = v.chunk(3)
        noise_pred = cfg_combine(v_neg, v_edit, guidance)
        b, c, fr, h, w = latents.shape
        latents = latents.permute(0, 2, 1, 3, 4).reshape(b * fr, c, h, w)
        noise_pred = noise_pred.permute(0, 2, 1, 3, 4).reshape(b * fr, c, h, w)
        z = None
        if eta > 0:  # DDIMScheduler.step's draw: randn_tensor(model_output.shape, generator=generator, dtype=model_output.dtype)
            z = randn_tensor(noise_pred.shape, generator=generator, device=noise_pred.device, dtype=noise_dtype).to(noise_pred.dtype)
        latents = step(sched, noise_pred, t, latents, eta=eta, variance_noise=z)[0]
        latents = latents[None, :].reshape(b, fr, c, h, w).permute(0, 2, 1, 3, 4)
        if callback is not None:
            callback(i, int(t), latents)
    return latents
