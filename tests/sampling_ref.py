"""TEST INFRASTRUCTURE — stochastic DDIM (eta > 0) and the image-to-video call for the tests of `I2VGenXLPipeline.__call__`;
nothing outside tests/ imports it.

1. Oracle: diffusers 0.26.3 `DDIMScheduler.step` with eta and `_get_variance`, and `randn_tensor` [recalled: diffusers is not
   vendored], with the fp16 rounding model of oracle/schedulers_ref.py (one rounding per PyTorch op); the sigma is the one of
   the reference's seine/diffusion/gaussian_diffusion.py:585-589.  ``call_loop`` is the denoising loop of the reference's
   `__call__` (pipeline_i2vgen_xl.py:805-874) over pre-encoded conditioning and the oracle UNet of oracle/unet_ref.py.
2. Contract of `ops.ddim_step_eta` (csrc/elementwise.cu, ddim_step_kernel<true>) in the style of tests/kernel_contracts.py;
   ``patch_ops`` swaps it in next to the ``emulated_ops`` fixture.
"""
from __future__ import annotations

import torch

import kernel_contracts
from oracle import schedulers_ref
from oracle.schedulers_ref import _add, _mul, cfg_combine


# ------------------------------------------------------------------------------------------------------------- oracle
def randn_tensor(shape, generator=None, device=None, dtype=None):
    """diffusers.utils.torch_utils.randn_tensor"""
    rand_device = device
    batch_size = shape[0]
    device = device or torch.device("cpu")
    if generator is not None:
        gen_device_type = generator.device.type if not isinstance(generator, list) else generator[0].device.type
        if gen_device_type != torch.device(device).type and gen_device_type == "cpu":
            rand_device = "cpu"
        elif gen_device_type != torch.device(device).type and gen_device_type == "cuda":
            raise ValueError(f"Cannot generate a {device} tensor from a generator of type {gen_device_type}.")
    if isinstance(generator, list) and len(generator) == 1:
        generator = generator[0]
    if isinstance(generator, list):
        shape = (1,) + tuple(shape[1:])
        latents = [torch.randn(shape, generator=generator[i], device=rand_device, dtype=dtype) for i in range(batch_size)]
        return torch.cat(latents, dim=0).to(device)
    return torch.randn(shape, generator=generator, device=rand_device, dtype=dtype).to(device)


def alpha_pair(sched: schedulers_ref.DDIMScheduler, timestep):
    t = int(timestep)
    prev_timestep = t - schedulers_ref.CONFIG["num_train_timesteps"] // sched.num_inference_steps
    alpha_prod_t = sched.alphas_cumprod[t]
    alpha_prod_t_prev = sched.alphas_cumprod[prev_timestep] if prev_timestep >= 0 else sched.final_alpha_cumprod
    return alpha_prod_t, alpha_prod_t_prev


def get_variance(sched, timestep):
    """DDIMScheduler._get_variance"""
    alpha_prod_t, alpha_prod_t_prev = alpha_pair(sched, timestep)
    beta_prod_t = 1 - alpha_prod_t
    beta_prod_t_prev = 1 - alpha_prod_t_prev
    return (beta_prod_t_prev / beta_prod_t) * (1 - alpha_prod_t / alpha_prod_t_prev)


def eta_coefficients(sched, timestep, eta):
    """(std_dev_t, (1 - alpha_prod_t_prev - std_dev_t ** 2) ** 0.5): fp32 0-dim tensors, as DDIMScheduler.step makes them"""
    _, alpha_prod_t_prev = alpha_pair(sched, timestep)
    std_dev_t = eta * get_variance(sched, timestep) ** (0.5)
    return std_dev_t, (1 - alpha_prod_t_prev - std_dev_t ** 2) ** (0.5)


def step(sched, model_output, timestep, sample, eta=0.0, generator=None, variance_noise=None):
    """DDIMScheduler.step (v_prediction, no clipping / thresholding) -> (prev_sample, pred_original_sample)"""
    alpha_prod_t, alpha_prod_t_prev = alpha_pair(sched, timestep)
    beta_prod_t = 1 - alpha_prod_t
    pred_original_sample = _add(_mul(alpha_prod_t ** 0.5, sample), _mul(beta_prod_t ** 0.5, model_output), -1.0)
    pred_epsilon = _add(_mul(alpha_prod_t ** 0.5, model_output), _mul(beta_prod_t ** 0.5, sample))
    std_dev_t, direction_coef = eta_coefficients(sched, timestep, eta)
    pred_sample_direction = _mul(direction_coef, pred_epsilon)
    prev_sample = _add(_mul(alpha_prod_t_prev ** 0.5, pred_original_sample), pred_sample_direction)
    if eta > 0:
        if variance_noise is not None and generator is not None:
            raise ValueError("Cannot pass both generator and variance_noise. Please make sure that either `generator` or"
                             " `variance_noise` stays `None`.")
        if variance_noise is None:
            variance_noise = randn_tensor(model_output.shape, generator=generator, device=model_output.device,
                                          dtype=model_output.dtype)
        variance = _mul(std_dev_t, variance_noise)
        prev_sample = _add(prev_sample, variance)
    return prev_sample, pred_original_sample


@torch.no_grad()
def call_loop(unet, latents, prompt_embeds, negative_prompt_embeds, image_latents, image_embeddings, target_fps, n_steps,
              guidance_scale, eta=0.0, generator=None, t_idx=1, num_videos=1, num_frames=None, dtype=torch.float32,
              callback=None, noise_at=None, max_steps=None):
    """pipeline_i2vgen_xl.py:805-874 over conditioning of batch 1; ``unet(x, t, fps, image_latents, image_embeddings,
    prompts)`` is the oracle UNet's call.  ``latents`` None: prepare_latents (:595-621) draws them from ``generator``.
    ``noise_at(i)`` (teacher forcing): the variance noise of step i instead of a draw; ``max_steps``: stop after that many
    steps.  Returns the final latents."""
    cfg = guidance_scale > 1
    n = num_videos
    rep = lambda x: x.repeat(n, *([1] * (x.dim() - 1)))
    prompts = torch.cat([rep(negative_prompt_embeds), rep(prompt_embeds)]) if cfg else rep(prompt_embeds)
    img_emb = rep(image_embeddings)
    if cfg:
        img_emb = torch.cat([torch.zeros_like(img_emb), img_emb])
    img_lat = rep(image_latents)
    if cfg:
        img_lat = torch.cat([img_lat] * 2)
    fps = (torch.tensor([target_fps, target_fps]) if cfg else torch.tensor([target_fps])).to(img_lat.device)
    fps = fps.repeat(n, 1).ravel()
    sched = schedulers_ref.DDIMScheduler()
    sched.set_timesteps(n_steps)
    timesteps = sched.timesteps[t_idx:]
    if max_steps is not None:
        timesteps = timesteps[:max_steps]
    if latents is None:
        f = num_frames or image_latents.shape[2]
        shape = (n, 4, f) + tuple(image_latents.shape[-2:])
        latents = randn_tensor(shape, generator=generator, device=image_latents.device, dtype=dtype)
    for i, t in enumerate(timesteps):
        latent_model_input = torch.cat([latents] * 2) if cfg else latents
        noise_pred = unet(latent_model_input, torch.tensor([int(t)], device=latents.device), fps, img_lat, img_emb, prompts)[0]
        if cfg:
            noise_pred_uncond, noise_pred_text = noise_pred.chunk(2)
            noise_pred = cfg_combine(noise_pred_uncond, noise_pred_text, guidance_scale)
        b, c, fr, h, w = latents.shape
        latents = latents.permute(0, 2, 1, 3, 4).reshape(b * fr, c, h, w)
        noise_pred = noise_pred.permute(0, 2, 1, 3, 4).reshape(b * fr, c, h, w)
        z = None if noise_at is None else noise_at(i)
        latents = step(sched, noise_pred, t, latents, eta=eta, generator=None if z is not None else generator,
                       variance_noise=z)[0]
        latents = latents[None, :].reshape(b, fr, c, h, w).permute(0, 2, 1, 3, 4)
        if callback is not None:
            callback(i, int(t), latents)
    return latents


# ------------------------------------------------------------------------------------------------------------- contract
def ddim_step_eta(x, v_neg, v_edit, noise, guidance, ca, cb, cc, cd, cs, out=None, coef_dev=None):
    """csrc/elementwise.cu ddim_step_kernel<true>: the eta = 0 contract, then fp16(y + fp16(cs * noise)) with fp32 scalars"""
    kernel_contracts._f16(noise, "ddim_eta.noise")
    assert noise.numel() == x.numel()
    if coef_dev is not None:
        ca, cb, cc, cd, guidance, cs = (float(v) for v in coef_dev[:6].tolist())
    y = kernel_contracts.ddim_step(x, v_neg, v_edit, guidance, ca, cb, cc, cd).float()  # counts the launch
    r16 = lambda t: t.to(torch.float16).to(torch.float32)
    res = r16(y + r16(torch.tensor(cs, dtype=torch.float32) * noise.float().view(y.shape)))
    return kernel_contracts._store(out, res, x.shape)


def patch_ops(monkeypatch):
    """ops.ddim_step_eta -> the contract for one test (use together with the emulated_ops fixture)"""
    from anyv2v_b200 import ops
    monkeypatch.setattr(ops, "ddim_step_eta", ddim_step_eta)
