"""Group runner, phase 2 — drop-in for the reference's ``i2vgen-xl/run_group_pnp_edit.py``.

Same CLI (``--template_config``, ``--configs_json``; reference :186-192), same YAML / JSON keys and override
semantics (template merged with each JSON entry, ``"active": false`` skips; :74-81), same ``init_pnp`` arithmetic
(:35-48), same ``ddim_latents_{t}.pt`` inputs and the same output directory naming (:154-168).
What changes: clips are sharded one-per-GPU when launched under torchrun (the reference loops over them on one
device, :74) and the models are this package's UNet / VAE plus the ``transformers`` CLIP towers.  The runner consumes
the REAL inputs like the reference (:95-150): source frames ``{video_dir}/{video_name}/%05d.png`` (mp4 fallback), the edited
first frame, the prompts; it decodes the result with the VAE and writes ``video.mp4`` / ``video.gif`` / ``video_%05d.png``
(:169-183) plus ``edited_latents.pt``.  Weights: ``model_name`` may name a local diffusers-layout checkpoint directory
(``unet/ vae/ text_encoder/ image_encoder/ tokenizer/ feature_extractor/``); there is no network on the build / bench boxes,
so otherwise every model is seeded random-init (logged).  ``synthetic: true`` (explicit opt-in, config key or JSON entry)
replaces CLIP / VAE by the seeded stand-ins of SURVEY 8d and writes latents only — the benchmark's workload.
"""
from __future__ import annotations

import argparse
import json
import logging
import os
from pathlib import Path

import torch

from .config import OmegaConf
from .latent_store import LatentStore, load_ddim_latents_at_t
from .pipeline import I2VGenXLPipeline, frame_position_latents
from .pnp_utils import register_conv_injection, register_spatial_attention_pnp, register_temp_attention_pnp
from .schedulers import DDIMScheduler, DPMSolverMultistepScheduler

logger = logging.getLogger(__name__)


def seed_everything(seed: int) -> None:
    """i2vgen-xl/utils.py:17-22."""
    import random

    import numpy as np
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed)
    random.seed(seed)
    np.random.seed(seed)


def pnp_schedules(scheduler, config):
    """reference :36-45 — k = int(n_steps * frac); schedule = first k entries of the FULL descending timestep list;
    a negative fraction gives an empty schedule."""
    out = []
    for frac in (config.pnp_f_t, config.pnp_spatial_attn_t, config.pnp_temp_attn_t):
        k = int(config.n_steps * frac)
        out.append(scheduler.timesteps[:k] if k >= 0 else [])
    return out


def init_pnp(pipe, scheduler, config):
    conv_t, spa_t, tmp_t = pnp_schedules(scheduler, config)
    register_conv_injection(pipe, conv_t)
    register_spatial_attention_pnp(pipe, spa_t)
    register_temp_attention_pnp(pipe, tmp_t)
    logger.debug("conv_injection_timesteps: %s", conv_t)
    logger.debug("spatial_attn_qk_injection_timesteps: %s", spa_t)
    logger.debug("temp_attn_qk_injection_timesteps: %s", tmp_t)


def synthetic_conditioning(n_frames: int, h: int, w: int, cross_dim: int, seed: int, device, dtype=torch.float16):
    """Seeded stand-ins for the CLIP / VAE outputs (SURVEY 8d); same generator order as oracle.loops_ref."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g).to(device=device, dtype=dtype)
    c = {}
    c["video_latents"] = rn(1, 4, n_frames, h, w)
    c["src_image_latents"] = frame_position_latents(rn(1, 4, h, w), n_frames)
    c["edit_image_latents"] = frame_position_latents(rn(1, 4, h, w), n_frames)
    c["inv_prompt"], c["neg_prompt"], c["edit_prompt"] = rn(1, 77, cross_dim), rn(1, 77, cross_dim), rn(1, 77, cross_dim)
    c["src_image_emb"], c["edit_image_emb"] = rn(1, 1, cross_dim), rn(1, 1, cross_dim)
    return c


def config_suffix(config) -> str:
    """reference :154-167; an edit with ``scheduler: dpmsolver++`` adds "_dpmsolver++", so that it does not overwrite the
    DDIM edit of the same settings."""
    suffix = ("ddim_init_latents_t_idx_" + str(config.ddim_init_latents_t_idx) + "_nsteps_" + str(config.n_steps) + "_cfg_"
              + str(config.cfg) + "_pnpf" + str(config.pnp_f_t) + "_pnps" + str(config.pnp_spatial_attn_t) + "_pnpt"
              + str(config.pnp_temp_attn_t))
    return suffix + ("" if scheduler_name(config) == "ddim" else "_" + scheduler_name(config))


#: the edit schedulers of the optional config key ``scheduler``
EDIT_SCHEDULERS = ("ddim", "dpmsolver++")


def scheduler_name(config) -> str:
    name = str(config.get("scheduler", "ddim") if hasattr(config, "get") else getattr(config, "scheduler", "ddim"))
    if name not in EDIT_SCHEDULERS:
        raise ValueError(f"config key `scheduler`: {name!r} is not one of {list(EDIT_SCHEDULERS)}")
    return name


def edit_scheduler(ddim_scheduler, config):
    """the scheduler the edit samples with: ``scheduler: ddim`` (the default) the runner's DDIMScheduler, ``dpmsolver++`` a
    DPMSolverMultistepScheduler on the same config.  The inversion the edit reads stays DDIM: its store must hold every
    timestep of the edit's schedule (a 50-step inversion serves a 25-step DPM-Solver++ edit)."""
    if scheduler_name(config) == "ddim":
        return ddim_scheduler
    return DPMSolverMultistepScheduler.from_config(ddim_scheduler.config)


def load_source_frames(config):
    """reference :95-106: the PNG frames, else decode the mp4 (and save the frames next to it)."""
    from . import image_io
    try:
        logger.info("Loading frames from: %s", config.video_frames_path)
        _, frame_list = image_io.load_video_frames(config.video_frames_path, config.n_frames, config.image_size)
    except (OSError, ValueError) as e:
        logger.error("Failed to load frames from: %s (%s)", config.video_frames_path, e)
        logger.info("Converting mp4 video to frames: %s", config.video_path)
        frame_list = image_io.convert_video_to_frames(config.video_path, config.image_size, save_frames=True)[: config.n_frames]
    return frame_list


def start_latents(pipe, ddim_scheduler, config, device):
    """reference :113-132: x_t at ``ddim_init_latents_t_idx`` blended with ``random_ratio`` of noise from the global RNG,
    then the PnP hooks (:35-48) and the edit scheduler registered on the pipeline."""
    ddim_scheduler.set_timesteps(config.n_steps)
    logger.info("ddim_scheduler.timesteps: %s", ddim_scheduler.timesteps)
    t0 = int(ddim_scheduler.timesteps[config.ddim_init_latents_t_idx])
    ddim_latents_at_t = load_ddim_latents_at_t(t0, config.ddim_latents_path, map_location=device)
    random_latents = torch.randn_like(ddim_latents_at_t)
    logger.info("Blending random_ratio (1 means random latent): %s", config.random_ratio)
    mixed = random_latents * config.random_ratio + ddim_latents_at_t * (1 - config.random_ratio)
    init_pnp(pipe, ddim_scheduler, config)
    pipe.register_modules(scheduler=ddim_scheduler)
    return mixed


def clip_key(config, rank_seed_offset: int = 0):
    """what the source branch of an entry's edit is computed from, as the config names it: entries with equal keys edit the
    same clip from the same inversion.  Synthetic entries draw their source stand-ins from their own seed."""
    key = (config.ddim_latents_path, config.video_dir, config.video_name, tuple(config.image_size), config.n_frames,
           config.target_fps, config.n_steps, config.seed, config.get("synthetic", False))
    if config.get("synthetic", False):
        return key + (rank_seed_offset,)
    return key + (config.ddim_inv_prompt,)


class SharedSourceFeatures:
    """``share_source_features: true``: one SourceFeatureCache for consecutive entries of the same clip and inversion
    (clip_key), dropped when the clip changes.  ``source_features_max_gb`` (default 24) bounds it."""

    def __init__(self):
        self.key, self.cache = None, None

    def for_entry(self, pipe, config, rank_seed_offset: int = 0):
        if not config.get("share_source_features", False):
            return None
        key = clip_key(config, rank_seed_offset)
        if key != self.key:
            self.cache = None  # the previous clip's features are released before the next ones are made
            self.key, self.cache = key, pipe.source_feature_cache(int(float(config.get("source_features_max_gb", 24)) * 2**30))
        return self.cache


def edit_one(pipe, ddim_scheduler, config, device, rank_seed_offset: int = 0, source_features=None):
    ddim_scheduler = edit_scheduler(ddim_scheduler, config)
    config.video_path = os.path.join(config.video_dir, config.video_name + ".mp4")
    config.video_frames_path = os.path.join(config.video_dir, config.video_name)
    config.edited_first_frame_path = os.path.join(config.data_dir, config.edited_first_frame_path)
    for k, v in config.items():
        if "ReplaceMe" in str(v):
            logger.error("Field %s contains 'ReplaceMe'", k)
    if not config.get("synthetic", False):
        return edit_one_real(pipe, ddim_scheduler, config, device, source_features)
    h, w = config.image_size[1] // 8, config.image_size[0] // 8
    cross_dim = pipe.unet.config["cross_attention_dim"]
    cond = synthetic_conditioning(config.n_frames, h, w, cross_dim, config.seed + rank_seed_offset, device)
    mixed = start_latents(pipe, ddim_scheduler, config, device)
    store = LatentStore(config.ddim_latents_path, write_files=False)
    out = pipe.sample_with_pnp(
        latents=mixed, prompt_embeds=cond["edit_prompt"], negative_prompt_embeds=cond["neg_prompt"],
        ddim_inv_prompt_embeds=cond["inv_prompt"], image_embeddings=cond["edit_image_emb"],
        image_latents=cond["edit_image_latents"], ddim_inv_image_embeddings=cond["src_image_emb"],
        ddim_inv_image_latents=cond["src_image_latents"], num_frames=config.n_frames,
        num_inference_steps=config.n_steps, guidance_scale=config.cfg, target_fps=config.target_fps,
        ddim_init_latents_t_idx=config.ddim_init_latents_t_idx, ddim_inv_latents_path=config.ddim_latents_path,
        latent_store=store, output_type="latent", source_features=source_features).frames
    output_dir = os.path.join(config.output_dir, config_suffix(config))
    os.makedirs(output_dir, exist_ok=True)
    torch.save(out.cpu(), os.path.join(output_dir, "edited_latents.pt"))
    logger.info("Saved edited latents to: %s", output_dir)
    return out


def edit_one_real(pipe, ddim_scheduler, config, device, source_features=None):
    """reference :95-183 on real inputs: frames + edited first frame + prompts -> edited video files."""
    from . import image_io
    Image = image_io._pil()
    if pipe.encoders is None or pipe.vae is None:
        raise ValueError("real inputs need `encoders` and `vae` on the pipeline (build_pipeline(..., with_encoders=True)); set "
                         "`synthetic: true` in the config for the seeded stand-ins")
    size = tuple(int(v) for v in config.image_size)
    src_frame_list = load_source_frames(config)
    src_1st_frame = src_frame_list[0]
    edited_1st_frame = image_io.load_image(config.edited_first_frame_path).resize(size, resample=Image.Resampling.LANCZOS)
    mixed = start_latents(pipe, ddim_scheduler, config, device)
    latents = pipe.sample_with_pnp(
        prompt=config.editing_prompt, image=edited_1st_frame, height=size[1], width=size[0], num_frames=config.n_frames,
        num_inference_steps=config.n_steps, guidance_scale=config.cfg, negative_prompt=config.editing_negative_prompt,
        target_fps=config.target_fps, latents=mixed, generator=torch.Generator(device=device).manual_seed(config.seed),
        return_dict=True, ddim_init_latents_t_idx=config.ddim_init_latents_t_idx,
        ddim_inv_latents_path=config.ddim_latents_path, ddim_inv_prompt=config.ddim_inv_prompt,
        ddim_inv_1st_frame=src_1st_frame, output_type="latent", source_features=source_features).frames
    video = pipe.decode_latents(latents)                                  # [1, 3, f, H, W] in [-1, 1]
    frames = image_io.frames_to_pil(video[0].permute(1, 0, 2, 3))
    output_dir = os.path.join(config.output_dir, config_suffix(config))
    os.makedirs(output_dir, exist_ok=True)
    frames = [f.resize(size, resample=Image.LANCZOS) for f in frames]
    name = "video"
    image_io.export_to_video(frames, os.path.join(output_dir, f"{name}.mp4"), fps=config.target_fps)
    image_io.export_to_gif(frames, os.path.join(output_dir, f"{name}.gif"))
    for i, frame in enumerate(frames):
        frame.save(os.path.join(output_dir, f"{name}_{i:05d}.png"))
    torch.save(latents.cpu(), os.path.join(output_dir, "edited_latents.pt"))
    logger.info("Saved video, gif, %d frames and the edited latents to: %s", len(frames), output_dir)
    return latents


def load_checkpoint_into(module: torch.nn.Module, folder: str) -> bool:
    """diffusers-layout weights (``diffusion_pytorch_model[.fp16].safetensors`` / ``.bin``) -> ``module`` (same parameter
    names as diffusers, so the state_dict loads unchanged).  False when the folder has no weight file."""
    for name in ("diffusion_pytorch_model.fp16.safetensors", "diffusion_pytorch_model.safetensors",
                 "diffusion_pytorch_model.fp16.bin", "diffusion_pytorch_model.bin"):
        path = os.path.join(folder, name)
        if not os.path.exists(path):
            continue
        if path.endswith(".safetensors"):
            from safetensors.torch import load_file
            sd = load_file(path)
        else:
            sd = torch.load(path, map_location="cpu")
        # pre-0.20 VAE attention names
        ren = {"query": "to_q", "key": "to_k", "value": "to_v", "proj_attn": "to_out.0"}
        sd = {".".join(ren.get(p, p) if ".attentions." in k else p for p in k.split(".")): v for k, v in sd.items()}
        module.load_state_dict(sd, strict=True)
        logger.info("loaded %s", path)
        return True
    return False


def vae_sample_size(folder: str) -> dict:
    """``{"sample_size": ...}`` from a diffusers-layout ``vae/config.json`` (the tile size of VAE tiling), or {} without one"""
    path = os.path.join(folder, "config.json")
    if not os.path.exists(path):
        return {}
    with open(path) as f:
        cfg = json.load(f)
    return {"sample_size": cfg["sample_size"]} if "sample_size" in cfg else {}


def build_pipeline(device, unet_config=None, seed: int = 8888, broadcast: bool = True, with_encoders: bool = False,
                   model_dir: str | None = None, vae_config=None, clip_arch=None):
    """The pipeline of reference :59-66 (``I2VGenXLPipeline.from_pretrained("ali-vilab/i2vgen-xl", fp16)``).  ``model_dir``
    = a local diffusers-layout checkpoint directory; without one (no network here) every model is seeded random-init.
    Under torchrun rank 0 builds the UNet weights and every other rank receives them by ONE NCCL broadcast of the flat
    fp16 buffer (anyv2v_b200.distributed).  ``with_encoders`` adds the VAE and the CLIP towers (real-input path)."""
    from . import distributed
    from .unet_i2vgen_xl import I2VGEN_XL_CONFIG, I2VGenXLUNet
    cfg = dict(unet_config or I2VGEN_XL_CONFIG)
    have_ckpt = bool(model_dir) and os.path.isdir(model_dir)
    unet = distributed.build_unet_replicated(I2VGenXLUNet, cfg, seed, device, broadcast=broadcast,
                                             checkpoint_dir=os.path.join(model_dir, "unet") if have_ckpt else None)
    if not have_ckpt:
        logger.warning("no local checkpoint directory (model_name=%r): seeded RANDOM-INIT weights", model_dir)
    pipe = I2VGenXLPipeline(unet, DDIMScheduler())
    if with_encoders:
        from .encoders import ClipEncoders
        from .vae import SD_VAE_CONFIG as KL_F8_CONFIG, AutoencoderKL
        vae_kwargs = dict(vae_config or KL_F8_CONFIG)
        if have_ckpt and "sample_size" not in vae_kwargs:
            vae_kwargs.update(vae_sample_size(os.path.join(model_dir, "vae")))
        state = torch.random.get_rng_state()
        torch.manual_seed(seed + 7)
        try:
            vae = AutoencoderKL(**vae_kwargs)
        finally:
            torch.random.set_rng_state(state)
        if have_ckpt:
            load_checkpoint_into(vae, os.path.join(model_dir, "vae"))
            enc = ClipEncoders.from_pretrained(model_dir, device=device)
        else:
            enc = ClipEncoders.random_init(cfg["cross_attention_dim"], seed=seed + 11, device=device, arch=clip_arch)
        pipe.vae = vae.to(device=device, dtype=torch.float16).eval()
        pipe.encoders = enc
    return pipe


def _model_dir(template_config):
    """``model_name`` is a hub id in the reference's templates ("i2vgen-xl"); a local directory is used when it is one,
    optionally relative to ``data_dir``."""
    name = str(template_config.get("model_name", "") or "")
    for cand in (name, os.path.join(str(template_config.get("data_dir", ".")), name)):
        if cand and os.path.isdir(os.path.join(cand, "unet")):
            return cand
    return None


def run_sharded(build, template_config, configs_list, device, run_entry, unet_config=None, pipeline_kwargs=None):
    """The group loop of both runners (reference :74-81): one pipeline from ``build`` (``build_pipeline`` as the calling
    runner module names it, so either runner's builder can be replaced on its own) for every entry, with the CLIP towers
    and the VAE when any active entry takes real inputs, and ``run_entry(pipe, config, i)`` on the template merged with the
    i-th active entry.  Entry i runs on rank i % world.  Returns the results that are not None."""
    from . import distributed
    rank, world = distributed.rank_world()
    active = [e for e in configs_list if e.get("active", True)]
    need_real = any(not OmegaConf.merge(template_config, OmegaConf.create(e)).get("synthetic", False) for e in active)
    pipe = build(device, unet_config, seed=template_config.seed, with_encoders=need_real,
                 model_dir=_model_dir(template_config), **(pipeline_kwargs or {}))
    for e in configs_list:
        if not e.get("active", True):
            logger.info("Skipping config_entry: %s", e)
    results = []
    for i, entry in enumerate(active):
        if i % world != rank:  # clips shard one-per-GPU; no data-path collective (SURVEY 8e)
            continue
        logger.info("Processing config_entry: %s", entry)
        out = run_entry(pipe, OmegaConf.merge(template_config, OmegaConf.create(entry)), i)
        if out is not None:
            results.append(out)
    return results


def main(template_config, configs_list, device, unet_config=None, pipeline_kwargs=None):
    ddim_scheduler = DDIMScheduler.from_pretrained("ali-vilab/i2vgen-xl", subfolder="scheduler")
    shared = SharedSourceFeatures()
    return run_sharded(build_pipeline, template_config, configs_list, device,
                       lambda pipe, config, i: edit_one(pipe, ddim_scheduler, config, device, rank_seed_offset=i,
                                                        source_features=shared.for_entry(pipe, config, i)),
                       unet_config, pipeline_kwargs)


def cli(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("--template_config", type=str, default="./configs/group_pnp_edit/template.yaml")
    parser.add_argument("--configs_json", type=str, default="./configs/group_config.json")
    args = parser.parse_args(argv)
    template_config = OmegaConf.load(args.template_config)
    logging.basicConfig(level=logging.DEBUG if template_config.debug else logging.INFO,
                        format="%(asctime)s - %(levelname)s - [%(funcName)s] - %(message)s")
    logger.info("template_config: %s", OmegaConf.to_yaml(template_config))
    assert Path(args.configs_json).exists()
    with open(args.configs_json, "r") as fh:
        configs_list = json.load(fh)
    logger.info("Loaded %d configs from %s", len(configs_list), args.configs_json)
    from . import distributed
    device = distributed.pick_device(template_config.device)
    torch.set_grad_enabled(False)
    seed_everything(template_config.seed)
    return main(template_config, configs_list, device)


if __name__ == "__main__":
    cli()
