"""Group runner, phase 1 — drop-in for the reference's ``i2vgen-xl/run_group_ddim_inversion.py``.

Same CLI (:195-198), same template keys (configs/group_ddim_inversion/template.yaml: ``inverse_config.{cfg,
target_fps, prompt, negative_prompt, n_steps, output_dir, ...}``, ``recon_config.*``), same skip rule (existing
``output_dir`` and not ``force_recompute_latents``; :118-120) and the same per-timestep ``ddim_latents_{t}.pt`` files
(pipeline :1424-1428).  ``ddim_inversion(config, first_frame, frame_list, pipe, inverse_scheduler, g)`` keeps the
reference signature (:29) and return value (``[steps, c, f, h, w]``, :54): with PIL ``first_frame`` / ``frame_list`` it runs
the real path (VAE-encode the frames, CLIP-encode prompt and first frame — the pipeline must carry ``encoders`` and
``vae``); ``cond=`` (pre-encoded tensors) is the ``synthetic: true`` opt-in of SURVEY 8d.  The source frames are read like the
reference does (:125-139; png frames, mp4 fallback), incl. ``inverse_static_video`` / ``null_image_inversion`` (:143-151).
"""
from __future__ import annotations

import argparse
import json
import logging
import os
from pathlib import Path

import torch

from .config import OmegaConf
from .pipeline import I2VGenXLPipeline
from .run_group_pnp_edit import build_pipeline, load_source_frames, run_sharded, seed_everything, synthetic_conditioning
from .schedulers import DDIMInverseScheduler, DDIMScheduler

logger = logging.getLogger(__name__)


def ddim_inversion(config, first_frame, frame_list, pipe: I2VGenXLPipeline, inverse_scheduler, g, cond=None):
    """reference :29-55.  Returns the inverted latents of the clip, [steps, c, f, h, w] (descending t), like :54."""
    pipe.scheduler = inverse_scheduler
    if cond is not None:  # synthetic opt-in: pre-encoded conditioning
        return pipe.invert(
            latents=cond["video_latents"], prompt_embeds=cond["inv_prompt"], negative_prompt_embeds=cond.get("neg_prompt"),
            image_latents=cond["src_image_latents"], image_embeddings=cond["src_image_emb"], num_frames=config.n_frames,
            num_inference_steps=config.n_steps, guidance_scale=config.cfg, target_fps=config.target_fps,
            output_dir=config.output_dir, return_dict=False)[0]
    if first_frame is None or frame_list is None:
        raise ValueError("ddim_inversion needs the source frames (PIL) or `cond=` (pre-encoded, `synthetic: true`)")
    width, height = int(config.image_size[0]), int(config.image_size[1])
    video_latents_at_0 = pipe.encode_vae_video(frame_list, device=pipe._execution_device, height=height, width=width, generator=g)
    return pipe.invert(
        prompt=config.prompt, image=first_frame, height=height, width=width, num_frames=config.n_frames,
        num_inference_steps=config.n_steps, guidance_scale=config.cfg, negative_prompt=config.negative_prompt,
        target_fps=config.target_fps, latents=video_latents_at_0, generator=g, return_dict=False,
        output_dir=config.output_dir)[0]


def ddim_sampling(config, first_frame, ddim_latents_path, pipe, ddim_scheduler, ddim_init_latents_t_idx, g, cond=None):
    """reference :58-77 (DDIM reconstruction, the authors' sanity check): ``pipe(...)`` from x_t, without hooks.  Returns the
    reconstructed latents [1, 4, F, h, w]; with PIL ``first_frame`` (real inputs) also the decoded frames, else None."""
    from .latent_store import load_ddim_latents_at_t
    ddim_scheduler.set_timesteps(config.n_steps)
    t0 = ddim_scheduler.timesteps.tolist()[ddim_init_latents_t_idx]
    latents = load_ddim_latents_at_t(t0, ddim_latents_path, map_location=pipe.device)
    pipe.scheduler = ddim_scheduler
    common = dict(num_frames=config.n_frames, num_inference_steps=config.n_steps, guidance_scale=config.cfg,
                  target_fps=config.target_fps, latents=latents, generator=g, ddim_init_latents_t_idx=ddim_init_latents_t_idx,
                  output_type="latent", return_dict=True)
    if cond is not None:  # synthetic opt-in: pre-encoded conditioning
        rec = pipe(prompt_embeds=cond["inv_prompt"], negative_prompt_embeds=cond["neg_prompt"],
                   image_embeddings=cond["src_image_emb"], image_latents=cond["src_image_latents"], **common).frames
        return rec, None
    from .pipeline import tensor2vid
    rec = pipe(prompt=config.prompt, image=first_frame, height=int(config.image_size[1]), width=int(config.image_size[0]),
               negative_prompt=config.negative_prompt, **common).frames
    return rec, tensor2vid(pipe.decode_latents(rec, decode_chunk_size=1), "pil")[0]


def main(template_config, configs_list, device, unet_config=None, pipeline_kwargs=None):
    assert len(configs_list) > 0
    g = torch.Generator(device=device).manual_seed(template_config.seed)
    inverse_scheduler = DDIMInverseScheduler.from_pretrained("ali-vilab/i2vgen-xl", subfolder="scheduler")
    ddim_scheduler = DDIMScheduler.from_pretrained("ali-vilab/i2vgen-xl", subfolder="scheduler")

    def run_entry(pipe, config, i):
        config.video_path = os.path.join(config.video_dir, config.video_name + ".mp4")
        config.video_frames_path = os.path.join(config.video_dir, config.video_name)
        if os.path.exists(config.output_dir) and not config.get("force_recompute_latents", False):
            logger.info("= Inverted latents already exist at %s. Skip.", config.output_dir)
            return None
        if config.get("synthetic", False):
            h, w = config.image_size[1] // 8, config.image_size[0] // 8
            cond = synthetic_conditioning(config.n_frames, h, w, pipe.unet.config["cross_attention_dim"], config.seed + i, device)
            inv = ddim_inversion(config.inverse_config, None, None, pipe, inverse_scheduler, g, cond=cond)
        else:
            from PIL import Image

            from . import image_io
            cond = None
            frame_list = load_source_frames(config)
            if not os.path.exists(os.path.join(config.video_frames_path, config.video_name + ".gif")):
                try:  # reference :137-141 saves the source frames as a gif next to them
                    image_io.export_to_gif(frame_list, os.path.join(config.video_frames_path, config.video_name + ".gif"))
                except OSError as e:
                    logger.info("source gif not written (%s)", e)
            first_frame = frame_list[0]
            if config.inverse_config.get("inverse_static_video", False):
                logger.info("### Inverse a static video!")
                frame_list = [frame_list[0]] * config.n_frames
            if config.inverse_config.get("null_image_inversion", False):
                logger.info("### Inverse a null image!")
                first_frame = Image.new("RGB", (config.image_size[0], config.image_size[1]), (0, 0, 0))
            inv = ddim_inversion(config.inverse_config, first_frame, frame_list, pipe, inverse_scheduler, g)
        rc = config.recon_config
        if rc.enable_recon:
            rec, frames = ddim_sampling(rc, None if cond is not None else first_frame, rc.ddim_latents_path, pipe,
                                        ddim_scheduler, rc.ddim_init_latents_t_idx, g, cond=cond)
            os.makedirs(os.path.join(config.output_dir, "ddim_reconstruction"), exist_ok=True)
            torch.save(rec.cpu(), os.path.join(config.output_dir, "ddim_reconstruction", "latents.pt"))
            if frames is not None:  # reference :180-192: down-sampled for space, mp4 at 10 fps + gif
                from PIL import Image

                from . import image_io
                frames = [f.resize((512, 512), resample=Image.LANCZOS) for f in frames]
                image_io.export_to_video(frames, os.path.join(config.output_dir, "ddim_reconstruction.mp4"), fps=10)
                image_io.export_to_gif(frames, os.path.join(config.output_dir, "ddim_reconstruction.gif"))
                logger.info("Saved reconstructed video to %s", config.output_dir)
        return inv
    return run_sharded(build_pipeline, template_config, configs_list, device, run_entry, unet_config, pipeline_kwargs)


def cli(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("--template_config", type=str, default="./configs/group_ddim_inversion/template.yaml")
    parser.add_argument("--configs_json", type=str, default="./configs/group_ddim_inversion/group_config.json")
    args = parser.parse_args(argv)
    template_config = OmegaConf.load(args.template_config)
    logging.basicConfig(level=logging.DEBUG if template_config.debug else logging.INFO,
                        format="%(asctime)s - %(levelname)s - [%(funcName)s] - %(message)s")
    assert Path(args.configs_json).exists()
    with open(args.configs_json, "r") as fh:
        configs_list = json.load(fh)
    from . import distributed
    device = distributed.pick_device(template_config.device)
    torch.set_grad_enabled(False)
    seed_everything(template_config.seed)
    return main(template_config, configs_list, device)


if __name__ == "__main__":
    cli()
