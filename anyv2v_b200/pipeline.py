"""I2VGen-XL sampling loops, H100-native: ``invert``, ``sample_with_pnp`` and the image-to-video call ``pipe(...)``.

Drop-in for the hot loops of the reference's ``I2VGenXLPipeline`` (i2vgen-xl/pipelines/pipeline_i2vgen_xl.py):
  invert            :1197-1439 (loop :1385-1433)
  sample_with_pnp   :892-1195  (loop :1131-1179; also eta > 0)
  __call__          :652-890   (loop :839-874; also eta > 0)
with the same keyword surface for everything that reaches the loops.  Differences, none of which changes a result:
  * no host sync inside the loop: timesteps are Python ints (the reference calls ``t.item()`` at :1143 and runs
    ``t in tensor`` membership kernels inside every hook), inverted latents stay in HBM (anyv2v_b200.latent_store)
    instead of ``torch.save``/``torch.load`` per step (:1134, :1424-1428);
  * conditioning that does not depend on t (fps embedding, 145-token context, image-latent stem) is computed once
    per clip (``unet.precompute_conditioning``) instead of once per step;
  * CFG + scheduler step is one fused kernel (``scheduler.step(..., model_output_cond=...)``);
  * on steps where no injection fires, the source branch — whose prediction the reference discards at :1160 — is
    not run at all (every norm is per-sample, so the edit branches do not depend on it).
CLIP / VAE encoders are outside the hot path and the metric (SURVEY 8d, 8f rank 4): the loops take pre-encoded
tensors (``prompt_embeds``, ``image_embeddings``, ``image_latents`` ...) or — with ``encoders=`` (anyv2v_b200.encoders)
and ``vae=`` attached — the reference's raw inputs (prompt strings, PIL first frames), encoded once per clip.
"""
from __future__ import annotations

import gc
import logging
import os
from types import SimpleNamespace
from typing import Callable, Optional

import torch

from .latent_store import LatentStore
from .pnp_utils import _PNP_SITES, _fires, register_time
from .schedulers import randn_tensor
from .unet_i2vgen_xl import SourceFeature

logger = logging.getLogger(__name__)


def frame_position_latents(first_frame_latent: torch.Tensor, num_frames: int) -> torch.Tensor:
    """prepare_image_latents (pipeline :532-562) minus the VAE: [b,4,h,w] -> [b,4,F,h,w], frame k>=1 = k/(F-1)."""
    x = first_frame_latent.unsqueeze(2)
    if num_frames == 1:
        return x
    scale = torch.arange(1, num_frames, device=x.device, dtype=torch.float32) / (num_frames - 1)
    mask = torch.ones_like(x).expand(-1, -1, num_frames - 1, -1, -1) * scale.view(1, 1, -1, 1, 1).to(x.dtype)
    return torch.cat([x, mask], dim=2)


class _GraphedIteration:
    """One loop iteration captured as a CUDA graph (streams + graphs instead of a tracing compiler).

    The iteration body reads only static device buffers (latents, source latent, timestep, scheduler coefficients) so
    the same graph is replayed for every timestep with the same hook flags and FreeU setting.  The first use runs eagerly
    (allocates workspaces / packed weights, builds nothing under capture), the second captures, later ones replay."""

    def __init__(self, body, on_cuda: bool = True, pool=None):
        self.body = body      # () -> None, operating on static buffers
        self.graph = None
        self.calls = 0
        self.on_cuda = bool(on_cuda)   # where the body's tensors live (NOT whether the box has a GPU)
        self.pool = pool               # shared memory pool of the per-hook-flag graphs of one loop

    def run(self):
        self.calls += 1
        if self.calls == 1 or not self.on_cuda:
            self.body()
            return
        if self.graph is None:
            g = torch.cuda.CUDAGraph()
            # no cyclic garbage collection inside the capture: a finished loop's state is a reference cycle (its iterations'
            # bodies close over it), and collecting it there would destroy its CUDA graphs, which invalidates the capture
            gc_was_on = gc.isenabled()
            gc.disable()
            try:
                # thread_local: the latent-store writer thread may call cudaEventSynchronize while this thread captures
                with torch.cuda.graph(g, pool=self.pool, capture_error_mode="thread_local"):
                    self.body()
            finally:
                if gc_was_on:
                    gc.enable()
            self.graph = g
        self.graph.replay()


def _loop_state(latents, timesteps, scheduler, guidance_scale: float, device, eta: float = 0.0,
                **fields) -> SimpleNamespace:
    """What the three sampling loops keep per clip: the latents the steps update in place (a copy: the captured graphs read
    this tensor for the life of the state), the per-step timestep / scheduler-coefficient tables, the static buffers the
    step body reads them from, and the loop iterations (``I2VGenXLPipeline._run``) with their shared activation pool.  A
    multistep scheduler (DPMSolverMultistepScheduler) also gets ``x0_prev``, the previous step's x0 that its step reads and
    rewrites in place, allocated once so that the captured graphs keep its address; DDIM loops have none."""
    st = SimpleNamespace(latents=latents.to(device).contiguous().clone(), timesteps=timesteps, scheduler=scheduler, eta=eta,
                         **fields)
    st.t_table = torch.tensor(timesteps, device=device, dtype=torch.int64)
    st.coef_table = scheduler.coefficient_table(timesteps, guidance_scale, device, eta=eta)
    st.g_t = torch.zeros(1, device=device, dtype=torch.int64)
    st.g_coef = torch.zeros(st.coef_table.shape[-1], device=device, dtype=torch.float32)
    st.g_noise = torch.zeros_like(st.latents) if eta > 0 else None  # the step noise of eta > 0 (I2VGenXLPipeline._draw_noise)
    st.x0_prev = torch.zeros_like(st.latents) if getattr(scheduler, "multistep", False) else None
    st.iterations = {}  # graph key of the loop -> _GraphedIteration
    st.graph_pool = torch.cuda.graph_pool_handle() if st.latents.is_cuda else None
    return st


def _pnp_sites(unet):
    """[(name, site)] of the 17 PnP injection sites: the conv-injected resnet, then the spatial and the temporal attn1
    processors of up_blocks[1..3] (pnp_utils.py:130, 235, 340)"""
    sites = [("conv", unet.up_blocks[1].resnets[1])]
    for kind, attr in (("spatial", "attentions"), ("temporal", "temp_attentions")):
        for res, blocks in _PNP_SITES.items():
            for blk in blocks:
                sites.append((f"{kind}{res}.{blk}", getattr(unet.up_blocks[res], attr)[blk].transformer_blocks[0].attn1.processor))
    return sites


class SourceFeatureCache:
    """The source branch's features at the PnP injection sites, kept from one edit of an inverted clip for the later edits of
    the same clip (``I2VGenXLPipeline.source_feature_cache``; ``sample_with_pnp(..., source_features=cache)``).

    Branch 0 of the edit's [source, uncond, cond] batch runs the UNet on the stored inverted latents with the inversion's
    prompt and first frame: nothing of it depends on the edit, and only its features at the firing injection sites are read.
    An edit step whose (t, firing sites, FreeU state) the cache holds therefore runs the UNet on [uncond, cond] only, with the
    injection sites fed from the cache; any other injected step runs the three branches as without the cache and stores its
    source features, as long as they fit in ``max_bytes``.  Either way the edit's latents are bit-identical to those of the
    same edit without the cache.  What the cache stores per site: the normed tokens at the spatial and temporal attn1 sites
    (Q and K are re-projected from them), conv2's input at the conv site; about 430 MB for a step with all three injections
    at 16 x 512 x 512, in proportion to frames x h x w.

    The cache belongs to one clip and one inversion: its first edit records the latent store (or ``ddim_inv_latents_path``),
    the inversion prompt, first-frame embeddings and latents, ``target_fps``, the latents' frames x h x w and the UNet, and
    an edit that differs in any of them raises ValueError.  The edit prompt, the edited first frame, the injection schedules,
    guidance and eta may change from edit to edit."""

    def __init__(self, unet, max_bytes: int):
        if max_bytes < 0:
            raise ValueError(f"max_bytes must be >= 0, got {max_bytes}")
        self.unet = unet
        self.max_bytes = int(max_bytes)
        self.nbytes = 0
        self.entries = {}     # (t, firing sites, FreeU state) -> {site name: feature}
        self.features = {}    # site name -> SourceFeature: the static buffers the (captured) steps read and write
        self._identity = None

    def __len__(self):
        return len(self.entries)

    def bind(self, store_id, prompt_embeds, image_embeddings, image_latents, target_fps, frames_hw, unet):
        """records what the source branch is computed from on the first edit; raises ValueError when a later edit differs"""
        tensors = (prompt_embeds, image_embeddings, image_latents)
        if unet is not self.unet:
            raise ValueError("source_features: the cache was made for another UNet")
        if self._identity is None:
            self._identity = (store_id, tuple(t.detach().clone() for t in tensors), int(target_fps), tuple(frames_hw))
            return
        sid, ref, fps, fhw = self._identity
        same_store = sid[0] == store_id[0] and (sid[1] == store_id[1] if sid[0] == "path" else sid[1] is store_id[1])
        if not same_store:
            raise ValueError("source_features: the cache holds the features of another inversion (latent store / "
                             "ddim_inv_latents_path differs)")
        for name, a, b in zip(("ddim_inv_prompt_embeds", "ddim_inv_image_embeddings", "ddim_inv_image_latents"), ref, tensors):
            if a.shape != b.shape or not torch.equal(a, b.to(device=a.device, dtype=a.dtype)) or a.dtype != b.dtype:
                raise ValueError(f"source_features: `{name}` differs from the edit the cache was filled by")
        if fps != int(target_fps):
            raise ValueError(f"source_features: target_fps {target_fps} differs from the cache's {fps}")
        if fhw != tuple(frames_hw):
            raise ValueError(f"source_features: frames x h x w {tuple(frames_hw)} differs from the cache's {fhw}")

    def _feature(self, name):
        f = self.features.get(name)
        if f is None:
            f = self.features[name] = SourceFeature()
        return f

    def begin_step(self, key, sites):
        """-> "replay" (the cache holds ``key``: its features are copied to the static buffers), "capture" (the firing sites
        store their source features) or None (they would not fit); attaches the sites' features in that mode"""
        firing = [name for (name, _), f in zip(sites, key[1]) if f]
        entry = self.entries.get(key)
        if entry is not None:
            mode = "replay"
            for name in firing:
                self.features[name].buf.copy_(entry[name])
        else:
            known = [self.features[n].buf for n in firing if n in self.features and self.features[n].buf is not None]
            need = sum(b.numel() * b.element_size() for b in known)
            mode = "capture" if self.nbytes + need <= self.max_bytes else None
        for name, site in sites:
            feat = self._feature(name)
            feat.mode = mode
            site.source_feature = feat
        return mode

    def end_step(self, key, sites, mode):
        """detaches the sites; after a capture, keeps the step's features if they fit"""
        for _, site in sites:
            site.source_feature = None
        if mode != "capture":
            return
        firing = [name for (name, _), f in zip(sites, key[1]) if f]
        bufs = {n: self.features[n].buf for n in firing}
        need = sum(b.numel() * b.element_size() for b in bufs.values())
        if self.nbytes + need <= self.max_bytes:
            self.entries[key] = {n: b.clone() for n, b in bufs.items()}
            self.nbytes += need


def tensor2vid(video: torch.Tensor, output_type: str = "np"):
    """pipeline_i2vgen_xl.py:79-97 with diffusers' `VaeImageProcessor.postprocess` (do_normalize=True) inlined:
    video [b, 3, f, H, W] in [-1, 1] -> "pt": [b, f, 3, H, W] in [0, 1]; "np": float32 [b, f, H, W, 3]; "pil": list (per
    batch entry) of lists of PIL images."""
    if output_type not in ("np", "pt", "pil"):
        raise ValueError(f"{output_type} does not exist. Please choose one of ['np', 'pt', 'pil]")
    outputs = []
    for batch_vid in video.permute(0, 2, 1, 3, 4):             # [f, 3, H, W] per batch entry
        img = (batch_vid / 2 + 0.5).clamp(0, 1)
        if output_type == "pt":
            outputs.append(img)
            continue
        arr = img.detach().cpu().permute(0, 2, 3, 1).float().numpy()
        if output_type == "np":
            outputs.append(arr)
        else:
            from PIL import Image
            outputs.append([Image.fromarray(a) for a in (arr * 255).round().astype("uint8")])
    if output_type == "np":
        import numpy as np
        return np.stack(outputs)
    if output_type == "pt":
        return torch.stack(outputs)
    return outputs


class I2VGenXLPipeline:
    #: replay loop iterations as CUDA graphs (set False to run every kernel launch eagerly)
    use_cuda_graphs = os.environ.get("AV2V_CUDA_GRAPHS", "1") != "0"

    def __init__(self, unet, scheduler=None, encoders: Optional[SimpleNamespace] = None, vae=None):
        self.unet = unet
        self.scheduler = scheduler
        self.vae = vae  # optional anyv2v_b200.vae.AutoencoderKL (or any module with diffusers' encode/decode protocol)
        self.encoders = encoders  # optional: .encode_prompt(str)->[1,77,D], .encode_image(img)->[1,1,D], .encode_vae(img)->[1,4,h,w]
        self.latent_store: Optional[LatentStore] = None
        self._guidance_scale = 1.0

    # -- small diffusers-pipeline surface the runners touch ---------------------------------------------------------
    @property
    def device(self):
        return next(self.unet.parameters()).device

    _execution_device = device

    @property
    def do_classifier_free_guidance(self):
        return self._guidance_scale > 1

    def to(self, device):
        self.unet.to(device)
        return self

    # -- the steps either side of the loops (SURVEY 8f row 4) ------------------------------------------------------
    def decode_latents(self, latents, decode_chunk_size=None):
        """pipeline_i2vgen_xl.py:443-463."""
        if self.vae is None:
            raise ValueError("decode_latents needs a VAE: construct the pipeline with `vae=` (anyv2v_b200.vae.AutoencoderKL)")
        from . import vae as vae_mod
        return vae_mod.decode_latents(self.vae, latents, decode_chunk_size)

    def encode_vae_video(self, video, device=None, height: Optional[int] = None, width: Optional[int] = None, generator=None):
        """pipeline_i2vgen_xl.py:565-592: ``video`` is the reference's list of PIL frames (each center-cropped-wide to
        (width, height) and mapped to [-1, 1], :578-580) or an already pre-processed tensor [f, 3, H, W] in [-1, 1];
        -> video latents [1, 4, f, H/8, W/8].  All frames go through the VAE in one batch."""
        if self.vae is None:
            raise ValueError("encode_vae_video needs a VAE: construct the pipeline with `vae=`")
        from . import image_io
        from . import vae as vae_mod
        if not torch.is_tensor(video):
            if height is None or width is None:
                width, height = video[0].size
            video = image_io.preprocess(image_io.center_crop_wide(list(video), (width, height)))
        p0 = next(self.vae.parameters())
        return vae_mod.encode_vae_video(self.vae, video.to(device=p0.device, dtype=p0.dtype), generator)

    # -- once-per-clip conditioning from raw inputs (pipeline :1318-1352 / :1014-1094) ----------------------------
    def encode_prompt(self, prompt):
        """pipeline :219-394 for this path (one prompt string, no LoRA, no clip_skip) -> [1, 77, D]."""
        if self.encoders is None:
            raise ValueError("a prompt STRING was given but the pipeline has no `encoders` (anyv2v_b200.encoders.ClipEncoders): "
                             "attach them or pass `prompt_embeds`")
        return self.encoders.encode_prompt(prompt).to(self.device)

    def encode_first_frame(self, image, height: int, width: int, num_frames: int, generator=None):
        """The image half of the conditioning: CLIP image embedding of the square crop (:1318-1322, `_encode_image`
        :395-412) and the VAE latent of the (width, height) crop with the frame-position planes appended
        (`prepare_image_latents` :532-562) -> (image_embeddings [1, 1, D], image_latents [1, 4, F, h, w])."""
        if self.encoders is None or self.vae is None:
            raise ValueError("a first-frame IMAGE was given but the pipeline lacks `encoders` and/or `vae`: attach them or pass "
                             "`image_embeddings` / `image_latents`")
        from . import image_io
        emb = self.encoders.encode_image(image, width).to(self.device)
        x = image_io.preprocess(image_io.center_crop_wide(image, (width, height))).to(device=self.device, dtype=next(self.vae.parameters()).dtype)
        lat = self.vae.encode(x).latent_dist.sample(generator) * self.vae.config.scaling_factor
        return emb, frame_position_latents(lat.to(emb.dtype), num_frames)

    def _size_of(self, image, height, width):
        if (height is None or width is None) and image is not None and hasattr(image, "size"):
            width, height = image.size
        return height, width

    def _encode(self, prompt, negative_prompt, image, height, width, num_frames, generator, need_negative: bool,
                prompt_embeds=None, negative_prompt_embeds=None, image_embeddings=None, image_latents=None):
        """-> (prompt_embeds, negative_prompt_embeds, image_embeddings, image_latents), each encoded from the raw input
        unless given.  The negative prompt ("" when None, :348-352) is encoded only when ``need_negative``; ``generator``
        samples the first-frame VAE latent."""
        if prompt_embeds is None and prompt is not None:
            prompt_embeds = self.encode_prompt(prompt)
        if need_negative and negative_prompt_embeds is None:
            negative_prompt_embeds = self.encode_prompt(negative_prompt if negative_prompt is not None else "")
        if image is not None and (image_embeddings is None or image_latents is None):
            emb, lat = self.encode_first_frame(image, *self._size_of(image, height, width), num_frames, generator)
            image_embeddings = emb if image_embeddings is None else image_embeddings
            image_latents = lat if image_latents is None else image_latents
        return prompt_embeds, negative_prompt_embeds, image_embeddings, image_latents

    def enable_freeu(self, s1: float, s2: float, b1: float, b2: float):
        """FreeU (arXiv:2309.11497), pipeline_i2vgen_xl.py:623-650: forwarded to ``unet.enable_freeu``.  s1 / s2 scale the low
        frequencies of the skip features of up blocks 0 / 1, b1 / b2 the first half of their backbone channels.  Applies to
        ``invert`` and ``sample_with_pnp``, also when switched between steps (e.g. from ``callback``)."""
        if getattr(self, "unet", None) is None:
            raise ValueError("The pipeline must have `unet` for using FreeU.")
        self.unet.enable_freeu(s1=s1, s2=s2, b1=b1, b2=b2)

    def disable_freeu(self):
        """Disables FreeU if enabled (pipeline_i2vgen_xl.py:646-648)."""
        self.unet.disable_freeu()

    # -- VAE memory knobs (pipeline_i2vgen_xl.py:191-222), forwarded to the VAE ------------------------------------------
    def _require_vae(self):
        if self.vae is None:
            raise ValueError("The pipeline must have `vae` for VAE slicing / tiling: construct it with `vae=`")
        return self.vae

    def enable_vae_slicing(self):
        """Encode and decode one frame per VAE pass: the same frames, with the memory of one frame."""
        self._require_vae().enable_slicing()

    def disable_vae_slicing(self):
        """Back to one VAE pass for all frames."""
        self._require_vae().disable_slicing()

    def enable_vae_tiling(self):
        """Encode and decode frames larger than the VAE's ``tile_sample_min_size`` in overlapping tiles with blended seams
        (diffusers' tiled VAE): the memory of a VAE pass no longer grows with the frame size."""
        self._require_vae().enable_tiling()

    def disable_vae_tiling(self):
        """Back to whole-frame encode and decode."""
        self._require_vae().disable_tiling()

    def source_feature_cache(self, max_bytes: int) -> SourceFeatureCache:
        """A cache of the source branch's injection-site features for several PnP edits of one inverted clip: pass it as
        ``sample_with_pnp(..., source_features=cache)`` to every edit; after the first, the injected steps it holds run the UNet
        on two branches instead of three, with bit-identical results.  ``max_bytes`` bounds its device memory (about 430 MB
        per fully injected step at 16 x 512 x 512)."""
        return SourceFeatureCache(self.unet, max_bytes)

    def register_modules(self, **kwargs):
        for k, v in kwargs.items():
            setattr(self, k, v)

    def check_inputs(self, prompt_embeds, image_latents, image_embeddings, latents):
        # mirrors the ValueError convention of pipeline :483-530 for the tensors this path takes
        for name, t in (("prompt_embeds", prompt_embeds), ("image_latents", image_latents),
                        ("image_embeddings", image_embeddings), ("latents", latents)):
            if t is None:
                raise ValueError(f"`{name}` is required: pass it pre-encoded, or give the raw prompt / image to a pipeline built "
                                 f"with `encoders=` (anyv2v_b200.encoders.ClipEncoders) and `vae=`.")
        if latents.dim() != 5 or latents.shape[1] != self.unet.config["in_channels"]:
            raise ValueError(f"`latents` must be [b, {self.unet.config['in_channels']}, f, h, w], got {tuple(latents.shape)}")
        if image_latents.shape[2:] != latents.shape[2:]:
            raise ValueError("`image_latents` and `latents` must agree in (frames, h, w)")

    def _any_hook_fires(self, t) -> bool:
        mod = self.unet.up_blocks[1].resnets[1]
        if _fires(t, getattr(mod, "_injection_set", None)):
            return True
        for res in (1, 2, 3):
            up = self.unet.up_blocks[res]
            for blk in range(3):
                for proc in (up.attentions[blk].transformer_blocks[0].attn1.processor,
                             up.temp_attentions[blk].transformer_blocks[0].attn1.processor):
                    if _fires(t, getattr(proc, "_injection_set", None)):
                        return True
        return False

    # -- what the three loops share ----------------------------------------------------------------------------------
    def _run(self, st, i: int, key, make_body):
        """Step i's timestep and scheduler coefficients into the static buffers, then the loop iteration for ``key`` (what
        the captured graph bakes in: hook flags, FreeU setting ...; its body from ``make_body()`` on first use), replayed
        as a CUDA graph unless ``use_cuda_graphs`` is off."""
        st.g_t.copy_(st.t_table[i:i + 1])
        st.g_coef.copy_(st.coef_table[i])
        it = st.iterations.get(key)
        if it is None:
            it = st.iterations[key] = _GraphedIteration(make_body(), on_cuda=st.latents.is_cuda, pool=st.graph_pool)
        if self.use_cuda_graphs:
            it.run()
        else:
            it.body()
        return st.latents

    @staticmethod
    def _loop(st, step, callback, max_steps):
        """``step(st, i)`` for the first ``max_steps`` timesteps (all by default), each followed by ``callback(i, t, latents)``."""
        n = len(st.timesteps) if max_steps is None else min(max_steps, len(st.timesteps))
        for i in range(n):
            step(st, i)
            if callback is not None:
                callback(i, st.timesteps[i], st.latents)

    def _output(self, latents, output_type, return_dict, decode_chunk_size):
        """"latent" -> the latents; "pt" / "np" / "pil" -> the video decoded by the attached VAE."""
        if output_type == "latent":
            frames = latents
        else:
            frames = tensor2vid(self.decode_latents(latents, decode_chunk_size=decode_chunk_size), output_type)
        return SimpleNamespace(frames=frames) if return_dict else (frames,)

    # -- image-to-video sampling (pipeline :652-890) ------------------------------------------------------------------
    @torch.no_grad()
    def __call__(self, prompt=None, image=None, height: Optional[int] = 704, width: Optional[int] = 1280,
                 target_fps: int = 16, num_frames: int = 16, num_inference_steps: int = 50, guidance_scale: float = 9.0,
                 negative_prompt=None, eta: float = 0.0, num_videos_per_prompt: int = 1,
                 decode_chunk_size: Optional[int] = 1, generator=None, latents: Optional[torch.Tensor] = None,
                 prompt_embeds=None, negative_prompt_embeds=None, output_type: str = "pil", return_dict: bool = True,
                 ddim_init_latents_t_idx: int = 1, image_embeddings=None, image_latents=None,
                 callback: Optional[Callable] = None, max_steps: Optional[int] = None, **_ignored):
        """Image-to-video DDIM sampling with CFG (pipeline :652-890), the reference's keyword surface and defaults.  Note the
        reference's ``ddim_init_latents_t_idx=1``: the first timestep is skipped (:812-813).  ``eta > 0`` samples
        stochastically, drawing sigma_t * z from ``generator`` at every step as diffusers' DDIMScheduler does.  Raw inputs
        (``prompt`` strings, PIL ``image``) need ``encoders=`` and ``vae=``; pre-encoded ``prompt_embeds`` /
        ``negative_prompt_embeds`` / ``image_embeddings`` / ``image_latents`` (batch 1) are accepted instead.
        ``output_type`` "latent" returns the latents [N, 4, F, h, w]; "pt" / "np" / "pil" decode them with the attached VAE.
        ``pipe.scheduler = DPMSolverMultistepScheduler.from_config(pipe.scheduler.config)`` samples with DPM-Solver++(2M)
        (eta = 0 only), typically with half the steps."""
        if isinstance(prompt, list):
            if len(prompt) != 1:  # the reference builds its image latents per video, not per prompt (:797-802)
                raise ValueError(f"one prompt per call (got {len(prompt)}): use num_videos_per_prompt for several videos")
            prompt = prompt[0]
        if isinstance(negative_prompt, list):
            if len(negative_prompt) != 1:
                raise ValueError(f"one negative prompt per call (got {len(negative_prompt)})")
            negative_prompt = negative_prompt[0]
        if height is None or width is None:
            height, width = self._size_of(image, height, width)
        if height is not None and width is not None and (height % 8 != 0 or width % 8 != 0):
            raise ValueError(f"`height` and `width` have to be divisible by 8 but are {height} and {width}.")
        n_videos = int(num_videos_per_prompt)
        if isinstance(generator, list):
            if len(generator) != n_videos:
                raise ValueError(f"You have passed a list of generators of length {len(generator)}, but requested an effective "
                                 f"batch size of {n_videos}. Make sure the batch size matches the length of the generators.")
            if eta > 0 and len(generator) > 1:  # the reference's step noise would index the list per frame (:868)
                raise ValueError("eta > 0 draws the step noise from one generator: pass a single torch.Generator")
        self._guidance_scale = guidance_scale
        # the reference samples the first-frame latent with the global RNG (:540 passes no generator)
        prompt_embeds, negative_prompt_embeds, image_embeddings, image_latents = self._encode(
            prompt, negative_prompt, image, height, width, num_frames, None,
            self.do_classifier_free_guidance and (negative_prompt is not None or prompt is not None),
            prompt_embeds, negative_prompt_embeds, image_embeddings, image_latents)
        if latents is None and prompt_embeds is not None and image_latents is not None:  # prepare_latents :595-621
            shape = (n_videos, self.unet.config["in_channels"], num_frames) + tuple(image_latents.shape[-2:])
            latents = randn_tensor(shape, generator=generator, device=self.device, dtype=prompt_embeds.dtype)
        st = self.prepare_call(latents, prompt_embeds, image_latents, image_embeddings, target_fps, num_inference_steps,
                               guidance_scale, negative_prompt_embeds, eta, generator, ddim_init_latents_t_idx)
        self._loop(st, self.call_step, callback, max_steps)
        return self._output(st.latents, output_type, return_dict, decode_chunk_size)

    def prepare_call(self, latents, prompt_embeds, image_latents, image_embeddings, target_fps=16, num_inference_steps=50,
                     guidance_scale=9.0, negative_prompt_embeds=None, eta=0.0, generator=None, ddim_init_latents_t_idx=1):
        """Everything of ``__call__`` that happens once per clip (pipeline :742-834): ``latents`` [N, 4, F, h, w] and the
        conditioning of one prompt / first frame (batch 1), repeated for the N videos.  With CFG the UNet batch is
        [uncond x N, cond x N] (:783, :437-439, :559-560)."""
        self._guidance_scale = guidance_scale
        self.check_inputs(prompt_embeds, image_latents, image_embeddings, latents)
        cfg = self.do_classifier_free_guidance
        if cfg and negative_prompt_embeds is None:
            raise ValueError("`negative_prompt_embeds` (or a `negative_prompt` string + encoders) is required when guidance_scale > 1")
        if eta < 0:
            raise ValueError(f"eta must be >= 0, got {eta}")
        for name, t in (("prompt_embeds", prompt_embeds), ("negative_prompt_embeds", negative_prompt_embeds),
                        ("image_embeddings", image_embeddings), ("image_latents", image_latents)):
            if t is not None and t.shape[0] != 1:
                raise ValueError(f"`{name}` must hold one prompt / first frame (batch 1), got {tuple(t.shape)}: "
                                 "num_videos_per_prompt repeats it")
        dev = self.device
        n_videos = latents.shape[0]
        rep = lambda x: x.to(dev).repeat(n_videos, *([1] * (x.dim() - 1)))
        if cfg:
            prompts = torch.cat([rep(negative_prompt_embeds), rep(prompt_embeds)])
            img_emb = torch.cat([torch.zeros_like(rep(image_embeddings)), rep(image_embeddings)])
            img_lat = torch.cat([rep(image_latents)] * 2)
        else:
            prompts, img_emb, img_lat = rep(prompt_embeds), rep(image_embeddings), rep(image_latents)
        fps = torch.tensor([target_fps] * img_lat.shape[0], device=dev)
        cond = self.unet.precompute_conditioning(fps, img_lat, img_emb, prompts)
        self.scheduler.set_timesteps(num_inference_steps, device=dev)
        self.scheduler.timesteps = self.scheduler.timesteps[ddim_init_latents_t_idx:]
        ts = self.scheduler.timesteps.tolist()
        logger.info("Sampling starts from latents_at_t=%s", ts[0] if ts else None)
        st = _loop_state(latents, ts, self.scheduler, guidance_scale if cfg else 1.0, dev, eta=float(eta), cond=cond,
                         generator=generator, n_videos=n_videos)
        # uncond and cond of one video have the same latents, image latents, fps and timestep: they share the UNet prefix
        # up to the first cross-attention.  With N > 1 the last two branches are different videos.
        st.shared_prefix = cfg and n_videos == 1

        if cfg:
            def body():
                v = self.unet(torch.cat([st.latents, st.latents]), st.g_t, cond=st.cond, shared_edit_prefix=st.shared_prefix)[0]
                st.scheduler.step(v[:n_videos], None, st.latents, eta=st.eta, model_output_cond=v[n_videos:], out=st.latents,
                                  coef_dev=st.g_coef, variance_noise=st.g_noise, x0_prev=st.x0_prev)
        else:
            def body():
                v = self.unet(st.latents, st.g_t, cond=st.cond)[0]
                st.scheduler.step(v, None, st.latents, eta=st.eta, out=st.latents, coef_dev=st.g_coef,
                                  variance_noise=st.g_noise, x0_prev=st.x0_prev)

        st.body = body
        return st

    @staticmethod
    def _draw_noise(st):
        """With eta > 0, the variance noise of one step: drawn eagerly from ``st.generator`` in the reference's
        [N*F, C, h, w] order (the step runs on the frame-major reshape, pipeline :864-868 / :1168-1176), so that the draws
        are those of the reference, and copied into the buffer ``st.g_noise`` the (captured) step reads.  Nothing with eta = 0."""
        if st.g_noise is not None:
            n, c, f, h, w = st.latents.shape
            z = randn_tensor((n * f, c, h, w), generator=st.generator, device=st.latents.device, dtype=st.latents.dtype)
            st.g_noise.copy_(z.view(n, f, c, h, w).permute(0, 2, 1, 3, 4))

    def call_step(self, st, i: int):
        """One iteration of the sampling loop (pipeline :839-874): UNet on [uncond, cond] -> CFG + DDIM step, in place."""
        self._draw_noise(st)
        return self._run(st, i, (self.unet.freeu_state(), st.eta > 0), lambda: st.body)

    # -- phase 1 --------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def invert(self, prompt=None, image=None, height=None, width=None, target_fps: int = 16, num_frames: int = 16,
               num_inference_steps: int = 50, guidance_scale: float = 1.0, negative_prompt=None, eta: float = 0.0,
               latents: Optional[torch.Tensor] = None, prompt_embeds=None, negative_prompt_embeds=None,
               image_embeddings=None, image_latents=None, output_dir: Optional[str] = None, return_dict: bool = False,
               write_files: bool = True, callback: Optional[Callable] = None, max_steps: Optional[int] = None,
               host_resident: bool = False, **_ignored):
        """DDIM inversion x_0 -> x_T (pipeline :1385-1433).  Returns [b, steps, c, f, h, w] in DESCENDING-t order like
        the reference (:1436); every x_t is kept in ``self.latent_store`` (and written as ddim_latents_{t}.pt)."""
        prompt_embeds, negative_prompt_embeds, image_embeddings, image_latents = self._encode(
            prompt, negative_prompt, image, height, width, num_frames, None, guidance_scale > 1,
            prompt_embeds, negative_prompt_embeds, image_embeddings, image_latents)
        st = self.prepare_invert(latents, prompt_embeds, image_latents, image_embeddings, target_fps,
                                 num_inference_steps, guidance_scale, output_dir, write_files, host_resident,
                                 negative_prompt_embeds=negative_prompt_embeds)
        inverted = []

        def step(st, i):
            self.invert_step(st, i)
            inverted.append(st.store.get(st.timesteps[i], device=st.latents.device))
        self._loop(st, step, callback, max_steps)
        st.store.flush()
        stacked = torch.stack(list(reversed(inverted)), 1)
        return SimpleNamespace(frames=stacked) if return_dict else stacked

    def prepare_invert(self, latents, prompt_embeds, image_latents, image_embeddings, target_fps, num_inference_steps,
                       guidance_scale=1.0, output_dir=None, write_files=True, host_resident=False,
                       negative_prompt_embeds=None):
        """Everything of ``invert`` that happens once per clip (pipeline :1316-1382).  With ``guidance_scale > 1`` the
        step runs the UNet on [uncond, cond] (:1387-1388: negative prompt, zero image embedding :420-422, same image
        latents :559-560) and combines them (:1407-1410) inside the fused inverse-DDIM kernel."""
        if getattr(self.scheduler, "multistep", False):
            raise ValueError(f"invert runs DDIM inversion: set `pipe.scheduler` to a DDIMInverseScheduler (got "
                             f"{type(self.scheduler).__name__}; a multistep solver is for sampling and editing only)")
        self._guidance_scale = guidance_scale
        self.check_inputs(prompt_embeds, image_latents, image_embeddings, latents)
        cfg = self.do_classifier_free_guidance
        if cfg and negative_prompt_embeds is None:
            raise ValueError("`negative_prompt_embeds` (or a `negative_prompt` string + encoders) is required when guidance_scale > 1")
        dev = self.device
        if cfg and latents.shape[0] != 1:
            raise ValueError("inversion with guidance handles one clip per call (the reference's batch is always 1, :571)")
        d = lambda x: x.to(dev)
        if cfg:
            fps = torch.tensor([target_fps] * 2, device=dev)
            cond = self.unet.precompute_conditioning(fps, torch.cat([d(image_latents)] * 2),
                                                     torch.cat([torch.zeros_like(d(image_embeddings)), d(image_embeddings)]),
                                                     torch.cat([d(negative_prompt_embeds), d(prompt_embeds)]))
        else:
            fps = torch.tensor([target_fps], device=dev).repeat(latents.shape[0])
            cond = self.unet.precompute_conditioning(fps, d(image_latents), d(image_embeddings), d(prompt_embeds))
        self.scheduler.set_timesteps(num_inference_steps, device=dev)
        ts = self.scheduler.timesteps.tolist()
        store = LatentStore(output_dir, write_files=write_files, host_resident=host_resident)
        self.latent_store = store
        st = _loop_state(latents, ts, self.scheduler, guidance_scale if cfg else 1.0, dev, cond=cond, store=store)

        if cfg:
            def body():
                v = self.unet(torch.cat([st.latents, st.latents]), st.g_t, cond=st.cond)[0]
                st.scheduler.step(v[0:1], None, st.latents, model_output_cond=v[1:2], out=st.latents, coef_dev=st.g_coef)
        else:
            def body():
                v = self.unet(st.latents, st.g_t, cond=st.cond)[0]
                st.scheduler.step(v, None, st.latents, out=st.latents, coef_dev=st.g_coef)  # in place: x_t -> x_{t+1}

        st.body = body
        return st

    def invert_step(self, st, i: int):
        """One iteration of the inversion loop (pipeline :1385-1433): UNet (B = 1) -> inverse DDIM step -> keep x_t."""
        self._run(st, i, self.unet.freeu_state(), lambda: st.body)
        st.store.put(st.timesteps[i], st.latents)
        return st.latents

    # -- phase 2 --------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def sample_with_pnp(self, prompt=None, image=None, height=None, width=None, target_fps: int = 16,
                        num_frames: int = 16, num_inference_steps: int = 50, guidance_scale: float = 9.0,
                        negative_prompt=None, eta: float = 0.0, generator=None, latents: Optional[torch.Tensor] = None,
                        prompt_embeds=None, negative_prompt_embeds=None, output_type: str = "latent",
                        return_dict: bool = True, ddim_init_latents_t_idx: int = 1,
                        ddim_inv_latents_path: Optional[str] = None, ddim_inv_prompt=None, ddim_inv_1st_frame=None,
                        ddim_inv_prompt_embeds=None, image_embeddings=None, image_latents=None,
                        ddim_inv_image_embeddings=None, ddim_inv_image_latents=None,
                        latent_store: Optional[LatentStore] = None, skip_dead_source_branch: bool = True,
                        callback: Optional[Callable] = None, max_steps: Optional[int] = None,
                        decode_chunk_size: Optional[int] = None, source_features: Optional[SourceFeatureCache] = None,
                        **_ignored):
        """PnP edit loop (pipeline :1131-1179) over the branches [source, uncond, cond]; `output_type` "latent" returns
        the latents, "pt" / "np" / "pil" decode them with the attached VAE (:1180-1194).  ``eta > 0`` edits stochastically:
        every step, dead-source steps included, adds sigma_t * z with z drawn from ``generator`` as diffusers' DDIMScheduler
        draws it (:1126, :1173).  ``source_features`` (``source_feature_cache()``): reuse the source branch's features of
        earlier edits of the same inverted clip, and keep this edit's; the result does not change.  With a
        ``DPMSolverMultistepScheduler`` as ``pipe.scheduler`` the edit takes DPM-Solver++(2M) steps (e.g. 25 instead of 50);
        the inversion store must hold the source latents of each of its timesteps (a 50-step DDIM inversion holds those of
        25 steps)."""
        # raw inputs (the reference's only interface, :1014-1094) are encoded once per clip when encoders / VAE are attached;
        # the source first frame is cropped to the size of the edited one
        height, width = self._size_of(image, height, width)
        prompt_embeds, negative_prompt_embeds, image_embeddings, image_latents = self._encode(
            prompt, negative_prompt, image, height, width, num_frames, generator,
            negative_prompt is not None or prompt is not None,
            prompt_embeds, negative_prompt_embeds, image_embeddings, image_latents)
        ddim_inv_prompt_embeds, _, ddim_inv_image_embeddings, ddim_inv_image_latents = self._encode(
            ddim_inv_prompt, None, ddim_inv_1st_frame, height, width, num_frames, generator, False,
            ddim_inv_prompt_embeds, None, ddim_inv_image_embeddings, ddim_inv_image_latents)
        st = self.prepare_edit(latents, prompt_embeds, negative_prompt_embeds, ddim_inv_prompt_embeds, image_embeddings,
                               image_latents, ddim_inv_image_embeddings, ddim_inv_image_latents, target_fps,
                               num_inference_steps, guidance_scale, ddim_init_latents_t_idx, ddim_inv_latents_path,
                               latent_store, skip_dead_source_branch, eta, generator, source_features)
        self._loop(st, self.edit_step, callback, max_steps)
        return self._output(st.latents, output_type, return_dict, decode_chunk_size)

    def prepare_edit(self, latents, prompt_embeds, negative_prompt_embeds, ddim_inv_prompt_embeds, image_embeddings,
                     image_latents, ddim_inv_image_embeddings, ddim_inv_image_latents, target_fps, num_inference_steps,
                     guidance_scale, ddim_init_latents_t_idx=0, ddim_inv_latents_path=None, latent_store=None,
                     skip_dead_source_branch=True, eta=0.0, generator=None, source_features=None):
        """Everything of ``sample_with_pnp`` that happens once per clip (pipeline :1014-1128).  ``eta > 0``: the step noise
        is drawn from ``generator`` (one generator, or a list of one).  ``source_features``: a SourceFeatureCache, checked
        against this edit's source inputs."""
        self._guidance_scale = guidance_scale
        if not self.do_classifier_free_guidance:
            raise NotImplementedError("the PnP edit path runs with classifier-free guidance (cfg 9.0)")
        if eta < 0:
            raise ValueError(f"eta must be >= 0, got {eta}")
        if eta > 0 and isinstance(generator, list) and len(generator) > 1:  # the reference's step noise would index it per frame
            raise ValueError("eta > 0 draws the step noise from one generator: pass a single torch.Generator")
        self.check_inputs(prompt_embeds, image_latents, image_embeddings, latents)
        for name, t in (("negative_prompt_embeds", negative_prompt_embeds), ("ddim_inv_prompt_embeds", ddim_inv_prompt_embeds),
                        ("ddim_inv_image_embeddings", ddim_inv_image_embeddings), ("ddim_inv_image_latents", ddim_inv_image_latents)):
            if t is None:
                raise ValueError(f"`{name}` is required (pre-encoded)")
        dev = self.device
        # explicit arguments win: a store left on the pipeline by an earlier invert() of ANOTHER clip must not shadow the
        # path the caller names (the reference only knows `ddim_inv_latents_path`, pipeline :1134)
        if latent_store is not None:
            store = latent_store
            # a store read from a directory is identified by the directory, one kept in memory by the object
            store_id = (("path", os.path.abspath(store.output_dir)) if store.output_dir is not None else ("store", store))
        elif ddim_inv_latents_path is not None:
            mine = self.latent_store
            same = (mine is not None and mine.output_dir is not None
                    and os.path.abspath(mine.output_dir) == os.path.abspath(ddim_inv_latents_path))
            store = mine if same else LatentStore(ddim_inv_latents_path, write_files=False)
            store_id = ("path", os.path.abspath(ddim_inv_latents_path))
        elif self.latent_store is not None:
            store = self.latent_store
            store_id = (("path", os.path.abspath(store.output_dir)) if store.output_dir is not None else ("store", store))
        else:
            raise ValueError("need `latent_store` or `ddim_inv_latents_path`")
        if getattr(self.scheduler, "multistep", False):
            # a multistep edit reads the inversion at its own timesteps (25 steps: 961, 921, ..., 1, every other timestep of
            # a 50-step inversion); a store that lacks one is refused before anything runs rather than at that step
            self.scheduler.set_timesteps(num_inference_steps, device=dev)
            missing = [t for t in self.scheduler.timesteps.tolist()[ddim_init_latents_t_idx:] if t not in store]
            if missing:
                raise ValueError(f"the inversion store lacks the source latents of timestep(s) {missing} of the "
                                 f"{num_inference_steps}-step {type(self.scheduler).__name__} schedule: invert with a number "
                                 "of steps whose timesteps include them (e.g. 50 for a 25-step edit)")
        if source_features is not None:
            source_features.bind(store_id, ddim_inv_prompt_embeds, ddim_inv_image_embeddings, ddim_inv_image_latents,
                                 target_fps, (latents.shape[2], latents.shape[3], latents.shape[4]), self.unet)
        d = lambda x: x.to(dev)
        # [source, uncond, cond] stacks (:1043-1046, :1093-1101); uncond image embedding is zeros (:438)
        prompts3 = torch.cat([d(ddim_inv_prompt_embeds), d(negative_prompt_embeds), d(prompt_embeds)])
        img_emb3 = torch.cat([d(ddim_inv_image_embeddings), torch.zeros_like(d(image_embeddings)), d(image_embeddings)])
        img_lat3 = torch.cat([d(ddim_inv_image_latents), d(image_latents), d(image_latents)])
        fps3 = torch.tensor([target_fps] * 3, device=dev)
        cond3 = self.unet.precompute_conditioning(fps3, img_lat3, img_emb3, prompts3)
        self.scheduler.set_timesteps(num_inference_steps, device=dev)
        ts = self.scheduler.timesteps.tolist()[ddim_init_latents_t_idx:]
        logger.info("Sampling starts from latents_at_t=%s", ts[0] if ts else None)
        fires = [self._any_hook_fires(t) for t in ts]
        cond2 = None
        if (skip_dead_source_branch and not all(fires)) or source_features is not None:
            cond2 = {k: v[v.shape[0] // 3:].contiguous() for k, v in cond3.items()}  # every entry is branch-major
        st = _loop_state(latents, ts, self.scheduler, guidance_scale, dev, eta=float(eta), cond3=cond3, cond2=cond2, store=store,
                         fires=fires, guidance=guidance_scale, skip=skip_dead_source_branch, generator=generator,
                         source_features=source_features)
        st.g_src = torch.zeros_like(st.latents)
        # uncond and cond are the same latents + image latents -> they share the UNet prefix up to the first cross-attention
        # (I2VGenXLUNet.forward, shared_edit_prefix); the source branch is dropped after the last injection site that fires in
        # the step (its prediction is discarded, pipeline :1160).  Both leave the result unchanged
        # (`skip_dead_source_branch=False` runs the reference's full batch instead)
        st.shared_prefix = bool(skip_dead_source_branch)
        st.prune_source = bool(skip_dead_source_branch)
        return st

    def _hook_flags(self, t):
        """Which of the three injections fire at t (decided on the host; baked into the captured graph)."""
        mod = self.unet.up_blocks[1].resnets[1]
        up = self.unet.up_blocks[3]
        spa = up.attentions[2].transformer_blocks[0].attn1.processor
        tmp = up.temp_attentions[2].transformer_blocks[0].attn1.processor
        return (_fires(t, getattr(mod, "_injection_set", None)), _fires(t, getattr(spa, "_injection_set", None)),
                _fires(t, getattr(tmp, "_injection_set", None)))

    @staticmethod
    def _prune_site(flags):
        """(conv, spatial, temporal) flags of a step -> the last site at which the source branch is still read
        (UNet order inside a layer: resnet -> temp_conv -> spatial transformer -> temporal transformer; the hooks sit on
        up_blocks[1].resnets[1] and on attentions / temp_attentions of up_blocks[1..3], pnp_utils.py:130,235,340)."""
        conv, spatial, temporal = flags
        if temporal:
            return (3, 2, "temporal")
        if spatial:
            return (3, 2, "spatial")
        if conv:
            return (1, 1, "resnet")
        return None

    def edit_step(self, st, i: int):
        """One iteration of the PnP edit loop (pipeline :1131-1179).  With eta > 0 every step, dead-source steps included,
        draws its noise before the UNet runs (``_draw_noise``)."""
        t = st.timesteps[i]
        register_time(self, t)
        dead_source = st.skip and not st.fires[i]
        flags = self._hook_flags(t)
        cache, mode = st.source_features, None
        if cache is not None and st.fires[i]:
            sites = _pnp_sites(self.unet)
            cache_key = (t, tuple(_fires(t, getattr(s, "_injection_set", None)) for _, s in sites), self.unet.freeu_state())
            mode = cache.begin_step(cache_key, sites)
        two_branch = dead_source or mode == "replay"  # a replayed step injects into [uncond, cond] from the cache

        def make_body():
            if two_branch:
                # a replayed step passes where the three-branch step would drop the source (_ReplayedSource)
                replay = dict(source_replay=True, prune_source_after=self._prune_site(flags) if st.prune_source else None) \
                    if mode == "replay" else {}

                def body():
                    v = self.unet(torch.cat([st.latents, st.latents]), st.g_t, cond=st.cond2,
                                  shared_edit_prefix=st.shared_prefix, **replay)[0]
                    st.scheduler.step(v[0:1], None, st.latents, eta=st.eta, model_output_cond=v[1:2], out=st.latents,
                                      coef_dev=st.g_coef, variance_noise=st.g_noise, x0_prev=st.x0_prev)
                return body
            site = self._prune_site(flags) if st.prune_source else None
            lo = 0 if site is not None else 1  # the pruned forward returns [uncond, cond] only

            def body():
                v = self.unet(torch.cat([st.g_src, st.latents, st.latents]), st.g_t, cond=st.cond3,
                              shared_edit_prefix=st.shared_prefix, prune_source_after=site)[0]
                st.scheduler.step(v[lo:lo + 1], None, st.latents, eta=st.eta, model_output_cond=v[lo + 1:lo + 2],
                                  out=st.latents, coef_dev=st.g_coef, variance_noise=st.g_noise, x0_prev=st.x0_prev)
            return body
        if not two_branch:
            st.g_src.copy_(st.store.get(t, device=st.latents.device), non_blocking=True)
        self._draw_noise(st)
        # the eta = 0 keys are those of the loop without eta; eta > 0 is marked, as in call_step's key; so is a step that
        # captures or replays source features
        key = (dead_source, flags, self.unet.freeu_state()) + ((True,) if st.eta > 0 else ()) + ((mode,) if mode else ())
        if cache is None or not st.fires[i]:
            return self._run(st, i, key, make_body)
        try:
            out = self._run(st, i, key, make_body)
        except BaseException:
            cache.end_step(cache_key, sites, None)  # detach; keep nothing of a step that did not complete
            raise
        cache.end_step(cache_key, sites, mode)
        return out
