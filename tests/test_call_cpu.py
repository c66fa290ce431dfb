"""The image-to-video call `I2VGenXLPipeline.__call__` (pipeline_i2vgen_xl.py:652-890) and stochastic DDIM (eta > 0) without a
GPU: the scheduler's coefficients against diffusers' fp32 formula, the kernel contract against the oracle step, the product call
on the tiny UNet (kernels replaced by their contracts) against the fp32 oracle loop, the generator's draws against the reference
loop's, and the reconstruction runner that now goes through `pipe(...)`.  Oracle and contract: tests/sampling_ref.py."""
import ctypes
import os
import subprocess

import pytest
import torch

import sampling_ref
from test_host_model_cpu import F_, _close, _models

N_STEPS = 4


@pytest.fixture
def emu(emulated_ops, monkeypatch):
    """the kernel contracts in place of anyv2v_b200.ops, ops.ddim_step_eta included"""
    sampling_ref.patch_ops(monkeypatch)
    return emulated_ops


def _sched_pair(n):
    from anyv2v_b200.schedulers import DDIMScheduler
    from oracle import schedulers_ref
    ours, ref = DDIMScheduler(), schedulers_ref.DDIMScheduler()
    ours.set_timesteps(n)
    ref.set_timesteps(n)
    return ours, ref


@pytest.mark.parametrize("n", [10, 50, 500, 1000])
@pytest.mark.parametrize("eta", [0.0, 0.3, 1.0])
def test_eta_coefficients_equal_the_fp32_formula(n, eta):
    ours, ref = _sched_pair(n)
    ts = [t for t in ours.timesteps.tolist() if t < 1000]  # "leading" spacing at n = 1000 also yields t = 1000
    if n == 1000:
        assert 999 in ts and float(ours.alphas_cumprod[999]) == 0.0
    for t in ts:
        c = ours.coefficients(t, eta)
        assert all(map(lambda v: v == v and abs(v) < float("inf"), c)), (t, c)
        if eta == 0.0:
            assert c == ours.coefficients(t) and len(c) == 4
            continue
        sigma, cd = sampling_ref.eta_coefficients(ref, t, eta)
        assert len(c) == 5 and c[:3] == ours.coefficients(t)[:3]
        assert c[4] == float(sigma) and c[3] == float(cd), t
    last = ts[-1]
    if last - 1000 // n < 0:                                          # at n = 1000 the last step still has t_prev = 0
        assert ours.coefficients(last, eta)[4:] in ((), (0.0,))      # sigma = 0 at the last step (a_prev = 1)
    table = ours.coefficient_table(ts[:3], 9.0, "cpu", eta=eta)
    assert table.shape == (3, 5 if eta == 0 else 6) and bool((table[:, 4] == 9.0).all())
    if eta == 0:
        assert torch.equal(table, ours.coefficient_table(ts[:3], 9.0, "cpu"))


def test_inverse_scheduler_has_no_eta():
    from anyv2v_b200.schedulers import DDIMInverseScheduler
    s = DDIMInverseScheduler()
    s.set_timesteps(10)
    with pytest.raises(ValueError):
        s.coefficients(int(s.timesteps[0]), eta=0.5)


@pytest.mark.parametrize("n", [1, 7, 8, 1001])
@pytest.mark.parametrize("cfg", [False, True])
def test_eta_contract_is_bit_exact_against_the_oracle_step(emu, n, cfg):
    from oracle.schedulers_ref import cfg_combine
    ours, ref = _sched_pair(50)
    torch.manual_seed(n + cfg)
    x, vn, ve = (torch.randn(n).half() for _ in range(3))
    z = (torch.randn(n) * 2).clamp(-5, 5).half()
    for t in (981, 501, 21, 1):
        for eta in (0.3, 1.0):
            v = cfg_combine(vn, ve, 9.0) if cfg else vn
            want, _ = sampling_ref.step(ref, v, t, x, eta=eta, variance_noise=z)
            got = ours.step(vn, t, x, eta=eta, model_output_cond=ve if cfg else None, guidance_scale=9.0 if cfg else 1.0,
                            variance_noise=z).prev_sample
            assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (t, eta)
    with pytest.raises(ValueError):
        ours.step(vn, 981, x, eta=1.0, generator=torch.Generator(), variance_noise=z)
    with pytest.raises(ValueError):
        sampling_ref.step(ref, vn, 981, x, eta=1.0, generator=torch.Generator(), variance_noise=z)


def test_randn_tensor_device_rule():
    from anyv2v_b200.schedulers import randn_tensor
    g1, g2 = torch.Generator().manual_seed(3), torch.Generator().manual_seed(3)
    a = randn_tensor((2, 3, 4), generator=g1, device=torch.device("cpu"), dtype=torch.float16)
    assert a.dtype == torch.float16 and torch.equal(a, torch.randn((2, 3, 4), generator=g2, dtype=torch.float16))
    gl = [torch.Generator().manual_seed(s) for s in (1, 2)]
    b = randn_tensor((2, 3), generator=gl, device="cpu")
    assert torch.equal(b[1], torch.randn((1, 3), generator=torch.Generator().manual_seed(2))[0])
    assert torch.equal(b, sampling_ref.randn_tensor((2, 3), generator=[torch.Generator().manual_seed(s) for s in (1, 2)]))


# ---------------------------------------------------------------------------------------------------------- __call__
def _conditioning(h, w, dtype, device="cpu"):
    from oracle import loops_ref
    return loops_ref.synthetic_inputs(F_, h, w, cross_dim=64, dtype=dtype, device=device)


def _spy_draws(monkeypatch):
    """record every randn_tensor draw of the product pipeline, in order"""
    from anyv2v_b200 import pipeline as pl
    draws = []
    real = pl.randn_tensor

    def spy(*a, **kw):
        z = real(*a, **kw)
        draws.append(z.clone())
        return z
    monkeypatch.setattr(pl, "randn_tensor", spy)
    return draws


def run_call_teacher_forced(ref32, ours, eta, guidance, n_videos, h, w, device, draws, rms=6e-3, mx=3e-2):
    """the product __call__ (default ddim_init_latents_t_idx = 1) against the fp32 oracle loop, teacher-forced per step with
    the latents and the step noise of the product; returns the product's final latents"""
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.schedulers import DDIMScheduler
    ns16, ns32 = _conditioning(h, w, torch.float16, device), _conditioning(h, w, torch.float32, device)
    lat = torch.randn(n_videos, 4, F_, h, w, generator=torch.Generator().manual_seed(11)).half().to(device)
    pipe = I2VGenXLPipeline(ours, DDIMScheduler())
    seen = []
    out = pipe(prompt_embeds=ns16.edit_prompt, negative_prompt_embeds=ns16.neg_prompt, image_embeddings=ns16.edit_image_emb,
               image_latents=ns16.edit_image_latents, latents=lat, num_inference_steps=N_STEPS, guidance_scale=guidance,
               eta=eta, num_videos_per_prompt=n_videos, target_fps=8, output_type="latent",
               generator=torch.Generator(device=device).manual_seed(5),
               callback=lambda i, t, x: seen.append((i, t, x.clone()))).frames
    assert out.shape == (n_videos, 4, F_, h, w) and len(seen) == N_STEPS - 1       # the first timestep is skipped
    assert len(draws) == (len(seen) if eta > 0 else 0)
    assert all(z.shape == (n_videos * F_, 4, h, w) for z in draws)              # the reference's [N*F, C, h, w] order
    x_prev = lat.float()
    for i, t, x_ours in seen:
        z = draws[i].float() if eta > 0 else None
        want = sampling_ref.call_loop(ref32, x_prev, ns32.edit_prompt, ns32.neg_prompt, ns32.edit_image_latents,
                                      ns32.edit_image_emb, 8, N_STEPS, guidance, eta=eta, t_idx=1 + i, num_videos=n_videos,
                                      noise_at=lambda _i: z, max_steps=1)
        _close(x_ours, want, f"call step {i} (t={t}) eta={eta} g={guidance} N={n_videos}", rms=rms, mx=mx)
        x_prev = x_ours.float()
    return out


@torch.no_grad()
@pytest.mark.parametrize("eta", [0.0, 1.0])
@pytest.mark.parametrize("guidance", [1.0, 9.0])
@pytest.mark.parametrize("n_videos", [1, 2])
def test_call_matches_the_oracle_loop_teacher_forced(emu, monkeypatch, eta, guidance, n_videos):
    draws = _spy_draws(monkeypatch)
    ref32, ours = _models()
    run_call_teacher_forced(ref32, ours, eta, guidance, n_videos, 16, 16, "cpu", draws)


@torch.no_grad()
def test_call_on_a_non_square_latent(emu, monkeypatch):
    draws = _spy_draws(monkeypatch)
    ref32, ours = _models()
    run_call_teacher_forced(ref32, ours, 1.0, 9.0, 2, 16, 24, "cpu", draws)


@torch.no_grad()
def test_batch_order_of_several_videos(emu):
    """N = 2 (batch [uncond x 2, cond x 2], no shared prefix) gives each video what N = 1 gives it alone (the float64
    contracts are batch-invariant, so this is bit for bit)"""
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.schedulers import DDIMScheduler
    _, ours = _models()
    ns = _conditioning(16, 16, torch.float16)
    lat = torch.randn(2, 4, F_, 16, 16, generator=torch.Generator().manual_seed(2)).half()
    pipe = I2VGenXLPipeline(ours, DDIMScheduler())
    kw = dict(prompt_embeds=ns.edit_prompt, negative_prompt_embeds=ns.neg_prompt, image_embeddings=ns.edit_image_emb,
              image_latents=ns.edit_image_latents, num_inference_steps=N_STEPS, target_fps=8, output_type="latent")
    both = pipe(latents=lat, num_videos_per_prompt=2, **kw).frames
    for k in range(2):
        alone = pipe(latents=lat[k:k + 1], **kw).frames
        assert torch.equal(both[k:k + 1], alone), k
    assert not torch.equal(both[0], both[1])


@torch.no_grad()
@pytest.mark.parametrize("consume", [False, True])
def test_generator_draws_equal_the_reference_loop(emu, monkeypatch, consume):
    """with equal seeds the product draws what the reference loop draws, in the same order: the initial latents and one
    [N*F, C, h, w] noise per step; ``consume``: a callback also draws from the generator between steps"""
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.schedulers import DDIMScheduler
    draws = _spy_draws(monkeypatch)
    _, ours = _models()
    ns = _conditioning(16, 16, torch.float16)
    g_ours, g_ref = torch.Generator().manual_seed(77), torch.Generator().manual_seed(77)
    side = {"ours": [], "ref": []}

    def cb(key, g):
        return (lambda i, t, x: side[key].append(torch.randn(3, generator=g))) if consume else None
    pipe = I2VGenXLPipeline(ours, DDIMScheduler())
    pipe(prompt_embeds=ns.edit_prompt, negative_prompt_embeds=ns.neg_prompt, image_embeddings=ns.edit_image_emb,
         image_latents=ns.edit_image_latents, num_inference_steps=N_STEPS, target_fps=8, output_type="latent", eta=1.0,
         num_frames=F_, generator=g_ours, callback=cb("ours", g_ours))
    ref_draws = []
    real = sampling_ref.randn_tensor

    def spy(*a, **kw):
        z = real(*a, **kw)
        ref_draws.append(z.clone())
        return z
    monkeypatch.setattr(sampling_ref, "randn_tensor", spy)
    zero_unet = lambda x, *a: (torch.zeros_like(x),)   # the draws do not depend on the model
    sampling_ref.call_loop(zero_unet, None, ns.edit_prompt, ns.neg_prompt, ns.edit_image_latents, ns.edit_image_emb, 8, N_STEPS,
                           9.0, eta=1.0, generator=g_ref, dtype=torch.float16, callback=cb("ref", g_ref))
    assert len(draws) == len(ref_draws) == N_STEPS                       # latents + one noise per step (first step skipped)
    for a, b in zip(draws, ref_draws):
        assert a.shape == b.shape and torch.equal(a, b)
    assert all(torch.equal(a, b) for a, b in zip(side["ours"], side["ref"]))


@torch.no_grad()
@pytest.mark.parametrize("eta", [0.0, 1.0])
def test_shared_prefix_is_bit_identical_and_eta_adds_no_launch(emu, eta):
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.schedulers import DDIMScheduler
    _, ours = _models()
    ns = _conditioning(16, 16, torch.float16)
    lat = torch.randn(1, 4, F_, 16, 16, generator=torch.Generator().manual_seed(4)).half()
    pipe = I2VGenXLPipeline(ours, DDIMScheduler())
    outs, launches = [], []
    for shared in (True, False):
        st = pipe.prepare_call(lat, ns.edit_prompt, ns.edit_image_latents, ns.edit_image_emb, 8, N_STEPS, 9.0,
                               ns.neg_prompt, eta, torch.Generator().manual_seed(9))
        assert st.shared_prefix
        st.shared_prefix = shared
        for i in range(len(st.timesteps)):
            n0 = emu.launch_count()
            pipe.call_step(st, i)
            launches.append(emu.launch_count() - n0)
        outs.append(st.latents.clone())
    assert torch.equal(outs[0], outs[1])
    st0 = pipe.prepare_call(lat, ns.edit_prompt, ns.edit_image_latents, ns.edit_image_emb, 8, N_STEPS, 9.0, ns.neg_prompt, 0.0)
    n0 = emu.launch_count()
    pipe.call_step(st0, 0)
    assert launches[0] == emu.launch_count() - n0      # an eta > 0 step launches as many kernels as an eta = 0 step


def test_call_refusals():
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    _, ours = _models()
    ns = _conditioning(16, 16, torch.float16)
    pipe = I2VGenXLPipeline(ours)
    kw = dict(prompt_embeds=ns.edit_prompt, negative_prompt_embeds=ns.neg_prompt, image_embeddings=ns.edit_image_emb,
              image_latents=ns.edit_image_latents, num_inference_steps=N_STEPS)
    with pytest.raises(ValueError, match="one prompt"):
        pipe(prompt=["a", "b"], **kw)
    with pytest.raises(ValueError, match="single torch.Generator"):
        pipe(eta=1.0, num_videos_per_prompt=2, generator=[torch.Generator(), torch.Generator()], **kw)
    with pytest.raises(ValueError, match="length"):
        pipe(num_videos_per_prompt=2, generator=[torch.Generator()] * 3, **kw)
    with pytest.raises(ValueError, match="VAE"):
        pipe.decode_latents(ns.video_latents)


# ---------------------------------------------------------------------------------------------------------- runner
def _old_inline_reconstruction(pipe, config, cond, latents_path):
    """the reconstruction loop of run_group_ddim_inversion.ddim_sampling before it called pipe(...): eager UNet on
    [latents, latents] with [neg, cond] prompts and [0, emb] image embeddings, by-value scheduler coefficients"""
    from anyv2v_b200.latent_store import load_ddim_latents_at_t
    from anyv2v_b200.schedulers import DDIMScheduler
    s = DDIMScheduler()
    s.set_timesteps(config["n_steps"])
    ts = s.timesteps.tolist()[config["ddim_init_latents_t_idx"]:]
    latents = load_ddim_latents_at_t(ts[0], latents_path, map_location=pipe.device)
    dev = pipe.device
    prompts = torch.cat([cond["neg_prompt"], cond["inv_prompt"]])
    img_emb = torch.cat([torch.zeros_like(cond["src_image_emb"]), cond["src_image_emb"]])
    img_lat = torch.cat([cond["src_image_latents"]] * 2)
    c2 = pipe.unet.precompute_conditioning(torch.tensor([config["target_fps"]] * 2, device=dev), img_lat, img_emb, prompts)
    for t in ts:
        v = pipe.unet(torch.cat([latents, latents]), torch.tensor([t], device=dev), cond=c2)[0]
        latents = s.step(v[0:1], t, latents, model_output_cond=v[1:2], guidance_scale=config["cfg"]).prev_sample
    return latents


def run_reconstruction_runner(tmp_path, device, monkeypatch):
    """run_group_ddim_inversion with recon_config.enable_recon (synthetic inputs): latents.pt == the old inline loop"""
    import yaml
    from test_gpu_runners import INV_TEMPLATE
    from anyv2v_b200 import run_group_ddim_inversion as inv
    from anyv2v_b200.config import OmegaConf
    from anyv2v_b200.run_group_pnp_edit import synthetic_conditioning
    from oracle.unet_ref import TINY_CONFIG
    data = str(tmp_path)
    (tmp_path / "inv.yaml").write_text(yaml.safe_dump(dict(INV_TEMPLATE, data_dir=data, device=str(device))))
    built = []
    real = inv.build_pipeline
    monkeypatch.setattr(inv, "build_pipeline", lambda *a, **kw: built.append(real(*a, **kw)) or built[-1])
    entries = [{"active": True, "video_name": "clipA"}]
    inv.main(OmegaConf.load(str(tmp_path / "inv.yaml")), entries, device, unet_config=TINY_CONFIG)
    clip = os.path.join(data, "inversions", "i2vgen-xl", "clipA")
    got = torch.load(os.path.join(clip, "ddim_reconstruction", "latents.pt"))
    rc = INV_TEMPLATE["recon_config"]
    cond = synthetic_conditioning(INV_TEMPLATE["n_frames"], 16, 16, 64, INV_TEMPLATE["seed"], device)
    want = _old_inline_reconstruction(built[0], rc, cond, os.path.join(clip, "ddim_latents")).cpu()
    assert got.shape == (1, 4, INV_TEMPLATE["n_frames"], 16, 16) and torch.isfinite(got.float()).all()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))


def test_reconstruction_runner_is_bit_identical_to_the_inline_loop(emu, tmp_path, monkeypatch):
    prev = torch.is_grad_enabled()
    torch.set_grad_enabled(False)
    try:
        run_reconstruction_runner(tmp_path, torch.device("cpu"), monkeypatch)
    finally:
        torch.set_grad_enabled(prev)


def run_real_input_reconstruction(tmp_path, device):
    """the real input path (png frames, prompt strings -> VAE / CLIP) with recon_config.enable_recon: pipe(prompt=...,
    image=first_frame) -> ddim_reconstruction/latents.pt, ddim_reconstruction.mp4 (fps 10) and .gif at 512 x 512"""
    import yaml
    from PIL import Image
    from test_gpu_runners import INV_TEMPLATE, TINY_VAE, write_demo_clip
    from anyv2v_b200 import run_group_ddim_inversion as inv
    from anyv2v_b200.config import OmegaConf
    from oracle.unet_ref import TINY_CONFIG
    data = str(tmp_path)
    write_demo_clip(data)
    t = dict(INV_TEMPLATE, data_dir=data, device=str(device), synthetic=False)
    t["inverse_config"] = dict(t["inverse_config"], prompt="a man", negative_prompt="blurry")
    t["recon_config"] = dict(t["recon_config"], prompt="a man", negative_prompt="blurry")
    (tmp_path / "inv.yaml").write_text(yaml.safe_dump(t))
    entries = [{"active": True, "video_name": "clipA"}]
    inv.main(OmegaConf.load(str(tmp_path / "inv.yaml")), entries, device, unet_config=TINY_CONFIG,
             pipeline_kwargs=dict(vae_config=TINY_VAE))
    clip = os.path.join(data, "inversions", "i2vgen-xl", "clipA")
    rec = torch.load(os.path.join(clip, "ddim_reconstruction", "latents.pt"))
    assert rec.shape == (1, 4, 4, 16, 16) and torch.isfinite(rec.float()).all()
    gif = Image.open(os.path.join(clip, "ddim_reconstruction.gif"))
    assert gif.size == (512, 512) and gif.n_frames == 4
    try:
        import cv2  # noqa: F401  (image_io writes mp4 through OpenCV)
    except ImportError:
        return
    assert os.path.getsize(os.path.join(clip, "ddim_reconstruction.mp4")) > 0


def test_reconstruction_runner_on_real_inputs(emu, tmp_path):
    prev = torch.is_grad_enabled()
    torch.set_grad_enabled(False)
    try:
        run_real_input_reconstruction(tmp_path, torch.device("cpu"))
    finally:
        torch.set_grad_enabled(prev)


def test_ddim_eta_args_struct_matches_the_c_header(tmp_path):
    """ctypes mirror of av2v_ddim_eta_args against the layout gcc gives include/anyv2v_b200.h"""
    from anyv2v_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cls = _lib.DdimEtaArgs
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "anyv2v_b200.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(av2v_ddim_eta_args));']
    lines += [f'  printf("{f} %zu\\n", offsetof(av2v_ddim_eta_args, {f}));' for f, _ in cls._fields_]
    lines += ['  return 0;', '}']
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(out["size"]) == ctypes.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(out[f]) == getattr(cls, f).offset, f
