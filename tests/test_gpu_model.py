"""GPU parity tests, model level: the sm_90a UNet + hooks + loops against the oracle (run on the same GPU with torch
ops, fp32 and fp16) on identical seeded weights / latents."""
from types import SimpleNamespace

import pytest
import torch

from parity_utils import assert_fp16_close, err_stats

pytestmark = pytest.mark.gpu
dev = "cuda"
F_, H_, W_ = 4, 16, 16


@pytest.fixture(scope="module")
def models():
    from anyv2v_b200.unet_i2vgen_xl import I2VGenXLUNet
    from oracle import unet_ref
    ref32 = unet_ref.seeded_unet(unet_ref.TINY_CONFIG, seed=8888, dtype=torch.float32, device=dev)
    ref16 = unet_ref.seeded_unet(unet_ref.TINY_CONFIG, seed=8888, dtype=torch.float16, device=dev)
    ours = I2VGenXLUNet(**unet_ref.TINY_CONFIG)
    ours.load_state_dict(ref32.state_dict())  # same names, same shapes as diffusers
    ours = ours.to(device=dev, dtype=torch.float16).eval()
    return SimpleNamespace(ref32=ref32, ref16=ref16, ours=ours)


def _inputs(dtype):
    from oracle import loops_ref
    ns = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, seed=8888, dtype=dtype, device=dev)
    prompts, img_lat, img_emb, fps = loops_ref.edit_conditioning(ns)
    g = torch.Generator().manual_seed(8895)
    x3 = torch.randn(3, 4, F_, H_, W_, generator=g).to(device=dev, dtype=dtype)
    return ns, x3, prompts, img_lat, img_emb, fps


def _check_vs_oracles(got, ref32, ref16, what, slack=3.0):
    """`got` (our fp16) must be as close to the fp32 oracle as the oracle's own fp16 run is (x slack)."""
    assert torch.isfinite(got).all()
    e_ours = err_stats(got, ref32)
    e_ref = err_stats(ref16, ref32)
    print(f"{what}: ours-vs-fp32 {e_ours}  |  torch-fp16-vs-fp32 {e_ref}")
    assert e_ours["rms_rel"] <= max(slack * e_ref["rms_rel"], 2e-3), (what, e_ours, e_ref)
    assert e_ours["rel_to_max"] <= max(slack * e_ref["rel_to_max"], 5e-3), (what, e_ours, e_ref)


@torch.no_grad()
def test_unet_forward_matches_oracle(models):
    outs = {}
    for name, net, dt in (("ref32", models.ref32, torch.float32), ("ref16", models.ref16, torch.float16), ("ours", models.ours, torch.float16)):
        _, x3, prompts, img_lat, img_emb, fps = _inputs(dt)
        outs[name] = net(x3, torch.tensor([981], device=dev), fps, img_lat, img_emb, prompts)[0]
    assert outs["ours"].shape == outs["ref32"].shape == (3, 4, F_, H_, W_)
    _check_vs_oracles(outs["ours"], outs["ref32"], outs["ref16"], "tiny UNet forward")


@torch.no_grad()
@pytest.mark.parametrize("t,expect_inject", [(901, True), (101, False), (1000, True)])
def test_hooks_match_oracle(models, t, expect_inject):
    from anyv2v_b200 import pnp_utils as ours_hooks
    from oracle import pnp_hooks_ref, schedulers_ref
    s = schedulers_ref.DDIMScheduler()
    s.set_timesteps(10)
    schedule = s.timesteps[:5]
    outs = {}
    for name, net, dt, hooks in (("ref32", models.ref32, torch.float32, pnp_hooks_ref), ("ref16", models.ref16, torch.float16, pnp_hooks_ref),
                                 ("ours", models.ours, torch.float16, ours_hooks)):
        pipe = SimpleNamespace(unet=net)
        hooks.register_conv_injection(pipe, schedule)
        hooks.register_spatial_attention_pnp(pipe, schedule)
        hooks.register_temp_attention_pnp(pipe, schedule)
        hooks.register_time(pipe, t)
        _, x3, prompts, img_lat, img_emb, fps = _inputs(dt)
        outs[name] = net(x3, torch.tensor([t], device=dev), fps, img_lat, img_emb, prompts)[0]
    _check_vs_oracles(outs["ours"], outs["ref32"], outs["ref16"], f"hooked UNet t={t}")
    proc = models.ours.up_blocks[2].attentions[1].transformer_blocks[0].attn1.processor
    assert proc.inject_now() == expect_inject and proc.t == t
    # un-register for the other tests (empty schedule == unpatched model, Appendix C.5)
    for net, hooks in ((models.ref32, pnp_hooks_ref), (models.ref16, pnp_hooks_ref), (models.ours, ours_hooks)):
        pipe = SimpleNamespace(unet=net)
        hooks.register_conv_injection(pipe, [])
        hooks.register_spatial_attention_pnp(pipe, [])
        hooks.register_temp_attention_pnp(pipe, [])
        hooks.register_time(pipe, -1)  # t == 1000 would keep forcing injection (pnp_utils.py:109), even with []


@torch.no_grad()
def test_inversion_and_edit_loops(models, tmp_path):
    """Both loops end to end on the tiny model: teacher-forced per-step parity + reported free-running drift."""
    from anyv2v_b200 import pnp_utils as ours_hooks
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.schedulers import DDIMInverseScheduler, DDIMScheduler
    from oracle import loops_ref, pnp_hooks_ref, schedulers_ref
    n_steps = 4
    for net, hooks in ((models.ref32, pnp_hooks_ref), (models.ref16, pnp_hooks_ref), (models.ours, ours_hooks)):
        p0 = SimpleNamespace(unet=net)  # module-scoped models: make sure no stale hook state leaks into the inversion
        hooks.register_conv_injection(p0, [])
        hooks.register_spatial_attention_pnp(p0, [])
        hooks.register_temp_attention_pnp(p0, [])
        hooks.register_time(p0, -1)
    ns32 = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float32, device=dev)
    ns16 = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float16, device=dev)
    inv_ref = loops_ref.invert_loop(models.ref32, ns32.video_latents, ns32.inv_prompt, ns32.src_image_latents, ns32.src_image_emb, ns32.fps, n_steps)
    pipe = I2VGenXLPipeline(models.ours, DDIMInverseScheduler())
    out_dir = str(tmp_path / "ddim_latents")
    stacked = pipe.invert(latents=ns16.video_latents, prompt_embeds=ns16.inv_prompt, image_latents=ns16.src_image_latents,
                          image_embeddings=ns16.src_image_emb, target_fps=8, num_inference_steps=n_steps, guidance_scale=1.0,
                          output_dir=out_dir)
    assert stacked.shape == (1, n_steps, 4, F_, H_, W_)
    store = pipe.latent_store
    ts = sorted(inv_ref)
    assert store.timesteps() == ts
    # free-running drift, calibrated against the oracle's own fp16 run (the "reference PyTorch fp16 pipeline")
    inv_ref16 = loops_ref.invert_loop(models.ref16, ns16.video_latents, ns16.inv_prompt, ns16.src_image_latents, ns16.src_image_emb, ns16.fps, n_steps)
    for t in ts:
        e, e16 = err_stats(store.get(t), inv_ref[t]), err_stats(inv_ref16[t], inv_ref[t])
        print(f"inversion drift t={t}: ours {e['rms_rel']:.3e}  torch-fp16 {e16['rms_rel']:.3e}")
        assert e["rms_rel"] <= max(3.0 * e16["rms_rel"], 2e-3)
    # teacher-forced: feed the oracle's x_t into ONE of our steps (UNet + fused inverse DDIM update)
    inv_s = DDIMInverseScheduler()
    inv_s.set_timesteps(n_steps)
    cond = models.ours.precompute_conditioning(ns16.fps, ns16.src_image_latents, ns16.src_image_emb, ns16.inv_prompt)
    prev = ns32.video_latents
    for t in ts:
        v = models.ours(prev.half(), torch.tensor([t], device=dev), cond=cond)[0]
        got = inv_s.step(v, t, prev.half()).prev_sample
        e = err_stats(got, inv_ref[t])
        print(f"teacher-forced inversion step t={t}: {e}")
        assert e["rms_rel"] < 3e-3
        prev = inv_ref[t]
    # reference-format files were written (ddim_latents_{t}.pt, [1,4,F,h,w] fp16)
    from anyv2v_b200.latent_store import load_ddim_latents_at_T, load_ddim_latents_at_t
    f = load_ddim_latents_at_t(ts[0], out_dir, map_location="cpu")
    assert f.shape == (1, 4, F_, H_, W_) and f.dtype == torch.float16 and torch.equal(f, store.get(ts[0]).cpu())
    assert torch.equal(load_ddim_latents_at_T(out_dir, "cpu"), store.get(ts[-1]).cpu())

    # edit: oracle fp32 loop with the oracle's inverted latents vs our loop with ours
    sref = schedulers_ref.DDIMScheduler()
    sref.set_timesteps(n_steps)
    pipe_ref = SimpleNamespace(unet=models.ref32)
    pnp_hooks_ref.init_pnp(pipe_ref, sref, n_steps, 1.0, 0.5, 0.5)
    prompts, img_lat, img_emb, fps = loops_ref.edit_conditioning(ns32)
    ref_final = loops_ref.pnp_edit_loop(pipe_ref, pnp_hooks_ref.register_time, inv_ref, inv_ref[ts[-1]].clone(), prompts, img_lat, img_emb, fps, n_steps, 9.0)
    sch = DDIMScheduler()
    sch.set_timesteps(n_steps)
    from anyv2v_b200.run_group_pnp_edit import init_pnp
    pipe.register_modules(scheduler=sch)
    init_pnp(pipe, sch, SimpleNamespace(n_steps=n_steps, pnp_f_t=1.0, pnp_spatial_attn_t=0.5, pnp_temp_attn_t=0.5))
    res = pipe.sample_with_pnp(latents=store.get(ts[-1]).clone(), prompt_embeds=ns16.edit_prompt, negative_prompt_embeds=ns16.neg_prompt,
                               ddim_inv_prompt_embeds=ns16.inv_prompt, image_embeddings=ns16.edit_image_emb, image_latents=ns16.edit_image_latents,
                               ddim_inv_image_embeddings=ns16.src_image_emb, ddim_inv_image_latents=ns16.src_image_latents,
                               target_fps=8, num_inference_steps=n_steps, guidance_scale=9.0, ddim_init_latents_t_idx=0, latent_store=store)
    e = err_stats(res.frames, ref_final)
    print(f"edit loop free-running drift after {n_steps}+{n_steps} steps (ours fp16 vs oracle fp32): {e}")
    assert torch.isfinite(res.frames).all() and e["rms_rel"] < 0.25  # reported, not a parity bar: a random-init UNet amplifies fp16 noise
    # skipping the dead source branch on non-injected steps must not change the result
    res2 = pipe.sample_with_pnp(latents=store.get(ts[-1]).clone(), prompt_embeds=ns16.edit_prompt, negative_prompt_embeds=ns16.neg_prompt,
                                ddim_inv_prompt_embeds=ns16.inv_prompt, image_embeddings=ns16.edit_image_emb, image_latents=ns16.edit_image_latents,
                                ddim_inv_image_embeddings=ns16.src_image_emb, ddim_inv_image_latents=ns16.src_image_latents,
                                target_fps=8, num_inference_steps=n_steps, guidance_scale=9.0, ddim_init_latents_t_idx=0, latent_store=store,
                                skip_dead_source_branch=False)
    assert torch.equal(res.frames, res2.frames)
    for net, hooks in ((models.ref32, pnp_hooks_ref), (models.ours, ours_hooks)):
        p = SimpleNamespace(unet=net)
        hooks.register_conv_injection(p, [])
        hooks.register_spatial_attention_pnp(p, [])
        hooks.register_temp_attention_pnp(p, [])


@torch.no_grad()
def test_shared_prefix_and_source_pruning_on_gpu():
    """shared_edit_prefix (set by the edit loop): the UNet prefix up to the first cross-attention computed once for the identical uncond / cond
    pair.  Every kernel is deterministic per element; only the GroupNorm partial-sum slicing depends on the batch, so the
    result may differ from the plain forward by fp32 rounding of the statistics (far below one fp16 ulp of the output)."""
    from types import SimpleNamespace
    from anyv2v_b200 import pnp_utils
    from anyv2v_b200.unet_i2vgen_xl import I2VGenXLUNet
    from oracle import loops_ref, schedulers_ref, unet_ref
    F_, H_, W_ = 4, 16, 16
    ref32 = unet_ref.seeded_unet(unet_ref.TINY_CONFIG, seed=8888, dtype=torch.float32, device=dev)
    net = I2VGenXLUNet(**unet_ref.TINY_CONFIG)
    net.load_state_dict(ref32.state_dict())
    net = net.to(device=dev, dtype=torch.float16).eval()
    pipe = SimpleNamespace(unet=net)
    s = schedulers_ref.DDIMScheduler()
    s.set_timesteps(10)
    for reg in (pnp_utils.register_conv_injection, pnp_utils.register_spatial_attention_pnp, pnp_utils.register_temp_attention_pnp):
        reg(pipe, s.timesteps[:5])
    ns = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, seed=8888, dtype=torch.float16, device=dev)
    prompts, img_lat, img_emb, fps = loops_ref.edit_conditioning(ns)
    g = torch.Generator().manual_seed(8895)
    x2 = torch.randn(2, 4, F_, H_, W_, generator=g).to(device=dev, dtype=torch.float16)
    x3 = torch.cat([x2, x2[1:2]])
    img_lat = torch.cat([img_lat[:2], img_lat[1:2]])
    for t in (901, 101):
        pnp_utils.register_time(pipe, t)
        for b0 in (0, 1):
            args = (x3[b0:], torch.tensor([t], device=dev), fps[b0:], img_lat[b0:], img_emb[b0:], prompts[b0:])
            plain = net(*args)[0]
            shared = net(*args, shared_edit_prefix=True)[0]
            assert_fp16_close(shared, plain.float(), f"shared prefix t={t} B={3 - b0}", rtol=2e-3, atol_frac=2e-3)
    # prune_source_after: the source branch dropped after the last firing site; [uncond, cond] must not change
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    t = 901
    pnp_utils.register_time(pipe, t)
    args = (x3, torch.tensor([t], device=dev), fps, img_lat, img_emb, prompts)
    plain = net(*args)[0]
    for site in ((3, 2, "temporal"), (3, 2, "spatial"), (1, 1, "resnet")):
        # every hook fires at t = 901, so only the temporal site is the true last one; the earlier sites are still valid
        # prune points for the layers behind them only if nothing fires later — check the true one exactly, and that the
        # others run (shapes, finiteness)
        pruned = net(*args, prune_source_after=site)[0]
        assert pruned.shape[0] == 2 and torch.isfinite(pruned).all()
        if site == I2VGenXLPipeline._prune_site((True, True, True)):
            assert_fp16_close(pruned, plain[1:].float(), f"source pruning at {site}", rtol=2e-3, atol_frac=2e-3)
            both = net(*args, prune_source_after=site, shared_edit_prefix=True)[0]
            assert_fp16_close(both, plain[1:].float(), f"source pruning + shared prefix at {site}", rtol=2e-3, atol_frac=2e-3)


@torch.no_grad()
def test_long_clip_128_frames_hooked_step(models):
    """BASELINE configs[4]: a 128-frame clip through the whole (tiny-topology) UNet with every hook firing — temporal sequences of
    128 frames, temporal convolutions over 128 frames, clip-level GroupNorm samples 32x larger than at 4 frames"""
    from anyv2v_b200 import pnp_utils as ours_hooks
    from oracle import loops_ref, pnp_hooks_ref, schedulers_ref
    F, H, W = 128, 16, 16
    s = schedulers_ref.DDIMScheduler()
    s.set_timesteps(10)
    schedule, t = s.timesteps[:5], 901
    outs = {}
    for name, net, dt, hooks in (("ref32", models.ref32, torch.float32, pnp_hooks_ref), ("ref16", models.ref16, torch.float16, pnp_hooks_ref),
                                 ("ours", models.ours, torch.float16, ours_hooks)):
        pipe = SimpleNamespace(unet=net)
        hooks.register_conv_injection(pipe, schedule)
        hooks.register_spatial_attention_pnp(pipe, schedule)
        hooks.register_temp_attention_pnp(pipe, schedule)
        hooks.register_time(pipe, t)
        ns = loops_ref.synthetic_inputs(F, H, W, cross_dim=64, seed=8888, dtype=dt, device=dev)
        prompts, img_lat, img_emb, fps = loops_ref.edit_conditioning(ns)
        g = torch.Generator().manual_seed(8895)
        x3 = torch.randn(3, 4, F, H, W, generator=g).to(device=dev, dtype=dt)
        outs[name] = net(x3, torch.tensor([t], device=dev), fps, img_lat, img_emb, prompts)[0]
    _check_vs_oracles(outs["ours"], outs["ref32"], outs["ref16"], "tiny UNet, 128 frames, hooked step")
    for net, hooks in ((models.ref32, pnp_hooks_ref), (models.ref16, pnp_hooks_ref), (models.ours, ours_hooks)):
        pipe = SimpleNamespace(unet=net)
        hooks.register_conv_injection(pipe, [])
        hooks.register_spatial_attention_pnp(pipe, [])
        hooks.register_temp_attention_pnp(pipe, [])
        hooks.register_time(pipe, -1)
