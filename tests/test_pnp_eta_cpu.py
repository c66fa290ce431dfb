"""Stochastic DDIM (eta > 0) in the PnP edit, `I2VGenXLPipeline.sample_with_pnp(eta=..., generator=...)`, without a GPU: the
product loop on the tiny UNet (kernels replaced by their contracts) against the reference's edit loop with
`DDIMScheduler.step(..., eta, generator)` (tests/pnp_eta_ref.py), in every step body (pruned source,
full three-branch, dead source); the generator's draws; eta = 0 bit for bit as the loop was before it took eta; the
refusals.  tests/test_gpu_pnp_eta.py runs ``run_edit_teacher_forced`` on the GPU kernels."""
from types import SimpleNamespace

import pytest
import torch

import pnp_eta_ref
import sampling_ref
from test_host_model_cpu import F_, H_, W_, _close, _models

N_STEPS = 4
#: conv injection on steps 0-2, spatial attention on 0-1, temporal attention on step 0 only, so that with
#: skip_dead_source_branch the source is pruned after the temporal (step 0), spatial (1) and resnet (2) sites and step 3
#: runs the dead-source two-branch body
PNP = SimpleNamespace(n_steps=N_STEPS, pnp_f_t=0.75, pnp_spatial_attn_t=0.5, pnp_temp_attn_t=0.25)
FLAGS = [(True, True, True), (True, True, False), (True, False, False), (False, False, False)]


@pytest.fixture
def emu(emulated_ops, monkeypatch):
    """the kernel contracts in place of anyv2v_b200.ops, ops.ddim_step_eta included"""
    sampling_ref.patch_ops(monkeypatch)
    return emulated_ops


def _store(device):
    """random source latents at every timestep of the schedule (what an inversion would have stored)"""
    from anyv2v_b200.latent_store import LatentStore
    from anyv2v_b200.schedulers import DDIMScheduler
    s = DDIMScheduler()
    s.set_timesteps(N_STEPS)
    store = LatentStore(None, write_files=False)
    g = torch.Generator().manual_seed(5)
    for t in s.timesteps.tolist():
        store.put(int(t), torch.randn(1, 4, F_, H_, W_, generator=g).half().to(device))
    return store


def _edit_pipeline(ours):
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp
    from anyv2v_b200.schedulers import DDIMScheduler
    sched = DDIMScheduler()
    sched.set_timesteps(N_STEPS)
    pipe = I2VGenXLPipeline(ours, sched)
    init_pnp(pipe, sched, PNP)
    return pipe


def _edit_kwargs(ns, store):
    return dict(prompt_embeds=ns.edit_prompt, negative_prompt_embeds=ns.neg_prompt, ddim_inv_prompt_embeds=ns.inv_prompt,
                image_embeddings=ns.edit_image_emb, image_latents=ns.edit_image_latents,
                ddim_inv_image_embeddings=ns.src_image_emb, ddim_inv_image_latents=ns.src_image_latents, target_fps=8,
                num_inference_steps=N_STEPS, guidance_scale=9.0, ddim_init_latents_t_idx=0, latent_store=store)


def _capture_states(pipe):
    """the loop states ``sample_with_pnp`` builds, so that a test can look at the graphs they keyed"""
    states = []
    real = pipe.prepare_edit
    pipe.prepare_edit = lambda *a, **kw: states.append(real(*a, **kw)) or states[-1]
    return states


def run_edit_teacher_forced(ref32, ours, eta, skip, device, rms=6e-3, mx=3e-2, seed=8888):
    """``sample_with_pnp(eta=eta, generator=torch.Generator().manual_seed(seed))`` against the reference's stochastic edit
    loop on the fp32 oracle UNet with the reference's hooks, teacher-forced per step with the product's latents; the oracle
    draws its own noise from an equally seeded generator, so every step also checks that the product drew the same noise.
    -> (product's final latents, its loop state)"""
    from oracle import loops_ref, pnp_hooks_ref, schedulers_ref
    ns16 = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float16, device=device)
    ns32 = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float32, device=device)
    store = _store(device)
    pipe = _edit_pipeline(ours)
    states = _capture_states(pipe)
    g_ours, g_ref = torch.Generator().manual_seed(seed), torch.Generator().manual_seed(seed)
    seen = []
    out = pipe.sample_with_pnp(latents=ns16.video_latents.clone(), eta=eta, generator=g_ours, skip_dead_source_branch=skip,
                               callback=lambda i, t, x: seen.append((i, t, x.clone())), return_dict=False,
                               **_edit_kwargs(ns16, store))[0]
    st = states[0]
    assert len(seen) == N_STEPS and [pipe._hook_flags(t) for t in st.timesteps] == FLAGS
    sref = schedulers_ref.DDIMScheduler()
    sref.set_timesteps(N_STEPS)
    rp = SimpleNamespace(unet=ref32)
    pnp_hooks_ref.init_pnp(rp, sref, N_STEPS, PNP.pnp_f_t, PNP.pnp_spatial_attn_t, PNP.pnp_temp_attn_t)
    inv32 = {t: store.get(t, device=device).float() for t in st.timesteps}
    prompts, img_lat, img_emb, fps3 = loops_ref.edit_conditioning(ns32)
    x_prev = ns16.video_latents.float()
    for i, t, x_ours in seen:
        want = pnp_eta_ref.pnp_edit_loop_eta(rp, pnp_hooks_ref.register_time, inv32, x_prev, prompts, img_lat, img_emb, fps3,
                                              N_STEPS, 9.0, eta, generator=g_ref, t_idx=i, max_steps=1)
        _close(x_ours, want, f"edit step {i} (t={t}) eta={eta} skip={skip}", rms=rms, mx=mx)
        x_prev = x_ours.float()
    assert torch.equal(g_ours.get_state(), g_ref.get_state())      # both made the same draws, dead-source steps included
    return out, st


@torch.no_grad()
@pytest.mark.parametrize("skip", [True, False])
@pytest.mark.parametrize("eta", [0.5, 1.0])
def test_stochastic_edit_matches_the_reference_loop(emu, eta, skip):
    ref32, ours = _models()
    _, st = run_edit_teacher_forced(ref32, ours, eta, skip, "cpu")
    fs = ours.freeu_state()
    dead = [skip and not any(f) for f in FLAGS]
    assert set(st.iterations) == {(d, f, fs, True) for d, f in zip(dead, FLAGS)}
    assert st.g_noise is not None and st.coef_table.shape == (N_STEPS, 6)


@torch.no_grad()
def test_noise_is_drawn_every_step_in_the_reference_order(emu, monkeypatch):
    """one [F, C, h, w] draw per step, dead-source steps included, each landing in the latents' [1, C, F, h, w] order"""
    from anyv2v_b200 import pipeline as pl
    from oracle import loops_ref
    draws = []
    real = pl.randn_tensor

    def spy(*a, **kw):
        z = real(*a, **kw)
        draws.append(z.clone())
        return z
    monkeypatch.setattr(pl, "randn_tensor", spy)
    _, ours = _models()
    ns = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float16, device="cpu")
    pipe = _edit_pipeline(ours)
    st = pipe.prepare_edit(ns.video_latents.clone(), ns.edit_prompt, ns.neg_prompt, ns.inv_prompt, ns.edit_image_emb,
                           ns.edit_image_latents, ns.src_image_emb, ns.src_image_latents, 8, N_STEPS, 9.0, 0, None, _store("cpu"),
                           True, 1.0, torch.Generator().manual_seed(3))
    for i in range(N_STEPS):
        pipe.edit_step(st, i)
        assert len(draws) == i + 1 and draws[-1].shape == (F_, 4, H_, W_)
        assert torch.equal(st.g_noise[0], draws[-1].transpose(0, 1))
    assert st.fires == [True, True, True, False]                     # the last step ran the dead-source body


def _parent_edit_step(pipe, st, i):
    """``edit_step`` as it was before the loop took eta: the reference for eta = 0"""
    from anyv2v_b200.pnp_utils import register_time
    t = st.timesteps[i]
    register_time(pipe, t)
    dead_source = st.skip and not st.fires[i]
    flags = pipe._hook_flags(t)

    def make_body():
        if dead_source:
            def body():
                v = pipe.unet(torch.cat([st.latents, st.latents]), st.g_t, cond=st.cond2,
                              shared_edit_prefix=st.shared_prefix)[0]
                st.scheduler.step(v[0:1], None, st.latents, model_output_cond=v[1:2], out=st.latents, coef_dev=st.g_coef)
            return body
        site = pipe._prune_site(flags) if st.prune_source else None
        lo = 0 if site is not None else 1

        def body():
            v = pipe.unet(torch.cat([st.g_src, st.latents, st.latents]), st.g_t, cond=st.cond3,
                          shared_edit_prefix=st.shared_prefix, prune_source_after=site)[0]
            st.scheduler.step(v[lo:lo + 1], None, st.latents, model_output_cond=v[lo + 1:lo + 2], out=st.latents,
                              coef_dev=st.g_coef)
        return body
    if not dead_source:
        st.g_src.copy_(st.store.get(t, device=st.latents.device), non_blocking=True)
    return pipe._run(st, i, (dead_source, flags, pipe.unet.freeu_state()), make_body)


@torch.no_grad()
@pytest.mark.parametrize("skip", [True, False])
def test_eta_zero_is_the_loop_without_eta(emu, skip):
    """eta = 0 (with a generator given): no noise buffer, no draw, the same launches, the same graph keys and bit for bit
    the latents of the loop before it took eta"""
    from oracle import loops_ref
    _, ours = _models()
    ns = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float16, device="cpu")
    store = _store("cpu")
    pipe = _edit_pipeline(ours)
    states = _capture_states(pipe)
    g = torch.Generator().manual_seed(8888)
    g0 = g.get_state()
    n0 = emu.launch_count()
    got = pipe.sample_with_pnp(latents=ns.video_latents.clone(), eta=0.0, generator=g, skip_dead_source_branch=skip,
                               return_dict=False, **_edit_kwargs(ns, store))[0]
    launches = emu.launch_count() - n0
    st = states[0]
    assert st.g_noise is None and torch.equal(g.get_state(), g0)
    assert torch.equal(st.coef_table, pipe.scheduler.coefficient_table(st.timesteps, 9.0, "cpu"))
    n0 = emu.launch_count()
    old = pipe.prepare_edit(ns.video_latents.clone(), ns.edit_prompt, ns.neg_prompt, ns.inv_prompt, ns.edit_image_emb,
                            ns.edit_image_latents, ns.src_image_emb, ns.src_image_latents, 8, N_STEPS, 9.0, 0, None, store, skip)
    for i in range(N_STEPS):
        _parent_edit_step(pipe, old, i)
    assert emu.launch_count() - n0 == launches
    assert set(st.iterations) == set(old.iterations)
    assert torch.isfinite(got.float()).all() and torch.equal(got, old.latents)


def test_refusals(emu):
    from oracle import loops_ref
    _, ours = _models()
    ns = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float16, device="cpu")
    pipe = _edit_pipeline(ours)
    kw = _edit_kwargs(ns, _store("cpu"))
    with pytest.raises(ValueError, match="eta must be >= 0"):
        pipe.sample_with_pnp(latents=ns.video_latents.clone(), eta=-0.1, **kw)
    with pytest.raises(ValueError, match="single torch.Generator"):
        pipe.sample_with_pnp(latents=ns.video_latents.clone(), eta=1.0,
                             generator=[torch.Generator().manual_seed(1), torch.Generator().manual_seed(2)], **kw)
    # a list of one generator is that generator
    g = torch.Generator().manual_seed(4)
    a = pipe.sample_with_pnp(latents=ns.video_latents.clone(), eta=1.0, generator=[g], max_steps=1, return_dict=False, **kw)[0]
    b = pipe.sample_with_pnp(latents=ns.video_latents.clone(), eta=1.0, generator=torch.Generator().manual_seed(4), max_steps=1,
                             return_dict=False, **kw)[0]
    assert torch.equal(a, b)
