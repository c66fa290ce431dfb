"""Source-feature sharing between PnP edits of one inverted clip (`I2VGenXLPipeline.source_feature_cache`,
`sample_with_pnp(..., source_features=cache)`) without a GPU: the tiny UNet with the kernel contracts in place of the kernels.
A second edit of the same inversion, with another prompt, edited first frame and injection schedule, must be bit for bit the
same edit run without the cache at every step: with partial coverage, an exhausted budget, FreeU switched between steps and
eta = 1.  tests/test_gpu_source_cache.py runs the same on the kernels at full size."""
from types import SimpleNamespace

import pytest
import torch

import freeu_ref
import sampling_ref
import source_cache_ref
from test_host_model_cpu import F_, H_, W_, _models

N_STEPS = 5
#: the first edit injects on fewer steps than the second, so the second replays some injected steps and captures others
SCHED_A = SimpleNamespace(n_steps=N_STEPS, pnp_f_t=0.6, pnp_spatial_attn_t=0.4, pnp_temp_attn_t=0.2)
SCHED_B = SimpleNamespace(n_steps=N_STEPS, pnp_f_t=0.8, pnp_spatial_attn_t=0.6, pnp_temp_attn_t=0.4)


@pytest.fixture
def emu(emulated_ops, monkeypatch):
    sampling_ref.patch_ops(monkeypatch)
    freeu_ref.patch_ops(monkeypatch)
    source_cache_ref.patch_ops(monkeypatch)
    return emulated_ops


def _store(device, seed=5):
    """random source latents at every timestep of the schedule (what an inversion would have stored)"""
    from anyv2v_b200.latent_store import LatentStore
    from anyv2v_b200.schedulers import DDIMScheduler
    s = DDIMScheduler()
    s.set_timesteps(N_STEPS)
    store = LatentStore(None, write_files=False)
    g = torch.Generator().manual_seed(seed)
    for t in s.timesteps.tolist():
        store.put(int(t), torch.randn(1, 4, F_, H_, W_, generator=g).half().to(device))
    return store


def _inputs(seed):
    """the source conditioning of the synthetic clip, and an edit (prompt, edited first frame) drawn from `seed`"""
    from oracle import loops_ref
    ns = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float16, device="cpu")
    g = torch.Generator().manual_seed(seed)
    rn = lambda t: (t.float() + torch.randn(t.shape, generator=g)).half()
    ns.edit_prompt, ns.edit_image_emb, ns.edit_image_latents = rn(ns.edit_prompt), rn(ns.edit_image_emb), rn(ns.edit_image_latents)
    return ns


def _pipeline(ours):
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.schedulers import DDIMScheduler
    sched = DDIMScheduler()
    sched.set_timesteps(N_STEPS)
    return I2VGenXLPipeline(ours, sched)


def _edit(pipe, ns, store, sched, cache=None, eta=0.0, seed=11, freeu_from=None, **kw):
    """one edit with the injection schedule `sched`; FreeU switched on after step `freeu_from` (and off at the end).
    -> (latents after every step, the graph keys of the loop)"""
    from anyv2v_b200.run_group_pnp_edit import init_pnp
    init_pnp(pipe, pipe.scheduler, sched)
    states, real = [], pipe.prepare_edit
    pipe.prepare_edit = lambda *a, **k: states.append(real(*a, **k)) or states[-1]
    seen = []

    def cb(i, t, x):
        seen.append(x.clone())
        if freeu_from is not None and i == freeu_from:
            pipe.enable_freeu(s1=0.9, s2=0.2, b1=1.2, b2=1.4)
    try:
        pipe.sample_with_pnp(latents=ns.video_latents.clone(), prompt_embeds=ns.edit_prompt, negative_prompt_embeds=ns.neg_prompt,
                             ddim_inv_prompt_embeds=ns.inv_prompt, image_embeddings=ns.edit_image_emb,
                             image_latents=ns.edit_image_latents, ddim_inv_image_embeddings=ns.src_image_emb,
                             ddim_inv_image_latents=ns.src_image_latents, target_fps=8, num_inference_steps=N_STEPS,
                             guidance_scale=9.0, ddim_init_latents_t_idx=0, latent_store=store, eta=eta,
                             generator=torch.Generator().manual_seed(seed), source_features=cache, callback=cb, **kw)
    finally:
        pipe.prepare_edit = real
        pipe.disable_freeu()
    return seen, set(states[0].iterations)


def _modes(keys):
    return sorted(k[-1] for k in keys if k[-1] in ("capture", "replay"))


def _assert_same(got, want):
    assert len(got) == len(want) == N_STEPS
    for i, (a, b) in enumerate(zip(got, want)):
        assert torch.isfinite(a.float()).all() and torch.equal(a, b), f"step {i} differs from the edit without the cache"


@torch.no_grad()
@pytest.mark.parametrize("eta", [0.0, 1.0])
def test_second_edit_equals_the_uncached_edit(emu, eta):
    _, ours = _models()
    pipe = _pipeline(ours)
    store = _store("cpu")
    cache = pipe.source_feature_cache(max_bytes=1 << 40)
    _, keys_a = _edit(pipe, _inputs(1), store, SCHED_A, cache, eta=eta, seed=1)
    assert _modes(keys_a) == ["capture"] * 3      # three distinct injected step kinds, all captured
    filled = len(cache)
    assert filled == 3 and cache.nbytes > 0
    ns_b = _inputs(2)
    got, keys_b = _edit(pipe, ns_b, store, SCHED_B, cache, eta=eta, seed=2)
    want, keys_plain = _edit(pipe, ns_b, store, SCHED_B, None, eta=eta, seed=2)
    _assert_same(got, want)
    assert "replay" in _modes(keys_b) and "capture" in _modes(keys_b)   # partial coverage: some steps replay, some capture
    assert len(cache) > filled
    assert not any(k[-1] in ("capture", "replay") for k in keys_plain)
    # a third edit finds every injected step of its schedule in the cache
    ns_c = _inputs(3)
    got, keys_c = _edit(pipe, ns_c, store, SCHED_B, cache, eta=eta, seed=3)
    want, _ = _edit(pipe, ns_c, store, SCHED_B, None, eta=eta, seed=3)
    _assert_same(got, want)
    assert set(_modes(keys_c)) == {"replay"}
    # the sites are left without features: a plain edit afterwards is the plain edit
    from anyv2v_b200.pipeline import _pnp_sites
    assert all(getattr(s, "source_feature", None) is None for _, s in _pnp_sites(ours))


@torch.no_grad()
def test_exhausted_budget(emu):
    """a budget of one step's features: the first edit keeps one step, the rest run as without the cache"""
    _, ours = _models()
    pipe = _pipeline(ours)
    store = _store("cpu")
    probe = pipe.source_feature_cache(max_bytes=1 << 40)
    _edit(pipe, _inputs(1), store, SCHED_B, probe)
    one = max(sum(f.numel() * f.element_size() for f in e.values()) for e in probe.entries.values())
    cache = pipe.source_feature_cache(max_bytes=one)
    _edit(pipe, _inputs(1), store, SCHED_B, cache)
    assert len(cache) == 1 and cache.nbytes <= one
    ns_b = _inputs(2)
    got, keys = _edit(pipe, ns_b, store, SCHED_B, cache, seed=2)
    want, _ = _edit(pipe, ns_b, store, SCHED_B, None, seed=2)
    _assert_same(got, want)
    assert "replay" in _modes(keys) and len(cache) == 1
    empty = pipe.source_feature_cache(max_bytes=0)
    got, keys = _edit(pipe, ns_b, store, SCHED_B, empty, seed=2)
    _assert_same(got, want)
    assert len(empty) == 0 and "replay" not in _modes(keys)


@torch.no_grad()
def test_freeu_switched_between_steps(emu):
    """FreeU is part of what a cached step is: features captured without it are not replayed with it"""
    _, ours = _models()
    pipe = _pipeline(ours)
    store = _store("cpu")
    cache = pipe.source_feature_cache(max_bytes=1 << 40)
    _edit(pipe, _inputs(1), store, SCHED_B, cache, freeu_from=0)          # FreeU from step 1 on
    ns_b = _inputs(2)
    got, keys = _edit(pipe, ns_b, store, SCHED_B, cache, seed=2, freeu_from=1)   # FreeU from step 2 on
    want, _ = _edit(pipe, ns_b, store, SCHED_B, None, seed=2, freeu_from=1)
    _assert_same(got, want)
    # step 0 (no FreeU) and steps >= 2 (FreeU) were captured by the first edit; step 1 ran without FreeU this time
    assert _modes(keys).count("capture") == 1 and "replay" in _modes(keys)
    # the same edit with the cache again, FreeU never on: step 0 replays, the others capture
    got, _ = _edit(pipe, ns_b, store, SCHED_B, cache, seed=2)
    want, _ = _edit(pipe, ns_b, store, SCHED_B, None, seed=2)
    _assert_same(got, want)


@torch.no_grad()
def test_refuses_another_inversion(emu):
    _, ours = _models()
    pipe = _pipeline(ours)
    store = _store("cpu")
    cache = pipe.source_feature_cache(max_bytes=1 << 40)
    ns = _inputs(1)
    _edit(pipe, ns, store, SCHED_A, cache, max_steps=1)
    with pytest.raises(ValueError, match="another inversion"):
        _edit(pipe, ns, _store("cpu"), SCHED_A, cache, max_steps=1)
    other = _inputs(1)
    other.inv_prompt = other.inv_prompt + 1
    with pytest.raises(ValueError, match="ddim_inv_prompt_embeds"):
        _edit(pipe, other, store, SCHED_A, cache, max_steps=1)
    other = _inputs(1)
    other.src_image_latents = other.src_image_latents.clone()
    other.src_image_latents[0, :, 0] += 1
    with pytest.raises(ValueError, match="ddim_inv_image_latents"):
        _edit(pipe, other, store, SCHED_A, cache, max_steps=1)
    other = _inputs(1)
    other.src_image_emb = other.src_image_emb + 1
    with pytest.raises(ValueError, match="ddim_inv_image_embeddings"):
        _edit(pipe, other, store, SCHED_A, cache, max_steps=1)
    _, other_unet = _models()
    with pytest.raises(ValueError, match="another UNet"):
        _edit(_pipeline(other_unet), ns, store, SCHED_A, cache, max_steps=1)
    with pytest.raises(ValueError, match="max_bytes"):
        pipe.source_feature_cache(max_bytes=-1)
    # what the edit changes does not invalidate it
    _edit(pipe, _inputs(7), store, SCHED_B, cache, eta=1.0, max_steps=1, seed=4)
