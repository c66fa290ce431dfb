"""Clips of any frame count on the GPU: the frames-mode attention kernels at frame counts that do not divide 128 (packed with an
empty tail of slots) and that are not multiples of 128 (unpacked with a ragged last tile), then the full-size UNet, one audited
edit step and the three sampling loops at those counts.

- Kernels: guarded float64-contract checks (tests/guarded.py via test_gpu_contracts._run), last pixel tile ragged, row
  strides above C.
- Full width: the criterion of test_gpu_fullwidth._check (ours against fp32 within 3 x torch-fp16's error).
- Audit: every kernel call of an injected 512^2 edit step at F = 24 against its float64 contract (tests/call_audit.py).
  The audit synchronises after each call, so the step runs eagerly; the loops below check that graph replay equals eager.
- Loops: invert, sample_with_pnp and pipe(...) at 512^2 and F = 24 on the CUDA-graph path.
"""
from types import SimpleNamespace

import pytest
import torch

import test_gpu_contracts as gc
import test_gpu_fullwidth as fw
from test_gpu_step_audit import CONFIG3, _expect, _Pass

pytestmark = pytest.mark.gpu
dev = "cuda"


# ------------------------------------------------------------------------------------------------------------- kernels
def _ragged_hw(F):
    """a pixel count whose last tile of floor(128 / F) pixels is partly empty (one pixel per tile from F = 65: 3 tiles)"""
    ppt = 128 // F if F <= 128 else 1
    return 2 * ppt + 1 if ppt > 1 else 3


@pytest.mark.parametrize("nv", [1, 3])
@pytest.mark.parametrize("F", [3, 5, 24, 40, 48, 56, 72, 96, 120])
def test_attention_frames_packed_any_count_guarded(F, nv):
    """packed frames with floor(128 / F) pixels per CTA and slots floor(128 / F) * F .. 127 empty"""
    gc.test_attention_frames_guarded((2, 2, F, _ragged_hw(F), nv))


@pytest.mark.parametrize("nv", [1, 3])
@pytest.mark.parametrize("F", [136, 200])
def test_attention_frames_unpacked_ragged_tile_guarded(F, nv):
    """F > 128 and not a multiple of 128: the last query tile is partly empty and keys past F are masked"""
    gc.test_attention_frames_guarded((1, 2, F, 2, nv))


@pytest.mark.parametrize("nv", [1, 3])
@pytest.mark.parametrize("Cx", [64, 320])
@pytest.mark.parametrize("F", [3, 24, 40, 48, 72, 120])
def test_temporal_attention_fused_any_count_guarded(F, Cx, nv):
    """the fused projection + attention with an empty slot tail, pixels straddling the 64-slot halves (both warpgroups visit
    both key tiles), a ragged last pixel tile, ldx > Cx with a NaN gap, ldo > C"""
    heads, src = 2, 2
    C = heads * 64
    HW = _ragged_hw(F)
    clips = src * nv
    rows = clips * F * HW
    torch.manual_seed(F * 7 + Cx + nv)
    x = gc.gin(gc.rnd(rows, Cx), ld=Cx + 8, guard=128 * (Cx + 8))
    out = gc.gout((rows, C), ld=C + 8)
    gc._run("temporal_attention_fused", [x, gc.gin(gc._w(3 * C, Cx)), heads, F, HW, clips, out], dict(scale=0.3, n_v=nv),
            [out], atol_frac=2e-3)


# ------------------------------------------------------------------------------------------------------------- full width
@pytest.fixture(scope="module")
def full():
    m = fw.build_models(dev)
    yield m
    del m
    torch.cuda.empty_cache()


@torch.no_grad()
def test_fullwidth_24_frames_hooked_edit_and_inversion_forward(full):
    """F = 24 at 32 x 32: a hooked step with conv, spatial and temporal injection (B = 3), then the unhooked B = 1 forward"""
    F = 24
    _, schedule = fw._schedule()
    fw._register(full, schedule, 901)
    outs = {}
    for name, net, dt in (("ours", full.ours, torch.float16), ("ref32", full.ref32, torch.float32), ("ref16", full.ref16, torch.float16)):
        _, x3, prompts, img_lat, img_emb, fps = fw._inputs(dt, F)
        outs[name] = net(x3, torch.tensor([901], device=dev), fps, img_lat, img_emb, prompts)[0]
    assert outs["ours"].shape == (3, 4, F, fw.H_, fw.W_)
    assert full.ours.up_blocks[3].temp_attentions[2].transformer_blocks[0].attn1.processor.inject_now()
    fw._check(outs["ours"], outs["ref32"], outs["ref16"], "full-width hooked UNet step, 24 frames")
    fw._register(full, [], -1)
    for name, net, dt in (("ours", full.ours, torch.float16), ("ref32", full.ref32, torch.float32), ("ref16", full.ref16, torch.float16)):
        ns, _, _, _, _, _ = fw._inputs(dt, F)
        outs[name] = net(ns.video_latents, torch.tensor([21], device=dev), ns.fps, ns.src_image_latents, ns.src_image_emb, ns.inv_prompt)[0]
    fw._check(outs["ours"], outs["ref32"], outs["ref16"], "full-width inversion-geometry forward, 24 frames")


@torch.no_grad()
def test_fullwidth_72_frames_forward(full):
    """F = 72: one pixel per CTA with 56 empty slots, in the fused kernel and in every temporal layer"""
    F = 72
    fw._register(full, [], -1)
    outs = {}
    for name, net, dt in (("ours", full.ours, torch.float16), ("ref32", full.ref32, torch.float32), ("ref16", full.ref16, torch.float16)):
        ns, _, _, _, _, _ = fw._inputs(dt, F)
        outs[name] = net(ns.video_latents, torch.tensor([501], device=dev), ns.fps, ns.src_image_latents, ns.src_image_emb, ns.inv_prompt)[0]
        torch.cuda.empty_cache()
    fw._check(outs["ours"], outs["ref32"], outs["ref16"], "full-width forward, 72 frames")


@torch.no_grad()
def test_fullwidth_finest_level_block_alone_24_frames(full):
    """up_blocks[3] (320 channels) at 64 x 64 with F = 24, all three hooks firing: 4096 pixels, 5 per fused-kernel CTA"""
    from anyv2v_b200.unet_i2vgen_xl import to_nhwc
    B, F, H, W = 3, 24, 64, 64
    _, schedule = fw._schedule()
    fw._register(full, schedule, 901)
    g = torch.Generator().manual_seed(2424)
    rn = lambda *s: torch.randn(*s, generator=g).to(dev)
    c0, c1 = fw._config()["block_out_channels"][:2]
    x = rn(B * F, c1, H, W)
    skips = [rn(B * F, c0, H, W) for _ in range(3)]
    emb = rn(B * F, 4 * c0)
    ctx = rn(B, 145, fw._config()["cross_attention_dim"])
    outs = {}
    for name, net, dt in (("ref32", full.ref32, torch.float32), ("ref16", full.ref16, torch.float16)):
        c = lambda z: z.to(dt)
        outs[name] = net.up_blocks[3](c(x), tuple(c(s) for s in skips), c(emb), c(ctx).repeat_interleave(F, dim=0), F)
        torch.cuda.empty_cache()
    h = lambda z: z.half()
    y = full.ours.up_blocks[3].forward_nhwc(to_nhwc(h(x)), [to_nhwc(h(s)) for s in skips], h(emb).contiguous(), h(ctx).contiguous(), F)
    fw._check(y.permute(0, 3, 1, 2), outs["ref32"], outs["ref16"], "up_blocks[3] alone at 64x64, 24 frames, injected")
    fw._register(full, [], -1)


# ------------------------------------------------------------------------------------------------------------- 512^2, F = 24
F24 = 24


@pytest.fixture(scope="module")
def unet():
    from anyv2v_b200 import distributed
    from anyv2v_b200.unet_i2vgen_xl import I2VGEN_XL_CONFIG, I2VGenXLUNet
    net = distributed.build_unet_replicated(I2VGenXLUNet, I2VGEN_XL_CONFIG, 8888, torch.device(dev))
    yield net
    del net
    torch.cuda.empty_cache()


def _conditioning():
    from anyv2v_b200.run_group_pnp_edit import synthetic_conditioning
    return {k: v.to(dev) for k, v in synthetic_conditioning(F24, 64, 64, 1024, 8888, "cpu").items()}


def _unhook(net):
    from anyv2v_b200 import pnp_utils
    pipe = SimpleNamespace(unet=net)
    for reg in (pnp_utils.register_conv_injection, pnp_utils.register_spatial_attention_pnp, pnp_utils.register_temp_attention_pnp):
        reg(pipe, [])
    pnp_utils.register_time(pipe, -1)


def _store(timesteps):
    from anyv2v_b200.latent_store import LatentStore
    store = LatentStore(None, write_files=False)
    g = torch.Generator().manual_seed(3)
    for t in timesteps:
        store.put(int(t), torch.randn(1, 4, F24, 64, 64, generator=g).half().to(dev))
    return store


@torch.no_grad()
def test_audited_edit_step_24_frames(unet, monkeypatch):
    """edit step 0 of BASELINE config 3 (conv, spatial and temporal injection) at 24 x 512^2: every call against its contract"""
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp
    from anyv2v_b200.schedulers import DDIMScheduler
    c = _conditioning()
    sched = DDIMScheduler()
    sched.set_timesteps(CONFIG3.n_steps)
    pipe = I2VGenXLPipeline(unet, sched)
    pipe.use_cuda_graphs = False
    pipe.disable_freeu()
    init_pnp(pipe, sched, CONFIG3)
    st = pipe.prepare_edit(c["video_latents"].clone(), c["edit_prompt"], c["neg_prompt"], c["inv_prompt"], c["edit_image_emb"],
                           c["edit_image_latents"], c["src_image_emb"], c["src_image_latents"], 8, CONFIG3.n_steps, 9.0, 0, None,
                           _store(sched.timesteps.tolist()), True)
    assert pipe._hook_flags(st.timesteps[0]) == (True, True, True)
    p = _Pass(monkeypatch, "edit step 0 (all injections), 24 frames", seed=24)
    pipe.edit_step(st, 0)
    a = p.finish()
    _expect(a, "temporal_attention_fused", n_v=3, F=F24, HW=4096)
    _expect(a, "temporal_attention_fused", n_v=1, F=F24)
    _expect(a, "attention", mode="rows", n_v=3, seq=4096)
    _expect(a, "tconv3", F=F24)
    assert not a.seen("attention", mode="frames")
    _unhook(unet)


@torch.no_grad()
def test_loops_24_frames_graph_replay_equals_eager(unet):
    """invert and sample_with_pnp for 3 steps each (every hook fires on the edit steps), eager and on the CUDA-graph path"""
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp
    from anyv2v_b200.schedulers import DDIMInverseScheduler, DDIMScheduler
    c = _conditioning()
    n = 3
    results = {}
    _unhook(unet)
    for graphs in (False, True):
        pipe = I2VGenXLPipeline(unet, DDIMInverseScheduler())
        pipe.use_cuda_graphs = graphs
        pipe.disable_freeu()
        inv = pipe.invert(latents=c["video_latents"], prompt_embeds=c["inv_prompt"], image_latents=c["src_image_latents"],
                          image_embeddings=c["src_image_emb"], target_fps=8, num_inference_steps=n, guidance_scale=1.0,
                          write_files=False)
        store = pipe.latent_store
        es = DDIMScheduler()
        es.set_timesteps(n)
        pipe.scheduler = es
        init_pnp(pipe, es, SimpleNamespace(n_steps=n, pnp_f_t=1.0, pnp_spatial_attn_t=1.0, pnp_temp_attn_t=1.0))
        out = pipe.sample_with_pnp(latents=store.get(es.timesteps.tolist()[0]).clone(), prompt_embeds=c["edit_prompt"],
                                   negative_prompt_embeds=c["neg_prompt"], ddim_inv_prompt_embeds=c["inv_prompt"],
                                   image_embeddings=c["edit_image_emb"], image_latents=c["edit_image_latents"],
                                   ddim_inv_image_embeddings=c["src_image_emb"], ddim_inv_image_latents=c["src_image_latents"],
                                   target_fps=8, num_inference_steps=n, guidance_scale=9.0, ddim_init_latents_t_idx=0,
                                   latent_store=store).frames
        torch.cuda.synchronize()
        results[graphs] = (inv.clone(), out.clone())
        _unhook(unet)
    inv, out = results[True]
    assert inv.shape[-3:] == (F24, 64, 64) and out.shape == (1, 4, F24, 64, 64)
    assert torch.isfinite(inv).all() and torch.isfinite(out).all()
    assert torch.equal(results[False][0], inv), "inversion: graph replay differs from eager launches"
    assert torch.equal(results[False][1], out), "edit: graph replay differs from eager launches"


@torch.no_grad()
def test_image_to_video_call_24_frames(unet):
    """pipe(..., num_frames=24, output_type="latent"), 2 steps on the CUDA-graph path (the second replays), against eager"""
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.schedulers import DDIMScheduler
    c = _conditioning()
    pipe = I2VGenXLPipeline(unet, DDIMScheduler())
    pipe.disable_freeu()
    outs = {}
    for graphs in (False, True):
        pipe.use_cuda_graphs = graphs
        outs[graphs] = pipe(prompt_embeds=c["edit_prompt"], negative_prompt_embeds=c["neg_prompt"],
                            image_embeddings=c["edit_image_emb"], image_latents=c["edit_image_latents"],
                            latents=c["video_latents"], num_frames=F24, target_fps=8, output_type="latent",
                            generator=torch.Generator(device=dev).manual_seed(1), max_steps=2).frames.clone()
    torch.cuda.synchronize()
    assert outs[True].shape == (1, 4, F24, 64, 64) and torch.isfinite(outs[True]).all()
    assert torch.equal(outs[True], outs[False])
