"""GPU parity at BASELINE width: the full I2VGEN_XL_CONFIG (all 1 420 469 224 parameters: BN = 160 / 256 tile plans,
pair mode, GEGLU N = 2560 ... 10240, the 2560 -> 1280 three-slot injection conv) against the oracle on identical seeded
weights and inputs.  Reference call: i2vgen-xl/pipelines/pipeline_i2vgen_xl.py:1146-1155 with the hooks of
i2vgen-xl/pnp_utils.py:109-115 (conv), :189-196 (spatial), :295-302 (temporal).

The oracle runs on the same GPU with torch ops in strict fp32 (TF32 off, see conftest) and in fp16; criterion as in
test_gpu_model.py: our fp16 result must be as close to the fp32 oracle as torch's own fp16 run of the oracle is (x 3).
Geometry: B = 3 branches, F = 4 frames, 32 x 32 latents (levels 32 / 16 / 8 / 4) for the whole-model steps; the finest
level (4096-token sites, the injected N = 4096 attention with shared probabilities) is covered by running up_blocks[3]
alone at 64 x 64."""
import copy
from types import SimpleNamespace

import pytest
import torch

from parity_utils import err_stats

pytestmark = pytest.mark.gpu
dev = "cuda"
F_, H_, W_ = 4, 32, 32
#: None = the full-size I2VGEN_XL_CONFIG.  tests/test_host_model_cpu.py re-runs these functions on CPU with the tiny
#: topology-equivalent config and the float64 kernel contracts, so that the host-side wiring of this module is exercised
#: before any GPU minute is spent on it.
CONFIG_OVERRIDE = None


def _config():
    from oracle import unet_ref
    return CONFIG_OVERRIDE or unet_ref.I2VGEN_XL_CONFIG


def build_models(device, config=None):
    """config: None = this module's _config() (other modules pass their own override)"""
    from anyv2v_b200.unet_i2vgen_xl import I2VGEN_XL_CONFIG, I2VGenXLUNet
    from oracle import unet_ref
    assert I2VGEN_XL_CONFIG == unet_ref.I2VGEN_XL_CONFIG
    cfg = config or _config()
    ref32 = unet_ref.seeded_unet(cfg, seed=8888, dtype=torch.float32, device="cpu")
    if cfg == unet_ref.I2VGEN_XL_CONFIG:
        n_params = sum(p.numel() for p in ref32.parameters())
        assert n_params == 1_420_469_224, n_params
    with torch.device("meta"):
        ours = I2VGenXLUNet(**cfg)
    ours.load_state_dict(ref32.state_dict(), assign=True)  # same names / shapes as diffusers
    ours = ours.to(device=device, dtype=torch.float16).eval()
    ref16 = copy.deepcopy(ref32).to(device=device, dtype=torch.float16).eval()
    ref32 = ref32.to(device)
    for net in (ours, ref16, ref32):
        for p in net.parameters():
            p.requires_grad_(False)
    return SimpleNamespace(ref32=ref32, ref16=ref16, ours=ours)


@pytest.fixture(scope="module")
def full():
    return build_models(dev)


def _inputs(dtype, F=F_, H=H_, W=W_):
    from oracle import loops_ref
    ns = loops_ref.synthetic_inputs(F, H, W, cross_dim=_config()["cross_attention_dim"], seed=8888, dtype=dtype, device=dev)
    prompts, img_lat, img_emb, fps = loops_ref.edit_conditioning(ns)
    g = torch.Generator().manual_seed(8895)
    x3 = torch.randn(3, 4, F, H, W, generator=g).to(device=dev, dtype=dtype)
    return ns, x3, prompts, img_lat, img_emb, fps


def _check(got, ref32, ref16, what, slack=3.0):
    assert torch.isfinite(got).all(), what
    e_ours, e_ref = err_stats(got, ref32), err_stats(ref16, ref32)
    print(f"{what}: ours-vs-fp32 {e_ours}  |  torch-fp16-vs-fp32 {e_ref}")
    assert e_ours["rms_rel"] <= max(slack * e_ref["rms_rel"], 2e-3), (what, e_ours, e_ref)
    assert e_ours["rel_to_max"] <= max(slack * e_ref["rel_to_max"], 5e-3), (what, e_ours, e_ref)
    return e_ours, e_ref


def _register(full, schedule, t):
    from anyv2v_b200 import pnp_utils as ours_hooks
    from oracle import pnp_hooks_ref
    for net, hooks in ((full.ref32, pnp_hooks_ref), (full.ref16, pnp_hooks_ref), (full.ours, ours_hooks)):
        pipe = SimpleNamespace(unet=net)
        hooks.register_conv_injection(pipe, schedule)
        hooks.register_spatial_attention_pnp(pipe, schedule)
        hooks.register_temp_attention_pnp(pipe, schedule)
        hooks.register_time(pipe, t)


def _schedule():
    from oracle import schedulers_ref
    s = schedulers_ref.DDIMScheduler()
    s.set_timesteps(50)
    return s, s.timesteps[:25]  # 981 ... 501


@torch.no_grad()
@pytest.mark.parametrize("t,expect_inject", [(901, True), (101, False), (1000, True)])
def test_fullwidth_hooked_step_matches_oracle(full, t, expect_inject):
    """one hooked UNet step of the full-size model: injected (conv + spatial + temporal), non-injected, t == 1000"""
    from anyv2v_b200 import ops
    _, schedule = _schedule()
    _register(full, schedule, t)
    outs = {}
    c0 = ops.launch_count()
    for name, net, dt in (("ours", full.ours, torch.float16), ("ref32", full.ref32, torch.float32), ("ref16", full.ref16, torch.float16)):
        _, x3, prompts, img_lat, img_emb, fps = _inputs(dt)
        outs[name] = net(x3, torch.tensor([t], device=dev), fps, img_lat, img_emb, prompts)[0]
    assert CONFIG_OVERRIDE is not None or ops.launch_count() - c0 > 500  # the step ran on this package's kernels
    assert outs["ours"].shape == outs["ref32"].shape == (3, 4, F_, H_, W_)
    _check(outs["ours"], outs["ref32"], outs["ref16"], f"full-width hooked UNet step t={t}")
    proc = full.ours.up_blocks[3].temp_attentions[2].transformer_blocks[0].attn1.processor
    assert proc.inject_now() == expect_inject and proc.t == t
    if expect_inject:
        # Appendix C.5: with conv injection active the patched resnet's h is identical across branches; the edit
        # branches still differ through their contexts, and the source output is the plain forward of the source
        assert not torch.equal(outs["ours"][1], outs["ours"][2])
    _register(full, [], -1)


@torch.no_grad()
def test_fullwidth_unhooked_forward_and_inversion_batch(full):
    """B = 1 (the inversion step's geometry) on the unpatched full-size model"""
    _register(full, [], -1)
    outs = {}
    for name, net, dt in (("ours", full.ours, torch.float16), ("ref32", full.ref32, torch.float32), ("ref16", full.ref16, torch.float16)):
        ns, _, _, _, _, _ = _inputs(dt)
        outs[name] = net(ns.video_latents, torch.tensor([21], device=dev), ns.fps, ns.src_image_latents, ns.src_image_emb, ns.inv_prompt)[0]
    _check(outs["ours"], outs["ref32"], outs["ref16"], "full-width inversion-geometry forward (B=1)")


@torch.no_grad()
def test_fullwidth_teacher_forced_edit_and_inversion_steps(full):
    """one iteration of each loop through the PRODUCT pipeline (UNet + fused CFG / DDIM kernels, CUDA-graph machinery off)
    fed with the oracle's state, against the oracle's own iteration (pipeline :1131-1179 and :1385-1433)"""
    from anyv2v_b200 import pnp_utils as ours_hooks
    from anyv2v_b200.latent_store import LatentStore
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp
    from anyv2v_b200.schedulers import DDIMInverseScheduler, DDIMScheduler
    from oracle import loops_ref, pnp_hooks_ref, schedulers_ref
    n_steps = 50
    ns32, _, _, _, _, _ = _inputs(torch.float32)
    ns16, _, _, _, _, _ = _inputs(torch.float16)
    # ---- inversion: first two steps of the oracle loop; ours is fed the oracle's x_t at each step
    _register(full, [], -1)
    inv_ref = schedulers_ref.DDIMInverseScheduler()
    inv_ref.set_timesteps(n_steps)
    pipe = I2VGenXLPipeline(full.ours, DDIMInverseScheduler())
    pipe.use_cuda_graphs = False
    st = pipe.prepare_invert(ns16.video_latents, ns16.inv_prompt, ns16.src_image_latents, ns16.src_image_emb, 8, n_steps,
                             1.0, None, False, False)
    x32 = ns32.video_latents
    inverted = {}
    for i in range(2):
        t = int(inv_ref.timesteps[i])
        v = full.ref32(x32, torch.tensor([t], device=dev), ns32.fps, ns32.src_image_latents, ns32.src_image_emb, ns32.inv_prompt)[0]
        want, _ = inv_ref.step(v, t, x32)
        v16 = full.ref16(x32.half(), torch.tensor([t], device=dev), ns16.fps, ns16.src_image_latents, ns16.src_image_emb, ns16.inv_prompt)[0]
        want16, _ = inv_ref.step(v16, t, x32.half())
        st.latents.copy_(x32.half())
        got = pipe.invert_step(st, i).clone()
        _check(got, want, want16, f"teacher-forced full-width inversion step t={t}")
        x32 = want
        inverted[t] = want
    # ---- edit: config-3 schedule (conv 0.8, spatial 0.5, temporal 0.5) at the first step (all three injections fire)
    sref = schedulers_ref.DDIMScheduler()
    sref.set_timesteps(n_steps)
    for net in (full.ref32, full.ref16):
        pnp_hooks_ref.init_pnp(SimpleNamespace(unet=net), sref, n_steps, 0.8, 0.5, 0.5)
    sch = DDIMScheduler()
    sch.set_timesteps(n_steps)
    pipe.register_modules(scheduler=sch)
    init_pnp(pipe, sch, SimpleNamespace(n_steps=n_steps, pnp_f_t=0.8, pnp_spatial_attn_t=0.5, pnp_temp_attn_t=0.5))
    prompts, img_lat, img_emb, fps = loops_ref.edit_conditioning(ns32)
    prompts16, img_lat16, img_emb16, fps16 = loops_ref.edit_conditioning(ns16)
    g = torch.Generator().manual_seed(77)
    ts = [int(t) for t in sref.timesteps]
    for i in (0, 30, 45):  # all three hooks / conv only / nothing fires (dead source branch)
        t = ts[i]
        src = torch.randn(1, 4, F_, H_, W_, generator=g).to(dev)
        x = torch.randn(1, 4, F_, H_, W_, generator=g).to(dev)
        pnp_hooks_ref.register_time(SimpleNamespace(unet=full.ref32), t)
        v = full.ref32(torch.cat([src, x, x]), torch.tensor([t], device=dev), fps, img_lat, img_emb, prompts)[0]
        want, _ = sref.step(schedulers_ref.cfg_combine(v[1:2], v[2:3], 9.0), t, x)
        pnp_hooks_ref.register_time(SimpleNamespace(unet=full.ref16), t)
        v16 = full.ref16(torch.cat([src, x, x]).half(), torch.tensor([t], device=dev), fps16, img_lat16, img_emb16, prompts16)[0]
        want16, _ = sref.step(schedulers_ref.cfg_combine(v16[1:2], v16[2:3], 9.0), t, x.half())
        store = LatentStore(None, write_files=False)
        store.put(t, src.half())
        st_e = pipe.prepare_edit(x.half(), ns16.edit_prompt, ns16.neg_prompt, ns16.inv_prompt, ns16.edit_image_emb,
                                 ns16.edit_image_latents, ns16.src_image_emb, ns16.src_image_latents, 8, n_steps, 9.0, 0, None,
                                 store, True)
        assert st_e.timesteps[i] == t
        got = pipe.edit_step(st_e, i).clone()
        flags = pipe._hook_flags(t)
        assert flags == (i < 40, i < 25, i < 25), (t, flags)
        _check(got, want, want16, f"teacher-forced full-width PnP edit step t={t} flags={flags}")
    _register(full, [], -1)


@torch.no_grad()
@pytest.mark.parametrize("inject", [True, False])
def test_fullwidth_finest_level_block_alone(full, inject):
    """up_blocks[3] (320 channels, 3 layers: resnet / temporal conv / spatial + temporal transformer) at 64 x 64: the
    4096-token attention sites and, when injected, the shared-probability N = 4096 kernel inside the model."""
    from anyv2v_b200.unet_i2vgen_xl import to_nhwc
    B, F, H, W = 3, 2, 64, 64
    t = 901 if inject else 101
    _, schedule = _schedule()
    _register(full, schedule, t)
    g = torch.Generator().manual_seed(4321)
    rn = lambda *s: torch.randn(*s, generator=g).to(dev)
    c0, c1 = _config()["block_out_channels"][:2]
    x = rn(B * F, c1, H, W)
    skips = [rn(B * F, c0, H, W) for _ in range(3)]
    emb = rn(B * F, 4 * c0)
    ctx = rn(B, 145, _config()["cross_attention_dim"])
    outs = {}
    for name, net, dt in (("ref32", full.ref32, torch.float32), ("ref16", full.ref16, torch.float16)):
        c = lambda z: z.to(dt)
        outs[name] = net.up_blocks[3](c(x), tuple(c(s) for s in skips), c(emb), c(ctx).repeat_interleave(F, dim=0), F)
    h = lambda z: z.half()
    y = full.ours.up_blocks[3].forward_nhwc(to_nhwc(h(x)), [to_nhwc(h(s)) for s in skips], h(emb).contiguous(), h(ctx).contiguous(), F)
    got = y.permute(0, 3, 1, 2)
    _check(got, outs["ref32"], outs["ref16"], f"up_blocks[3] alone at 64x64, inject={inject}")
    _register(full, [], -1)


@torch.no_grad()
def test_fullwidth_level_with_128_frames(full):
    """BASELINE configs[4] (128-frame long-video clip, gradio_demo.py:120-131,186-203): one full-width level — up_blocks[2] (640
    channels, spatial + temporal transformers, fused Upsample2D) at 32 x 32 with F = 128 and all three hooks firing.  Temporal sequences of
    128 frames = one whole 128-row tile per pixel in the fused temporal-attention kernel (ppt = 1, injected n_v = 3 variant)."""
    from anyv2v_b200.unet_i2vgen_xl import to_nhwc
    B, F, H, W = 3, 128, 32, 32
    _, schedule = _schedule()
    _register(full, schedule, 901)
    cfg = _config()
    c0, c1, c2 = cfg["block_out_channels"][0], cfg["block_out_channels"][1], cfg["block_out_channels"][2]
    g = torch.Generator().manual_seed(99)
    rn = lambda *s: torch.randn(*s, generator=g).to(dev)
    x = rn(B * F, c2, H, W)                                      # from up_blocks[1] (1280 channels, already up-sampled)
    skips = [rn(B * F, c0, H, W), rn(B * F, c1, H, W), rn(B * F, c1, H, W)]   # popped from the end: 640, 640, 320
    emb = rn(B * F, 4 * c0)
    ctx = rn(B, 145, cfg["cross_attention_dim"])
    outs = {}
    for name, net, dt in (("ref32", full.ref32, torch.float32), ("ref16", full.ref16, torch.float16)):
        c = lambda z: z.to(dt)
        outs[name] = net.up_blocks[2](c(x), tuple(c(s) for s in skips), c(emb), c(ctx).repeat_interleave(F, dim=0), F)
        torch.cuda.empty_cache()
    h = lambda z: z.half()
    y = full.ours.up_blocks[2].forward_nhwc(to_nhwc(h(x)), [to_nhwc(h(s)) for s in skips], h(emb).contiguous(), h(ctx).contiguous(), F)
    _check(y.permute(0, 3, 1, 2), outs["ref32"], outs["ref16"], "up_blocks[2] alone, 128 frames, 32x32, injected")
    _register(full, [], -1)
