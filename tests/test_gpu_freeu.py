"""FreeU on the GPU: ops.freeu against its float64 contract inside guarded buffers, the wrapper's refusals, the UNet with
FreeU against the fp32 oracle, a full-size edit step, and CUDA-graph replay of both loops with FreeU on and switched mid-loop."""
from types import SimpleNamespace

import pytest
import torch

import freeu_ref
from guarded import check_output, guarded_inout, guarded_input, guarded_output
from parity_utils import err_stats
from ulp_check import KAPPA_FREEU, assert_within_bound, cond_freeu

pytestmark = pytest.mark.gpu
dev = "cuda"
FREEU = dict(s1=0.9, s2=0.2, b1=1.5, b2=1.6)


def _check_freeu(hidden, skip, b, s):
    """ops.freeu on guarded CUDA views vs the contract on CPU copies: the filtered skip within the FreeU bound, hidden[..., :C/2]
    bit for bit against torch's fp16 `h * b` on the GPU, hidden[..., C/2:], the skip and every guard untouched"""
    from anyv2v_b200 import ops
    NF, H, W, Cs = skip.shape
    gh, gs, go = guarded_inout(hidden, device=dev), guarded_input(skip, device=dev), guarded_output(skip.shape, device=dev)
    h0 = gh.view.clone()
    s_bits = gs.buf.clone()
    want_half = h0[..., :hidden.shape[-1] // 2] * b
    ops.freeu(gh.view, gs.view, b, s, out=go.view)
    torch.cuda.synchronize()
    check_output(go, "freeu out")
    check_output(gh, "freeu hidden")
    assert torch.equal(gs.buf.view(torch.int16), s_bits.view(torch.int16)), "the skip input was written"
    half = hidden.shape[-1] // 2
    assert torch.equal(gh.view[..., :half].view(torch.int16), want_half.view(torch.int16)), "backbone half differs from torch h * b"
    assert torch.equal(gh.view[..., half:].view(torch.int16), h0[..., half:].view(torch.int16)), "second half of hidden was changed"
    h_host = hidden.clone()
    ref = freeu_ref.freeu(h_host, skip, b, s)
    assert torch.equal(gh.view.cpu(), h_host), "hidden differs from the contract"
    exact = freeu_ref.fourier_filter_closed_form(skip.double(), float(torch.tensor(s, dtype=torch.float32)))
    assert torch.equal(ref, exact.half())
    assert_within_bound(go.view.cpu(), exact, cond_freeu(skip, s), KAPPA_FREEU, f"freeu {tuple(skip.shape)} s={s}",
                        shape=tuple(skip.shape))


@pytest.mark.parametrize("shape,ch", [((48, 8, 8, 1280), 1280), ((48, 16, 16, 1280), 1280), ((48, 16, 16, 640), 1280),
                                      ((6, 5, 8, 1280), 1280), ((3, 9, 16, 640), 640), ((2, 1, 1, 64), 64), ((2, 2, 2, 64), 64),
                                      ((3, 5, 7, 72), 72), ((2, 3, 4, 72), 40)])
def test_freeu_against_contract_guarded(shape, ch):
    torch.manual_seed(sum(shape) + ch)
    NF, H, W, Cs = shape
    skip = (torch.randn(shape) + 0.5 * torch.randn(NF, 1, 1, Cs)).half()  # a per-plane offset makes the mode-0 term matter
    hidden = (torch.randn(NF, H, W, ch) * 20).half()
    _check_freeu(hidden, skip, 1.37, 0.2 if H > 8 else 0.9)


def test_freeu_large_skip_values_stay_finite():
    """planes reaching 3e4: their sums overflow fp16 (the kernel accumulates in fp32)"""
    torch.manual_seed(7)
    skip = (3e4 - 2e3 * torch.rand(2, 16, 16, 64)).half()
    hidden = torch.randn(2, 16, 16, 64).half()
    _check_freeu(hidden, skip, 1.5, 0.9)


def test_freeu_wrapper_refusals():
    from anyv2v_b200 import ops
    from anyv2v_b200._lib import Av2vError
    h = torch.randn(2, 4, 4, 64, device=dev).half()
    s = torch.randn(2, 4, 4, 64, device=dev).half()
    with pytest.raises(Av2vError):
        ops.freeu(h.cpu(), s.cpu(), 1.5, 0.9)
    with pytest.raises(Av2vError):
        ops.freeu(h, s.permute(0, 2, 1, 3), 1.5, 0.9)                              # non-contiguous skip
    with pytest.raises(Av2vError):
        ops.freeu(h, s, 1.5, 0.9, out=torch.empty(2, 4, 4, 32, device=dev, dtype=torch.float16))  # undersized out
    with pytest.raises(Av2vError):
        ops.freeu(h, torch.randn(2, 4, 4, 9, device=dev).half(), 1.5, 0.9)        # odd channel count
    with pytest.raises(Av2vError):
        ops.freeu(torch.randn(2, 4, 4, 12, device=dev).half(), s, 1.5, 0.9)       # not a multiple of 8
    torch.cuda.synchronize()


def _tiny_models():
    from anyv2v_b200.unet_i2vgen_xl import I2VGenXLUNet
    from oracle import unet_ref
    ref32 = unet_ref.seeded_unet(unet_ref.TINY_CONFIG, seed=8888, dtype=torch.float32, device=dev)
    ours = I2VGenXLUNet(**unet_ref.TINY_CONFIG)
    ours.load_state_dict(ref32.state_dict())
    return ref32, ours.to(device=dev, dtype=torch.float16).eval()


@torch.no_grad()
def test_tiny_unet_with_hooks_and_freeu_matches_fp32_oracle():
    from anyv2v_b200 import pnp_utils
    from oracle import loops_ref, pnp_hooks_ref, schedulers_ref
    ref32, ours = _tiny_models()
    s = schedulers_ref.DDIMScheduler()
    s.set_timesteps(10)
    outs = {}
    for name, net, dt, hooks in (("ref", ref32, torch.float32, pnp_hooks_ref), ("ours", ours, torch.float16, pnp_utils)):
        pipe = SimpleNamespace(unet=net)
        hooks.register_conv_injection(pipe, s.timesteps[:5])
        hooks.register_spatial_attention_pnp(pipe, s.timesteps[:5])
        hooks.register_temp_attention_pnp(pipe, s.timesteps[:5])
        hooks.register_time(pipe, 901)
        if net is ours:
            ours.enable_freeu(**FREEU)
        else:
            freeu_ref.enable_freeu(ref32, **FREEU)
        ns = loops_ref.synthetic_inputs(4, 16, 16, cross_dim=64, dtype=dt, device=dev)
        prompts, img_lat, img_emb, fps = loops_ref.edit_conditioning(ns)
        x3 = torch.randn(3, 4, 4, 16, 16, generator=torch.Generator().manual_seed(1)).to(device=dev, dtype=dt)
        outs[name] = net(x3, torch.tensor([901], device=dev), fps, img_lat, img_emb, prompts)[0]
    e = err_stats(outs["ours"], outs["ref"])
    print(f"tiny hooked UNet with FreeU vs fp32 oracle: {e}")
    assert torch.isfinite(outs["ours"]).all() and e["rms_rel"] < 1e-2


@torch.no_grad()
def test_full_size_edit_step_with_freeu_is_finite():
    """one 16-frame 512 x 512 PnP edit step (up_blocks[0] at 8 x 8, up_blocks[1] at 16 x 16) of the full-size UNet with FreeU"""
    from anyv2v_b200 import distributed
    from anyv2v_b200.latent_store import LatentStore
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp, synthetic_conditioning
    from anyv2v_b200.schedulers import DDIMScheduler
    from anyv2v_b200.unet_i2vgen_xl import I2VGEN_XL_CONFIG, I2VGenXLUNet
    unet = distributed.build_unet_replicated(I2VGenXLUNet, I2VGEN_XL_CONFIG, 8888, torch.device(dev))
    c = {k: v.to(dev) for k, v in synthetic_conditioning(16, 64, 64, 1024, 8888, "cpu").items()}
    sched = DDIMScheduler()
    sched.set_timesteps(50)
    pipe = I2VGenXLPipeline(unet, sched)
    init_pnp(pipe, sched, SimpleNamespace(n_steps=50, pnp_f_t=1.0, pnp_spatial_attn_t=1.0, pnp_temp_attn_t=0.0))
    pipe.enable_freeu(**FREEU)
    store = LatentStore(None, write_files=False)
    store.put(int(sched.timesteps[0]), torch.randn(1, 4, 16, 64, 64, generator=torch.Generator().manual_seed(3)).half().to(dev))
    st = pipe.prepare_edit(c["video_latents"].clone(), c["edit_prompt"], c["neg_prompt"], c["inv_prompt"], c["edit_image_emb"],
                           c["edit_image_latents"], c["src_image_emb"], c["src_image_latents"], 8, 50, 9.0, 0, None, store, True)
    x = pipe.edit_step(st, 0)
    torch.cuda.synchronize()
    assert x.shape == (1, 4, 16, 64, 64) and torch.isfinite(x).all()
    del unet, pipe, st
    torch.cuda.empty_cache()


def _run_loops(ours, graphs, toggle=False):
    """invert then sample_with_pnp, 6 steps each, on the tiny model with FreeU on.  Every edit step injects at the same sites, so
    with graphs the steps after the first two of a setting replay one graph.  toggle: the callback flips FreeU after every step
    (on, off, on, off, ...), so each of the two settings runs eagerly, is captured and is replayed in both loops."""
    from anyv2v_b200.latent_store import LatentStore
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp
    from anyv2v_b200.schedulers import DDIMInverseScheduler, DDIMScheduler
    from oracle import loops_ref
    n = 6
    ns = loops_ref.synthetic_inputs(4, 16, 16, cross_dim=64, dtype=torch.float16, device=dev)
    pipe = I2VGenXLPipeline(ours, DDIMInverseScheduler())
    pipe.use_cuda_graphs = graphs
    pipe.enable_freeu(**FREEU)

    def callback(i, t, x):
        if toggle and i % 2 == 0:
            pipe.disable_freeu()
        elif toggle:
            pipe.enable_freeu(**FREEU)

    inv = pipe.invert(latents=ns.video_latents, prompt_embeds=ns.inv_prompt, image_latents=ns.src_image_latents,
                      image_embeddings=ns.src_image_emb, target_fps=8, num_inference_steps=n, write_files=False, callback=callback)
    pipe.enable_freeu(**FREEU)
    sched = DDIMScheduler()
    sched.set_timesteps(n)
    pipe.scheduler = sched
    init_pnp(pipe, sched, SimpleNamespace(n_steps=n, pnp_f_t=1.0, pnp_spatial_attn_t=1.0, pnp_temp_attn_t=0.0))
    store = LatentStore(None, write_files=False)
    g = torch.Generator().manual_seed(5)
    for t in sched.timesteps.tolist():
        store.put(int(t), torch.randn(1, 4, 4, 16, 16, generator=g).half().to(dev))
    out = pipe.sample_with_pnp(latents=ns.video_latents.clone(), prompt_embeds=ns.edit_prompt, negative_prompt_embeds=ns.neg_prompt,
                               ddim_inv_prompt_embeds=ns.inv_prompt, image_embeddings=ns.edit_image_emb,
                               image_latents=ns.edit_image_latents, ddim_inv_image_embeddings=ns.src_image_emb,
                               ddim_inv_image_latents=ns.src_image_latents, target_fps=8, num_inference_steps=n,
                               guidance_scale=9.0, ddim_init_latents_t_idx=0, latent_store=store, callback=callback,
                               return_dict=False)[0]
    pipe.disable_freeu()
    return inv.clone(), out.clone()


@torch.no_grad()
@pytest.mark.parametrize("toggle", [False, True])
def test_cuda_graph_loops_with_freeu_equal_eager(toggle):
    _, ours = _tiny_models()
    eager = _run_loops(ours, graphs=False, toggle=toggle)
    graphed = _run_loops(ours, graphs=True, toggle=toggle)
    assert all(torch.isfinite(x).all() for x in eager)
    assert torch.equal(graphed[0], eager[0]) and torch.equal(graphed[1], eager[1])
    if toggle:  # the toggling does change the result, so the graphs did follow it
        steady = _run_loops(ours, graphs=False)
        assert not torch.equal(steady[0], eager[0]) and not torch.equal(steady[1], eager[1])
