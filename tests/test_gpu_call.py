"""Stochastic DDIM and the image-to-video call on the GPU: ops.ddim_step_eta against its contract inside guarded buffers, the
wrapper's refusals, `__call__` on the tiny UNet against the fp32 oracle, CUDA-graph replay against eager launches with FreeU
switched between steps, and the full-size UNet at 16 x 512^2 and at the reference default 704 x 1280."""
import pytest
import torch

import sampling_ref
from guarded import check_output, guarded_inout, guarded_input, guarded_output
from test_call_cpu import _spy_draws, run_call_teacher_forced

pytestmark = pytest.mark.gpu
dev = "cuda"
FREEU = dict(s1=0.9, s2=0.2, b1=1.5, b2=1.6)


def _coefs():
    """(ca, cb, cc, cd', cs) of t = 981 of 50 steps at eta = 1, with cs replaced by 1.0 (the largest sigma eta <= 1 gives)"""
    from anyv2v_b200.schedulers import DDIMScheduler
    s = DDIMScheduler()
    s.set_timesteps(50)
    ca, cb, cc, cd, _ = s.coefficients(981, 1.0)
    return ca, cb, cc, cd, 1.0


def _rnd(n, scale=1.0):
    return (torch.randn(n) * scale).half()


@pytest.mark.parametrize("n", [1, 7, 8, 1001, 4 * 16 * 64 * 64, 4 * 16 * 88 * 160])
@pytest.mark.parametrize("cfg", [False, True])
@pytest.mark.parametrize("coef", ["value", "device"])
def test_ddim_eta_against_contract_guarded(n, cfg, coef):
    """in place (out is x, as the pipeline calls it), noise up to |z| = 5, cs = 1; bit for bit against the contract"""
    from anyv2v_b200 import ops
    torch.manual_seed(n + 2 * cfg)
    x_host, vn_host, ve_host = _rnd(n), _rnd(n), _rnd(n)
    z_host = (torch.randn(n) * 2).clamp(-5, 5)
    z_host[: min(n, 2)] = torch.tensor([5.0, -5.0])[: min(n, 2)]
    z_host = z_host.half()
    ca, cb, cc, cd, cs = _coefs()
    x = guarded_inout(x_host.to(dev))
    vn, ve, z = guarded_input(vn_host, device=dev), guarded_input(ve_host, device=dev), guarded_input(z_host, device=dev)
    if coef == "device":
        table = torch.tensor([ca, cb, cc, cd, 9.0, cs], dtype=torch.float32, device=dev)
        ops.ddim_step_eta(x.view, vn.view, ve.view if cfg else None, z.view, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, out=x.view,
                          coef_dev=table)
    else:
        ops.ddim_step_eta(x.view, vn.view, ve.view if cfg else None, z.view, 9.0, ca, cb, cc, cd, cs, out=x.view)
    torch.cuda.synchronize()
    check_output(x, "ddim_step_eta in place")
    want = sampling_ref.ddim_step_eta(x_host, vn_host, ve_host if cfg else None, z_host, 9.0, ca, cb, cc, cd, cs)
    assert torch.equal(x.view.cpu().view(torch.int16), want.view(torch.int16))


def test_ddim_eta_out_of_place_equals_in_place():
    from anyv2v_b200 import ops
    n = 1001
    torch.manual_seed(3)
    x, vn, ve, z = (_rnd(n).to(dev) for _ in range(4))
    sep = guarded_output((n,), device=dev)
    ops.ddim_step_eta(x, vn, ve, z, 9.0, *_coefs(), out=sep.view)
    ops.ddim_step_eta(x, vn, ve, z, 9.0, *_coefs(), out=x)
    torch.cuda.synchronize()
    check_output(sep, "ddim_step_eta out")
    assert torch.equal(sep.view, x)


def _h(*shape, device=dev, dtype=torch.float16):
    return torch.zeros(*shape, device=device, dtype=dtype)


REFUSALS = {
    "noise dtype": lambda o: o.ddim_step_eta(_h(16), _h(16), None, _h(16, dtype=torch.float32), 1.0, 1, 0, 1, 0, 0),
    "noise device": lambda o: o.ddim_step_eta(_h(16), _h(16), None, _h(16, device="cpu"), 1.0, 1, 0, 1, 0, 0),
    "noise strided": lambda o: o.ddim_step_eta(_h(16), _h(16), None, _h(32)[::2], 1.0, 1, 0, 1, 0, 0),
    "noise size": lambda o: o.ddim_step_eta(_h(16), _h(16), None, _h(8), 1.0, 1, 0, 1, 0, 0),
    "out strided": lambda o: o.ddim_step_eta(_h(16), _h(16), None, _h(16), 1.0, 1, 0, 1, 0, 0, out=_h(32)[::2]),
    "out size": lambda o: o.ddim_step_eta(_h(16), _h(16), None, _h(16), 1.0, 1, 0, 1, 0, 0, out=_h(8)),
    "coef_dev dtype": lambda o: o.ddim_step_eta(_h(16), _h(16), None, _h(16), 1.0, 1, 0, 1, 0, 0,
                                                coef_dev=_h(6, dtype=torch.float64)),
    "coef_dev device": lambda o: o.ddim_step_eta(_h(16), _h(16), None, _h(16), 1.0, 1, 0, 1, 0, 0,
                                                 coef_dev=_h(6, device="cpu", dtype=torch.float32)),
    "coef_dev length": lambda o: o.ddim_step_eta(_h(16), _h(16), None, _h(16), 1.0, 1, 0, 1, 0, 0,
                                                 coef_dev=_h(5, dtype=torch.float32)),
}


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_ddim_eta_wrapper_refusals(case):
    from anyv2v_b200 import ops
    from anyv2v_b200._lib import Av2vError
    n0 = ops.launch_count()
    with pytest.raises(Av2vError):
        REFUSALS[case](ops)
    assert ops.launch_count() == n0
    torch.cuda.synchronize()


def _tiny_models():
    from anyv2v_b200.unet_i2vgen_xl import I2VGenXLUNet
    from oracle import unet_ref
    ref32 = unet_ref.seeded_unet(unet_ref.TINY_CONFIG, seed=8888, dtype=torch.float32, device=dev)
    ours = I2VGenXLUNet(**unet_ref.TINY_CONFIG)
    ours.load_state_dict(ref32.state_dict())
    return ref32, ours.to(device=dev, dtype=torch.float16).eval()


@torch.no_grad()
@pytest.mark.parametrize("eta,guidance,n_videos,hw", [(0.0, 9.0, 1, (16, 16)), (1.0, 9.0, 1, (16, 16)), (1.0, 1.0, 1, (16, 16)),
                                                      (1.0, 9.0, 2, (16, 24))])
def test_call_on_the_tiny_unet_matches_the_fp32_oracle(monkeypatch, eta, guidance, n_videos, hw):
    draws = _spy_draws(monkeypatch)
    ref32, ours = _tiny_models()
    run_call_teacher_forced(ref32, ours, eta, guidance, n_videos, hw[0], hw[1], dev, draws, rms=1e-2, mx=4e-2)


def _call(pipe, ns, eta, graphs, toggle, n_steps=6):
    pipe.use_cuda_graphs = graphs
    pipe.enable_freeu(**FREEU)

    def callback(i, t, x):
        if toggle and i % 2 == 0:
            pipe.disable_freeu()
        elif toggle:
            pipe.enable_freeu(**FREEU)
    out = pipe(prompt_embeds=ns.edit_prompt, negative_prompt_embeds=ns.neg_prompt, image_embeddings=ns.edit_image_emb,
               image_latents=ns.edit_image_latents, latents=ns.video_latents, num_frames=4, num_inference_steps=n_steps,
               eta=eta, target_fps=8, output_type="latent", generator=torch.Generator(device=dev).manual_seed(21),
               callback=callback).frames
    pipe.disable_freeu()
    return out.clone()


@torch.no_grad()
@pytest.mark.parametrize("eta", [0.0, 1.0])
def test_cuda_graph_call_equals_eager_with_freeu_switched(eta):
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.schedulers import DDIMScheduler
    from oracle import loops_ref
    _, ours = _tiny_models()
    ns = loops_ref.synthetic_inputs(4, 16, 16, cross_dim=64, dtype=torch.float16, device=dev)
    pipe = I2VGenXLPipeline(ours, DDIMScheduler())
    eager = _call(pipe, ns, eta, graphs=False, toggle=True)
    graphed = _call(pipe, ns, eta, graphs=True, toggle=True)
    assert torch.isfinite(eager).all() and torch.equal(graphed, eager)
    steady = _call(pipe, ns, eta, graphs=False, toggle=False)
    assert not torch.equal(steady, eager)  # the toggling changes the result, so the graphs did follow it


@torch.no_grad()
def test_call_with_raw_inputs_returns_pil_frames_at_the_default_size():
    """pipe(prompt=..., image=PIL) with encoders and a VAE attached (tiny random-init models): height / width default to the
    reference's 704 x 1280"""
    from PIL import Image
    from anyv2v_b200.run_group_pnp_edit import build_pipeline
    from oracle.unet_ref import TINY_CONFIG
    from test_gpu_runners import TINY_VAE
    pipe = build_pipeline(torch.device(dev), TINY_CONFIG, seed=3, broadcast=False, with_encoders=True, vae_config=TINY_VAE)
    image = Image.new("RGB", (640, 480), (120, 60, 200))
    frames = pipe(prompt="a man walking", image=image, num_frames=2, num_inference_steps=3, eta=1.0,
                  generator=torch.Generator(device=dev).manual_seed(0)).frames
    assert len(frames) == 1 and len(frames[0]) == 2
    assert all(isinstance(f, Image.Image) and f.size == (1280, 704) for f in frames[0])


@torch.no_grad()
@pytest.mark.parametrize("h,w,steps", [(64, 64, 2), (88, 160, 2)])
def test_full_size_call_steps_graph_equals_eager(h, w, steps):
    """the full-size UNet, CFG batch 2, 16 frames: 512 x 512 and the reference default 704 x 1280; the second step replays
    the captured graph"""
    from anyv2v_b200 import distributed
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import synthetic_conditioning
    from anyv2v_b200.schedulers import DDIMScheduler
    from anyv2v_b200.unet_i2vgen_xl import I2VGEN_XL_CONFIG, I2VGenXLUNet
    unet = distributed.build_unet_replicated(I2VGenXLUNet, I2VGEN_XL_CONFIG, 8888, torch.device(dev))
    c = {k: v.to(dev) for k, v in synthetic_conditioning(16, h, w, 1024, 8888, "cpu").items()}
    pipe = I2VGenXLPipeline(unet, DDIMScheduler())
    outs = {}
    for graphs in (False, True):
        pipe.use_cuda_graphs = graphs
        outs[graphs] = pipe(prompt_embeds=c["edit_prompt"], negative_prompt_embeds=c["neg_prompt"],
                            image_embeddings=c["edit_image_emb"], image_latents=c["edit_image_latents"],
                            latents=c["video_latents"], num_frames=16, eta=1.0, target_fps=8, output_type="latent",
                            generator=torch.Generator(device=dev).manual_seed(1), max_steps=steps).frames.clone()
    torch.cuda.synchronize()
    assert outs[True].shape == (1, 4, 16, h, w) and torch.isfinite(outs[True]).all()
    assert torch.equal(outs[True], outs[False])
    del unet, pipe
    torch.cuda.empty_cache()
