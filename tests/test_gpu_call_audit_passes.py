"""tests/call_audit.py over the full-size passes of the DPM-Solver++(2M) sampler, the SourceFeatureCache replay and the tiled
VAE: every kernel call checked element by element against its float64 contract at the arguments the model passes, the
mean error of each op over the pass against the bias bound, and every kernel launch audited.  16 x 64 x 64 latents, eager
(no CUDA graph); the VAE at 704 x 1280.  ``-s`` prints the per-signature table and the wall time of each pass and test."""
import time
from types import SimpleNamespace

import pytest
import torch

from test_gpu_step_audit import CONFIG3, _conditioning, _expect, _Pass

pytestmark = pytest.mark.gpu
dev = "cuda"
DPM_STEPS = 25
CONFIG3_DPM = SimpleNamespace(**{**vars(CONFIG3), "n_steps": DPM_STEPS})


@pytest.fixture(scope="module")
def unet():
    from anyv2v_b200 import distributed
    from anyv2v_b200.unet_i2vgen_xl import I2VGEN_XL_CONFIG, I2VGenXLUNet
    net = distributed.build_unet_replicated(I2VGenXLUNet, I2VGEN_XL_CONFIG, 8888, torch.device(dev))
    yield net
    del net
    torch.cuda.empty_cache()


@pytest.fixture
def wall(request):
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"\n{request.node.name}: {time.perf_counter() - t0:.1f} s wall")


def _ddim_store(n_steps=50, seed=3):
    """random source latents at every timestep of an n-step DDIM inversion"""
    from anyv2v_b200.latent_store import LatentStore
    from anyv2v_b200.schedulers import DDIMScheduler
    s = DDIMScheduler()
    s.set_timesteps(n_steps)
    store = LatentStore(None, write_files=False)
    g = torch.Generator().manual_seed(seed)
    for t in s.timesteps.tolist():
        store.put(int(t), torch.randn(1, 4, 16, 64, 64, generator=g).half().to(dev))
    return store


def _edit_pipeline(unet, sched, pnp):
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp
    sched.set_timesteps(pnp.n_steps)
    pipe = I2VGenXLPipeline(unet, sched)
    pipe.use_cuda_graphs = False
    pipe.disable_freeu()
    init_pnp(pipe, sched, pnp)
    return pipe


def _prepare_edit(pipe, c, n_steps, store, cache=None):
    return pipe.prepare_edit(c["video_latents"].clone(), c["edit_prompt"], c["neg_prompt"], c["inv_prompt"], c["edit_image_emb"],
                             c["edit_image_latents"], c["src_image_emb"], c["src_image_latents"], 8, n_steps, 9.0, 0, None,
                             store, True, source_features=cache)


@torch.no_grad()
def test_dpm_call_steps(unet, monkeypatch, wall):
    """image-to-video steps 0 (first order) and 1 (second order) of a 25-step DPM-Solver++(2M) call, CFG batch 2"""
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.schedulers import DPMSolverMultistepScheduler
    c = _conditioning(64, 64)
    pipe = I2VGenXLPipeline(unet, DPMSolverMultistepScheduler())
    pipe.use_cuda_graphs = False
    pipe.disable_freeu()
    st = pipe.prepare_call(c["video_latents"], c["edit_prompt"], c["edit_image_latents"], c["edit_image_emb"], 8, DPM_STEPS,
                           9.0, c["neg_prompt"])
    for i, order in ((0, 1), (1, 2)):
        p = _Pass(monkeypatch, f"DPM call step {i} (order {order})", seed=11 + i)
        pipe.call_step(st, i)
        a = p.finish()
        _expect(a, "dpmpp2m_step", order=order, cfg=True, n=4 * 16 * 64 * 64)
        _expect(a, "attention", mode="rows", seq=4096)
        monkeypatch.undo()


@torch.no_grad()
def test_dpm_edit_steps(unet, monkeypatch, wall):
    """BASELINE config 3 PnP edit, 25 DPM steps reading a 50-step DDIM inversion store: steps 0 (first order, every injection
    fires) and 1 (second order)"""
    from anyv2v_b200.schedulers import DPMSolverMultistepScheduler
    c = _conditioning(64, 64)
    pipe = _edit_pipeline(unet, DPMSolverMultistepScheduler(), CONFIG3_DPM)
    st = _prepare_edit(pipe, c, DPM_STEPS, _ddim_store())
    assert pipe._hook_flags(st.timesteps[0]) == (True, True, True)
    for i, order in ((0, 1), (1, 2)):
        p = _Pass(monkeypatch, f"DPM edit step {i} (order {order})", seed=13 + i)
        pipe.edit_step(st, i)
        a = p.finish()
        _expect(a, "dpmpp2m_step", order=order, cfg=True, in_place=True)
        _expect(a, "attention", mode="rows", n_v=3, seq=4096)
        _expect(a, "temporal_attention_fused", n_v=3)
        monkeypatch.undo()


@torch.no_grad()
def test_edit_steps_replayed_from_the_source_feature_cache(unet, monkeypatch, wall):
    """edit A's steps 0 and 30 (config 3, DDIM) fill a SourceFeatureCache; edit B (another prompt and first frame) replays
    them: step 0 with every injection (attention at n_v = 2, the fused temporal attention with Q / K from the cache, GroupNorm
    partitioned as the three-branch step), step 30 with the conv injection only"""
    from anyv2v_b200.schedulers import DDIMScheduler
    c = _conditioning(64, 64)
    pipe = _edit_pipeline(unet, DDIMScheduler(), CONFIG3)
    store = _ddim_store()
    cache = pipe.source_feature_cache(max_bytes=1 << 40)
    st = _prepare_edit(pipe, c, CONFIG3.n_steps, store, cache)
    for i in (0, 30):
        pipe.edit_step(st, i)
    assert len(cache) == 2
    g = torch.Generator().manual_seed(4)
    c_b = dict(c)
    for k in ("edit_prompt", "edit_image_emb", "edit_image_latents"):
        c_b[k] = (c[k].float() + torch.randn(c[k].shape, generator=g).to(dev)).half()
    st = _prepare_edit(pipe, c_b, CONFIG3.n_steps, store, cache)
    p = _Pass(monkeypatch, "replayed edit step 0 (all injections)", seed=15)
    pipe.edit_step(st, 0)
    a = p.finish()
    _expect(a, "attention", mode="rows", n_v=2, seq=4096)
    _expect(a, "temporal_attention_fused_qksrc", F=16)
    _expect(a, "groupnorm", partition_samples=lambda v: v > 0)
    assert not a.seen("attention", n_v=3) and not a.seen("temporal_attention_fused", n_v=3)
    monkeypatch.undo()
    p = _Pass(monkeypatch, "replayed edit step 30 (conv injection only)", seed=16)
    pipe.edit_step(st, 30)
    a = p.finish()
    assert not a.seen("attention", n_v=3) and not a.seen("temporal_attention_fused_qksrc")
    assert [k[-1] for k in st.iterations] == ["replay", "replay"]


@pytest.fixture(scope="module")
def tiled_vae():
    from anyv2v_b200 import vae as product
    from oracle import vae_ref
    ref32 = vae_ref.seeded_vae(vae_ref.SD_VAE_CONFIG, seed=8888, dtype=torch.float32)
    ours = product.AutoencoderKL(**vae_ref.SD_VAE_CONFIG, sample_size=768)
    ours.load_state_dict(ref32.state_dict())
    ours = ours.to(device=dev, dtype=torch.float16).eval()
    ours.enable_tiling()
    yield ours
    torch.cuda.empty_cache()


@torch.no_grad()
def test_tiled_vae_decode_704x1280(tiled_vae, monkeypatch, wall):
    from anyv2v_b200 import vae as product
    lat = torch.randn(1, 4, 2, 88, 160, generator=torch.Generator().manual_seed(17)).half().to(dev)
    p = _Pass(monkeypatch, "tiled VAE decode, 2 frames at 704 x 1280", seed=17)
    video = product.decode_latents(tiled_vae, lat, None)
    a = p.finish()
    assert video.shape == (1, 3, 2, 704, 1280) and torch.isfinite(video).all()
    _expect(a, "tile_stitch", N=2, C=3, H=704, W=1280, rows=2, cols=3)


@torch.no_grad()
def test_tiled_vae_encode_704x1280(tiled_vae, monkeypatch, wall):
    from anyv2v_b200 import vae as product
    frames = torch.randn(2, 3, 704, 1280, generator=torch.Generator().manual_seed(18)).clamp(-1, 1).half().to(dev)
    p = _Pass(monkeypatch, "tiled VAE encode, 2 frames at 704 x 1280", seed=18)
    z = product.encode_vae_video(tiled_vae, frames, torch.Generator(device=dev).manual_seed(3))
    a = p.finish()
    assert z.shape == (1, 4, 2, 88, 160) and torch.isfinite(z).all()
    _expect(a, "tile_stitch", N=2, C=8, H=88, W=160, rows=2, cols=3)
