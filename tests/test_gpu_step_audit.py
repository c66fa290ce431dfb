"""The production passes under tests/call_audit.py: every kernel call of a full-size inversion step, two PnP edit steps, an
edit step with FreeU, one image-to-video step at 704 x 1280 and the VAE at 512 x 512, checked element by element against its
float64 contract at the arguments the model passes, and the mean error of each op over the pass against the bias bound of
tests/bias_check.py.  All passes run eagerly (no CUDA graph: graph replay is tested
bit-equal to eager elsewhere).  Each test asserts that every call passed, that every kernel launch was audited, and that
the intended kinds of call were reached; ``-s`` prints the per-signature table."""
import time
from types import SimpleNamespace

import pytest
import torch

from call_audit import CallAudit

pytestmark = pytest.mark.gpu
dev = "cuda"
FREEU = dict(s1=0.9, s2=0.2, b1=1.5, b2=1.6)
CONFIG3 = SimpleNamespace(n_steps=50, pnp_f_t=0.8, pnp_spatial_attn_t=0.5, pnp_temp_attn_t=0.5)  # BASELINE config 3


@pytest.fixture(scope="module")
def unet():
    from anyv2v_b200 import distributed
    from anyv2v_b200.unet_i2vgen_xl import I2VGEN_XL_CONFIG, I2VGenXLUNet
    net = distributed.build_unet_replicated(I2VGenXLUNet, I2VGEN_XL_CONFIG, 8888, torch.device(dev))
    yield net
    del net
    torch.cuda.empty_cache()


def _conditioning(h, w):
    from anyv2v_b200.run_group_pnp_edit import synthetic_conditioning
    return {k: v.to(dev) for k, v in synthetic_conditioning(16, h, w, 1024, 8888, "cpu").items()}


class _Pass:
    """the audit installed for one pass: launches counted by ops.launch_count() over the same span"""

    def __init__(self, monkeypatch, what, seed):
        from anyv2v_b200 import ops
        self.ops, self.what = ops, what
        self.audit = CallAudit(seed=seed).install(monkeypatch)
        self.n0 = ops.launch_count()
        self.t0 = time.perf_counter()

    def finish(self):
        torch.cuda.synchronize()
        launches = self.ops.launch_count() - self.n0
        a = self.audit
        print(f"\n{self.what}: {len(a.records)} audited calls, {a.launches} audited launches, {launches} launches counted, "
              f"{time.perf_counter() - self.t0:.1f} s\n{a.table()}")
        bias = a.bias_by_op()
        for op, (calls, ulp, margin) in a.families().items():
            print(f"  {op:26s} {calls:5d} calls  worst {ulp:.3g} ulp16  min margin {margin:+.3g}  {bias[op].line()}")
        a.assert_clean()
        a.assert_unbiased()
        assert a.launches == launches > 0
        return a


def _expect(audit, op, **want):
    assert audit.seen(op, **want), f"no audited {op} call with {want}"


def _edit_state(unet, c, freeu=False):
    from anyv2v_b200.latent_store import LatentStore
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp
    from anyv2v_b200.schedulers import DDIMScheduler
    sched = DDIMScheduler()
    sched.set_timesteps(CONFIG3.n_steps)
    pipe = I2VGenXLPipeline(unet, sched)
    pipe.use_cuda_graphs = False
    init_pnp(pipe, sched, CONFIG3)
    if freeu:
        pipe.enable_freeu(**FREEU)
    else:
        pipe.disable_freeu()
    store = LatentStore(None, write_files=False)
    g = torch.Generator().manual_seed(3)
    for t in sched.timesteps.tolist():
        store.put(int(t), torch.randn(1, 4, 16, 64, 64, generator=g).half().to(dev))
    st = pipe.prepare_edit(c["video_latents"].clone(), c["edit_prompt"], c["neg_prompt"], c["inv_prompt"], c["edit_image_emb"],
                           c["edit_image_latents"], c["src_image_emb"], c["src_image_latents"], 8, CONFIG3.n_steps, 9.0, 0, None,
                           store, True)
    return pipe, st


@torch.no_grad()
def test_inversion_step(unet, monkeypatch):
    """one inversion step, B = 1, 16 x 64 x 64"""
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.schedulers import DDIMInverseScheduler
    c = _conditioning(64, 64)
    pipe = I2VGenXLPipeline(unet, DDIMInverseScheduler())
    pipe.use_cuda_graphs = False
    pipe.disable_freeu()
    p = _Pass(monkeypatch, "inversion step", seed=1)
    st = pipe.prepare_invert(c["video_latents"], c["inv_prompt"], c["src_image_latents"], c["src_image_emb"], 8, 50,
                             write_files=False)
    pipe.invert_step(st, 0)
    a = p.finish()
    _expect(a, "attention", mode="rows", n_v=1, seq=4096, batch=16)
    _expect(a, "attention", mode="rows", seq=4096, seq_kv=lambda v: v > 77, kv_batch_div=16)
    _expect(a, "temporal_attention_fused", n_v=1, F=16, HW=4096)
    _expect(a, "linear", geglu=True, N=10240)
    _expect(a, "groupnorm", two_source=True)
    _expect(a, "ddim_step", inverse=True)


@torch.no_grad()
def test_edit_steps(unet, monkeypatch):
    """BASELINE config 3: step 0 (conv, spatial and temporal injection fire) and step 30 (conv injection only, shared prefix
    and source pruning active)"""
    c = _conditioning(64, 64)
    pipe, st = _edit_state(unet, c)
    assert st.fires[0] and st.fires[30] and pipe._hook_flags(st.timesteps[30]) == (True, False, False)
    assert pipe._hook_flags(st.timesteps[0]) == (True, True, True)
    p = _Pass(monkeypatch, "edit step 0 (all injections)", seed=2)
    pipe.edit_step(st, 0)
    a = p.finish()
    _expect(a, "attention", mode="rows", n_v=3, seq=4096)
    _expect(a, "temporal_attention_fused", n_v=3)
    _expect(a, "attention", mode="rows", seq=4096, seq_kv=lambda v: v > 77, kv_batch_div=16, ldk_in_C=2)
    _expect(a, "conv3x3", slots=3, C=1280, Cout=1280, residual=True)
    _expect(a, "linear", K=2560, N=1280)
    _expect(a, "groupnorm", two_source=True, C=1920)
    _expect(a, "groupnorm", two_source=True, C=2560)
    _expect(a, "linear", geglu=True, N=10240)
    _expect(a, "ddim_step", inverse=False)
    p = _Pass(monkeypatch, "edit step 30 (conv injection only)", seed=3)
    pipe.edit_step(st, 30)
    a = p.finish()
    _expect(a, "conv3x3", slots=3, C=1280, Cout=1280, residual=True)
    assert not a.seen("attention", n_v=3) and not a.seen("temporal_attention_fused", n_v=3)


@torch.no_grad()
def test_edit_step_with_freeu(unet, monkeypatch):
    c = _conditioning(64, 64)
    pipe, st = _edit_state(unet, c, freeu=True)
    p = _Pass(monkeypatch, "edit step 0 with FreeU", seed=4)
    pipe.edit_step(st, 0)
    pipe.disable_freeu()
    a = p.finish()
    assert len(a.seen("freeu")) == 6
    _expect(a, "freeu", H=8, W=8)
    _expect(a, "freeu", H=16, W=16)


@torch.no_grad()
def test_call_step_704x1280_with_eta(unet, monkeypatch):
    """one image-to-video step at the reference's default 704 x 1280 (latents 88 x 160), CFG batch 2, eta = 1"""
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.schedulers import DDIMScheduler
    c = _conditioning(88, 160)
    pipe = I2VGenXLPipeline(unet, DDIMScheduler())
    pipe.use_cuda_graphs = False
    pipe.disable_freeu()
    st = pipe.prepare_call(c["video_latents"], c["edit_prompt"], c["edit_image_latents"], c["edit_image_emb"], 8, 50, 9.0,
                           c["neg_prompt"], 1.0, torch.Generator(device=dev).manual_seed(1), 1)
    p = _Pass(monkeypatch, "call step 704 x 1280, eta = 1", seed=5)
    pipe.call_step(st, 0)
    a = p.finish()
    _expect(a, "ddim_step_eta")
    _expect(a, "groupnorm", rows=225280)
    for seq in (3520, 880, 220):
        _expect(a, "attention", mode="rows", seq=seq)
    _expect(a, "attention", mode="rows", seq=14080)


@pytest.fixture(scope="module")
def sd_vae():
    from anyv2v_b200 import vae as product
    from oracle import vae_ref
    ref32 = vae_ref.seeded_vae(vae_ref.SD_VAE_CONFIG, seed=8888, dtype=torch.float32)
    ours = product.AutoencoderKL(**vae_ref.SD_VAE_CONFIG)
    ours.load_state_dict(ref32.state_dict())
    yield ours.to(device=dev, dtype=torch.float16).eval()
    torch.cuda.empty_cache()


@torch.no_grad()
def test_vae_decode_512(sd_vae, monkeypatch):
    from anyv2v_b200 import vae as product
    lat = torch.randn(1, 4, 2, 64, 64, generator=torch.Generator().manual_seed(11)).half().to(dev)
    p = _Pass(monkeypatch, "VAE decode, 2 frames at 512 x 512", seed=6)
    video = product.decode_latents(sd_vae, lat, None)
    a = p.finish()
    assert video.shape == (1, 3, 2, 512, 512) and torch.isfinite(video).all()
    _expect(a, "groupnorm", C=128, rows=262144, eps=1e-6)
    _expect(a, "conv3x3", C=512, H=256, W=256)
    _expect(a, "conv3x3", C=128, H=512, W=512)


@torch.no_grad()
def test_vae_encode_512(sd_vae, monkeypatch):
    from anyv2v_b200 import vae as product
    frames = torch.randn(2, 3, 512, 512, generator=torch.Generator().manual_seed(12)).clamp(-1, 1).half().to(dev)
    p = _Pass(monkeypatch, "VAE encode, 2 frames at 512 x 512", seed=7)
    z = product.encode_vae_video(sd_vae, frames, torch.Generator(device=dev).manual_seed(3))
    a = p.finish()
    assert z.shape == (1, 4, 2, 64, 64) and torch.isfinite(z).all()
    _expect(a, "groupnorm", C=128, rows=262144, eps=1e-6)
    _expect(a, "conv3x3", C=128, H=512, W=512)
