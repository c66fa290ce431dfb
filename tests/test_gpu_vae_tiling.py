"""VAE tiling and slicing on the GPU: the stitch kernel bit-exact against diffusers' sequential blend loop in torch CUDA fp16
inside guarded buffers; tiled encode / decode of the tiny and the full-size VAE against the fp32 oracle's tiled loop; slicing,
tile_batch grouping, the pipeline knobs, and peak memory that does not grow with the frame count."""
import pytest
import torch

import vae_tiling_ref as vt
from guarded import check_output, guarded_input, guarded_output
from parity_utils import err_stats

pytestmark = pytest.mark.gpu
dev = "cuda"


# -------------------------------------------------------------------------------------------------------- the kernel
def _tile_strides(k, C, h, w):
    """non-contiguous layouts, alternating: channels-last with padded rows, planar with padded rows and planes"""
    if k % 2 == 0:
        return (1, (w + 3) * C, C)
    return ((h + 1) * (w + 5), w + 5, 1)


# (N, C, H, W, tile, step, blend, row_limit): the 704 x 1280 decode (pixels) and encode (latents), and the 1160 x 648 encode
# (latent edge tiles 1 and 9 long, shorter than the blend extent)
STITCH = [(2, 3, 704, 1280, 768, 576, 192, 576), (3, 8, 88, 160, 96, 72, 24, 72), (2, 8, 145, 81, 96, 72, 24, 72)]


@torch.no_grad()
@pytest.mark.parametrize("geo", STITCH, ids=["decode704x1280", "encode704x1280", "encode1160x648"])
def test_stitch_kernel_equals_the_sequential_loop_guarded(geo):
    from anyv2v_b200 import ops
    N, C, H, W, tile, step, blend, row_limit = geo
    g = torch.Generator().manual_seed(H + W)
    ext_h = [min(tile, H - y) for y in range(0, H, step)]
    ext_w = [min(tile, W - x) for x in range(0, W, step)]
    vals = [[[(3 * torch.randn(C, h, w, generator=g)).half() for w in ext_w] for h in ext_h] for _ in range(N)]
    guards, k = [], 0
    tiles = []
    for img in vals:
        rows = []
        for row in img:
            cols = []
            for t in row:
                gi = guarded_input(t, strides=_tile_strides(k, *t.shape), device=dev)
                guards.append(gi)
                cols.append(gi.view)
                k += 1
            rows.append(cols)
        tiles.append(rows)
    go = guarded_output((N, C, H, W), strides=(H * W * C, 1, W * C, C), device=dev)
    ops.tile_stitch(tiles, H, W, tile, step, blend, row_limit, out=go.view)
    torch.cuda.synchronize()
    check_output(go, f"tile_stitch {geo}")
    rows = [[torch.stack([img[i][j] for img in vals]).to(dev) for j in range(len(ext_w))] for i in range(len(ext_h))]
    want = vt.blend_loop(rows, blend, row_limit)                       # diffusers' loop, torch CUDA fp16
    assert torch.equal(go.view, want), geo
    assert torch.equal(go.view.cpu(), vt.stitch_closed_form(vals, H, W, tile, step, blend, row_limit))


def test_stitch_wrapper_refusals():
    from anyv2v_b200 import ops
    from anyv2v_b200._lib import Av2vError
    t = [[[torch.zeros(3, 16, 16, device=dev, dtype=torch.float16)]]]
    with pytest.raises(Av2vError, match="expected"):
        ops.tile_stitch([[[torch.zeros(3, 16, 15, device=dev, dtype=torch.float16)]]], 16, 16, 16, 12, 4, 12)
    with pytest.raises(Av2vError, match="CUDA fp16"):
        ops.tile_stitch([[[torch.zeros(3, 16, 16, dtype=torch.float16)]]], 16, 16, 16, 12, 4, 12)
    with pytest.raises(Av2vError, match="kept parts"):
        ops.tile_stitch(t, 16, 16, 16, 16, 4, 12)
    assert torch.equal(ops.tile_stitch(t, 16, 16, 16, 16, 4, 16), t[0][0][0][None])


# ----------------------------------------------------------------------------------------------------- tiny VAE
def _as_close_as_fp16_torch(got, ref32, ref16, what, slack=3.0):
    """the slack of tests/test_gpu_vae.py: our error against fp32 within 3x fp16 torch's own"""
    assert torch.isfinite(got).all(), what
    e_ours, e_ref = err_stats(got, ref32), err_stats(ref16, ref32)
    assert e_ours["rms_rel"] <= max(slack * e_ref["rms_rel"], 2e-3), (what, e_ours, e_ref)


def _vaes(cfg, sample_size):
    from types import SimpleNamespace
    from anyv2v_b200 import vae as product
    from oracle import vae_ref
    ref32 = vae_ref.seeded_vae(cfg, seed=8888, dtype=torch.float32).to(dev)
    ref16 = vae_ref.seeded_vae(cfg, seed=8888, dtype=torch.float16).to(dev)
    ours = product.AutoencoderKL(**cfg, sample_size=sample_size)
    ours.load_state_dict(ref32.state_dict())
    ours = ours.to(device=dev, dtype=torch.float16).eval()
    t32, t16 = vt.DiffusersTiling(ref32, sample_size), vt.DiffusersTiling(ref16, sample_size)
    for m in (ours, t32, t16):
        m.enable_tiling()
    return SimpleNamespace(ref32=t32, ref16=t16, ours=ours)


@pytest.fixture(scope="module")
def tiny():
    from oracle import vae_ref
    return _vaes(vae_ref.TINY_VAE_CONFIG, 32)  # 32-pixel / 16-latent tiles: 3 x 3 grids below


@torch.no_grad()
def test_tiny_tiled_decode_and_encode_match_the_oracle(tiny):
    g = torch.Generator().manual_seed(21)
    z = torch.randn(3, 4, 32, 36, generator=g).to(dev)        # latent tiles at 0 / 12 / 24: 3 x 3
    x = torch.randn(3, 3, 64, 72, generator=g).clamp(-1, 1).to(dev)
    assert len(tiny.ours.decode_grid(32, 36).shapes()) == 4 and len(tiny.ours.encode_grid(64, 72).ys) == 3
    got = tiny.ours.decode(z.half()).sample
    _as_close_as_fp16_torch(got, tiny.ref32.decode(z).sample, tiny.ref16.decode(z.half()).sample, "tiny tiled decode")
    d, d32, d16 = tiny.ours.encode(x.half()).latent_dist, tiny.ref32.encode(x).latent_dist, tiny.ref16.encode(x.half()).latent_dist
    _as_close_as_fp16_torch(d.mean, d32.mean, d16.mean, "tiny tiled encode mean")
    _as_close_as_fp16_torch(d.logvar, d32.logvar, d16.logvar, "tiny tiled encode logvar")


@torch.no_grad()
def test_tiny_slicing_and_tile_batch_do_not_change_the_frames(tiny):
    g = torch.Generator().manual_seed(22)
    z = torch.randn(3, 4, 32, 36, generator=g).to(dev).half()
    x = torch.randn(3, 3, 64, 72, generator=g).clamp(-1, 1).to(dev).half()
    v = tiny.ours
    ref_dec, ref_enc = v.decode(z).sample, v.encode(x).latent_dist.mean
    try:
        v.enable_slicing()
        assert err_stats(v.decode(z).sample, ref_dec)["rms_rel"] < 2e-3
        v.disable_slicing()
        for tb in (1, 2):
            v.tile_batch = tb
            assert err_stats(v.decode(z).sample, ref_dec)["rms_rel"] < 2e-3, tb
            assert err_stats(v.encode(x).latent_dist.mean, ref_enc)["rms_rel"] < 2e-3, tb
        v.disable_tiling()
        small = z[:, :, :16, :16]
        whole = v.decode(small).sample
        v.enable_slicing()
        assert err_stats(v.decode(small).sample, whole)["rms_rel"] < 2e-3
    finally:
        v.tile_batch = 16
        v.disable_slicing()
        v.enable_tiling()


# ----------------------------------------------------------------------------------------------------- full size
@torch.no_grad()
def test_full_size_tiled_decode_and_encode_at_704x1280_match_the_oracle():
    from oracle import vae_ref
    full = _vaes(vae_ref.SD_VAE_CONFIG, 768)
    g = torch.Generator().manual_seed(23)
    z = torch.randn(2, 4, 88, 160, generator=g).to(dev)
    got = full.ours.decode(z.half()).sample
    assert got.shape == (2, 3, 704, 1280)
    _as_close_as_fp16_torch(got, full.ref32.decode(z).sample, full.ref16.decode(z.half()).sample, "full tiled decode")
    x = torch.randn(2, 3, 704, 1280, generator=g).clamp(-1, 1).to(dev)
    d, d32, d16 = full.ours.encode(x.half()).latent_dist, full.ref32.encode(x).latent_dist, full.ref16.encode(x.half()).latent_dist
    assert d.mean.shape == (2, 4, 88, 160)
    _as_close_as_fp16_torch(d.mean, d32.mean, d16.mean, "full tiled encode mean")
    _as_close_as_fp16_torch(d.logvar, d32.logvar, d16.logvar, "full tiled encode logvar")


@torch.no_grad()
def test_peak_memory_does_not_grow_with_frames_at_704x1280():
    """tiling + slicing: peak memory minus the output is the same for 4 and 32 frames (encode and decode)"""
    from anyv2v_b200 import vae as product
    from oracle import vae_ref
    v = product.AutoencoderKL(**vae_ref.SD_VAE_CONFIG).to(device=dev, dtype=torch.float16).eval()
    v.enable_tiling()
    v.enable_slicing()
    over = {}
    for f in (2, 4, 32):  # 2: warm-up (library workspaces, first-call allocations), not compared
        z = torch.randn(f, 4, 88, 160, device=dev).half()
        x = torch.randn(f, 3, 704, 1280, device=dev).clamp(-1, 1).half()
        for what, fn in (("decode", lambda: v.decode(z).sample), ("encode", lambda: product.encode_vae_video(v, x))):
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            out = fn()
            torch.cuda.synchronize()
            over[what, f] = torch.cuda.max_memory_allocated() - base - out.numel() * out.element_size()
            del out
        del z, x
    for what in ("decode", "encode"):
        assert abs(over[what, 32] - over[what, 4]) <= 0.10 * over[what, 4], (what, over)


# ------------------------------------------------------------------------------------------------------- pipeline
@torch.no_grad()
def test_pipeline_knobs_change_the_call_and_disable_restores_it():
    from PIL import Image
    from anyv2v_b200.run_group_pnp_edit import build_pipeline
    from oracle.unet_ref import TINY_CONFIG
    from test_gpu_runners import TINY_VAE
    pipe = build_pipeline(torch.device(dev), TINY_CONFIG, seed=3, broadcast=False, with_encoders=True, vae_config=TINY_VAE)
    image = Image.new("RGB", (640, 480), (120, 60, 200))
    video = torch.randn(2, 3, 704, 1280, generator=torch.Generator().manual_seed(4)).clamp(-1, 1)

    lat = torch.randn(1, 4, 2, 88, 160, generator=torch.Generator().manual_seed(5)).to(dev).half()

    def run():
        """(first-frame image latents, encode_vae_video latents, decode_latents video, pipe(...) frames) at 704 x 1280"""
        _, img_lat = pipe.encode_first_frame(image, 704, 1280, 2, generator=torch.Generator(device=dev).manual_seed(2))
        enc = pipe.encode_vae_video(video, generator=torch.Generator(device=dev).manual_seed(1))
        frames = pipe(prompt="a man walking", image=image, num_frames=2, num_inference_steps=3, output_type="np",
                      generator=torch.Generator(device=dev).manual_seed(0)).frames
        return img_lat, enc, pipe.decode_latents(lat), torch.as_tensor(frames)
    plain = run()
    pipe.enable_vae_tiling()
    tiled = run()
    pipe.enable_vae_slicing()
    both = run()
    pipe.disable_vae_tiling()
    sliced = run()
    pipe.disable_vae_slicing()
    again = run()
    # what the VAE computes is restored bit for bit.  The frames of pipe(...) are compared in shape only: its UNet steps
    # do not repeat bit for bit from one call to the next, with or without these knobs
    for a, b in zip(again[:3], plain[:3]):
        assert torch.equal(a, b)
    for knob in (tiled, both):
        assert all(k.shape == p.shape and torch.isfinite(k.float()).all() for k, p in zip(knob, plain))
        for a, b in zip(knob[:3], plain[:3]):
            assert not torch.equal(a, b)
    for a, b in zip(sliced[:3], plain[:3]):
        assert err_stats(a, b)["rms_rel"] < 2e-3
    for a, b in zip(both[:3], tiled[:3]):
        assert err_stats(a, b)["rms_rel"] < 2e-3
