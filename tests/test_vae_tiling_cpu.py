"""VAE tiling and slicing (diffusers `enable_tiling` / `enable_slicing`, pipeline_i2vgen_xl.py:191-222) without a GPU: the tile
geometry, the stitch kernel's four-tile closed form against diffusers' sequential in-place blend loop (both in
tests/vae_tiling_ref.py), the precondition checks, and the encode / decode dispatch of the oracle and of the product VAE."""
import ctypes
import os
import subprocess

import pytest
import torch

import vae_tiling_ref as vt


@pytest.fixture
def emu(emulated_ops, monkeypatch):
    """the kernel contracts in place of anyv2v_b200.ops, ops.tile_stitch included"""
    vt.patch_ops(monkeypatch)
    return emulated_ops


def _product_grid(h, w, sample_size, decode):
    from anyv2v_b200 import vae
    v = vae.AutoencoderKL.__new__(vae.AutoencoderKL)  # the geometry needs the attributes only, not the modules
    v.config = type("C", (), dict(block_out_channels=(128, 256, 512, 512)))
    v.tile_sample_min_size, v.tile_latent_min_size, v.tile_overlap_factor = sample_size, int(sample_size / 8), 0.25
    return v.decode_grid(h, w) if decode else v.encode_grid(h, w)


# ----------------------------------------------------------------------------------------------------------- geometry
@pytest.mark.parametrize("H, W, rows, cols, blend_px, blend_lat", [
    (704, 1280, [704, 128], [768, 704, 128], 192, 24),
    (720, 1280, [720, 144], [768, 704, 128], 192, 24),
    (512, 512, [512], [512], 192, 24),
    (1160, 648, [768, 584, 8], [648, 72], 192, 24),
])
def test_geometry_known_answers(H, W, rows, cols, blend_px, blend_lat):
    dec = vt.geometry(H // 8, W // 8, 768, decode=True)
    enc = vt.geometry(H, W, 768, decode=False)
    assert [8 * e for e in dec.in_h] == rows and [8 * e for e in dec.in_w] == cols
    assert enc.in_h == rows and enc.in_w == cols
    assert (dec.blend, dec.row_limit, enc.blend, enc.row_limit) == (blend_px, 576, blend_lat, 72)
    assert dec.ys == [72 * k for k in range(len(rows))] and enc.xs == [576 * k for k in range(len(cols))]
    for ref, decode in ((dec, True), (enc, False)):
        g = _product_grid(H // 8 if decode else H, W // 8 if decode else W, 768, decode)
        assert (list(g.ys), list(g.xs), list(g.in_h), list(g.in_w)) == (ref.ys, ref.xs, ref.in_h, ref.in_w)
        assert (g.blend, g.row_limit, g.H, g.W) == (ref.blend, ref.row_limit, H if decode else H // 8, W if decode else W // 8)
        assert list(g.out_h) == ([8 * e for e in ref.in_h] if decode else [e // 8 for e in ref.in_h])


def test_geometry_at_704x1280_six_shapes_and_shrunken_seams():
    g = _product_grid(88, 160, 768, decode=True)
    assert len(g.ys) * len(g.xs) == 6 and len(g.shapes()) == 6
    assert sorted((8 * h, 8 * w) for h, w in g.shapes()) == sorted(
        [(704, 768), (704, 704), (704, 128), (128, 768), (128, 704), (128, 128)])
    ev = min(g.out_h[0], g.out_h[1], g.blend)
    eh = [min(g.out_w[j - 1], g.out_w[j], g.blend) for j in (1, 2)]
    assert ev == 128 and eh == [192, 128]


# --------------------------------------------------------------------------------------------- closed form vs loop
def _random_tiles(N, C, H, W, tile, step, seed):
    g = torch.Generator().manual_seed(seed)
    ext_h = [min(tile, H - y) for y in range(0, H, step)]
    ext_w = [min(tile, W - x) for x in range(0, W, step)]
    return [[[(3 * torch.randn(C, h, w, generator=g)).half() for w in ext_w] for h in ext_h] for _ in range(N)]


def _loop(tiles, blend, row_limit, **kw):
    rows = [[torch.stack([img[i][j] for img in tiles]) for j in range(len(tiles[0][0]))] for i in range(len(tiles[0]))]
    return vt.blend_loop(rows, blend, row_limit, **kw)


# (H, W, tile, step, blend, row_limit): diffusers' own settings (tile 4b, step = row_limit = 3b) at small b, grids up to
# 4 x 4, last tiles longer and shorter than the blend extent, single rows / columns
GRIDS = [(38, 33, 16, 12, 4, 12), (48, 48, 16, 12, 4, 12), (37, 13, 16, 12, 4, 12), (10, 40, 16, 12, 4, 12),
         (50, 50, 24, 18, 6, 18), (44, 27, 32, 24, 8, 24), (26, 62, 8, 6, 2, 6)]


@pytest.mark.parametrize("grid", GRIDS)
def test_closed_form_equals_the_sequential_loop(grid):
    H, W, tile, step, blend, row_limit = grid
    tiles = _random_tiles(2, 3, H, W, tile, step, seed=H * W)
    got = vt.stitch_closed_form(tiles, H, W, tile, step, blend, row_limit)
    want = _loop(tiles, blend, row_limit)
    assert got.shape == want.shape == (2, 3, H, W)
    assert torch.equal(got, want)


@pytest.mark.parametrize("control", ["h_first", "raw_neighbours"])
def test_negative_controls_differ(control):
    H, W, tile, step, blend, row_limit = GRIDS[0]
    tiles = _random_tiles(1, 3, H, W, tile, step, seed=7)
    want = vt.stitch_closed_form(tiles, H, W, tile, step, blend, row_limit)
    bad = _loop(tiles, blend, row_limit, **{control: True})
    assert not torch.equal(bad, want)


def test_stitch_weights_round_like_torch_fp16_times_python_float():
    """the contract's blend is torch's `a * (1 - y/e) + b * (y/e)` on fp16 tensors, bit for bit"""
    g = torch.Generator().manual_seed(3)
    a, b = (5 * torch.randn(4, 7, generator=g)).half(), (5 * torch.randn(4, 7, generator=g)).half()
    for e in (3, 7, 24, 192):
        for y in range(min(e, 7)):
            want = a * (1 - y / e) + b * (y / e)
            got = vt._blend(a[:, y:y + 1], b[:, y:y + 1], [y], e, 1)
            assert torch.equal(got, want[:, y:y + 1]), (e, y)


# ------------------------------------------------------------------------------------------------- preconditions
def test_inconsistent_tile_latent_min_size_is_refused():
    from anyv2v_b200 import vae
    with pytest.raises(ValueError, match="disagree"):
        vae.tile_grid(88, 160, 64, 48, 192, 576, up=8)       # tile_latent_min_size 64 with tile_sample_min_size 768
    with pytest.raises(ValueError, match="disagree"):
        vae.tile_grid(704, 1280, 768, 576, 16, 48, down=8)  # latent blend / row_limit of a 64-pixel tile
    with pytest.raises(ValueError, match="whole output pixels"):
        vae.tile_grid(700, 1280, 768, 576, 24, 72, down=8)
    vae.tile_grid(88, 160, 96, 72, 192, 576, up=8)


def test_tile_stitch_abi_rejects_bad_grids_before_any_cuda_call():
    import __graft_entry__ as g
    g.build()
    from anyv2v_b200 import _lib
    lib = _lib.lib()
    ok = dict(tiles=64, out=128, on=1, oc=1, oy=1, ox=1, N=2, C=3, H=704, W=1280, tile_rows=2, tile_cols=3, tile=768, step=576,
              blend=192, row_limit=576)
    for bad in (dict(row_limit=512), dict(tile=512, step=384), dict(tile_rows=3), dict(tile_cols=2), dict(blend=400),
                dict(C=0), dict(tiles=None), dict(step=0)):
        a = _lib.TileStitchArgs(**dict(ok, **bad))
        assert lib.av2v_tile_stitch_f16(ctypes.byref(a), None) == _lib.AV2V_EINVAL, bad
    assert lib.av2v_tile_stitch_f16(None, None) == _lib.AV2V_EINVAL
    assert lib.av2v_tile_stitch_f16(ctypes.byref(_lib.TileStitchArgs(**dict(ok, N=0))), None) == _lib.AV2V_OK


def test_tile_stitch_args_struct_matches_the_c_header(tmp_path):
    """ctypes mirrors of av2v_tile_desc / av2v_tile_stitch_args against the layout gcc gives include/anyv2v_b200.h"""
    from anyv2v_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "anyv2v_b200.h"', 'int main(void) {']
    for c_name, cls in (("av2v_tile_desc", _lib.TileDesc), ("av2v_tile_stitch_args", _lib.TileStitchArgs)):
        lines.append(f'  printf("{c_name}.size %zu\\n", sizeof({c_name}));')
        lines += [f'  printf("{c_name}.{f} %zu\\n", offsetof({c_name}, {f}));' for f, _ in cls._fields_]
    lines += ['  return 0;', '}']
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    for c_name, cls in (("av2v_tile_desc", _lib.TileDesc), ("av2v_tile_stitch_args", _lib.TileStitchArgs)):
        assert int(out[f"{c_name}.size"]) == ctypes.sizeof(cls)
        for f, _ in cls._fields_:
            assert int(out[f"{c_name}.{f}"]) == getattr(cls, f).offset, (c_name, f)


# ---------------------------------------------------------------------------------------------------------- dispatch
@pytest.fixture(scope="module")
def tiny_oracle():
    from oracle import vae_ref
    return vae_ref.seeded_vae(vae_ref.TINY_VAE_CONFIG, seed=8888, dtype=torch.float32)


@torch.no_grad()
def test_oracle_dispatch_rules(tiny_oracle):
    """diffusers: tiling wins when the image exceeds the tile; slicing splits batches > 1; decode slices before it tiles"""
    d = vt.DiffusersTiling(tiny_oracle, sample_size=16)
    assert (d.tile_sample_min_size, d.tile_latent_min_size, d.tile_overlap_factor) == (16, 8, 0.25)
    big, small = torch.randn(2, 3, 32, 40), torch.randn(2, 3, 16, 16)
    zbig, zsmall = torch.randn(2, 4, 16, 20), torch.randn(2, 4, 8, 8)

    def path(fn, x):
        d.trace.clear()
        fn(x)
        return list(d.trace)
    assert path(d.encode, big) == ["encode"] and path(d.decode, zbig) == ["decode"]
    d.enable_slicing()
    assert path(d.encode, big) == ["sliced_encode"] and path(d.encode, big[:1]) == ["encode"]
    assert path(d.decode, zbig) == ["decode", "decode"]
    d.enable_tiling()
    assert path(d.encode, big) == ["tiled_encode"] and path(d.encode, small) == ["sliced_encode"]
    assert path(d.decode, zbig) == ["tiled_decode", "tiled_decode"] and path(d.decode, zsmall) == ["decode", "decode"]
    d.disable_slicing()
    assert path(d.decode, zbig) == ["tiled_decode"] and path(d.encode, big[:, :, :16, :17]) == ["tiled_encode"]
    d.disable_tiling()
    assert path(d.encode, big) == ["encode"]
    # slicing does not change the per-sample result; tiling changes it (the seams) but keeps the shapes
    ref = d.decode(zbig).sample
    d.enable_slicing()
    assert torch.allclose(d.decode(zbig).sample, ref, rtol=1e-5, atol=1e-5)
    d.enable_tiling()
    tiled = d.decode(zbig).sample
    assert tiled.shape == ref.shape and not torch.allclose(tiled, ref, rtol=1e-3, atol=1e-3)


def _product_tiny(tiny_oracle, sample_size=16):
    from anyv2v_b200 import vae
    from oracle import vae_ref
    ours = vae.AutoencoderKL(**vae_ref.TINY_VAE_CONFIG, sample_size=sample_size)
    ours.load_state_dict(tiny_oracle.state_dict())
    return ours.half().eval()


@torch.no_grad()
def test_product_dispatch_and_tiles_follow_the_oracle(emu, tiny_oracle, monkeypatch):
    """the product VAE on the kernel contracts: the same paths as diffusers for each knob, tiled results close to the fp32
    oracle's tiled loop, and independent of tile_batch"""
    from anyv2v_b200 import ops
    ours = _product_tiny(tiny_oracle)
    assert (ours.tile_sample_min_size, ours.tile_latent_min_size, ours.tile_overlap_factor, ours.tile_batch) == (16, 8, 0.25, 16)
    assert not ours.use_tiling and not ours.use_slicing
    d = vt.DiffusersTiling(tiny_oracle, sample_size=16)
    stitches = []
    monkeypatch.setattr(ops, "tile_stitch", lambda *a, **k: stitches.append(1) or vt.stitch_closed_form(*a, **k))
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 3, 32, 40, generator=g).clamp(-1, 1)
    z = torch.randn(2, 4, 16, 20, generator=g)
    for slicing in (False, True):
        for tiling in (False, True):
            for m in (ours, d):
                (m.enable_slicing if slicing else m.disable_slicing)()
                m.enable_tiling(tiling)
            stitches.clear()
            dec = ours.decode(z.half()).sample
            enc = ours.encode(x.half()).latent_dist
            assert len(stitches) == (3 if slicing else 2) * tiling, (slicing, tiling, len(stitches))
            want_dec = d.decode(z).sample
            want_enc = d.encode(x).latent_dist
            for got, want, what in ((dec, want_dec, "decode"), (enc.mean, want_enc.mean, "mean"), (enc.logvar, want_enc.logvar, "logvar")):
                assert got.shape == want.shape, what
                err = (got.float() - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt()
                assert err < 1e-2, (what, slicing, tiling, float(err))
    ours.disable_slicing()
    ours.enable_tiling()
    ref = ours.decode(z.half()).sample
    for tb in (1, 3):
        ours.tile_batch = tb
        got = ours.decode(z.half()).sample
        assert (got.float() - ref.float()).abs().max() <= 2e-3 * ref.float().abs().max(), tb


@torch.no_grad()
def test_encode_vae_video_with_slicing_keeps_the_draws(emu, tiny_oracle):
    from anyv2v_b200 import vae
    ours = _product_tiny(tiny_oracle)
    frames = torch.randn(3, 3, 16, 24, generator=torch.Generator().manual_seed(6)).clamp(-1, 1).half()
    want = vae.encode_vae_video(ours, frames, torch.Generator().manual_seed(3))
    ours.enable_slicing()
    got = vae.encode_vae_video(ours, frames, torch.Generator().manual_seed(3))
    assert got.shape == want.shape == (1, 4, 3, 8, 12)
    assert (got.float() - want.float()).abs().max() <= 2e-3 * want.float().abs().max()


def test_pipeline_vae_knobs_forward_to_the_vae():
    from types import SimpleNamespace
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    with pytest.raises(ValueError, match="vae"):
        I2VGenXLPipeline(unet=None).enable_vae_tiling()
    calls = []
    fake = SimpleNamespace(**{n: (lambda n=n: calls.append(n)) for n in ("enable_slicing", "disable_slicing", "enable_tiling",
                                                                          "disable_tiling")})
    pipe = I2VGenXLPipeline(unet=None, vae=fake)
    pipe.enable_vae_slicing()
    pipe.enable_vae_tiling()
    pipe.disable_vae_tiling()
    pipe.disable_vae_slicing()
    assert calls == ["enable_slicing", "enable_tiling", "disable_tiling", "disable_slicing"]


def test_build_pipeline_reads_the_vae_sample_size(tmp_path):
    import json
    from anyv2v_b200.run_group_pnp_edit import vae_sample_size
    assert vae_sample_size(str(tmp_path)) == {}
    (tmp_path / "config.json").write_text(json.dumps({"sample_size": 512, "block_out_channels": [128, 256, 512, 512]}))
    assert vae_sample_size(str(tmp_path)) == {"sample_size": 512}
    from anyv2v_b200.vae import AutoencoderKL
    v = AutoencoderKL(block_out_channels=(32, 32), norm_num_groups=32, layers_per_block=1, sample_size=[512, 512])
    assert (v.tile_sample_min_size, v.tile_latent_min_size) == (512, 256)
    assert AutoencoderKL(block_out_channels=(32, 32), norm_num_groups=32, layers_per_block=1).tile_sample_min_size == 768
