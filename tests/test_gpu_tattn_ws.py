"""The persistent, warp-specialized fused temporal attention (tattn_fused_kernel) against its float64 contract, in guarded
buffers (tests/guarded.py via test_gpu_contracts._run): the UNet's widths at F = 16, frame counts that leave an empty slot
tail or put a pixel across the 64-slot halves, a ragged last pixel tile, ldx > Cx with a NaN gap, launches with fewer items
than SMs and with many times more, and shared memory left full of NaN by a previous launch."""
import pytest
import torch

import test_gpu_contracts as gc

pytestmark = pytest.mark.gpu

# (Cx, heads) of the temporal transformers at the 64², 32², 16² and 8² levels and of transformer_in
WIDTHS = [(320, 5), (640, 10), (1280, 20), (1280, 20), (320, 8)]
LEVEL_HW = [1024, 1024, 256, 64, 1024]  # the 64² level and transformer_in at 32² pixels keep the float64 contract cheap


def _call(F, HW, Cx, heads, src, nv, seed, x_scale=1.0):
    """ops.temporal_attention_fused on guarded x (ldx = Cx + 8) and out (ldo = C + 8) against the contract"""
    C = heads * 64
    clips = src * nv
    rows = clips * F * HW
    torch.manual_seed(seed)
    x = gc.gin(gc.rnd(rows, Cx, scale=x_scale), ld=Cx + 8, guard=128 * (Cx + 8))
    out = gc.gout((rows, C), ld=C + 8)
    gc._run("temporal_attention_fused", [x, gc.gin(gc._w(3 * C, Cx)), heads, F, HW, clips, out], dict(scale=0.125, n_v=nv),
            [out], atol_frac=2e-3)


def _poison(F, HW, Cx, heads, nv):
    """one launch whose x is all NaN: every ring stage and Q / K / V tile of the SMs it ran on is left holding NaN"""
    from anyv2v_b200 import ops
    C = heads * 64
    rows = nv * F * HW
    x = torch.full((rows, Cx), float("nan"), dtype=torch.float16, device="cuda")
    w = torch.full((3 * C, Cx), float("nan"), dtype=torch.float16, device="cuda")
    ops.temporal_attention_fused(x, w, heads, F, HW, nv, torch.empty(rows, C, dtype=torch.float16, device="cuda"), n_v=nv)
    torch.cuda.synchronize()


@pytest.mark.parametrize("nv", [1, 3])
@pytest.mark.parametrize("level", range(len(WIDTHS)), ids=["64x64", "32x32", "16x16", "8x8", "transformer_in"])
def test_unet_widths(level, nv):
    """F = 16 at every (Cx, heads) the UNet runs the kernel at; items = heads x pixel tiles are many times the SM count"""
    Cx, heads = WIDTHS[level]
    _call(16, LEVEL_HW[level], Cx, heads, 1, nv, seed=level * 2 + nv)


@pytest.mark.parametrize("nv", [1, 3])
@pytest.mark.parametrize("F", [24, 72, 128])
def test_frame_counts_after_nan(F, nv):
    """F = 24 / 72 (slot tail, pixels across slot 64), F = 128 (one pixel per item), each after a launch that filled
    shared memory with NaN at F = 16 (every slot row written): the tail rows must be zero again, not stale"""
    ppt = 128 // F
    _poison(16, 2048, 320, 5, nv)
    _call(F, 40 * ppt + 1, 320, 5, 2, nv, seed=F + nv)


@pytest.mark.parametrize("nv", [1, 3])
def test_fewer_items_than_sms(nv):
    """2 heads x 3 pixel tiles (the last ragged): most SMs get no item"""
    _call(16, 17, 64, 2, 1, nv, seed=7 + nv)


@pytest.mark.parametrize("nv", [1, 3])
def test_many_items_per_cta(nv):
    """the 64² level at full size: 5 heads x 512 pixel tiles = 2560 items, about 19 per CTA"""
    _call(16, 4096, 320, 5, 1, nv, seed=11 + nv, x_scale=2.0)
