"""CPU tests of the conv A operand of the persistent GEMM kernel (csrc/gemm_ws.cu, gemm_ws_kernel<true>), through the
model of tools/kernel_models.py: per output tile and K block, the TMA box the producer loads (its origin, the tap walk and
TMA's zero-fill outside the tensor) holds element for element what gemm_wgmma_kernel's cp.async gather loads; and the
dispatch rule (conv_ws_box) sends the UNet's geometries where a box exists, the others to gemm_wgmma_kernel.  Negative
controls: a tap offset off by one, the phase offsets swapped, and an odd-F temporal conv at 8 x 8 let onto the TMA path."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _km():
    from tools import kernel_models as km
    km.conv_ws_rules()
    return km


@pytest.mark.parametrize("NF,H,W,Cin,chan", [
    (1, 64, 64, 64, 64),    # box 64 x 2 x 1: two image rows per tile
    (2, 32, 32, 128, 128),  # 32 x 4 x 1
    (3, 16, 16, 64, 64),    # 16 x 8 x 1
    (4, 8, 8, 128, 128),    # 8 x 8 x 2: two frames per tile
    (5, 8, 8, 64, 64),      # odd NF: the last tile is ragged, its box's second frame past the tensor
    (3, 4, 4, 64, 64),      # 4 x 4 x 8: one ragged tile
    (2, 32, 32, 64, 8),     # a_channels = 8: the box's channels past 8 read zeros
])
def test_conv3x3_tiles(NF, H, W, Cin, chan):
    assert _km().check_conv_tma_tiles("conv", NF=NF, H=H, W=W, Cin=Cin, chan=chan)


@pytest.mark.parametrize("phase", [1, 2, 3, 4])
@pytest.mark.parametrize("NF,H,W", [(1, 16, 16), (3, 8, 8)])
def test_up2_phase_tiles(phase, NF, H, W):
    assert _km().check_conv_tma_tiles("conv", NF=NF, H=H, W=W, Cin=64, phase=phase)


@pytest.mark.parametrize("B,F,HW", [(2, 3, 4096), (2, 5, 256), (2, 4, 64), (1, 16, 64)])
def test_tconv3_tiles(B, F, HW):
    assert _km().check_conv_tma_tiles("tconv", B=B, F=F, HW=HW, Cin=64)


def test_dispatch_rule():
    """the UNet's geometries at 512 x 512 (latents 64 / 32 / 16 / 8 wide) run on the TMA path; stride 2, widths that do not
    divide 128 (27 x 29, 720p's 88 x 160 levels), HW 400 and an odd F at 8 x 8 for the temporal conv do not"""
    km = _km()
    box = lambda mode, **g: km.conv_ws_box(km.conv_geometry(mode, **g))
    for hw in (64, 32, 16, 8):
        for nf in (16, 48):
            assert box("conv", NF=nf, H=hw, W=hw, Cin=64) == ((hw, 128 // hw, 1) if hw * hw >= 128 else (hw, hw, 128 // (hw * hw)))
            for ph in range(1, 5):
                assert box("conv", NF=nf, H=hw, W=hw, Cin=64, phase=ph) is not None
        assert box("tconv", B=3, F=16, HW=hw * hw, Cin=64) is not None
    assert box("conv", NF=16, H=64, W=64, Cin=64, stride=2) is None
    assert box("conv", NF=7, H=27, W=29, Cin=64) is None
    assert box("conv", NF=16, H=88, W=160, Cin=64) is None
    assert box("conv", NF=16, H=44, W=80, Cin=64) is None
    assert box("conv", NF=5, H=8, W=8, Cin=64) == (8, 8, 2)
    assert box("tconv", B=2, F=5, HW=64, Cin=64) is None
    assert box("tconv", B=2, F=3, HW=400, Cin=64) is None


@pytest.mark.parametrize("mode,geo,bad,match", [
    ("conv", dict(NF=2, H=16, W=16, Cin=64), dict(x_off=0), "TMA box holds"),                  # tap column off by one
    ("conv", dict(NF=2, H=16, W=16, Cin=64), dict(y_off=0), "TMA box holds"),                  # tap row off by one
    ("conv", dict(NF=2, H=8, W=8, Cin=64, phase=2), dict(swap_phase=True), "TMA box holds"),   # px and py exchanged
    ("tconv", dict(B=2, F=5, HW=64, Cin=64), dict(box=(64, 2, 1)), "TMA box holds"),         # a box across two clips
])
def test_negative_controls(mode, geo, bad, match):
    with pytest.raises(AssertionError, match=match):
        _km().check_conv_tma_tiles(mode, **geo, **bad)
