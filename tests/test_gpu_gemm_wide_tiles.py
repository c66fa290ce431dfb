"""GPU tests of gemm_ws_kernel's 160-column tiles (csrc/gemm_ws.cu, ws_tile_n: N a multiple of 160, with enough row tiles
that the wider tiles shorten the schedule) against the float64 contracts of tests/kernel_contracts.py, within
ulp16(ref) + kappa * cond (tests/ulp_check.py), on guarded buffers whose outputs start as NaN (tests/guarded.py).

Each case's shape is one that ws_tile_n sends to the 160-wide tiles on this GPU's SM count (tools/kernel_models.py restates
the rule and tests/test_gemm_wide_tiles_cpu.py pins it to the source), unless it says otherwise.  Covered: LINEAR with
bias, rowbias and a residual, ragged M, tile counts below and far above the SM count, a residual that aliases out, the up-block shortcut's two
sources (K = 640 / 960 split at 320 / 640); 3 x 3 convs with rowbias and a residual, a ragged last tile, three PnP slots,
N = 960, the four up2 phases and the temporal conv."""
import os
import sys

import pytest
import torch

import kernel_contracts as kc
from guarded import check_output, guarded_input, guarded_output
from test_gpu_gemm_conv_ws import _conv
from test_gpu_gemm_linear_ws import _run_linear
from ulp_check import KAPPA_GEMM, assert_within_bound, cond_conv_abs, cond_linear

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.kernel_models import ws_tile_n  # noqa: E402

pytestmark = pytest.mark.gpu
dev = "cuda"


def gin(t, **kw):
    return guarded_input(t, device=dev, **kw)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _w(N, K, g):
    return (torch.randn(N, K, generator=g) * K ** -0.5).half()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _width(M, N):
    return ws_tile_n(M, N, sms=_sms())


@pytest.mark.parametrize("N,K,row_tiles,width", [
    (320, 320, "1", 128),          # 3 tiles of 128 on 3 SMs end before 2 of 160
    (320, 320, "sms/2-1", 160),    # 2 x (SMs / 2 - 1) tiles: just below the SM count
    (320, 320, "3sms+1", 160),
    (960, 320, "1", 128),
    (960, 320, "sms/2-1", 160),    # 6 column tiles per row tile
    (1280, 1280, "sms/4", 160),    # 160 and 128 both exact
    (320, 1280, "sms/2-1", 160),   # K loops longer than the ring
    (320, 2880, "sms/2-1", 160),
])
def test_linear(N, K, row_tiles, width):
    """bias + rowbias + residual; the last row tile ragged"""
    sms = _sms()
    rows = {"1": 1, "sms/4": sms // 4, "sms/2-1": sms // 2 - 1, "3sms+1": 3 * sms + 1}[row_tiles]
    M = rows * 128 - 37
    assert _width(M, N) == width
    _run_linear(M, N, K, seed=rows * N + K)


def test_residual_aliases_out():
    from anyv2v_b200 import ops
    g = _gen(13)
    M, N, K = 3 * _sms() * 128 + 50, 960, 320
    assert _width(M, N) == 160
    a = torch.randn(M, K, generator=g).half()
    w = _w(N, K, g)
    bias = (torch.randn(N, generator=g) * 0.1).half()
    res = torch.randn(M, N, generator=g).half()
    out = guarded_output((M, N), device=dev)
    out.view.copy_(res)
    ops.linear(gin(a).view, gin(w).view, bias=gin(bias).view, residual=out.view, out=out.view)
    torch.cuda.synchronize()
    check_output(out, "linear residual in place")
    assert_within_bound(out.view.cpu(), kc.linear_exact(a, w, bias, residual=res), cond_linear(a, w, bias, residual=res),
                        KAPPA_GEMM, "linear residual in place", shape=(M, N))


@pytest.mark.parametrize("K1,K2", [(320, 320), (640, 320)])
def test_two_source(K1, K2):
    """the up-block shortcut: A = [hidden | skip] along K, split at k_split = K1"""
    from anyv2v_b200 import ops
    g = _gen(K1 + K2)
    M, N = 16000 + 3, 320
    assert _width(M, N) == 160
    a, a2 = torch.randn(M, K1, generator=g).half(), torch.randn(M, K2, generator=g).half()
    w = _w(N, K1 + K2, g)
    bias = (torch.randn(N, generator=g) * 0.1).half()
    out = guarded_output((M, N), device=dev)
    ag, a2g, wg, bg = gin(a, ld=K1 + 40).view, gin(a2, ld=K2 + 24).view, gin(w).view, gin(bias).view
    ops.linear(ag, wg, bias=bg, a2=a2g, out=out.view)
    torch.cuda.synchronize()
    check_output(out, "linear two-source")
    assert_within_bound(out.view.cpu(), kc.linear_exact(a, w, bias, a2=a2), cond_linear(a, w, bias, a2=a2), KAPPA_GEMM,
                        "linear two-source", shape=(M, N))


@pytest.mark.parametrize("NF,H,W,C,Cout,kw", [
    (2, 64, 64, 320, 320, {}),                 # the 64 x 64 level's resnet conv2: rowbias + residual
    (129, 8, 8, 128, 320, {}),                 # odd frame count: a ragged last tile
    (33, 16, 16, 64, 960, {}),                 # six column tiles
    (33, 16, 16, 128, 320, dict(slots=3)),     # PnP conv injection: three slots, each with its residual
    (33, 16, 16, 128, 320, dict(slots=3, residual=False)),
    (36, 32, 32, 64, 320, dict(alias=True)),       # out += conv(x) in place over 576 tiles
])
def test_conv3x3(NF, H, W, C, Cout, kw):
    assert _width(NF * H * W, Cout) == 160
    _conv(NF, H, W, C, Cout, seed=NF * H * W + C + Cout, **kw)


@pytest.mark.parametrize("NF,H,W", [(33, 16, 16), (129, 8, 8)])
def test_upsample_phases(NF, H, W):
    from anyv2v_b200 import ops
    g = _gen(NF * H * W)
    Cin, Cout = 128, 320
    assert _width(NF * H * W, Cout) == 160
    x = torch.randn(NF, H, W, Cin, generator=g).half()
    wph = ops.pack_upsample_weights((torch.randn(Cout, Cin, 3, 3, generator=g) * (9 * Cin) ** -0.5).half())
    bias = (torch.randn(Cout, generator=g) * 0.1).half()
    out = guarded_output((NF, 2 * H, 2 * W, Cout), device=dev)
    xg, wg, bg = gin(x).view, gin(wph).view, gin(bias).view
    ops.upsample2x_conv3x3(xg, wg, bias=bg, out=out.view)
    torch.cuda.synchronize()
    check_output(out, "upsample")
    assert_within_bound(out.view.cpu(), kc.upsample2x_conv3x3_exact(x, wph, bias),
                        cond_conv_abs(kc.upsample2x_conv3x3_exact, x, wph, bias), KAPPA_GEMM, f"upsample {NF}x{H}x{W}",
                        shape=tuple(out.view.shape))


@pytest.mark.parametrize("B,F_,HW,C", [(1, 4, 4096, 320), (6, 5, 256, 128), (20, 6, 64, 320)])
def test_tconv3(B, F_, HW, C):
    from anyv2v_b200 import ops
    g = _gen(B * F_ * HW + C)
    Cout = 320
    assert _width(B * F_ * HW, Cout) == 160
    x = torch.randn(B, F_ * HW, C, generator=g).half()
    w = _w(Cout, 3 * C, g)
    bias = (torch.randn(Cout, generator=g) * 0.1).half()
    res = torch.randn(B, F_ * HW, Cout, generator=g).half()
    out = guarded_output((B, F_ * HW, Cout), device=dev)
    xg, wg, bg, rg = gin(x).view, gin(w).view, gin(bias).view, gin(res).view
    ops.tconv3(xg, wg, F_, HW, bias=bg, residual=rg, out=out.view)
    torch.cuda.synchronize()
    check_output(out, "tconv3")
    ref = kc.tconv3_exact(x, w, F_, HW, bias, res).view(B, F_ * HW, Cout)
    cond = cond_conv_abs(kc.tconv3_exact, x, w, F_, HW, bias, res).view(B, F_ * HW, Cout)
    assert_within_bound(out.view.cpu(), ref, cond, KAPPA_GEMM, f"tconv3 B={B} F={F_} HW={HW}", shape=(B, F_ * HW, Cout))
