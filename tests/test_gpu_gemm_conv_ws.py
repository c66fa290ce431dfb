"""GPU tests of the conv modes on the persistent, TMA-fed GEMM kernel (csrc/gemm_ws.cu, gemm_ws_kernel<true>) against
the float64 contracts of tests/kernel_contracts.py, within ulp16(ref) + kappa * cond (tests/ulp_check.py), on guarded
buffers (tests/guarded.py).

A conv runs there iff every 128-row tile is one box of its input (conv_ws_box); each case also checks, with torch.profiler
on a few more calls into a scratch output, which kernel runs it, so both sides of the rule are covered: tile counts around the SM count, 3 x 3 convs at 64 / 32 / 16 / 8
pixels wide (two-frame boxes at 8 x 8; an odd frame count leaves a ragged last tile whose box runs past the last frame),
the four up2 phases, temporal convs at HW 4096 / 256 / 64 (an odd frame count at 64 goes to gemm_wgmma_kernel), K up to
11520, rowbias, three slots with a residual, a residual that aliases out, and padded
channels (a_channels = 8)."""
import pytest
import torch

import kernel_contracts as kc
from guarded import check_output, guarded_input, guarded_output
from ulp_check import KAPPA_GEMM, assert_within_bound, cond_conv_abs

pytestmark = pytest.mark.gpu
dev = "cuda"
WS, OLD = "gemm_ws_kernel", "gemm_wgmma_kernel"


def gin(t):
    return guarded_input(t, device=dev)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _w(N, K, g):
    return (torch.randn(N, K, generator=g) * K ** -0.5).half()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _kernels(fn, reps=3, sessions=3):
    """the GEMM kernels (WS, OLD) that fn launches, recorded by torch.profiler over a few calls (fn writes a scratch output).
    fn always launches kernels, so a session that recorded no device kernel at all lost its CUPTI activity records (seen on
    shared machines): that session says nothing about the dispatch and is recorded again.  Any recorded kernel counts, so a
    session in which fn ran something other than WS / OLD still returns (and fails the caller's check)."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    for _ in range(sessions):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if e.device_type == DeviceType.CUDA}
        if names:
            return {k for k in (WS, OLD) if any(k in n for n in names)}
    raise AssertionError(f"torch.profiler recorded no device kernel in {sessions} sessions of {reps} calls")


def _conv(NF, H, W, C, Cout, seed, *, Cin=None, rowbias=True, slots=1, residual=True, alias=False, kernel=WS):
    from anyv2v_b200 import ops
    g = _gen(seed)
    Cin = Cin or C
    x = torch.randn(NF, H, W, C, generator=g).half()
    wfull = _w(Cout, 9 * Cin, g)
    if C != Cin:  # weights of the missing channels are zero (ops pads them so)
        wfull = wfull.view(Cout, 9, Cin)
        wfull[:, :, C:] = 0
        wfull = wfull.reshape(Cout, 9 * Cin).contiguous()
    M = NF * H * W
    bias = (torch.randn(Cout, generator=g) * 0.1).half()
    rb = (torch.randn(NF, Cout, generator=g) * 0.25).half() if rowbias else None
    shape = (slots, M, Cout) if slots > 1 else (M, Cout)
    res = torch.randn(shape, generator=g).half() if residual else None
    out = guarded_output(shape, device=dev)
    kw = dict(bias=gin(bias).view, n_slots=slots, slot_stride=M * Cout)
    if rb is not None:
        kw.update(rowbias=gin(rb).view, rows_per_rowbias=H * W)
    if alias:
        out.view.copy_(res)
        kw["residual"] = out.view
    elif res is not None:
        kw["residual"] = gin(res).view
    xg = gin(x).view
    wg = gin(wfull).view
    ops.conv3x3(xg, wg, out=out.view, **kw)
    torch.cuda.synchronize()
    check_output(out, "conv3x3")
    scratch = dict(kw, residual=res.to(dev)) if res is not None else kw
    assert _kernels(lambda: ops.conv3x3(xg, wg, out=torch.empty(shape, dtype=torch.half, device=dev), **scratch)) == {kernel}
    xp = x if C == Cin else torch.cat([x, torch.zeros(NF, H, W, Cin - C, dtype=x.dtype)], dim=3)
    acc = kc.conv3x3_exact(xp, wfull, bias, rb, H * W)
    cond = cond_conv_abs(kc.conv3x3_exact, xp, wfull, bias, rb, H * W)
    if res is not None:
        acc, cond = acc + res.double(), cond + res.double().abs()
    else:
        acc, cond = acc.expand(shape), cond.expand(shape)
    assert_within_bound(out.view.cpu(), acc, cond, KAPPA_GEMM, f"conv3x3 {NF}x{H}x{W}x{C} -> {Cout}", shape=shape)


@pytest.mark.parametrize("n", ["1", "sms-1", "sms", "sms+1", "2sms+3"])
def test_tile_counts(n):
    """one column tile; the tile count is 2 NF of 16 x 16 frames when even, else of 8 x 8 frames that many pairs"""
    sms = _sms()
    tiles = {"1": 1, "sms-1": sms - 1, "sms": sms, "sms+1": sms + 1, "2sms+3": 2 * sms + 3}[n]
    if tiles % 2:  # 8 x 8 frames two per tile
        _conv(2 * tiles, 8, 8, 64, 128, seed=tiles)
    else:
        _conv(tiles // 2, 16, 16, 64, 128, seed=tiles)


@pytest.mark.parametrize("NF,H,W,C,Cout,kernel", [
    (2, 64, 64, 64, 320, WS),     # one tile = two image rows
    (3, 32, 32, 128, 256, WS),    # four rows
    (5, 16, 16, 192, 136, WS),    # eight rows; ragged column tile
    (6, 8, 8, 128, 320, WS),      # two whole frames
    (5, 8, 8, 128, 320, WS),      # odd frame count: the last tile is one frame, its box's second frame past NF
    (8, 4, 4, 64, 128, WS),       # 16-pixel frames, eight per tile
    (3, 4, 4, 64, 128, WS),       # ... one ragged tile of three
    (7, 27, 29, 64, 128, OLD),    # width does not divide 128
    (4, 12, 32, 64, 128, WS),     # 384 = 3 tiles per frame
    (2, 12, 16, 64, 128, OLD),    # 192 pixels: 1.5 tiles per frame, 128 does not divide H W
])
def test_conv3x3_geometries(NF, H, W, C, Cout, kernel):
    _conv(NF, H, W, C, Cout, seed=NF * H * W + C, kernel=kernel)


def test_long_k():
    """K = 9 x 1280 = 11520 (180 K blocks) at the 8 x 8 level"""
    _conv(4, 8, 8, 1280, 256, seed=11)


def test_no_rowbias_no_residual():
    _conv(4, 16, 16, 64, 320, seed=12, rowbias=False, residual=False)


def test_three_slots():
    """PnP conv injection: one accumulator tile, each slot with its own residual, through the one staging tile in turn"""
    _conv(6, 16, 16, 128, 320, seed=13, slots=3)


def test_three_slots_without_residual():
    _conv(6, 16, 16, 128, 256, seed=14, slots=3, residual=False)


def test_residual_aliases_out():
    """out += conv(x) in place, over more tiles than the SMs hold at once"""
    _conv(2 * _sms() // 8 + 3, 32, 32, 64, 320, seed=15, alias=True)


def test_padded_channels():
    """a_channels = 8 of Cin = 64: the box reads 8 channels and TMA zero-fills the rest of each K block"""
    _conv(4, 32, 32, 8, 320, seed=16, Cin=64)


@pytest.mark.parametrize("NF,H,W,kernel", [(3, 16, 16, WS), (4, 8, 8, WS), (3, 8, 8, WS), (2, 12, 20, OLD)])
def test_upsample_phases(NF, H, W, kernel):
    """the four phases of nearest-up x 2 + conv 3 x 3, each a 2 x 2 conv with its own input offsets and output pixels"""
    from anyv2v_b200 import ops
    g = _gen(NF * H * W)
    Cin, Cout = 128, 192
    x = torch.randn(NF, H, W, Cin, generator=g).half()
    wph = ops.pack_upsample_weights((torch.randn(Cout, Cin, 3, 3, generator=g) * (9 * Cin) ** -0.5).half())
    bias = (torch.randn(Cout, generator=g) * 0.1).half()
    out = guarded_output((NF, 2 * H, 2 * W, Cout), device=dev)
    xg, wg, bg = gin(x).view, gin(wph).view, gin(bias).view
    ops.upsample2x_conv3x3(xg, wg, bias=bg, out=out.view)
    torch.cuda.synchronize()
    check_output(out, "upsample")
    assert _kernels(lambda: ops.upsample2x_conv3x3(xg, wg, bias=bg, out=torch.empty_like(out.view))) == {kernel}
    assert_within_bound(out.view.cpu(), kc.upsample2x_conv3x3_exact(x, wph, bias),
                        cond_conv_abs(kc.upsample2x_conv3x3_exact, x, wph, bias), KAPPA_GEMM, f"upsample {NF}x{H}x{W}",
                        shape=tuple(out.view.shape))


@pytest.mark.parametrize("B,F_,HW,kernel", [
    (1, 4, 4096, WS),   # 64 x 64: 32 tiles per frame
    (2, 5, 256, WS),    # 16 x 16: 2 tiles per frame, odd F
    (2, 6, 64, WS),     # 8 x 8: two frames per tile
    (2, 5, 64, OLD),    # 8 x 8, odd F: a tile would cross clips
    (2, 3, 400, OLD),   # 20 x 20
])
def test_tconv3(B, F_, HW, kernel):
    from anyv2v_b200 import ops
    g = _gen(B * F_ * HW)
    C, Cout = 128, 320
    x = torch.randn(B, F_ * HW, C, generator=g).half()
    w = _w(Cout, 3 * C, g)
    bias = (torch.randn(Cout, generator=g) * 0.1).half()
    res = torch.randn(B, F_ * HW, Cout, generator=g).half()
    out = guarded_output((B, F_ * HW, Cout), device=dev)
    xg, wg, bg, rg = gin(x).view, gin(w).view, gin(bias).view, gin(res).view
    ops.tconv3(xg, wg, F_, HW, bias=bg, residual=rg, out=out.view)
    torch.cuda.synchronize()
    check_output(out, "tconv3")
    assert _kernels(lambda: ops.tconv3(xg, wg, F_, HW, bias=bg, residual=rg, out=torch.empty_like(out.view))) == {kernel}
    ref = kc.tconv3_exact(x, w, F_, HW, bias, res).view(B, F_ * HW, Cout)
    cond = cond_conv_abs(kc.tconv3_exact, x, w, F_, HW, bias, res).view(B, F_ * HW, Cout)
    assert_within_bound(out.view.cpu(), ref, cond, KAPPA_GEMM, f"tconv3 B={B} F={F_} HW={HW}", shape=(B, F_ * HW, Cout))
