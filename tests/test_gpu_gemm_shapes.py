"""GPU tests of the GEMM (csrc/gemm_wgmma.cu: the conv modes, csrc/gemm_ws.cu: LINEAR) against the float64
contracts of tests/kernel_contracts.py, within ulp16(ref) + kappa * cond (tests/ulp_check.py), on guarded buffers
(tests/guarded.py).

Every A mode and epilogue at full and ragged column tiles (N = 320, 384, 136, 256), shapes with many more tiles than the
resident CTAs, K loops shorter and longer than the stage ring (K = 64, 320, 1280), ragged M, and the step's full-size
shapes checked on a seeded subset of rows / frames."""
import pytest
import torch

import kernel_contracts as kc
from guarded import check_output, guarded_input, guarded_output
from ulp_check import KAPPA_GEGLU, KAPPA_GEMM, assert_within_bound, cond_conv_abs, cond_geglu, cond_linear

pytestmark = pytest.mark.gpu
dev = "cuda"


def gin(t):
    return guarded_input(t, device=dev)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _check(got, ref, cond, kappa, what):
    assert_within_bound(got, ref, cond, kappa, what, shape=tuple(got.shape))


def _w(N, K, g):
    return (torch.randn(N, K, generator=g) * K ** -0.5).half()


# --------------------------------------------------------------------------------------------------- LINEAR
@pytest.mark.parametrize("N", [320, 384, 136])  # ragged last column tile; full tiles; ragged
@pytest.mark.parametrize("K", [64, 320, 1280])  # 1, 5 and 20 K blocks
def test_linear_epilogues(N, K):
    from anyv2v_b200 import ops
    g = _gen(N * 7 + K)
    M = 130 * 128 + 77  # 131 row tiles, a ragged last one
    a = torch.randn(M, K, generator=g).half()
    w = _w(N, K, g)
    kw = dict(bias=(torch.randn(N, generator=g) * 0.1).half(), rowbias=(torch.randn(M // 97 + 1, N, generator=g) * 0.5).half(),
              rows_per_rowbias=97, residual=torch.randn(M, N, generator=g).half())
    out = guarded_output((M, N), device=dev)
    ops.linear(gin(a).view, gin(w).view, **{k: gin(v).view if isinstance(v, torch.Tensor) else v for k, v in kw.items()},
               out=out.view)
    torch.cuda.synchronize()
    check_output(out, "linear")
    ref = kc.linear_exact(a, w, **kw)
    cond = cond_linear(a, w, kw["bias"], kw["rowbias"], 97, kw["residual"])
    _check(out.view.cpu(), ref, cond, KAPPA_GEMM, f"linear N={N} K={K}")


@pytest.mark.parametrize("N", [320, 256])
def test_linear_two_source(N):
    from anyv2v_b200 import ops
    g = _gen(N)
    M, K1, K2 = 9000, 640, 320
    a, a2 = torch.randn(M, K1, generator=g).half(), torch.randn(M, K2, generator=g).half()
    w = _w(N, K1 + K2, g)
    bias = (torch.randn(N, generator=g) * 0.1).half()
    out = guarded_output((M, N), device=dev)
    ops.linear(gin(a).view, gin(w).view, bias=gin(bias).view, a2=gin(a2).view, out=out.view)
    torch.cuda.synchronize()
    check_output(out, "linear two-source")
    _check(out.view.cpu(), kc.linear_exact(a, w, bias, a2=a2), cond_linear(a, w, bias, a2=a2), KAPPA_GEMM, f"linear two-source N={N}")


@pytest.mark.parametrize("M,N,K", [(40000 + 51, 2560, 320), (9000, 640, 1280)])
def test_geglu(M, N, K):
    from anyv2v_b200 import ops
    g = _gen(M + N)
    a = torch.randn(M, K, generator=g).half()
    wp, bp = kc.geglu_pack(_w(N, K, g), (torch.randn(N, generator=g) * 0.5).half())
    out = guarded_output((M, N // 2), device=dev)
    ops.linear(gin(a).view, gin(wp).view, bias=gin(bp).view, out=out.view, geglu=True)
    torch.cuda.synchronize()
    check_output(out, "geglu")
    _check(out.view.cpu(), kc.linear_exact(a, wp, bp, geglu=True), cond_geglu(a, wp, bp), KAPPA_GEGLU, f"geglu {M}x{N}x{K}")


# --------------------------------------------------------------------------------------------------- CONV3X3 / TCONV3
@pytest.mark.parametrize("Cout", [320, 256])
@pytest.mark.parametrize("case", ["residual", "slots3", "stride2", "padded_channels", "ragged"])
def test_conv3x3(case, Cout):
    from anyv2v_b200 import ops
    g = _gen(len(case) * 1000 + Cout)
    NF, H, W, C = 12, 32, 32, 128
    stride = 2 if case == "stride2" else 1
    if case == "padded_channels":
        C = 8
    if case == "ragged":
        NF, H, W = 7, 27, 29  # M = 5481: a ragged last row tile, rows crossing frames
    Cin = 64 if C == 8 else C
    x = torch.randn(NF, H, W, C, generator=g).half()
    wfull = _w(Cout, 9 * Cin, g)
    if C != Cin:  # weights of the missing channels are zero (ops pads them so)
        wfull = wfull.view(Cout, 9, Cin)
        wfull[:, :, C:] = 0
        wfull = wfull.reshape(Cout, 9 * Cin).contiguous()
    bias = (torch.randn(Cout, generator=g) * 0.1).half()
    M = NF * (H // stride) * (W // stride)
    rowbias = (torch.randn(NF, Cout, generator=g) * 0.25).half()
    ns = 3 if case == "slots3" else 1
    shape = (ns, M, Cout) if ns > 1 else (M, Cout)
    res = torch.randn(shape, generator=g).half()
    out = guarded_output(shape, device=dev)
    ops.conv3x3(gin(x).view, gin(wfull).view, bias=gin(bias).view, rowbias=gin(rowbias).view, rows_per_rowbias=M // NF,
                residual=gin(res).view, out=out.view, n_slots=ns, slot_stride=M * Cout, stride=stride)
    torch.cuda.synchronize()
    check_output(out, f"conv3x3 {case}")
    xp = x if C == Cin else torch.cat([x, torch.zeros(NF, H, W, Cin - C, dtype=x.dtype)], dim=3)
    acc = kc.conv3x3_exact(xp, wfull, bias, rowbias, M // NF, stride)
    cond = cond_conv_abs(kc.conv3x3_exact, xp, wfull, bias, rowbias, M // NF, stride) + res.double().abs()
    _check(out.view.cpu(), acc + res.double(), cond, KAPPA_GEMM, f"conv3x3 {case} Cout={Cout}")


@pytest.mark.parametrize("Cout", [320, 256])
def test_upsample_phases(Cout):
    from anyv2v_b200 import ops
    g = _gen(Cout + 3)
    NF, H, W, Cin = 12, 16, 16, 320
    x = torch.randn(NF, H, W, Cin, generator=g).half()
    wph = ops.pack_upsample_weights((torch.randn(Cout, Cin, 3, 3, generator=g) * (9 * Cin) ** -0.5).half())
    bias = (torch.randn(Cout, generator=g) * 0.1).half()
    out = guarded_output((NF, 2 * H, 2 * W, Cout), device=dev)
    ops.upsample2x_conv3x3(gin(x).view, gin(wph).view, bias=gin(bias).view, out=out.view)
    torch.cuda.synchronize()
    check_output(out, "upsample")
    _check(out.view.cpu(), kc.upsample2x_conv3x3_exact(x, wph, bias), cond_conv_abs(kc.upsample2x_conv3x3_exact, x, wph, bias),
           KAPPA_GEMM, f"upsample Cout={Cout}")


@pytest.mark.parametrize("Cout", [320, 256])
def test_tconv3(Cout):
    from anyv2v_b200 import ops
    g = _gen(Cout + 5)
    B, F_, HW, C = 3, 16, 400, 192
    x = torch.randn(B, F_ * HW, C, generator=g).half()
    w = _w(Cout, 3 * C, g)
    bias = (torch.randn(Cout, generator=g) * 0.1).half()
    res = torch.randn(B, F_ * HW, Cout, generator=g).half()
    out = guarded_output((B, F_ * HW, Cout), device=dev)
    ops.tconv3(gin(x).view, gin(w).view, F_, HW, bias=gin(bias).view, residual=gin(res).view, out=out.view)
    torch.cuda.synchronize()
    check_output(out, "tconv3")
    ref = kc.tconv3_exact(x, w, F_, HW, bias, res).view(B, F_ * HW, Cout)
    cond = cond_conv_abs(kc.tconv3_exact, x, w, F_, HW, bias, res).view(B, F_ * HW, Cout)
    _check(out.view.cpu(), ref, cond, KAPPA_GEMM, f"tconv3 Cout={Cout}")


# --------------------------------------------------------------------------------------------------- full-size step shapes
def test_full_size_geglu_rows():
    """196608 x 2560 x 320 GEGLU of an edit step, checked on 4096 seeded rows"""
    from anyv2v_b200 import ops
    g = _gen(196608)
    M, N, K = 196608, 2560, 320
    a = torch.randn(M, K, generator=g).half()
    wp, bp = kc.geglu_pack(_w(N, K, g), (torch.randn(N, generator=g) * 0.5).half())
    out = ops.linear(a.to(dev), wp.to(dev), bias=bp.to(dev), geglu=True)
    torch.cuda.synchronize()
    rows = torch.randperm(M, generator=g)[:4096]
    ar = a[rows]
    _check(out[rows.to(dev)].cpu(), kc.linear_exact(ar, wp, bp, geglu=True), cond_geglu(ar, wp, bp), KAPPA_GEGLU, "geglu full size")


@pytest.mark.parametrize("NF,H,W,C,Cout", [(48, 64, 64, 320, 320), (48, 16, 16, 1280, 1280)])
def test_full_size_conv_residual_frames(NF, H, W, C, Cout):
    """196608 x 320 x 2880 and 12288 x 1280 x 11520 conv + residual, checked on two seeded frames (the conv is per frame)"""
    from anyv2v_b200 import ops
    g = _gen(NF * H * C)
    x = torch.randn(NF, H, W, C, generator=g).half()
    w = _w(Cout, 9 * C, g)
    bias = (torch.randn(Cout, generator=g) * 0.1).half()
    res = torch.randn(NF, H, W, Cout, generator=g).half()
    out = torch.empty(NF * H * W, Cout, device=dev, dtype=torch.float16)
    ops.conv3x3(x.to(dev), w.to(dev), bias=bias.to(dev), residual=res.to(dev).view(-1, Cout), out=out)
    torch.cuda.synchronize()
    frames = torch.randperm(NF, generator=g)[:2]
    xf, rf = x[frames], res[frames]
    acc = kc.conv3x3_exact(xf, w, bias).reshape(2, H, W, Cout)
    cond = cond_conv_abs(kc.conv3x3_exact, xf, w, bias).reshape(2, H, W, Cout) + rf.double().abs()
    _check(out.view(NF, H, W, Cout)[frames.to(dev)].cpu(), acc + rf.double(), cond, KAPPA_GEMM, f"conv3x3 full size C={C}")
