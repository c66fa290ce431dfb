"""CPU tests of tests/ulp_check.py: the bound itself at its edges (inf, subnormals, NaN), and its power to catch the faults
it is there for.  Each fault is restated in numpy fp32, in the order of operations of the kernel it models; the correct
restatement must pass the bound and the faulty one (one intermediate rounded to fp16, an absolute-error erf, unshifted
variance sums) must fail it."""
import math

import numpy as np
import pytest
import torch

import kernel_contracts as kc
from ulp_check import (KAPPA_FREEU, KAPPA_GEGLU, KAPPA_GEMM, KAPPA_NORM, assert_within_bound, cond_freeu, cond_layernorm,
                       cond_linear, measure, ulp16)

f32 = np.float32


def _fails(got, ref, cond, kappa):
    with pytest.raises(AssertionError, match="over the bound"):
        assert_within_bound(got, ref, cond, kappa, "negative control")


# ------------------------------------------------------------------------------------------------------------- the bound
def test_ulp16_spacing():
    ref = torch.tensor([1.0, 1.5, 2.0, 0.999, 65504.0, 2.0 ** -14, 2.0 ** -20, 0.0, -3.0], dtype=torch.float64)
    want = [2.0 ** -10, 2.0 ** -10, 2.0 ** -9, 2.0 ** -11, 32.0, 2.0 ** -24, 2.0 ** -24, 2.0 ** -24, 2.0 ** -9]
    assert ulp16(ref).tolist() == want
    # the spacing is the distance to the next fp16 value at every exponent
    h = torch.tensor([2.0 ** e for e in range(-14, 16)], dtype=torch.float16)
    nxt = (h.view(torch.int16) + 1).view(torch.float16)
    assert torch.equal(ulp16(h.double()), (nxt.double() - h.double()))


def test_correct_rounding_passes_everywhere():
    ref = torch.cat([torch.randn(10000, dtype=torch.float64) * 10.0 ** torch.randint(-9, 5, (10000,)),
                     torch.tensor([65519.9, -65519.9, 2.0 ** -25, -(2.0 ** -25), 0.0])])
    assert_within_bound(ref.to(torch.float16), ref, torch.zeros(()), 0.0, "rounded reference")


def test_overflow_boundary():
    ref = torch.tensor([65519.0, 65520.0, -65520.0, 7.0e4, -7.0e4], dtype=torch.float64)
    got = ref.to(torch.float16)
    assert torch.isinf(got[1:]).all() and got[0] == 65504.0
    assert_within_bound(got, ref, torch.zeros(()), 0.0, "overflow")
    for i, wrong in ((1, 65504.0), (2, -65504.0), (3, -math.inf), (0, math.inf)):
        bad = got.clone()
        bad[i] = wrong
        _fails(bad, ref, torch.zeros(()), 0.0)


def test_subnormal_reference():
    ref = torch.tensor([3.1e-8, 2.0 ** -24 * 5.4, -1.0e-6, 2.0 ** -15], dtype=torch.float64)
    got = ref.to(torch.float16)
    assert_within_bound(got, ref, torch.zeros(()), 0.0, "subnormal")
    off = (got.view(torch.int16) + 2).view(torch.float16)  # two subnormal steps away: more than one spacing of 2^-24
    _fails(off, ref, torch.zeros(()), 0.0)
    # a cond term admits it
    assert_within_bound(off, ref, torch.full((4,), 2.0 ** -22), 1.0, "subnormal with cond")


def test_nan_always_fails():
    ref = torch.ones(5, dtype=torch.float64)
    got = ref.to(torch.float16)
    got[3] = float("nan")
    _fails(got, ref, torch.full((5,), 1e30), 1.0)
    _fails(got, torch.full((5,), 1e6, dtype=torch.float64), torch.zeros(()), 0.0)  # also where ref overflows


def test_message_names_worst_element():
    ref = torch.linspace(1, 2, 12, dtype=torch.float64).view(3, 4)
    got = ref.to(torch.float16)
    got[2, 1] += 0.25
    with pytest.raises(AssertionError) as e:
        assert_within_bound(got, ref, torch.zeros(()), 0.0, "msg", shape=(3, 4))
    msg = str(e.value)
    assert "(2, 1)" in msg and "1 of 12 elements" in msg and "ulp" in msg


# ------------------------------------------------------------------------------------------------------------- GEMM
def _scaled_operands(M=256, N=192, K=1280, seed=0):
    """A rows and W output channels scaled by 2^-12 ... 2^4, bias on a third scale: magnitudes that differ by row and column"""
    g = torch.Generator().manual_seed(seed)
    rs = 2.0 ** torch.randint(-12, 5, (M, 1), generator=g)
    cs = 2.0 ** torch.randint(-12, 5, (N, 1), generator=g)
    a = (torch.randn(M, K, generator=g) * rs).half()
    w = (torch.randn(N, K, generator=g) * cs * K ** -0.5).half()
    bias = (torch.randn(N, generator=g) * 2.0 ** -6).half()
    return a, w, bias


def _gemm_fp32(a, w, bias, round_partial):
    """fp32 accumulation in K blocks of 64 (products of fp16 values are exact in fp32), fp32 epilogue; round_partial: the
    accumulator rounded to fp16 after every block"""
    an, wn = a.numpy().astype(f32), w.numpy().astype(f32)
    acc = np.zeros((a.shape[0], w.shape[0]), f32)
    for k0 in range(0, a.shape[1], 64):
        acc = (acc + an[:, k0:k0 + 64].astype(np.float64) @ wn[:, k0:k0 + 64].T.astype(np.float64)).astype(f32)
        if round_partial:
            acc = acc.astype(np.float16).astype(f32)
    return torch.from_numpy((acc + bias.numpy().astype(f32)).astype(np.float16))


def test_gemm_fp32_k_blocks_pass():
    a, w, bias = _scaled_operands()
    ref = kc.linear_exact(a, w, bias)
    assert_within_bound(_gemm_fp32(a, w, bias, False), ref, cond_linear(a, w, bias), KAPPA_GEMM, "gemm fp32")


def test_gemm_fp16_partial_sums_fail():
    a, w, bias = _scaled_operands()
    ref = kc.linear_exact(a, w, bias)
    _fails(_gemm_fp32(a, w, bias, True), ref, cond_linear(a, w, bias), KAPPA_GEMM)


# ------------------------------------------------------------------------------------------------------------- GEGLU
def _rcp(x):
    return (f32(1.0) / x).astype(f32)


def _ex2(x):
    return np.exp2(x.astype(f32)).astype(f32)


def gelu_as7125(g):
    """the GEGLU epilogue's gelu before the fix: erf from Abramowitz & Stegun 7.1.25 (absolute error 2.5e-5)"""
    g = g.astype(f32)
    u = (np.abs(g) * f32(0.70710678118654752)).astype(f32)
    t = _rcp((f32(0.47047) * u + f32(1.0)).astype(f32))
    poly = (t * f32(0.7478556) + f32(-0.0958798)).astype(f32)
    poly = (poly * t + f32(0.3480242)).astype(f32)
    poly = (poly * t).astype(f32)
    e = _ex2((u * u * f32(-1.4426950408889634)).astype(f32))
    erf_abs = (f32(1.0) - poly * e).astype(f32)
    hg = (f32(0.5) * g).astype(f32)
    return (np.abs(hg) * erf_abs + hg).astype(f32)


def gelu_erfcc(g):
    """the GEGLU epilogue's gelu: gelu = max(g, 0) - |g/2| * erfc(|g| / sqrt 2), erfc = t exp(-z^2 + P5(t)), t = 1 / (1 + z/2)
    (the form of Numerical Recipes' erfcc, P5 from tools/erfc_poly_fit.py)"""
    g = g.astype(f32)
    z = (np.abs(g) * f32(0.70710678118654752)).astype(f32)
    t = _rcp((f32(0.5) * z + f32(1.0)).astype(f32))
    p = (t * f32(0.22427836) + f32(-0.69402432)).astype(f32)
    for c in (0.45475456, 0.26681793, 1.01429605, -1.26611602):
        p = (p * t + f32(c)).astype(f32)
    e = (t * _ex2(((-z * z).astype(np.float64) + p).astype(f32) * f32(1.4426950408889634))).astype(f32)
    return (np.maximum(g, f32(0)) - np.abs(f32(0.5) * g) * e).astype(f32)


def _gelu64(g):
    g = torch.as_tensor(g, dtype=torch.float64)
    return 0.5 * g * torch.erfc(-g / math.sqrt(2))


def _gates(lo, hi):
    return np.linspace(lo, hi, 20001, dtype=np.float64).astype(np.float16).astype(f32)  # fp16 gates, as the GEMM sees sums


@pytest.mark.parametrize("lo,hi", [(-4.0, -3.0), (-3.0, -2.0)])
def test_gelu_abs_error_erf_fails(lo, hi):
    g = _gates(lo, hi)
    _fails(torch.from_numpy(gelu_as7125(g).astype(np.float16)), _gelu64(g), torch.zeros(()), KAPPA_GEGLU)


@pytest.mark.parametrize("lo,hi", [(-9.0, -4.0), (-4.0, -2.0), (-2.0, 0.0), (0.0, 9.0)])
def test_gelu_erfcc_passes(lo, hi):
    g = _gates(lo, hi)
    for h in (1.0, -7.5, 100.0):
        got = torch.from_numpy((f32(h) * gelu_erfcc(g)).astype(np.float16))
        assert_within_bound(got, h * _gelu64(g), torch.zeros(()), KAPPA_GEGLU, f"gelu erfcc, h = {h}, gates [{lo}, {hi}]")


# ------------------------------------------------------------------------------------------------------------- LayerNorm
def _layernorm_fp32(x, gamma, beta, eps, round_mean):
    """the two-pass LayerNorm kernel: fp32 sum -> mean, centred fp32 sum of squares -> rstd, (x - mean) * rstd * g + b"""
    xn = x.numpy().astype(f32)
    C = xn.shape[-1]
    mean = (np.cumsum(xn, axis=-1, dtype=f32)[:, -1:] * f32(1.0 / C)).astype(f32)
    if round_mean:
        mean = mean.astype(np.float16).astype(f32)
    d = (xn - mean).astype(f32)
    q = np.cumsum((d * d).astype(f32), axis=-1, dtype=f32)[:, -1:]
    rstd = (f32(1.0) / np.sqrt((q * f32(1.0 / C) + f32(eps)).astype(f32))).astype(f32)
    y = ((d * rstd).astype(f32) * gamma.numpy().astype(f32) + beta.numpy().astype(f32)).astype(f32)
    return torch.from_numpy(y.astype(np.float16))


def _ln_inputs(C, offset, seed=0):
    g = torch.Generator().manual_seed(seed)
    rows = 64
    mu = offset * (torch.rand(rows, 1, generator=g) * 2 - 1).sign()
    x = (torch.randn(rows, C, generator=g) + mu).half()
    return x, (torch.randn(C, generator=g) * 0.2 + 1).half(), (torch.randn(C, generator=g) * 0.2).half()


@pytest.mark.parametrize("offset", [0.0, 30.0, 300.0])
def test_layernorm_fp32_passes(offset):
    x, gm, bt = _ln_inputs(1280, offset)
    assert_within_bound(_layernorm_fp32(x, gm, bt, 1e-5, False), kc.layernorm_exact(x, gm, bt, 1e-5),
                        cond_layernorm(x, gm, bt, 1e-5), KAPPA_NORM, f"layernorm fp32, offset {offset}")


def test_layernorm_fp16_mean_fails():
    x, gm, bt = _ln_inputs(1280, 30.0)
    _fails(_layernorm_fp32(x, gm, bt, 1e-5, True), kc.layernorm_exact(x, gm, bt, 1e-5), cond_layernorm(x, gm, bt, 1e-5),
           KAPPA_NORM)


# ------------------------------------------------------------------------------------------------------------- GroupNorm
def _groupnorm_fp32(x, gamma, beta, groups, eps, shifted, lanes=16):
    """the statistics and affine map of csrc/groupnorm.cu for ONE sample [rows, C]: per-thread sequential fp32 sums over the
    rows of each of `lanes` row lanes, an fp32 fold over the lanes and then over the channels of a group, then in double
    mean / var; shifted: sums of x - k with k = the group's first channel in row 0 (the kernel), else of x (before the fix,
    var = E[x^2] - mean^2).  Then a = rstd * gamma, b = beta - mean * a in fp32 and y = fma(x, a, b)."""
    xn = x.numpy().astype(f32)
    rows, C = xn.shape
    cpg = C // groups
    k = np.repeat(xn[0, ::cpg], cpg) if shifted else np.zeros(C, f32)
    d = (xn - k).astype(f32)
    lane = d.reshape(rows // lanes, lanes, C)
    s1 = np.cumsum(lane, axis=0, dtype=f32)[-1]                           # [lanes, C]
    s2 = np.cumsum((lane * lane).astype(f32), axis=0, dtype=f32)[-1]      # fma(d, d, s) rounds once; d*d exact in fp32 here
    s1 = np.cumsum(s1, axis=0, dtype=f32)[-1].reshape(groups, cpg)        # fold over lanes
    s2 = np.cumsum(s2, axis=0, dtype=f32)[-1].reshape(groups, cpg)
    s1 = np.cumsum(s1, axis=1, dtype=f32)[:, -1].astype(np.float64)       # fold over the channels of a group
    s2 = np.cumsum(s2, axis=1, dtype=f32)[:, -1].astype(np.float64)
    cnt = float(rows * cpg)
    d1 = s1 / cnt
    mean = k[::cpg].astype(np.float64) + d1
    var = np.maximum(s2 / cnt - d1 * d1, 0.0)
    mean32 = np.repeat(mean.astype(f32), cpg)
    rstd32 = np.repeat((1.0 / np.sqrt(var + np.float64(f32(eps)))).astype(f32), cpg)
    a = (rstd32 * gamma.numpy().astype(f32)).astype(f32)
    b = (beta.numpy().astype(f32) - (mean32 * a).astype(f32)).astype(f32)
    y = (xn.astype(np.float64) * a + b).astype(f32)                       # fma: x * a is exact in double
    return torch.from_numpy(y.astype(np.float16))


def _gn_inputs(ratio, rows=4096, C=320, groups=32, seed=0):
    """one sample, every group with its own mean of |mean| / sigma = ratio (sigma = 1)"""
    g = torch.Generator().manual_seed(seed)
    sign = torch.where(torch.rand(groups, generator=g) < 0.5, -1.0, 1.0)
    mu = (ratio * sign * (1 + 0.1 * torch.rand(groups, generator=g))).repeat_interleave(C // groups)
    x = (torch.randn(rows, C, generator=g) + mu).half()
    return x, (torch.randn(C, generator=g) * 0.2 + 1).half(), (torch.randn(C, generator=g) * 0.2).half()


def _gn_check(x, gm, bt, shifted, what):
    ref = kc.groupnorm_exact(x[None], gm, bt, 32, 1e-5, False)[0]
    from ulp_check import cond_groupnorm
    cond = cond_groupnorm(x[None], gm, bt, 32, 1e-5, False)[0]
    return assert_within_bound(_groupnorm_fp32(x, gm, bt, 32, 1e-5, shifted), ref, cond, KAPPA_NORM, what)


def test_groupnorm_unshifted_sums_fail():
    x, gm, bt = _gn_inputs(300.0)
    with pytest.raises(AssertionError, match="over the bound"):
        _gn_check(x, gm, bt, False, "groupnorm E[x^2] - mean^2, |mean| / sigma = 300")


@pytest.mark.parametrize("ratio", [0.0, 30.0, 300.0, 1000.0])
def test_groupnorm_shifted_sums_pass(ratio):
    x, gm, bt = _gn_inputs(ratio)
    _gn_check(x, gm, bt, True, f"groupnorm shifted sums, |mean| / sigma = {ratio}")


# ------------------------------------------------------------------------------------------------------------- FreeU
def _freeu_filter(x, s, fp16_sums):
    """csrc/freeu.cu's filtered skip of one channels-last plane x[H, W, C]: seven plane sums of x * t over the H W pixels,
    accumulated one pixel after the other (fp32, or fp16 with fp16_sums), twiddles t = cos / sin of th_h, ph_w, th_h + ph_w
    rounded to fp32, then y = fp16(x + sum_j ((s - 1) / (H W) * S_j) * t_j)"""
    H, W, C = x.shape
    th = 2 * np.pi * np.arange(H)[:, None] / H + 0 * np.arange(W)[None, :]
    ph = 0 * np.arange(H)[:, None] + 2 * np.pi * np.arange(W)[None, :] / W
    t = [np.ones((H, W))] + [fn(a) for a in (th, ph, th + ph) for fn in (np.cos, np.sin)]
    t = [tj.reshape(H * W, 1).astype(f32) for tj in t]
    xs = x.numpy().astype(f32).reshape(H * W, C)
    acc = np.float16 if fp16_sums else f32
    k = f32(f32(s) - f32(1.0)) / f32(H * W)
    corr = np.zeros((H * W, C), f32)
    for tj in t:
        S = np.cumsum((xs * tj).astype(acc), axis=0, dtype=acc)[-1].astype(f32)
        corr = (corr + (k * S).astype(f32) * tj).astype(f32)
    return torch.from_numpy((xs + corr).astype(np.float16).reshape(H, W, C))


def _freeu_plane(seed=0, H=32, W=32, C=64):
    """planes with a per-channel offset of 2 +- 1, so the mode-0 sums are large: 2 H W"""
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(H, W, C, generator=g) + 2 + torch.rand(1, 1, C, generator=g) * 2 - 1).half()


@pytest.mark.parametrize("s", [0.2, 0.9, 1.6])
def test_freeu_fp32_plane_sums_pass(s):
    import freeu_ref
    x = _freeu_plane()
    ref = freeu_ref.fourier_filter_closed_form(x.double(), float(f32(s)))
    assert_within_bound(_freeu_filter(x, s, False), ref, cond_freeu(x, s), KAPPA_FREEU, f"freeu fp32 plane sums, s = {s}")


def test_freeu_fp16_plane_sums_fail():
    import freeu_ref
    x = _freeu_plane()
    ref = freeu_ref.fourier_filter_closed_form(x.double(), float(f32(0.2)))
    _fails(_freeu_filter(x, 0.2, True), ref, cond_freeu(x, 0.2), KAPPA_FREEU)


def test_measure_reports_margin():
    ref = torch.tensor([1.0, 2.0], dtype=torch.float64)
    m = measure(ref.half(), ref, torch.zeros(()), 0.0)
    assert m["n_bad"] == 0 and m["err_ulp"] == 0.0 and m["over_rel"] == -1.0
