"""GPU tests of the kernels' MEAN error: every kernel family that stores fp16 through its own rounding, at model shapes,
against its float64 contract with tests/bias_check.py.  The element-wise bound of tests/test_gpu_numerics.py grants each
element a full ulp, so a store that rounds in one direction passes it; here the mean of (got - ref) / ulp16(ref), and of
sign(ref) times it, pooled and per output channel, must stay within 1/16 ulp (1/8 per channel) with the power to see that.

Each case runs the ``ops`` wrapper on guarded CUDA buffers (tests/guarded.py), evaluates the ``kernel_contracts`` ``*_exact``
function and the ``cond_*`` scale of tests/ulp_check.py in float64 on the GPU, and compares at least 2^20 elements.  With -s
it prints both statistics, their standard errors, n, the excluded fraction and the worst channel.  Attention cases give V a
common offset per channel: over a diffuse softmax the output of zero-mean V is close to 0, where the arithmetic bound
exceeds the store's ulp and almost every element would be excluded.  The DDIM steps and FreeU's backbone scaling are not
here: they are compared bit for bit elsewhere."""
import pytest
import torch

import freeu_ref
import kernel_contracts as kc
from bias_check import assert_unbiased
from guarded import check_output, guarded_inout, guarded_input, guarded_output
from test_gpu_numerics import _affine, _gn_input, _pow2, _scaled_image, _scaled_linear
from ulp_check import (KAPPA_ATTN, KAPPA_FREEU, KAPPA_GEGLU, KAPPA_GEMM, KAPPA_NORM, cond_attention, cond_conv_abs, cond_freeu,
                       cond_geglu, cond_groupnorm, cond_layernorm, cond_linear)

pytestmark = pytest.mark.gpu
dev = "cuda"
MIN_ELEMENTS = 1 << 20


def gin(t, ld=None):
    return guarded_input(t, ld=ld, device=dev)


def gout(shape, ld=None):
    return guarded_output(shape, ld=ld, device=dev)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _d(t):
    """the CUDA copy the float64 contract is evaluated on"""
    return None if t is None else t.to(dev)


def _check(out, ref, cond, kappa, what):
    check_output(out, what)
    got = out.view
    assert got.numel() >= MIN_ELEMENTS, f"{what}: {got.numel()} elements compared, at least {MIN_ELEMENTS}"
    assert_unbiased(got, ref, cond, kappa, what)


# ------------------------------------------------------------------------------------------------------------- linear
@pytest.mark.parametrize("case", ["plain", "bias_rowbias_residual", "two_source"])
def test_linear(case):
    from anyv2v_b200 import ops
    g = _gen(101 + len(case))
    M, N, K = 4096, 640, 1280
    a, w = _scaled_linear(M, N, K, g)
    kw = dict(bias=(torch.randn(N, generator=g) * 2.0 ** -6).half())
    if case == "bias_rowbias_residual":
        kw.update(rowbias=(torch.randn(M // 256, N, generator=g) * 0.5).half(), rows_per_rowbias=256,
                  residual=(torch.randn(M, N, generator=g, dtype=torch.float64) * _pow2(M, g, -8, 2)[:, None]).half())
    a2 = None
    if case == "two_source":  # the K loop switches source at 640
        a, a2 = a[:, :640].contiguous(), a[:, 640:].contiguous()
    out = gout((M, N))
    ops.linear(gin(a).view, gin(w).view, **{k: gin(v).view if isinstance(v, torch.Tensor) else v for k, v in kw.items()},
               a2=None if a2 is None else gin(a2).view, out=out.view)
    torch.cuda.synchronize()
    kd = {k: _d(v) if isinstance(v, torch.Tensor) else v for k, v in kw.items()}
    ref = kc.linear_exact(_d(a), _d(w), a2=_d(a2), **kd)
    cond = cond_linear(_d(a), _d(w), kd.get("bias"), kd.get("rowbias"), kd.get("rows_per_rowbias", 0), kd.get("residual"), a2=_d(a2))
    _check(out, ref, cond, KAPPA_GEMM, f"linear {case} {M}x{N}x{K}")


def test_linear_geglu():
    """the feed-forward GEGLU of the 64 x 64 level: 16384 tokens, 320 -> 2 x 1280; gates N(0, 1.1), as the model's are"""
    from anyv2v_b200 import ops
    g = _gen(111)
    M, N, K = 16384, 2560, 320
    a = torch.randn(M, K, generator=g).half()
    w = (torch.randn(N, K, generator=g) * K ** -0.5).half()
    bias = (torch.randn(N, generator=g) * 0.5).half()
    wp, bp = kc.geglu_pack(w, bias)
    out = gout((M, N // 2))
    ops.linear(gin(a).view, gin(wp).view, bias=gin(bp).view, out=out.view, geglu=True)
    torch.cuda.synchronize()
    ref = kc.linear_exact(_d(a), _d(wp), _d(bp), geglu=True)
    _check(out, ref, cond_geglu(_d(a), _d(wp), _d(bp)), KAPPA_GEGLU, f"linear geglu {M}x{N}x{K}")


# ------------------------------------------------------------------------------------------------------------- conv
@pytest.mark.parametrize("case", ["stride1_residual", "stride2", "slots3", "padded_channels"])
def test_conv3x3(case):
    from anyv2v_b200 import ops
    g = _gen(121 + len(case))
    NF, H, W, C, Cout, Cin = 4, 32, 32, 320, 320, 320
    stride = 2 if case == "stride2" else 1
    if case == "stride2":
        H = W = 64
    if case == "padded_channels":  # 8 channels present in a 64-wide K block (the VAE's first conv, padded)
        NF, H, W, C, Cin, Cout = 16, 64, 64, 8, 64, 64
    x = _scaled_image(NF, H, W, C, g)
    w = (torch.randn(Cout, 9 * Cin, generator=g, dtype=torch.float64) * _pow2(Cout, g)[:, None] * (9 * C) ** -0.5).half()
    bias = (torch.randn(Cout, generator=g) * 2.0 ** -6).half()
    M = NF * (H // stride) * (W // stride)
    ns = 3 if case == "slots3" else 1
    res = None
    if case in ("stride1_residual", "slots3"):
        res = (torch.randn(ns, M, Cout, generator=g, dtype=torch.float64) * _pow2(M, g, -8, 2)[None, :, None]).half()
        res = res[0] if ns == 1 else res
    out = gout((ns, M, Cout) if ns > 1 else (M, Cout))
    ops.conv3x3(gin(x).view, gin(w).view, bias=gin(bias).view, residual=None if res is None else gin(res).view, out=out.view,
                n_slots=ns, slot_stride=M * Cout, stride=stride)
    torch.cuda.synchronize()
    ref = kc.conv3x3_exact(_d(x), _d(w), _d(bias), stride=stride)
    cond = cond_conv_abs(kc.conv3x3_exact, _d(x), _d(w), _d(bias), stride=stride)
    if res is not None:
        ref, cond = ref + _d(res).double(), cond + _d(res).double().abs()
    _check(out, ref, cond, KAPPA_GEMM, f"conv3x3 {case} NF={NF} {H}x{W} C={C} Cout={Cout}")


def test_upsample2x_conv3x3():
    from anyv2v_b200 import ops
    g = _gen(131)
    NF, H, W, Cin, Cout = 4, 16, 16, 640, 320
    x = _scaled_image(NF, H, W, Cin, g)
    wfull = torch.randn(Cout, Cin, 3, 3, generator=g, dtype=torch.float64) * (9 * Cin) ** -0.5
    wph = ops.pack_upsample_weights(wfull.half())
    bias = (torch.randn(Cout, generator=g) * 2.0 ** -6).half()
    out = gout((NF, 2 * H, 2 * W, Cout))
    ops.upsample2x_conv3x3(gin(x).view, gin(wph).view, bias=gin(bias).view, out=out.view)
    torch.cuda.synchronize()
    args = (_d(x), _d(wph), _d(bias))
    _check(out, kc.upsample2x_conv3x3_exact(*args), cond_conv_abs(kc.upsample2x_conv3x3_exact, *args), KAPPA_GEMM,
           f"upsample2x_conv3x3 NF={NF} {H}x{W} Cin={Cin} Cout={Cout}")


def test_tconv3():
    from anyv2v_b200 import ops
    g = _gen(141)
    B, F_, HW, C = 2, 16, 1024, 320
    x = _scaled_image(B, F_, HW, C, g).view(B, F_ * HW, C)
    w = (torch.randn(C, 3 * C, generator=g, dtype=torch.float64) * (3 * C) ** -0.5).half()
    bias = (torch.randn(C, generator=g) * 2.0 ** -6).half()
    res = (torch.randn(B, F_ * HW, C, generator=g) * 0.1).half()
    out = gout((B, F_ * HW, C))
    ops.tconv3(gin(x).view, gin(w).view, F_, HW, bias=gin(bias).view, residual=gin(res).view, out=out.view)
    torch.cuda.synchronize()
    args = (_d(x), _d(w), F_, HW, _d(bias), _d(res))
    _check(out, kc.tconv3_exact(*args).view(B, F_ * HW, C), cond_conv_abs(kc.tconv3_exact, *args).view(B, F_ * HW, C),
           KAPPA_GEMM, f"tconv3 B={B} F={F_} HW={HW} C={C}")


# ------------------------------------------------------------------------------------------------------------- norms
def _gn_run(x, gamma, beta, groups, eps, silu, what, x2=None):
    from anyv2v_b200 import ops
    n, rows = x.shape[:2]
    C = x.shape[2] + (0 if x2 is None else x2.shape[2])
    out = gout((n, rows, C))
    ops.groupnorm(gin(x).view, gin(gamma).view, gin(beta).view, groups, eps, silu, out=out.view,
                  x2=None if x2 is None else gin(x2).view)
    torch.cuda.synchronize()
    args = (_d(x), _d(gamma), _d(beta), groups, eps, silu)
    ref = kc.groupnorm_exact(*args, x2=_d(x2))
    _check(out, ref, cond_groupnorm(*args, x2=_d(x2)), KAPPA_NORM, what)


# No constant groups here (test_gpu_numerics.py has them): every row of a constant group is the same value, so a column of
# one holds one error repeated, not a sample of the rounding.  At sigma = 0 the kernel's y = x a + (beta - mean a) rounds
# beta - mean a with |mean a| = |mean| |gamma| / sqrt(eps) ~ 1e3, up to 1.5 ulp16 off beta (inside the element-wise bound,
# whose cond_norm holds that term), and the same in all 65536 rows of the per-clip sample.
@pytest.mark.parametrize("ratio,silu", [(0.0, False), (0.0, True), (300.0, False), (300.0, True)])
def test_groupnorm_per_frame(ratio, silu):
    """48 samples of 1024 x 320, 32 groups, |mean| / sigma = ratio"""
    g = _gen(151 + int(ratio) + silu)
    x = _gn_input(48, 1024, 320, 32, ratio, g, const_groups=0)
    gamma, beta = _affine(320, g)
    _gn_run(x, gamma, beta, 32, 1e-5, silu, f"groupnorm 48x1024x320 |mean|/sigma={ratio} silu={silu}")


def test_groupnorm_per_clip():
    g = _gen(161)
    x = _gn_input(1, 65536, 320, 32, 0.0, g, const_groups=0)
    gamma, beta = _affine(320, g)
    _gn_run(x, gamma, beta, 32, 1e-5, True, "groupnorm 1x65536x320 silu")


def test_groupnorm_two_source():
    """the up-block concat, 640 + 320 channels (group 21 straddles the sources)"""
    g = _gen(171)
    x = _gn_input(16, 1024, 640, 32, 0.0, g, const_groups=0)
    x2 = _gn_input(16, 1024, 320, 16, 0.0, g, const_groups=0)
    gamma, beta = _affine(960, g)
    _gn_run(x, gamma, beta, 32, 1e-5, True, "groupnorm two-source 16x1024x(640+320) silu", x2=x2)


@pytest.mark.parametrize("rows,C,ratio", [(65536, 320, 0.0), (16384, 1280, 30.0)])
def test_layernorm(rows, C, ratio):
    from anyv2v_b200 import ops
    g = _gen(181 + C)
    sign = torch.where(torch.rand(rows, 1, generator=g) < 0.5, -1.0, 1.0)
    x = (torch.randn(rows, C, generator=g) + ratio * sign * (1 + 0.1 * torch.rand(rows, 1, generator=g))).half()
    gamma, beta = _affine(C, g)
    out = gout((rows, C))
    ops.layernorm(gin(x).view, gin(gamma).view, gin(beta).view, 1e-5, out=out.view)
    torch.cuda.synchronize()
    args = (_d(x), _d(gamma), _d(beta), 1e-5)
    _check(out, kc.layernorm_exact(*args), cond_layernorm(*args), KAPPA_NORM, f"layernorm {rows}x{C} |mean|/sigma={ratio}")


# ------------------------------------------------------------------------------------------------------------- attention
def _offset_v(rows, C, g):
    """V = a per-channel offset of +-(1 ... 2), common to every key, plus N(0, 0.5^2)"""
    off = (1 + torch.rand(C, generator=g)) * torch.where(torch.rand(C, generator=g) < 0.5, -1.0, 1.0)
    return (off + 0.5 * torch.randn(rows, C, generator=g)).half()


def _attn_run(q, k, v, heads, seq, batch, out_rows, kw, what):
    from anyv2v_b200 import ops
    C = heads * 64
    out = gout((out_rows, C))
    ops.attention(gin(q).view, gin(k).view, gin(v).view, heads, seq, batch, out.view, **kw)
    torch.cuda.synchronize()
    o = torch.empty(out_rows, C, dtype=torch.float16, device=dev)
    ref, cond = kc.attention_exact(_d(q), _d(k), _d(v), heads, seq, batch, o, cond=cond_attention(kw.get("scale", 0.125)), **kw)
    _check(out, ref, cond, KAPPA_ATTN, what)


@pytest.mark.parametrize("nv", [1, 3])
@pytest.mark.parametrize("seq,batch", [(256, 32), (1024, 4)], ids=["attn_kernel_256keys", "attn_rows_kernel_1024keys"])
def test_attention_rows(seq, batch, nv):
    """self-attention, 5 heads: 256 keys run attn_kernel, 1024 keys the pipelined attn_rows_kernel"""
    g = _gen(191 + seq + nv)
    heads = 5
    C, rows = heads * 64, batch * seq
    q, k = (torch.randn(rows, C, generator=g) * 0.5).half(), (torch.randn(rows, C, generator=g) * 0.5).half()
    v = _offset_v(nv * rows, C, g)
    kw = dict(n_v=nv, v_branch_stride=rows * C if nv == 3 else 0, o_branch_stride=rows * C if nv == 3 else 0)
    _attn_run(q, k, v, heads, seq, batch, nv * rows, kw, f"attention rows seq={seq} batch={batch} nv={nv}")


def test_attention_cross_145_keys():
    """cross-attention of 16 frames of 1024 queries to one 145-key sequence (kv_batch_div = 16), 5 heads"""
    g = _gen(201)
    heads, seq, batch, nk = 5, 1024, 16, 145
    C = heads * 64
    q, k = (torch.randn(batch * seq, C, generator=g) * 0.5).half(), (torch.randn(nk, C, generator=g) * 0.5).half()
    v = _offset_v(nk, C, g)
    _attn_run(q, k, v, heads, seq, batch, batch * seq, dict(seq_kv=nk, kv_batch_div=batch), "attention cross 145 keys div=16")


@pytest.mark.parametrize("F,clips,HW", [(16, 2, 1024), (24, 2, 512), (136, 1, 64)])
def test_attention_frames(F, clips, HW):
    """temporal attention: packed pixels at F = 16 and 24, one pixel over two query tiles at F = 136"""
    g = _gen(211 + F)
    heads = 5
    C, rows = heads * 64, clips * F * HW
    q, k = (torch.randn(rows, C, generator=g) * 0.5).half(), (torch.randn(rows, C, generator=g) * 0.5).half()
    _attn_run(q, k, _offset_v(rows, C, g), heads, F, clips * HW, rows, dict(frames_mode=True, HW=HW),
              f"attention frames F={F} clips={clips} HW={HW}")


@pytest.mark.parametrize("nv", [1, 3])
@pytest.mark.parametrize("F,HW", [(16, 1024), (24, 512)])
def test_temporal_attention_fused(F, HW, nv):
    """the fused projection + temporal attention, 5 heads over Cx = 320; input channel 0 is a constant 4 that only the V
    projection reads, so V carries a per-channel offset of +-(1 ... 2)"""
    from anyv2v_b200 import ops
    g = _gen(221 + F + nv)
    heads, Cx = 5, 320
    C = heads * 64
    clips = 2 if nv == 1 else 3
    rows = clips * F * HW
    x = torch.randn(rows, Cx, generator=g)
    x[:, 0] = 4.0
    w = torch.randn(3 * C, Cx, generator=g) * Cx ** -0.5
    w[:C] *= 2  # Q: scores of order 1
    w[:2 * C, 0] = 0
    w[2 * C:, 0] = (1 + torch.rand(C, generator=g)) * torch.where(torch.rand(C, generator=g) < 0.5, -1.0, 1.0) / 4
    x, w = x.half(), w.half()
    out = gout((rows, C))
    ops.temporal_attention_fused(gin(x).view, gin(w).view, heads, F, HW, clips, out.view, n_v=nv)
    torch.cuda.synchronize()
    o = torch.empty(rows, C, dtype=torch.float16, device=dev)
    ref, cond = kc.temporal_attention_fused_exact(_d(x), _d(w), heads, F, HW, clips, o, 0.125, nv,
                                                  cond=cond_attention(0.125, rounded_operands=True))
    _check(out, ref, cond, KAPPA_ATTN, f"temporal attention fused F={F} HW={HW} nv={nv}")


# ------------------------------------------------------------------------------------------------------------- FreeU
@pytest.mark.parametrize("s", [0.9, 0.2])
def test_freeu_filtered_skip(s):
    """the filtered skip of up_blocks[0] (48 frames of 16 x 16 x 1280), channels with their own offset so that the low
    modes the filter scales are large"""
    from anyv2v_b200 import ops
    g = _gen(231 + int(10 * s))
    NF, H, W, C = 48, 16, 16, 1280
    skip = (torch.randn(NF, H, W, C, generator=g) + 4 * torch.rand(NF, 1, 1, C, generator=g) - 2).half()
    hidden = torch.randn(NF, H, W, C, generator=g).half()
    gh, out = guarded_inout(hidden, device=dev), gout((NF, H, W, C))
    ops.freeu(gh.view, gin(skip).view, 1.5, s, out=out.view)
    torch.cuda.synchronize()
    s32 = float(torch.tensor(s, dtype=torch.float32))
    ref = freeu_ref.fourier_filter_closed_form(_d(skip).double(), s32)
    _check(out, ref, cond_freeu(_d(skip), s), KAPPA_FREEU, f"freeu filtered skip {NF}x{H}x{W}x{C} s={s}")
