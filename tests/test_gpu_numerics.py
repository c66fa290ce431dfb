"""GPU tests of the kernels' VALUES: every output element against its float64 contract, within ulp16(ref) + kappa * cond
(tests/ulp_check.py), at the model's shapes and at the value ranges where fast arithmetic breaks: magnitudes that differ by
row and column, outputs that overflow fp16, GEGLU gates far below zero, GroupNorm / LayerNorm inputs with |mean| >> sigma and
constant groups, and softmax rows that are sharp, flat, or far from zero.

Each case runs the ``ops`` wrapper on guarded CUDA buffers (tests/guarded.py) and the ``kernel_contracts`` ``*_exact``
function on CPU copies of the same inputs, and prints its worst error in ulps and its margin to the bound (run with -s to
keep them in the log)."""
import pytest
import torch

import kernel_contracts as kc
from guarded import check_output, guarded_input, guarded_output
from ulp_check import (KAPPA_ATTN, KAPPA_GEGLU, KAPPA_GEMM, KAPPA_NORM, assert_within_bound, cond_attention, cond_conv_abs,
                       cond_geglu, cond_groupnorm, cond_layernorm, cond_linear)

pytestmark = pytest.mark.gpu
dev = "cuda"


def gin(t, ld=None):
    return guarded_input(t, ld=ld, device=dev)


def gout(shape, ld=None):
    return guarded_output(shape, ld=ld, device=dev)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _pow2(n, g, lo=-12, hi=4):
    return 2.0 ** torch.randint(lo, hi + 1, (n,), generator=g).double()


def _check(out, ref, cond, kappa, what):
    check_output(out, what)
    got = out.view.cpu()
    assert_within_bound(got, ref, cond, kappa, what, shape=tuple(got.shape))


# ------------------------------------------------------------------------------------------------------------- linear
def _scaled_linear(M, N, K, g):
    """A rows and W output channels scaled by 2^-12 ... 2^4 (W also by K^-1/2)"""
    a = (torch.randn(M, K, generator=g, dtype=torch.float64) * _pow2(M, g)[:, None]).half()
    w = (torch.randn(N, K, generator=g, dtype=torch.float64) * _pow2(N, g)[:, None] * K ** -0.5).half()
    return a, w


@pytest.mark.parametrize("case", ["plain", "rowbias_residual", "two_source", "overflow"])
def test_linear_magnitudes(case):
    from anyv2v_b200 import ops
    g = _gen(sum(map(ord, case)))
    M, N, K = 4096, 640, 1280
    if case == "overflow":  # outputs spread over [5.8e4, 7.0e4]: the switch to inf at 65520
        M, N, K = 1024, 256, 320
        a = (16 + 0.01 * torch.randn(M, K, generator=g)).half()
        w = (12.5 * (1 + 0.1 * (2 * torch.rand(N, 1, generator=g) - 1)) * (1 + 1e-3 * torch.randn(N, K, generator=g))).half()
    else:
        a, w = _scaled_linear(M, N, K, g)
    bias = (torch.randn(N, generator=g) * 2.0 ** -6).half()
    kw = dict(bias=bias)
    if case == "rowbias_residual":
        kw.update(rowbias=(torch.randn(M // 256, N, generator=g) * 0.5).half(), rows_per_rowbias=256,
                  residual=(torch.randn(M, N, generator=g, dtype=torch.float64) * _pow2(M, g, -8, 2)[:, None]).half())
    a2 = None
    if case == "two_source":
        a, a2 = a[:, :640].contiguous(), a[:, 640:].contiguous()
    out = gout((M, N))
    ops.linear(gin(a).view, gin(w).view, **{k: gin(v).view if isinstance(v, torch.Tensor) else v for k, v in kw.items()},
               a2=None if a2 is None else gin(a2).view, out=out.view)
    torch.cuda.synchronize()
    ref = kc.linear_exact(a, w, a2=a2, **kw)
    if case == "overflow":
        assert (ref.abs() >= 65520).any() and (ref.abs() < 65504).any()
    cond = cond_linear(a, w, kw.get("bias"), kw.get("rowbias"), kw.get("rows_per_rowbias", 0), kw.get("residual"), a2=a2)
    _check(out, ref, cond, KAPPA_GEMM, f"linear {case}")


# ------------------------------------------------------------------------------------------------------------- conv
def _scaled_image(NF, H, W, C, g):
    """pixels (the GEMM rows) scaled by 2^-12 ... 2^4"""
    s = _pow2(NF * H * W, g).view(NF, H, W, 1)
    return (torch.randn(NF, H, W, C, generator=g, dtype=torch.float64) * s).half()


@pytest.mark.parametrize("case", ["stride1", "stride2", "slots3"])
def test_conv3x3_magnitudes(case):
    from anyv2v_b200 import ops
    g = _gen(len(case))
    NF, H, W, C, Cout = 4, 32, 32, 320, 320
    stride = 2 if case == "stride2" else 1
    x = _scaled_image(NF, H, W, C, g)
    w = (torch.randn(Cout, 9 * C, generator=g, dtype=torch.float64) * _pow2(Cout, g)[:, None] * (9 * C) ** -0.5).half()
    bias = (torch.randn(Cout, generator=g) * 2.0 ** -6).half()
    M = NF * (H // stride) * (W // stride)
    rowbias = (torch.randn(NF, Cout, generator=g) * 0.25).half()
    rpr = M // NF
    ns = 3 if case == "slots3" else 1
    res = (torch.randn(ns, M, Cout, generator=g, dtype=torch.float64) * _pow2(M, g, -8, 2)[None, :, None]).half()
    if ns == 1:
        res = res[0]
    out = gout(res.shape)
    ops.conv3x3(gin(x).view, gin(w).view, bias=gin(bias).view, rowbias=gin(rowbias).view, rows_per_rowbias=rpr,
                residual=gin(res).view, out=out.view, n_slots=ns, slot_stride=M * Cout, stride=stride)
    torch.cuda.synchronize()
    acc = kc.conv3x3_exact(x, w, bias, rowbias, rpr, stride)
    ref = acc + res.double()
    cond = cond_conv_abs(kc.conv3x3_exact, x, w, bias, rowbias, rpr, stride) + res.double().abs()
    _check(out, ref, cond, KAPPA_GEMM, f"conv3x3 {case}")


def test_tconv3_magnitudes():
    from anyv2v_b200 import ops
    g = _gen(7)
    B, F_, HW, C = 2, 16, 256, 320
    x = _scaled_image(B, F_, HW, C, g).view(B, F_ * HW, C)
    w = (torch.randn(C, 3 * C, generator=g, dtype=torch.float64) * _pow2(C, g)[:, None] * (3 * C) ** -0.5).half()
    bias = (torch.randn(C, generator=g) * 2.0 ** -6).half()
    res = (torch.randn(B, F_ * HW, C, generator=g) * 0.1).half()
    out = gout((B, F_ * HW, C))
    ops.tconv3(gin(x).view, gin(w).view, F_, HW, bias=gin(bias).view, residual=gin(res).view, out=out.view)
    torch.cuda.synchronize()
    ref = kc.tconv3_exact(x, w, F_, HW, bias, res).view(B, F_ * HW, C)
    cond = cond_conv_abs(kc.tconv3_exact, x, w, F_, HW, bias, res).view(B, F_ * HW, C)
    _check(out, ref, cond, KAPPA_GEMM, "tconv3")


def test_upsample_phases_magnitudes():
    from anyv2v_b200 import ops
    g = _gen(8)
    NF, H, W, Cin, Cout = 4, 16, 16, 640, 320
    x = _scaled_image(NF, H, W, Cin, g)
    wfull = torch.randn(Cout, Cin, 3, 3, generator=g, dtype=torch.float64) * _pow2(Cout, g)[:, None, None, None] * (9 * Cin) ** -0.5
    wph = ops.pack_upsample_weights(wfull.half())
    bias = (torch.randn(Cout, generator=g) * 2.0 ** -6).half()
    out = gout((NF, 2 * H, 2 * W, Cout))
    ops.upsample2x_conv3x3(gin(x).view, gin(wph).view, bias=gin(bias).view, out=out.view)
    torch.cuda.synchronize()
    _check(out, kc.upsample2x_conv3x3_exact(x, wph, bias), cond_conv_abs(kc.upsample2x_conv3x3_exact, x, wph, bias),
           KAPPA_GEMM, "upsample2x_conv3x3")


# ------------------------------------------------------------------------------------------------------------- GEGLU
GATES = (-6.0, -4.0, -3.0, -2.0, -1.0, 0.0, 2.0, 5.0)


def test_geglu_gate_ranges():
    """the FF shape; whole gate columns at gates {-6, ..., 5} +- 0.3 (bias plus a small GEMM term), h of magnitude ~1 and ~100"""
    from anyv2v_b200 import ops
    g = _gen(11)
    M, N, K = 4096, 2560, 320
    inner = N // 2
    a = torch.randn(M, K, generator=g).half()
    w_h = torch.randn(inner, K, generator=g, dtype=torch.float64) * K ** -0.5
    w_h *= torch.where(torch.arange(inner) % 2 == 0, 1.0, 100.0).double()[:, None]
    w_g = torch.randn(inner, K, generator=g, dtype=torch.float64) * K ** -0.5 * 0.1
    b_h = torch.randn(inner, generator=g, dtype=torch.float64) * 0.1
    b_g = torch.tensor(GATES, dtype=torch.float64)[(torch.arange(inner) // 2) % len(GATES)]
    wp, bp = kc.geglu_pack(torch.cat([w_h, w_g]).half(), torch.cat([b_h, b_g]).half())
    out = gout((M, inner))
    ops.linear(gin(a).view, gin(wp).view, bias=gin(bp).view, out=out.view, geglu=True)
    torch.cuda.synchronize()
    ref = kc.linear_exact(a, wp, bp, geglu=True)
    cond = cond_geglu(a, wp, bp)
    check_output(out, "geglu")
    got = out.view.cpu()
    gate_col = b_g.view(-1)
    failures = []
    for gt in GATES:  # one verdict per gate value, so the log shows where an erf approximation breaks
        cols = (gate_col == gt).nonzero().view(-1)
        try:
            assert_within_bound(got[:, cols], ref[:, cols], cond[:, cols], KAPPA_GEGLU, f"geglu gates {gt:+.0f} +- 0.3")
        except AssertionError as e:
            failures.append(str(e))
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------------------- GroupNorm
def _gn_input(n, rows, C, groups, ratio, g, const_groups=2):
    """every (sample, group) with its own mean, |mean| / sigma = ratio * (1 ... 1.1), sigma = 1.  fp16 spaces values near |mean|
    by |mean| * 2^-10 or less, so sigma is >= 8 fp16 ulps of the mean up to ratio 128; beyond that the rounded values take a
    few dozen levels, which the contract's statistics see as they are.  The last ``const_groups`` groups of sample 0 are
    exactly constant."""
    cpg = C // groups
    sign = torch.where(torch.rand(n, 1, groups, 1, generator=g) < 0.5, -1.0, 1.0)
    mu = ratio * sign * (1 + 0.1 * torch.rand(n, 1, groups, 1, generator=g))
    x = (torch.randn(n, rows, groups, cpg, generator=g) + mu).half()
    if const_groups:
        x[0, :, groups - const_groups:] = (3.0 + ratio)
    return x.view(n, rows, C)


def _gn_run(x, gamma, beta, groups, eps, silu, what, x2=None):
    from anyv2v_b200 import ops
    n, rows = x.shape[:2]
    C = x.shape[2] + (0 if x2 is None else x2.shape[2])
    out = gout((n, rows, C))
    ops.groupnorm(gin(x).view, gin(gamma).view, gin(beta).view, groups, eps, silu, out=out.view,
                  x2=None if x2 is None else gin(x2).view)
    torch.cuda.synchronize()
    ref = kc.groupnorm_exact(x, gamma, beta, groups, eps, silu, x2=x2)
    cond = cond_groupnorm(x, gamma, beta, groups, eps, silu, x2=x2)
    _check(out, ref, cond, KAPPA_NORM, what)
    return out.view.cpu(), ref


def _affine(C, g):
    return (torch.randn(C, generator=g) * 0.2 + 1).half(), (torch.randn(C, generator=g) * 0.2).half()


@pytest.mark.parametrize("ratio,silu,eps", [(0.0, False, 1e-5), (30.0, True, 1e-6), (100.0, False, 1e-5),
                                            (300.0, True, 1e-5), (300.0, False, 1e-6), (1000.0, True, 1e-6)])
def test_groupnorm_offsets_per_frame(ratio, silu, eps):
    """the per-frame shape (48 samples of 4096 x 320, 32 groups); two constant groups give exactly beta (before SiLU)"""
    g = _gen(int(ratio) + silu)
    x = _gn_input(48, 4096, 320, 32, ratio, g)
    gamma, beta = _affine(320, g)
    got, ref = _gn_run(x, gamma, beta, 32, eps, silu, f"groupnorm 48x4096x320 |mean|/sigma={ratio} silu={silu} eps={eps}")
    if not silu:
        assert torch.equal(ref[0, :, -20:], beta[-20:].double().expand(4096, 20))


@pytest.mark.parametrize("ratio,silu", [(0.0, True), (300.0, False), (1000.0, True)])
def test_groupnorm_offsets_per_clip(ratio, silu):
    """the per-clip shape (one sample of 65536 x 320: larger than a chunk)"""
    g = _gen(int(ratio) + 7)
    x = _gn_input(1, 65536, 320, 32, ratio, g)
    gamma, beta = _affine(320, g)
    _gn_run(x, gamma, beta, 32, 1e-5, silu, f"groupnorm 1x65536x320 |mean|/sigma={ratio} silu={silu}")


@pytest.mark.parametrize("offset_on", ["x", "x2"])
def test_groupnorm_two_source_offset(offset_on):
    """the up-block rows and channels, 4096 x (640 + 320), for 16 frames; the offset on one of the two sources only (group 21
    straddles them)"""
    g = _gen(21 + len(offset_on))
    n, rows = 16, 4096
    x = _gn_input(n, rows, 640, 32, 300.0 if offset_on == "x" else 0.0, g, const_groups=0)
    x2 = _gn_input(n, rows, 320, 16, 300.0 if offset_on == "x2" else 0.0, g, const_groups=0)
    gamma, beta = _affine(960, g)
    _gn_run(x, gamma, beta, 32, 1e-5, True, f"groupnorm two-source, offset on {offset_on}", x2=x2)


# ------------------------------------------------------------------------------------------------------------- LayerNorm
@pytest.mark.parametrize("C", [320, 640, 1280])
@pytest.mark.parametrize("ratio", [0.0, 30.0, 300.0, 1000.0])
def test_layernorm_offsets(C, ratio):
    """rows with their own mean, |mean| / sigma = ratio; 16 constant rows give exactly beta"""
    from anyv2v_b200 import ops
    g = _gen(C + int(ratio))
    rows = 4096
    sign = torch.where(torch.rand(rows, 1, generator=g) < 0.5, -1.0, 1.0)
    x = (torch.randn(rows, C, generator=g) + ratio * sign * (1 + 0.1 * torch.rand(rows, 1, generator=g))).half()
    x[:16] = 2.0 + ratio
    gamma, beta = _affine(C, g)
    out = gout((rows, C))
    ops.layernorm(gin(x).view, gin(gamma).view, gin(beta).view, 1e-5, out=out.view)
    torch.cuda.synchronize()
    ref = kc.layernorm_exact(x, gamma, beta, 1e-5)
    assert torch.equal(ref[:16], beta.double().expand(16, C))
    _check(out, ref, cond_layernorm(x, gamma, beta, 1e-5), KAPPA_NORM, f"layernorm C={C} |mean|/sigma={ratio}")


# ------------------------------------------------------------------------------------------------------------- attention
def _scores_qk(kind, rows_q, rows_k, heads, key_of_row, g, dom_key):
    """Q, K [rows, heads * 64] whose scaled scores (scale 0.125) have the requested shape.
    dom<D>: channel 0 of every head carries q = 32 on queries and k = 8 D / 32 on the dominant key (0 elsewhere), so that key
            leads each row by D nats over scores of order 1;
    uniform: q = 0, every score 0;
    far:    q = 40, k = -31.25 + (0 ... 12) fp16 steps of 1 / 64: scores in [-1e4, -1e4 + 1]."""
    C = heads * 64
    if kind == "uniform":
        return torch.zeros(rows_q, C).half(), torch.randn(rows_k, C, generator=g).half()
    if kind == "far":
        q = torch.full((rows_q, C), 40.0)
        k = torch.full((rows_k, C), -31.25)
        steps = (torch.rand(rows_k, C, generator=g) < 12.0 / 64).float() / 64
        return q.half(), (k + steps).half()
    D = float(kind[3:])
    q = torch.randn(rows_q, C, generator=g) * 0.35
    k = torch.randn(rows_k, C, generator=g) * 0.35
    q[:, ::64] = 32.0
    k[:, ::64] = 0.0
    k[dom_key, ::64] = 8 * D / 32
    return q.half(), k.half()


def _attn_run(q, k, v, heads, seq, batch, out_rows, kw, what):
    from anyv2v_b200 import ops
    C = heads * 64
    out = gout((out_rows, C))
    ops.attention(gin(q).view, gin(k).view, gin(v).view, heads, seq, batch, out.view, **kw)
    torch.cuda.synchronize()
    o = torch.empty(out_rows, C, dtype=torch.float16)
    ref, cond = kc.attention_exact(q, k, v, heads, seq, batch, o, cond=cond_attention(kw.get("scale", 0.125)), **kw)
    _check(out, ref, cond, KAPPA_ATTN, what)


ATTN_KINDS = ["dom20", "dom60", "dom140", "uniform", "far", "dom60_last_tile"]


@pytest.mark.parametrize("nv", [1, 3])
@pytest.mark.parametrize("kind", ATTN_KINDS)
def test_attention_rows_softmax(kind, nv):
    """rows mode, seq = 4096 keys for the flat softmax (l = 4096), 1000 keys (a ragged last tile) otherwise; the dominant key in
    the middle, or in the last, ragged key tile"""
    g = _gen(len(kind) * 10 + nv)
    heads, batch = (1, 1) if kind == "uniform" else (2, 2)
    seq = 4096 if kind == "uniform" else 1000
    dom = seq - 5 if kind.endswith("last_tile") else seq // 3
    base = kind.split("_")[0]
    rows = batch * seq
    q, k = _scores_qk(base, rows, rows, heads, None, g, torch.arange(batch) * seq + dom)
    v = torch.randn(nv * rows, heads * 64, generator=g).half()
    kw = dict(n_v=nv, v_branch_stride=rows * heads * 64 if nv == 3 else 0, o_branch_stride=rows * heads * 64 if nv == 3 else 0)
    _attn_run(q, k, v, heads, seq, batch, nv * rows, kw, f"attention rows {kind} nv={nv}")


@pytest.mark.parametrize("nv", [1, 3])
@pytest.mark.parametrize("kind", ["dom20", "dom140", "uniform", "far"])
@pytest.mark.parametrize("F", [16, 128])
def test_attention_frames_softmax(F, kind, nv):
    """frames mode (temporal attention) at F = 16 (packed pixels) and 128 (one pixel per CTA): the dominant key is frame F - 1"""
    g = _gen(F + len(kind) + nv)
    heads, clips, HW = 2, 2, 64
    rows = clips * F * HW
    dom = ((torch.arange(rows) // HW) % F == F - 1).nonzero().view(-1)
    q, k = _scores_qk(kind, rows, rows, heads, None, g, dom)
    v = torch.randn(nv * rows, heads * 64, generator=g).half()
    kw = dict(n_v=nv, v_branch_stride=rows * heads * 64 if nv == 3 else 0, o_branch_stride=rows * heads * 64 if nv == 3 else 0,
              frames_mode=True, HW=HW)
    _attn_run(q, k, v, heads, F, clips * HW, nv * rows, kw, f"attention frames F={F} {kind} nv={nv}")


@pytest.mark.parametrize("nv", [1, 3])
@pytest.mark.parametrize("F", [16, 128])
def test_temporal_attention_fused_bound(F, nv):
    """the fused projection + temporal attention against the same bound; Q / K / V are the fp16-rounded projections"""
    from anyv2v_b200 import ops
    g = _gen(F * 3 + nv)
    heads, Cx, HW, src = 2, 320, 32, 2
    C = heads * 64
    clips = src * nv
    rows = clips * F * HW
    x = torch.randn(rows, Cx, generator=g).half()
    wqkv = (torch.randn(3 * C, Cx, generator=g) * Cx ** -0.5 * 2).half()
    out = gout((rows, C))
    ops.temporal_attention_fused(gin(x).view, gin(wqkv).view, heads, F, HW, clips, out.view, n_v=nv)
    torch.cuda.synchronize()
    qkv = (x.double() @ wqkv.double().t()).half()
    if nv == 1:
        args = (qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], heads, F, clips * HW, torch.empty(rows, C).half())
        kw = dict(frames_mode=True, HW=HW)
    else:
        sr = src * F * HW
        args = (qkv[:sr, :C], qkv[:sr, C:2 * C], qkv[:, 2 * C:], heads, F, src * HW, torch.empty(rows, C).half())
        kw = dict(n_v=3, v_branch_stride=sr * qkv.stride(0), o_branch_stride=sr * C, frames_mode=True, HW=HW)
    ref, cond = kc.attention_exact(*args, cond=cond_attention(0.125, rounded_operands=True), **kw)
    _check(out, ref, cond, KAPPA_ATTN, f"temporal attention fused F={F} nv={nv}")
