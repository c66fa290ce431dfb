"""Element-wise error bound of an fp16 kernel output against its float64 contract.

    |got - ref| <= ulp16(ref) + kappa * cond          for every element

``ref`` is the contract's float64 value BEFORE the store rounds it to fp16 (the ``*_exact`` functions of kernel_contracts).
``ulp16(ref)`` is the fp16 spacing at |ref| (2^-24 in the subnormal range): the store's own rounding takes half of it, the
other half is left for arithmetic errors that are small relative to the result.  ``cond`` is the op's condition scale per
element, in float64: the size of the terms whose rounding errors the kernel can not avoid (the operands of a sum that
cancels), and ``kappa`` is the relative precision the kernel's arithmetic keeps on them.  A bound relative to the largest
element of the output (``assert_fp16_close``) lets any error at a small element through; this one does not.

Where |ref| >= 65520 (rounds to inf in fp16) ``got`` must be inf of the same sign; a NaN in ``got`` always fails.
"""
from __future__ import annotations

import math

import torch

# ------------------------------------------------------------------------------------------------------------- kappa per op
# GEMM family (linear, conv3x3, tconv3, upsample phases): fp32 accumulation.  wgmma adds each product of two fp16 values
# exactly and keeps the running sum in fp32; over the K loop and the fp32 epilogue the error stays within 64 fp32 ulps of the
# sum of |terms|, 2^-24 * 64 = 2^-18.  An operand or a partial sum rounded to fp16 costs 2^-11 and fails by a wide margin.
KAPPA_GEMM = 2.0 ** -18
# GEGLU: the same accumulation in the h and gate columns, carried through h * gelu(g) by the first-order terms of cond.
KAPPA_GEGLU = 2.0 ** -18
# GroupNorm / LayerNorm: fp32 statistics of centred (or shifted) values, so mean and rstd carry a few fp32 ulps of sigma and of
# rstd, and the affine map y = x * a + (beta - mean * a) is exact to a few fp32 ulps of |x| * rstd * |gamma| and
# |mean| * rstd * |gamma|: 16 ulps, 2^-20, on cond_norm (which therefore holds sigma * rstd * |gamma| as well).
KAPPA_NORM = 2.0 ** -20
# attention: P is rounded to fp16 before the PV product by design (the wgmma A fragment is fp16), a relative error of
# 2^-11 per weight of |V|: 2^-10 covers it and the fp32 exponentials.
KAPPA_ATTN = 2.0 ** -10
# FreeU's filtered skip, y = x + (s - 1) / (H W) * sum_j S_j t_j (tests/freeu_ref.py): each of the seven plane sums S_j adds
# H W fp32 products x * t with |t| <= 1, so it keeps (H W) 2^-24 of sum |x|; the twiddles t carry <= 3 * 2^-24 in both passes,
# and (s - 1) / (H W) cancels the H W: |err| <= 2^-24 (|x| + 7 |s - 1| sum |x| (1 + 3 + 3 + 1)) <= 2^-21 * cond_freeu.
KAPPA_FREEU = 2.0 ** -20

FP16_MAX_FINITE_EDGE = 65520.0  # values at or above this magnitude round to inf in fp16


def ulp16(ref: torch.Tensor) -> torch.Tensor:
    """fp16 spacing at |ref| (float64): 2^(floor(log2|ref|) - 10) in the normal range, 2^-24 below 2^-14"""
    _, e = torch.frexp(ref.to(torch.float64).abs().clamp_min(2.0 ** -14))  # |ref| = m * 2^e, m in [0.5, 1)
    return torch.pow(2.0, (e - 11).to(torch.float64))


def measure(got16: torch.Tensor, ref64: torch.Tensor, cond64: torch.Tensor, kappa: float) -> dict:
    """worst element statistics: error in ulps, error over the bound (negative = margin), fraction over the bound"""
    ref64 = torch.as_tensor(ref64).detach().to(torch.float64)  # evaluated on ref64's device
    got = torch.as_tensor(got16).detach().to(ref64.device, torch.float64).reshape(-1)
    cond = torch.broadcast_to(torch.as_tensor(cond64, dtype=torch.float64).to(ref64.device), ref64.shape).reshape(-1)
    ref = ref64.reshape(-1)
    assert got.shape == ref.shape == cond.shape, (got.shape, ref.shape, cond.shape)
    assert torch.isfinite(ref).all() and torch.isfinite(cond).all(), "reference or condition scale not finite"
    u = ulp16(ref)
    bound = u + kappa * cond
    overflow = ref.abs() >= FP16_MAX_FINITE_EDGE
    err = (got - ref).abs()
    # an element that must be inf: error 0 if it is inf of ref's sign, else infinite
    want_inf = torch.where(ref > 0, math.inf, -math.inf)
    err = torch.where(overflow, torch.where(got == want_inf, 0.0, math.inf), err)
    err = torch.where(torch.isnan(got), math.inf, err)  # NaN always fails
    err = torch.where(~overflow & torch.isinf(got), math.inf, err)
    over = err - bound
    bad = over > 0
    i = int(torch.argmax(torch.where(torch.isnan(over), math.inf, over))) if over.numel() else 0
    return dict(n=ref.numel(), n_bad=int(bad.sum()), worst=i, got=float(got[i]) if got.numel() else 0.0,
                ref=float(ref[i]) if ref.numel() else 0.0, err_ulp=float((err / u).max()) if err.numel() else 0.0,
                worst_ulp_err=float(err[i] / u[i]) if err.numel() else 0.0, bound_ulp=float(bound[i] / u[i]) if err.numel() else 0.0,
                over_bound=float(over.max()) if over.numel() else 0.0, over_rel=float((over / bound).max()) if over.numel() else 0.0)


def assert_within_bound(got16, ref64, cond64, kappa: float, what: str, shape=None, quiet: bool = False) -> dict:
    """fails with the worst element (index, got, ref, error in ulps, bound in ulps) and the fraction over the bound"""
    m = measure(got16, ref64, cond64, kappa)
    idx = m["worst"] if shape is None else tuple(int(v) for v in torch.unravel_index(torch.tensor(m["worst"]), shape))
    line = (f"{what}: max err {m['err_ulp']:.3g} ulp16; worst vs bound at {idx}: got {m['got']!r} ref {m['ref']!r} "
            f"err {m['worst_ulp_err']:.3g} ulp, bound {m['bound_ulp']:.3g} ulp, (err - bound) / bound = {m['over_rel']:+.3g}")
    if not quiet:
        print(line)
    assert m["n_bad"] == 0, f"{line}; {m['n_bad']} of {m['n']} elements ({m['n_bad'] / max(m['n'], 1):.2%}) over the bound"
    return m


# ------------------------------------------------------------------------------------------------------------- cond per op
def _d(t):
    """float64 on the tensor's own device"""
    return None if t is None else torch.as_tensor(t).detach().to(torch.float64)


def cond_linear(a, w, bias=None, rowbias=None, rows_per_rowbias=0, residual=None, a2=None):
    """|A| |W|^T + |bias| + |rowbias| + |residual| per element: the sum of the magnitudes of the terms the output adds"""
    a = _d(a) if a2 is None else torch.cat([_d(a), _d(a2)], dim=1)
    c = a.abs() @ _d(w).abs().t()
    if bias is not None:
        c = c + _d(bias).abs()
    if rowbias is not None:
        c = c + _d(rowbias).abs()[torch.arange(c.shape[0], device=c.device) // rows_per_rowbias]
    if residual is not None:
        c = c + _d(residual).abs().reshape(c.shape)
    return c


def cond_geglu(a, w_packed, bias_packed):
    """|gelu(g)| * cond_h + |h * gelu'(g)| * cond_g: first-order propagation of the two accumulations through h * gelu(g)"""
    a, w, b = _d(a), _d(w_packed), _d(bias_packed)
    M, N = a.shape[0], w.shape[0]
    y = (a @ w.t() + b).view(M, N // 64, 2, 32)
    c = (a.abs() @ w.abs().t() + b.abs()).view(M, N // 64, 2, 32)
    h, g, ch, cg = y[:, :, 0], y[:, :, 1], c[:, :, 0], c[:, :, 1]
    phi = torch.exp(-0.5 * g * g) / math.sqrt(2 * math.pi)
    cdf = 0.5 * torch.erfc(-g / math.sqrt(2))
    return ((g * cdf).abs() * ch + (h * (cdf + g * phi)).abs() * cg).reshape(M, N // 2)


def cond_conv_abs(fn, *args, **kwargs):
    """the conv ops' |A| |W|^T: the same contract evaluated on |x| and |w| (bias / rowbias / residual passed as |.|)"""
    ab = lambda t: t.abs() if isinstance(t, torch.Tensor) and t.is_floating_point() else t
    return fn(*[ab(v) for v in args], **{k: ab(v) for k, v in kwargs.items()})


def cond_norm(x, mean, rstd, gamma, beta, sigma):
    """(|x| + |mean| + sigma) * rstd * |gamma| + |beta| per element; mean / rstd / sigma broadcast against x.  |x| and |mean|
    are the operands of the affine map; sigma is the scale of the statistics' own error: an fp32 sum of x - mean (or of x - k)
    knows the mean to a few ulps of sigma, not of |mean|, and that error moves an output at x ~ mean by sigma * rstd * |gamma|"""
    return (_d(x).abs() + mean.abs() + sigma) * rstd * _d(gamma).abs() + _d(beta).abs()


def cond_groupnorm(x, gamma, beta, groups, eps, silu, x2=None):
    """cond_norm with the group statistics; + SiLU: times |d silu / dy| at the fp16-rounded GroupNorm value"""
    x = _d(x) if x2 is None else torch.cat([_d(x), _d(x2)], dim=2)
    n, rows, C = x.shape
    xf = x.view(n, rows, groups, C // groups)
    mean = xf.mean(dim=(1, 3), keepdim=True)
    var = xf.var(dim=(1, 3), unbiased=False, keepdim=True)
    rstd = torch.rsqrt(var + eps)
    c = cond_norm(xf, mean, rstd, 1.0, 0.0, var.sqrt()).view(n, rows, C) * _d(gamma).abs() + _d(beta).abs()
    if silu:
        # the contract rounds the GroupNorm value to fp16 before SiLU, as the reference does (two ops).  Any error in the kernel's
        # GroupNorm value, however small, can move that rounding by one fp16 step where the exact value lies near a midpoint, so
        # the bound holds one step of the intermediate carried through SiLU: |d silu| * ulp16(g) / KAPPA_NORM in cond units
        yn = ((xf - mean) * rstd).view(n, rows, C) * _d(gamma) + _d(beta)
        g = yn.to(torch.float16).double()
        s = torch.sigmoid(g)
        ds = (s * (1 + g * (1 - s))).abs()
        c = c * ds + ds * ulp16(g) / KAPPA_NORM
    return c


def cond_layernorm(x, gamma, beta, eps):
    xd = _d(x)
    mean = xd.mean(dim=-1, keepdim=True)
    var = xd.var(dim=-1, unbiased=False, keepdim=True)
    return cond_norm(xd, mean, torch.rsqrt(var + eps), gamma, beta, var.sqrt())


def cond_attention(scale, rounded_operands=False):
    """for kernel_contracts.attention_exact: P |V| per element, P the exact softmax; plus the scores' own fp32 accumulation
    error carried through the softmax, sum_k P_k |V_k - o| * |dS_k| with |dS_k| <= 2^-18 * scale * |q| . |k| (the GEMM bound of
    QK^T), written as 2^-8 * ... so that KAPPA_ATTN * cond holds it: at scores of 1e4 that term is the larger one"""
    def cond(p, qh, kh, vh, o):
        # p [..., heads, Lq, Lk]; qh / kh / vh [..., L, heads, 64]; o [..., Lq, heads, 64]
        pv = torch.einsum("...hqk,...khd->...qhd", p, vh.abs())
        sabs = torch.einsum("...qhd,...khd->...hqk", qh.abs(), kh.abs()) * abs(scale)
        # sum_k P_qk sabs_qk |V_kd - o_qd| <= sum_k P sabs |V_kd| + |o_qd| sum_k P sabs
        w = p * sabs
        dev = torch.einsum("...hqk,...khd->...qhd", w, vh.abs()) + o.abs() * w.sum(-1).transpose(-1, -2).unsqueeze(-1)
        if rounded_operands:
            # the fused temporal kernel projects Q / K / V in fp32 and rounds them to fp16 itself; the contract rounds the exact
            # projection.  Where a projection lies near a rounding midpoint the two differ by one fp16 step (2^-10 relative at
            # most): up to 2^-10 * P |V| through V and 2^-10 * 2 * scale |q| . |k| per score through Q and K, in cond units
            # (KAPPA_ATTN = 2^-10) that is P |V| + 2 * the score term over 2^-8
            return 2 * pv + (2.0 ** -8 + 2.0) * dev
        return pv + 2.0 ** -8 * dev
    return cond


def cond_freeu(skip, s):
    """|x| + 7 |s - 1| sum_plane |x| per element of channels-last planes skip[..., H, W, C]: the operand of the final add and
    the magnitudes the seven plane sums add, carried through (s - 1) / (H W) (H W cancels against fp32 accumulation over H W
    terms, see KAPPA_FREEU); s is the fp32 value the kernel receives"""
    x = _d(skip).abs()
    s32 = float(torch.tensor(s, dtype=torch.float32))
    return x + 7.0 * abs(s32 - 1.0) * x.sum(dim=(-3, -2), keepdim=True)
