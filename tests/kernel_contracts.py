"""TEST INFRASTRUCTURE — CPU restatement of the CONTRACT of every C-ABI op in anyv2v_b200.ops (include/anyv2v_b200.h).

The product has no CPU path (ops.* raise on CPU tensors).  For the `-m "not gpu"` tests this module states what each
kernel is specified to compute — same arguments, same layouts (channels-last activations, packed weights, branch slots,
row-strided views), exact (float64) arithmetic on the fp16 inputs, one rounding to fp16 at the store — in plain PyTorch
(float64 rather than the kernels' fp32 accumulation makes the emulation independent of how a batch is split, so the
de-duplication / pruning switches can be checked for bit-identical results), and the
``emulated_ops`` fixture (tests/conftest.py) swaps it in for the duration of ONE test.  That lets the host logic that sits
on top of the kernels (the channels-last UNet wiring, the PnP de-duplication, hooks, loops, latent store) run on CPU and
be compared with the oracle.  tests/test_gpu_contracts.py runs every kernel against these functions on the GPU (guarded
buffers, same views and strides), so the contract the CPU tests rely on is the one the kernels implement;
tests/test_gpu_kernels.py checks them against inline fp32 formulas as well.  Every function computes on its inputs' device,
so tests/call_audit.py evaluates the same contracts on the GPU for the calls of a full-size pass.  Nothing outside tests/
imports this file.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

_launches = 0


def _count(n=1):
    global _launches
    _launches += n


def launch_count():
    return _launches


def _f16(t, name):
    assert t.dtype == torch.float16, f"{name}: the C ABI takes fp16 tensors, got {t.dtype}"


def _store(out, y32, shape=None):
    y16 = y32.to(torch.float16).contiguous()  # the kernels write freshly allocated, contiguous outputs
    if out is None:
        return y16 if shape is None else y16.view(shape)
    out.copy_(y16.view(out.shape))
    return out


# ------------------------------------------------------------------------------------------------------------- K7
def ddim_step(x, v_neg, v_edit, guidance, ca, cb, cc, cd, out=None, inverse=False, coef_dev=None):
    """csrc/elementwise.cu ddim_one: every product / sum rounded to fp16 separately, fp32 scalars."""
    _f16(x, "ddim.x")
    if coef_dev is not None:
        ca, cb, cc, cd, guidance = (float(v) for v in coef_dev[:5].tolist())
    f32 = lambda s: torch.tensor(s, dtype=torch.float32)
    r16 = lambda t: t.to(torch.float16).to(torch.float32)
    xf, vn = x.float(), v_neg.float()
    v = vn
    if v_edit is not None:
        d0 = r16(v_edit.float() - vn)
        d1 = r16(f32(guidance) * d0)
        v = r16(vn + d1)
    x0 = r16(r16(f32(ca) * xf) - r16(f32(cb) * v))
    ep = r16(r16(f32(ca) * v) + r16(f32(cb) * xf))
    direction = r16(f32(cd) * ep)
    res = r16(r16(f32(cc) * x0) + direction)
    _count()
    return _store(out, res, x.shape)


# ------------------------------------------------------------------------------------------------------------- K6
def groupnorm(x, gamma, beta, groups, eps, silu, out=None, x2=None):
    y = groupnorm_exact(x, gamma, beta, groups, eps, silu, x2=x2)
    _count(1)
    return _store(out, y, y.shape)


def groupnorm_exact(x, gamma, beta, groups, eps, silu, x2=None):
    """the float64 value ``groupnorm`` rounds to fp16 at the store, [n, rows, C]"""
    _f16(x, "groupnorm.x")
    assert x.dim() == 3 and x.is_contiguous()
    if x2 is not None:  # two-source input: the logical tensor is [x | x2] along the channels
        _f16(x2, "groupnorm.x2")
        assert x2.is_contiguous() and x2.shape[:2] == x.shape[:2] and x.shape[2] % 8 == 0
        x = torch.cat([x, x2], dim=2)
    n, rows, C = x.shape
    xf = x.double().view(n, rows, groups, C // groups)
    mean = xf.mean(dim=(1, 3), keepdim=True)
    var = xf.var(dim=(1, 3), unbiased=False, keepdim=True)
    y = ((xf - mean) * torch.rsqrt(var + eps)).view(n, rows, C) * gamma.double() + beta.double()
    if silu:
        y = y.to(torch.float16).double()  # the reference rounds the GroupNorm output before SiLU (two ops)
        y = y * torch.sigmoid(y)
    return y.view(x.shape)


def layernorm(x, gamma, beta, eps=1e-5, out=None):
    y = layernorm_exact(x, gamma, beta, eps)
    _count()
    return _store(out, y, x.shape)


def layernorm_exact(x, gamma, beta, eps=1e-5):
    _f16(x, "layernorm.x")
    assert x.is_contiguous()
    return F.layer_norm(x.double(), (x.shape[-1],), gamma.double(), beta.double(), eps)


# ------------------------------------------------------------------------------------------------------------- GEMM
def geglu_pack(w, bias):
    n2, k = w.shape
    inner = n2 // 2
    assert inner % 32 == 0
    wp = torch.stack([w[:inner].view(inner // 32, 32, k), w[inner:].view(inner // 32, 32, k)], dim=1).reshape(n2, k)
    bp = torch.stack([bias[:inner].view(inner // 32, 32), bias[inner:].view(inner // 32, 32)], dim=1).reshape(n2)
    return wp.contiguous(), bp.contiguous()


def _epilogue(y, bias, rowbias, rows_per_rowbias, residual2d):
    if bias is not None:
        y = y + bias.double()
    if rowbias is not None:
        idx = torch.arange(y.shape[0], device=y.device) // rows_per_rowbias
        y = y + rowbias.double()[idx]
    if residual2d is not None:
        y = y + residual2d.double()
    return y


def linear(a, w, bias=None, residual=None, out=None, rowbias=None, rows_per_rowbias=0, geglu=False, a2=None):
    y = linear_exact(a, w, bias, residual, rowbias, rows_per_rowbias, geglu, a2)
    _count()
    if out is None:
        return y.to(torch.float16).contiguous()
    assert out.stride(1) == 1
    out.copy_(y.to(torch.float16))
    return out


def linear_exact(a, w, bias=None, residual=None, rowbias=None, rows_per_rowbias=0, geglu=False, a2=None):
    """the float64 value ``linear`` rounds to fp16 at the store, [M, N] (GEGLU: [M, N / 2])"""
    _f16(a, "linear.a")
    if a2 is not None:  # two-source K loop: the logical A is [a | a2]
        _f16(a2, "linear.a2")
        assert a.shape[1] % 64 == 0 and a2.shape[0] == a.shape[0]
        a = torch.cat([a, a2], dim=1)
    assert a.dim() == 2 and a.stride(1) == 1 and w.is_contiguous() and w.shape[1] == a.shape[1]
    M, N = a.shape[0], w.shape[0]
    y = a.double() @ w.double().t()
    if geglu:
        assert residual is None and rowbias is None and N % 64 == 0
        y = _epilogue(y, bias, None, 0, None).view(M, N // 64, 2, 32)
        y = (y[:, :, 0] * F.gelu(y[:, :, 1])).reshape(M, N // 2)  # exact (erf) GELU, one rounding at the store
    else:
        y = _epilogue(y, bias, rowbias, rows_per_rowbias, residual)
    return y


def conv3x3(x, w_packed, bias=None, rowbias=None, rows_per_rowbias=0, residual=None, out=None, n_slots=1, slot_stride=0, stride=1):
    y = conv3x3_exact(x, w_packed, bias, rowbias, rows_per_rowbias, stride)
    NF, H, W = x.shape[0], x.shape[1] // stride, x.shape[2] // stride
    M, Cout = y.shape
    _count()
    if out is None:
        assert n_slots == 1
        if residual is not None:
            y = y + residual.double().reshape(M, Cout)
        return y.to(torch.float16).contiguous().view(NF, H, W, Cout)
    # slot s, row m lives at s * slot_stride + m * ld (ld = the row stride of out; the residual has out's layout)
    rows = lambda t, s: t.as_strided((M, Cout), (t.stride(-2), 1), t.storage_offset() + s * slot_stride)
    for s in range(n_slots):  # one accumulator tile, n_slots stores (+ each slot's own residual): fused PnP injection
        ys = y if residual is None else y + rows(residual, s).double()
        rows(out, s).copy_(ys.to(torch.float16))
    return out


def conv3x3_exact(x, w_packed, bias=None, rowbias=None, rows_per_rowbias=0, stride=1):
    """the float64 accumulator tile of ``conv3x3`` with bias and rowbias, [M, Cout]; each slot's residual is added to it before
    the store rounds to fp16"""
    _f16(x, "conv3x3.x")
    assert x.dim() == 4 and x.is_contiguous()
    NF, H, W, C = x.shape
    Cout = w_packed.shape[0]
    Cin = w_packed.shape[1] // 9
    assert w_packed.shape[1] == 9 * Cin and C <= Cin and H % stride == 0 and W % stride == 0
    w = w_packed.double().view(Cout, 3, 3, Cin).permute(0, 3, 1, 2)[:, :C]  # [Cout][ky][kx][Cin] -> OIHW; padded channels read zeros
    H, W = H // stride, W // stride
    y = F.conv2d(x.double().permute(0, 3, 1, 2), w, None, stride=stride, padding=1).permute(0, 2, 3, 1).reshape(NF * H * W, Cout)
    return _epilogue(y, bias, rowbias, rows_per_rowbias, None)


def upsample2x_conv3x3(x, w_phases, bias=None, out=None):
    """the four 2 x 2 phase convolutions of nearest-up x 2 + conv 3 x 3, interleaved into the [NF, 2H, 2W, Cout] image"""
    y = upsample2x_conv3x3_exact(x, w_phases, bias)
    _count(4)
    return _store(out, y, y.shape)


def upsample2x_conv3x3_exact(x, w_phases, bias=None):
    _f16(x, "upsample2x_conv3x3.x")
    NF, H, W, Cin = x.shape
    Cout = w_phases.shape[1]
    xp = F.pad(x.double().permute(0, 3, 1, 2), (1, 1, 1, 1))  # zero border: input offsets -1 .. +1
    y = torch.zeros(NF, 2 * H, 2 * W, Cout, dtype=torch.float64, device=x.device)
    for ph in range(4):
        py, px = ph >> 1, ph & 1
        w = w_phases[ph].double().view(Cout, 2, 2, Cin).permute(0, 3, 1, 2)  # OIHW, tap (a, b) reads input (i + a - 1 + py, j + b - 1 + px)
        acc = F.conv2d(xp[:, :, py:py + H + 1, px:px + W + 1], w, None if bias is None else bias.double())  # [NF, Cout, H, W]
        y[:, py::2, px::2, :] = acc.permute(0, 2, 3, 1)
    return y


def tconv3(x, w_packed, F_, HW, bias=None, residual=None, out=None):
    y = tconv3_exact(x, w_packed, F_, HW, bias, residual)
    _count()
    return _store(out, y, (x.shape[0], x.shape[1], y.shape[1]))


def tconv3_exact(x, w_packed, F_, HW, bias=None, residual=None):
    """the float64 value ``tconv3`` rounds to fp16 at the store, [B * F * HW, Cout]"""
    _f16(x, "tconv3.x")
    assert x.dim() == 3 and x.is_contiguous() and x.shape[1] == F_ * HW
    B, R, Cin = x.shape
    Cout = w_packed.shape[0]
    w = w_packed.double().view(Cout, 3, Cin).permute(0, 2, 1)[:, :, :, None, None]  # [Cout][kt][Cin] -> [O, I, kt, 1, 1]
    x5 = x.double().view(B, F_, HW, 1, Cin).permute(0, 4, 1, 2, 3)
    y = F.conv3d(x5, w, None, padding=(1, 0, 0)).permute(0, 2, 3, 4, 1).reshape(B * R, Cout)
    return _epilogue(y, bias, None, 0, None if residual is None else residual.reshape(B * R, Cout))


# ------------------------------------------------------------------------------------------------------------- attention
def attention(q, k, v, heads, seq, batch, out, scale=0.125, n_v=1, v_branch_stride=0, o_branch_stride=0,
              frames_mode=False, HW=0, seq_kv=0, kv_batch_div=0):
    def store(rows, o, c):
        out[rows, :o.shape[1]] = o.to(torch.float16)

    _attention(q, k, v, heads, seq, batch, out, scale, n_v, v_branch_stride, o_branch_stride, frames_mode, HW, seq_kv,
               kv_batch_div, store)
    _count()
    return out


def attention_exact(q, k, v, heads, seq, batch, out, scale=0.125, n_v=1, v_branch_stride=0, o_branch_stride=0,
                    frames_mode=False, HW=0, seq_kv=0, kv_batch_div=0, cond=None):
    """the float64 values ``attention`` rounds to fp16 at the store, as a float64 [out rows, heads * 64] matrix (NaN where
    nothing is stored).  cond(p, qh, kh, vh, o) -> a tensor like o: computed from the exact softmax p [..., heads, Lq, Lk] and
    the same operands, returned in the same layout as a second matrix (None without ``cond``)"""
    C = heads * 64
    ref = torch.full((out.shape[0], C), float("nan"), dtype=torch.float64, device=q.device)
    cnd = torch.full_like(ref, float("nan")) if cond is not None else None

    def store(rows, o, c):
        ref[rows] = o
        if c is not None:
            cnd[rows] = c

    _attention(q, k, v, heads, seq, batch, out, scale, n_v, v_branch_stride, o_branch_stride, frames_mode, HW, seq_kv,
               kv_batch_div, store, cond)
    return ref, cnd


def _attention(q, k, v, heads, seq, batch, out, scale, n_v, v_branch_stride, o_branch_stride, frames_mode, HW, seq_kv,
               kv_batch_div, store, cond=None):
    for name, t in (("q", q), ("k", k), ("v", v), ("o", out)):
        _f16(t, "attention." + name)
        assert t.dim() == 2 and t.stride(1) == 1
    C = heads * 64
    ldv, ldo = v.stride(0), out.stride(0)

    def sdpa(qh, kh, vh):  # [..., L, heads, 64] -> (o, cond(...) or None)
        p = torch.softmax(torch.einsum("...qhd,...khd->...hqk", qh.double(), kh.double()) * scale, dim=-1)
        o = torch.einsum("...hqk,...khd->...qhd", p, vh.double())
        return o, (None if cond is None else cond(p, qh.double(), kh.double(), vh.double(), o))

    # n_v = 3: V / out of [source, uncond, cond]; n_v = 2: of [uncond, cond] (a step replayed from cached source Q / K).
    # Either way branch b reads V and writes out at b * its branch stride, with the P of the one Q / K
    branches = range(n_v)
    if not frames_mode:
        div = kv_batch_div if kv_batch_div > 0 else 1
        nk = seq_kv if seq_kv > 0 else seq
        kvb = batch // div
        qh = q[:batch * seq, :C].reshape(batch, seq, heads, 64)
        kh = k[:kvb * nk, :C].reshape(kvb, nk, heads, 64).repeat_interleave(div, dim=0)
        vrows = v_branch_stride // ldv if n_v > 1 else 0
        orows = o_branch_stride // ldo if n_v > 1 else 0
        for b in branches:
            vh = v[b * vrows:b * vrows + kvb * nk, :C].reshape(kvb, nk, heads, 64).repeat_interleave(div, dim=0)
            o, c = sdpa(qh, kh, vh)
            store(slice(b * orows, b * orows + batch * seq), o.reshape(batch * seq, C),
                  None if c is None else c.reshape(batch * seq, C))
    else:
        assert batch % HW == 0 and (seq_kv <= 0 or seq_kv == seq) and kv_batch_div <= 1
        clips, Fr = batch // HW, seq
        rows = clips * Fr * HW
        to_seq = lambda t: t.reshape(clips, Fr, HW, heads, 64).permute(0, 2, 1, 3, 4)  # [clips, HW, F, heads, 64]
        qh, kh = to_seq(q[:rows, :C]), to_seq(k[:rows, :C])
        vrows = v_branch_stride // ldv if n_v > 1 else 0
        orows = o_branch_stride // ldo if n_v > 1 else 0
        for b in branches:
            vh = to_seq(v[b * vrows:b * vrows + rows, :C])
            o, c = sdpa(qh, kh, vh)
            back = lambda t: t.permute(0, 2, 1, 3, 4).reshape(rows, C)  # back to frame-major tokens
            store(slice(b * orows, b * orows + rows), back(o), None if c is None else back(c))


def _tattn_operands(x, wqkv, heads, F_, HW, clips, out, scale, n_v):
    """Q/K/V projection (rounded to fp16, as the QKV GEMM would store them) and the frames-mode ``attention`` arguments that
    read them; n_v = 3: Q, K of every clip from the source clip of the same index (clips ordered [source | uncond | cond])"""
    _f16(x, "temporal_attention_fused.x")
    C = heads * 64
    qkv = (x.double() @ wqkv.double().t()).to(torch.float16)
    if n_v == 1:
        return (qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], heads, F_, clips * HW, out), dict(scale=scale, frames_mode=True, HW=HW)
    assert n_v == 3 and clips % 3 == 0
    src_rows = (clips // 3) * F_ * HW
    return ((qkv[:src_rows, :C], qkv[:src_rows, C:2 * C], qkv[:, 2 * C:], heads, F_, (clips // 3) * HW, out),
            dict(scale=scale, n_v=3, v_branch_stride=src_rows * qkv.stride(0), o_branch_stride=src_rows * out.stride(0),
                 frames_mode=True, HW=HW))


def temporal_attention_fused(x, wqkv, heads, F_, HW, clips, out, scale=0.125, n_v=1):
    """the fused projection + temporal attention: ``attention`` on the fp16-rounded projections (_tattn_operands)"""
    args, kw = _tattn_operands(x, wqkv, heads, F_, HW, clips, out, scale, n_v)
    return attention(*args, **kw)


def temporal_attention_fused_exact(x, wqkv, heads, F_, HW, clips, out, scale=0.125, n_v=1, cond=None):
    """the float64 values ``temporal_attention_fused`` rounds to fp16 at the store, as ``attention_exact`` returns them"""
    args, kw = _tattn_operands(x, wqkv, heads, F_, HW, clips, out, scale, n_v)
    return attention_exact(*args, cond=cond, **kw)


CONTRACTS = dict(upsample2x_conv3x3=upsample2x_conv3x3, temporal_attention_fused=temporal_attention_fused, ddim_step=ddim_step, groupnorm=groupnorm, layernorm=layernorm, geglu_pack=geglu_pack, linear=linear,
                 conv3x3=conv3x3, tconv3=tconv3, attention=attention, launch_count=launch_count)
