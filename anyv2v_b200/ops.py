"""Tensor-level wrappers over the C ABI: PyTorch is used for device memory and streams only.

Every function enqueues hand-written sm_90a kernels on the current CUDA stream; none has a PyTorch fallback.
Activations are channels-last (see include/anyv2v_b200.h).  ``launch_count()`` reports how many of OUR kernels
were launched (bench.py's ``gpu_launches``).
"""
from __future__ import annotations

import ctypes
from typing import Optional

import torch

from . import _lib as L

_launches = 0
_gn_ws: dict = {}
_gn_ws_keepalive: list = []


def launch_count() -> int:
    return _launches


# -- optional in-situ timing (development aid): CUDA events around every wrapper call, keyed by op + shape
_prof = None


def profile_begin():
    global _prof
    _prof = []


def profile_end():
    """-> {key: (calls, total_ms)} sorted by time; synchronises."""
    global _prof
    torch.cuda.synchronize()
    out = {}
    for key, e0, e1 in _prof or []:
        c, t = out.get(key, (0, 0.0))
        out[key] = (c + 1, t + e0.elapsed_time(e1))
    _prof = None
    return dict(sorted(out.items(), key=lambda kv: -kv[1][1]))


class _timed:
    def __init__(self, key):
        self.key = key

    def __enter__(self):
        if _prof is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()

    def __exit__(self, *exc):
        if _prof is not None:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            _prof.append((self.key, self.e0, e1))


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _f16_cuda(t: torch.Tensor, name: str) -> None:
    if not (t.is_cuda and t.dtype == torch.float16):
        raise L.Av2vError(f"{name}: expected a CUDA fp16 tensor, got {t.device}/{t.dtype} (no CPU fallback exists)")


def _require(cond: bool, msg: str) -> None:
    if not cond:
        raise L.Av2vError(msg)


def _row_layout(t: torch.Tensor, name: str, rows: int, cols: int, slots: int = 1, slot_stride: int = 0) -> int:
    """Row stride `ld` of `t` when t addresses element (s, m, n) at s * slot_stride + m * ld + n for s < slots, m < rows,
    n < cols: the layout the kernels store (and read residuals) in.  Leading dims that nest exactly are merged, so an
    [NF, H, W, C] image with a row stride, or a [slots, M, N] stack with a gap between slots, qualifies."""
    _f16_cuda(t, name)
    _require(t.dim() >= 2 and t.shape[-1] == cols and t.stride(-1) == 1,
             f"{name}: expected [..., {cols}] with unit column stride, got shape {tuple(t.shape)} strides {t.stride()}")
    groups = []  # (size, stride) of the leading dims, innermost first
    for size, st in zip(reversed(t.shape[:-1]), reversed(t.stride()[:-1])):
        if size == 1:
            continue
        if groups and st == groups[-1][0] * groups[-1][1]:
            groups[-1] = (groups[-1][0] * size, groups[-1][1])
        else:
            groups.append((size, st))
    groups = groups[::-1]
    if rows == 1:
        ld = cols
        ok = groups == ([(slots, slot_stride)] if slots > 1 else [])
    else:
        ld = groups[-1][1] if groups else 0
        ok = groups == ([(slots, slot_stride), (rows, ld)] if slots > 1 else [(rows, ld)]) or (
            slots > 1 and groups == [(slots * rows, ld)] and slot_stride == rows * ld)
    _require(ok and ld >= cols, f"{name}: shape {tuple(t.shape)} strides {t.stride()} does not hold "
                                f"{slots} x [{rows}, {cols}] rows (slot stride {slot_stride})")
    return ld


def _vector(t: Optional[torch.Tensor], name: str, n: int) -> None:
    if t is not None:
        _f16_cuda(t, name)
        _require(t.is_contiguous() and t.numel() == n, f"{name}: expected {n} contiguous elements, got shape {tuple(t.shape)}")


def _rowbias(t: Optional[torch.Tensor], M: int, N: int, rows_per_rowbias: int) -> None:
    if t is not None:
        _f16_cuda(t, "rowbias")
        _require(rows_per_rowbias > 0, "rowbias needs rows_per_rowbias > 0")
        want = (-(-M // rows_per_rowbias), N)
        _require(t.is_contiguous() and tuple(t.shape) == want, f"rowbias: expected a contiguous {want}, got {tuple(t.shape)}")


# ----------------------------------------------------------------------------------------------------------- K7
def ddim_step(x, v_neg, v_edit, guidance: float, ca: float, cb: float, cc: float, cd: float, out=None,
              inverse: bool = False, coef_dev=None):
    """Fused CFG + v-prediction DDIM update (pipeline_i2vgen_xl.py:1159-1176 / :1407-1420). Elementwise."""
    global _launches
    _f16_cuda(x, "ddim_step.x")
    _f16_cuda(v_neg, "ddim_step.v_neg")
    assert x.is_contiguous() and v_neg.is_contiguous() and x.numel() == v_neg.numel()
    if v_edit is not None:
        _f16_cuda(v_edit, "ddim_step.v_edit")
        assert v_edit.is_contiguous() and v_edit.numel() == x.numel()
    if out is None:
        out = torch.empty_like(x)
    _f16_cuda(out, "ddim_step.out")
    _require(out.is_contiguous() and out.numel() == x.numel(), f"ddim_step.out: expected {x.numel()} contiguous elements")
    if coef_dev is not None:
        assert coef_dev.is_cuda and coef_dev.dtype == torch.float32 and coef_dev.numel() >= 5
    a = L.DdimArgs(_p(x), _p(v_neg), _p(v_edit), _p(out), x.numel(), guidance, ca, cb, cc, cd, _p(coef_dev))
    fn = L.lib().av2v_ddim_inverse_step_f16 if inverse else L.lib().av2v_ddim_step_cfg_f16
    with _timed("ddim_step"):
        L.check(fn(ctypes.byref(a), _stream()), "av2v_ddim_step")
    _launches += 1
    return out


def ddim_step_eta(x, v_neg, v_edit, noise, guidance: float, ca: float, cb: float, cc: float, cd: float, cs: float, out=None,
                  coef_dev=None):
    """``ddim_step`` with DDIM's variance noise (eta > 0): out = fp16(update + fp16(cs * noise)), cd = sqrt(1 - a_prev - cs^2).
    ``noise`` is in x's element order.  ``coef_dev``: device {ca, cb, cc, cd, guidance, cs}."""
    global _launches
    n = x.numel()
    _vector(x, "ddim_step_eta.x", n)
    _vector(v_neg, "ddim_step_eta.v_neg", n)
    _vector(v_edit, "ddim_step_eta.v_edit", n)
    _f16_cuda(noise, "ddim_step_eta.noise")
    _require(noise.device == x.device, f"ddim_step_eta.noise: on {noise.device}, x on {x.device}")
    _vector(noise, "ddim_step_eta.noise", n)
    if out is None:
        out = torch.empty_like(x)
    _f16_cuda(out, "ddim_step_eta.out")
    _require(out.device == x.device, f"ddim_step_eta.out: on {out.device}, x on {x.device}")
    _vector(out, "ddim_step_eta.out", n)
    if coef_dev is not None:
        _require(coef_dev.device == x.device and coef_dev.dtype == torch.float32 and coef_dev.numel() >= 6,
                 f"ddim_step_eta.coef_dev: expected >= 6 fp32 values on {x.device}, got {coef_dev.numel()} "
                 f"{coef_dev.dtype} on {coef_dev.device}")
    a = L.DdimEtaArgs(_p(x), _p(v_neg), _p(v_edit), _p(noise), _p(out), n, guidance, ca, cb, cc, cd, cs, _p(coef_dev))
    with _timed("ddim_step_eta"):
        L.check(L.lib().av2v_ddim_step_eta_f16(ctypes.byref(a), _stream()), "av2v_ddim_step_eta")
    _launches += 1
    return out


def _overlap(a: torch.Tensor, b: Optional[torch.Tensor]) -> bool:
    """whether the byte ranges of two contiguous tensors intersect"""
    if b is None or a.numel() == 0 or b.numel() == 0:
        return False
    a0, b0 = a.data_ptr(), b.data_ptr()
    return a0 < b0 + b.numel() * b.element_size() and b0 < a0 + a.numel() * a.element_size()


def dpmpp2m_step(x, v_neg, v_edit, x0_prev, guidance: float, alpha: float, sigma: float, a: float, b: float, c: float,
                 out=None, coef_dev=None):
    """Fused CFG + DPM-Solver++(2M) step (csrc/elementwise.cu dpm_step_kernel): x0 = alpha*x - sigma*v is written to
    ``x0_prev`` (which holds the previous step's x0 on entry), out = a*x + b*(x0 + c*(x0 - x0_prev)).  ``out`` may be x;
    ``x0_prev`` must not overlap any other operand.  ``coef_dev``: device {alpha, sigma, a, b, c, guidance}."""
    global _launches
    n = x.numel()
    _vector(x, "dpmpp2m_step.x", n)
    _vector(v_neg, "dpmpp2m_step.v_neg", n)
    _vector(v_edit, "dpmpp2m_step.v_edit", n)
    _f16_cuda(x0_prev, "dpmpp2m_step.x0_prev")
    _vector(x0_prev, "dpmpp2m_step.x0_prev", n)
    if out is None:
        out = torch.empty_like(x)
    _f16_cuda(out, "dpmpp2m_step.out")
    _vector(out, "dpmpp2m_step.out", n)
    for name, t in (("v_neg", v_neg), ("v_edit", v_edit), ("x0_prev", x0_prev), ("out", out)):
        _require(t is None or t.device == x.device, f"dpmpp2m_step.{name}: on {t.device if t is not None else None}, x on {x.device}")
    for name, t in (("x", x), ("v_neg", v_neg), ("v_edit", v_edit), ("out", out)):
        _require(not _overlap(x0_prev, t), f"dpmpp2m_step.x0_prev overlaps {name}")
    for name, t in (("v_neg", v_neg), ("v_edit", v_edit)):
        _require(not _overlap(out, t), f"dpmpp2m_step.out overlaps {name} (only x may be updated in place)")
    _require(out.data_ptr() == x.data_ptr() or not _overlap(out, x), "dpmpp2m_step.out partly overlaps x")
    if coef_dev is not None:
        _require(coef_dev.device == x.device and coef_dev.dtype == torch.float32 and coef_dev.numel() >= 6,
                 f"dpmpp2m_step.coef_dev: expected >= 6 fp32 values on {x.device}, got {coef_dev.numel()} "
                 f"{coef_dev.dtype} on {coef_dev.device}")
    args = L.DpmArgs(_p(x), _p(v_neg), _p(v_edit), _p(x0_prev), _p(out), n, guidance, alpha, sigma, a, b, c, _p(coef_dev))
    with _timed("dpmpp2m_step"):
        L.check(L.lib().av2v_dpmpp2m_step_f16(ctypes.byref(args), _stream()), "av2v_dpmpp2m_step")
    _launches += 1
    return out


# ----------------------------------------------------------------------------------------------------------- K6
def groupnorm(x, gamma, beta, groups: int, eps: float, silu: bool, out=None, x2=None, partition_samples: int = 0):
    """GroupNorm(+SiLU) over x[n_samples, rows, C] (channels-last). pnp_utils.py:48-49,92,104.
    x2: second source — the logical input is [x | x2] along the channels (skip-concat without torch.cat); out is [n, rows, C1 + C2].
    partition_samples (>= n_samples): reduce each sample as a call of that many samples would, so that its statistics are
    bit for bit those of that call."""
    global _launches
    _f16_cuda(x, "groupnorm.x")
    assert x.dim() == 3 and x.is_contiguous()
    n, rows, C = x.shape
    C1 = C
    if x2 is not None:
        _f16_cuda(x2, "groupnorm.x2")
        assert x2.dim() == 3 and x2.is_contiguous() and x2.shape[:2] == x.shape[:2]
        C = C1 + x2.shape[2]
    if out is None:
        out = torch.empty((n, rows, C), dtype=x.dtype, device=x.device)
    _f16_cuda(out, "groupnorm.out")
    _require(out.is_contiguous() and tuple(out.shape) == (n, rows, C), f"groupnorm.out: expected a contiguous {(n, rows, C)}")
    _vector(gamma, "groupnorm.gamma", C)
    _vector(beta, "groupnorm.beta", C)
    need = L.lib().av2v_groupnorm_workspace_floats(n, C)
    key = x.device.index
    ws = _gn_ws.get(key)
    if ws is None or ws.numel() < need:
        # never free an old workspace: a captured CUDA graph may still hold its address
        _gn_ws_keepalive.append(ws)
        ws = torch.empty(max(need, 1 << 22), dtype=torch.float32, device=x.device)
        _gn_ws[key] = ws
    a = L.GroupNormArgs(_p(x), _p(out), _p(gamma), _p(beta), _p(ws), n, rows, C, groups, eps, 1 if silu else 0, _p(x2), C1)
    with _timed(f"groupnorm n={n} rows={rows} C={C}"):
        if partition_samples:
            L.check(L.lib().av2v_groupnorm_silu_part_f16(ctypes.byref(a), partition_samples, _stream()),
                    "av2v_groupnorm_silu_part_f16")
        else:
            L.check(L.lib().av2v_groupnorm_silu_f16(ctypes.byref(a), _stream()), "av2v_groupnorm_silu_f16")
    _launches += 1
    return out


# ----------------------------------------------------------------------------------------------------------- GEMM
def _gemm(args: L.GemmArgs):
    global _launches
    kind = ("linear", "conv3x3", "tconv3")[args.mode] + ("+geglu" if args.geglu else "") + ("+res" if args.residual else "")
    with _timed(f"{kind} M={args.M} N={args.N} K={args.K} slots={args.n_slots}"):
        L.check(L.lib().av2v_gemm_f16(ctypes.byref(args), _stream()), "av2v_gemm_f16")
    _launches += 1


def linear(a, w, bias=None, residual=None, out=None, rowbias=None, rows_per_rowbias: int = 0, geglu: bool = False, a2=None):
    """out[M,N] = a[M,K] @ w[N,K]^T (+bias) (+rowbias[m//rpr]) (+residual). a may be a row-strided view.
    geglu=True: w/bias are block-32 interleaved [h|gate] (see geglu_pack) and out is [M, N/2] = h * gelu_erf(gate).
    a2: second source of the K loop — the logical A is [a | a2] along K (a.shape[1] % 64 == 0): the skip-connection concat of
    the up blocks without a materialised torch.cat."""
    _f16_cuda(a, "linear.a")
    assert a.dim() == 2 and a.stride(1) == 1 and w.is_contiguous()
    M, K = a.shape
    if a2 is not None:
        _f16_cuda(a2, "linear.a2")
        assert a2.dim() == 2 and a2.stride(1) == 1 and a2.shape[0] == M and K % 64 == 0
        K = K + a2.shape[1]
    _f16_cuda(w, "linear.w")
    N = w.shape[0]
    assert w.shape[1] == K
    if out is None:
        out = torch.empty((M, N // 2 if geglu else N), dtype=torch.float16, device=a.device)
    ldo = _row_layout(out, "linear.out", M, N // 2 if geglu else N)
    if residual is not None:
        _require(_row_layout(residual, "linear.residual", M, N) == ldo, "linear.residual: row stride differs from out's")
    _vector(bias, "linear.bias", N)
    _rowbias(rowbias, M, N, rows_per_rowbias)
    g = L.GemmArgs()
    g.mode = L.A_LINEAR
    g.a, g.w, g.M, g.N, g.K, g.lda = _p(a), _p(w), M, N, K, a.stride(0)
    g.bias, g.rowbias, g.rows_per_rowbias = _p(bias), _p(rowbias), rows_per_rowbias
    g.residual, g.out, g.ldo, g.n_slots, g.slot_stride = _p(residual), _p(out), ldo, 1, 0
    g.geglu = 1 if geglu else 0
    if a2 is not None:
        g.a2, g.k_split, g.lda2 = _p(a2), a.shape[1], a2.stride(0)
    _gemm(g)
    return out


def geglu_pack(w, bias):
    """Interleave the h / gate halves of GEGLU.proj in blocks of 32 output features (layout of av2v_gemm_args.geglu)."""
    n2, k = w.shape
    inner = n2 // 2
    assert inner % 32 == 0
    wp = torch.stack([w[:inner].view(inner // 32, 32, k), w[inner:].view(inner // 32, 32, k)], dim=1).reshape(n2, k)
    bp = torch.stack([bias[:inner].view(inner // 32, 32), bias[inner:].view(inner // 32, 32)], dim=1).reshape(n2)
    return wp.contiguous(), bp.contiguous()


def layernorm(x, gamma, beta, eps: float = 1e-5, out=None):
    """LayerNorm over the last dim of a contiguous [..., C] tensor."""
    global _launches
    _f16_cuda(x, "layernorm.x")
    assert x.is_contiguous()
    C = x.shape[-1]
    rows = x.numel() // C
    if out is None:
        out = torch.empty_like(x)
    _f16_cuda(out, "layernorm.out")
    _require(out.is_contiguous() and out.shape == x.shape, f"layernorm.out: expected a contiguous {tuple(x.shape)}")
    _vector(gamma, "layernorm.gamma", C)
    _vector(beta, "layernorm.beta", C)
    a = L.LayerNormArgs(_p(x), _p(out), _p(gamma), _p(beta), rows, C, eps)
    with _timed(f"layernorm rows={rows} C={C}"):
        L.check(L.lib().av2v_layernorm_f16(ctypes.byref(a), _stream()), "av2v_layernorm_f16")
    _launches += 1
    return out


def conv3x3(x, w_packed, bias=None, rowbias=None, rows_per_rowbias: int = 0, residual=None, out=None,
            n_slots: int = 1, slot_stride: int = 0, stride: int = 1):
    """3x3 / pad 1 convolution as an implicit GEMM. x: [NF,H,W,C] contiguous (channels-last),
    w_packed: [Cout, 9*Cin] (= conv.weight.permute(0,2,3,1).reshape). out: [n_slots][NF*(H/stride)*(W/stride), Cout].
    out (and residual, in the same layout) may have a row stride; with n_slots > 1, slot s starts slot_stride elements after
    slot s - 1.  stride 2 = Downsample2D (each A row gathers the taps at twice the output coordinates).  C < Cin (conv_in: 8
    channels): the weights are zero-padded per tap to Cin = 64 and the missing channels of every K block are zero-filled by
    the cp.async channel predicate, as are out-of-image taps."""
    _f16_cuda(x, "conv3x3.x")
    assert x.dim() == 4 and x.is_contiguous()
    NF, H, W, C = x.shape
    Cout = w_packed.shape[0]
    assert w_packed.shape[1] % 9 == 0 and w_packed.is_contiguous()
    Cin = w_packed.shape[1] // 9
    assert C <= Cin and C % 8 == 0
    M = NF * (H // stride) * (W // stride)
    if out is None:
        assert n_slots == 1
        out = torch.empty((NF, H // stride, W // stride, Cout), dtype=torch.float16, device=x.device)
    ldo = _row_layout(out, "conv3x3.out", M, Cout, n_slots, slot_stride)
    if residual is not None:
        _require(_row_layout(residual, "conv3x3.residual", M, Cout, n_slots, slot_stride) == ldo,
                 "conv3x3.residual: row stride differs from out's")
    _vector(bias, "conv3x3.bias", Cout)
    _rowbias(rowbias, M, Cout, rows_per_rowbias)
    g = L.GemmArgs()
    g.mode = L.A_CONV3X3
    g.a, g.w, g.M, g.N, g.K = _p(x), _p(w_packed), M, Cout, 9 * Cin
    g.NF, g.H, g.W, g.Cin = NF, H, W, Cin
    g.stride, g.a_channels = stride, (C if C != Cin else 0)
    g.bias, g.rowbias, g.rows_per_rowbias = _p(bias), _p(rowbias), rows_per_rowbias
    g.residual, g.out, g.ldo, g.n_slots, g.slot_stride = _p(residual), _p(out), ldo, n_slots, slot_stride
    _gemm(g)
    return out


def upsample2x_conv3x3(x, w_phases, bias=None, out=None):
    """Upsample2D = nearest-neighbour x 2 followed by a 3x3 / pad 1 convolution (SURVEY A.7; twin at seine/models/resnet.py:24-76)
    WITHOUT the up-sampled tensor: output pixel (2i+py, 2j+px) only sees a 2 x 2 neighbourhood of the input, with the 3 x 3 taps
    that land on the same input pixel pre-summed (``pack_upsample_weights``).  x: [NF,H,W,Cin]; w_phases: [4][Cout, 4*Cin];
    -> [NF, 2H, 2W, Cout].  Four launches of the implicit GEMM (K = 4*Cin each): 4/9 of the direct layer's FLOPs, and the 4x
    larger intermediate is neither written nor read."""
    _f16_cuda(x, "upsample2x_conv3x3.x")
    assert x.dim() == 4 and x.is_contiguous() and w_phases.dim() == 3 and w_phases.shape[0] == 4 and w_phases.is_contiguous()
    NF, H, W, Cin = x.shape
    Cout = w_phases.shape[1]
    assert w_phases.shape[2] == 4 * Cin
    if out is None:
        out = torch.empty((NF, 2 * H, 2 * W, Cout), dtype=torch.float16, device=x.device)
    ldo = _row_layout(out, "upsample2x_conv3x3.out", NF * 4 * H * W, Cout)
    _require(out.dim() == 4 and tuple(out.shape[:3]) == (NF, 2 * H, 2 * W), f"upsample2x_conv3x3.out: expected {(NF, 2 * H, 2 * W, Cout)}")
    _vector(bias, "upsample2x_conv3x3.bias", Cout)
    for ph in range(4):
        g = L.GemmArgs()
        g.mode = L.A_CONV3X3
        g.a, g.w, g.M, g.N, g.K = _p(x), _p(w_phases[ph]), NF * H * W, Cout, 4 * Cin
        g.NF, g.H, g.W, g.Cin = NF, H, W, Cin
        g.bias, g.out, g.ldo, g.n_slots, g.slot_stride = _p(bias), _p(out), ldo, 1, 0
        g.up2_phase = ph + 1
        _gemm(g)
    return out


def pack_upsample_weights(w):
    """conv weight [Cout, Cin, 3, 3] -> [4][Cout, 2*2*Cin]: for output phase (py, px) the tap (a, b) of the 2 x 2 neighbourhood
    (input offsets a - 1 + py, b - 1 + px) carries the sum of the 3 x 3 taps that read the same input pixel after the nearest
    up-sampling: rows {0 | 1,2} for py = 0, {0,1 | 2} for py = 1 (columns alike).  Summed in fp32, rounded to fp16 once."""
    sets = {0: ((0,), (1, 2)), 1: ((0, 1), (2,))}
    wf = w.float()
    co, ci = w.shape[0], w.shape[1]
    out = torch.empty((4, co, 2, 2, ci), dtype=torch.float32, device=w.device)
    for py in (0, 1):
        for px in (0, 1):
            for a in (0, 1):
                for b in (0, 1):
                    acc = 0
                    for ky in sets[py][a]:
                        for kx in sets[px][b]:
                            acc = acc + wf[:, :, ky, kx]
                    out[py * 2 + px, :, a, b, :] = acc
    return out.reshape(4, co, 4 * ci).to(w.dtype).contiguous()


def tconv3(x, w_packed, F: int, HW: int, bias=None, residual=None, out=None):
    """Conv3d (3,1,1) / pad (1,0,0) over frames. x: [B, F*HW, Cin] contiguous (frame-major channels-last),
    w_packed: [Cout, 3*Cin] (= conv.weight[:, :, :, 0, 0].permute(0,2,1).reshape)."""
    _f16_cuda(x, "tconv3.x")
    assert x.dim() == 3 and x.is_contiguous() and x.shape[1] == F * HW
    B, R, Cin = x.shape
    Cout = w_packed.shape[0]
    assert w_packed.shape[1] == 3 * Cin and w_packed.is_contiguous()
    if out is None:
        out = torch.empty((B, R, Cout), dtype=torch.float16, device=x.device)
    ldo = _row_layout(out, "tconv3.out", B * R, Cout)
    if residual is not None:
        _require(_row_layout(residual, "tconv3.residual", B * R, Cout) == ldo, "tconv3.residual: row stride differs from out's")
    _vector(bias, "tconv3.bias", Cout)
    g = L.GemmArgs()
    g.mode = L.A_TCONV3
    g.a, g.w, g.M, g.N, g.K = _p(x), _p(w_packed), B * R, Cout, 3 * Cin
    g.B, g.rows_per_clip, g.HW, g.Cin = B, R, HW, Cin
    g.bias, g.residual, g.out, g.ldo, g.n_slots, g.slot_stride = _p(bias), _p(residual), _p(out), ldo, 1, 0
    _gemm(g)
    return out


# ----------------------------------------------------------------------------------------------------------- FreeU
def freeu(hidden, skip, b: float, s: float, out=None):
    """FreeU at one skip connection of up_blocks[0] / [1] (diffusers `apply_freeu`, csrc/freeu.cu): scales hidden[..., :Ch/2]
    by b IN PLACE and returns fourier_filter(skip, threshold=1, scale=s).  hidden: [NF,H,W,Ch]; skip, out: [NF,H,W,Cs];
    all contiguous (channels-last frames)."""
    global _launches
    _f16_cuda(hidden, "freeu.hidden")
    _f16_cuda(skip, "freeu.skip")
    _require(skip.dim() == 4 and skip.is_contiguous(), f"freeu.skip: expected a contiguous [NF, H, W, C], got shape "
                                                        f"{tuple(skip.shape)} strides {skip.stride()}")
    NF, H, W, Cs = skip.shape
    _require(hidden.dim() == 4 and hidden.is_contiguous() and tuple(hidden.shape[:3]) == (NF, H, W),
             f"freeu.hidden: expected a contiguous [{NF}, {H}, {W}, C], got shape {tuple(hidden.shape)} strides {hidden.stride()}")
    if out is None:
        out = torch.empty_like(skip)
    _f16_cuda(out, "freeu.out")
    _require(out.is_contiguous() and out.shape == skip.shape, f"freeu.out: expected a contiguous {tuple(skip.shape)}, got shape "
                                                               f"{tuple(out.shape)} strides {out.stride()}")
    _require(hidden.device == skip.device == out.device, "freeu: hidden, skip and out must be on the same device")
    a = L.FreeUArgs(_p(hidden), _p(skip), _p(out), NF, H, W, hidden.shape[3], Cs, b, s)
    with _timed(f"freeu NF={NF} H={H} W={W} Ch={hidden.shape[3]} Cs={Cs}"):
        L.check(L.lib().av2v_freeu_f16(ctypes.byref(a), _stream()), "av2v_freeu_f16")
    _launches += 1
    return out


# ----------------------------------------------------------------------------------------------------------- VAE tiles
def tile_stitch(tiles, H: int, W: int, tile: int, step: int, blend: int, row_limit: int, out=None):
    """The seams of diffusers' tiled VAE encode / decode (csrc/vae_tiles.cu): ``tiles[n][i][j]`` is the RAW output [C, t_i, t_j]
    (any strides) of tile (i, j) of image n, with t_k = min(tile, L - k * step); -> [N, C, H, W] (channels-last unless ``out``
    is given), the tiles blended as the reference's in-place loop does and their first ``row_limit`` pixels kept."""
    global _launches
    N = len(tiles)
    _require(N > 0 and all(len(r) == len(tiles[0]) for r in tiles) and len(tiles[0]) > 0 and tiles[0][0],
             "tile_stitch: expected a non-empty [N][rows][cols] table of tiles")
    rows, cols = len(tiles[0]), len(tiles[0][0])
    C = tiles[0][0][0].shape[0]
    dev = tiles[0][0][0].device
    ext_h = [min(tile, H - i * step) for i in range(rows)]
    ext_w = [min(tile, W - j * step) for j in range(cols)]
    table = []
    for n, image in enumerate(tiles):
        for i, row in enumerate(image):
            _require(len(row) == cols, f"tile_stitch: image {n} row {i} has {len(row)} tiles, expected {cols}")
            for j, t in enumerate(row):
                _f16_cuda(t, f"tile_stitch.tiles[{n}][{i}][{j}]")
                _require(t.device == dev and tuple(t.shape) == (C, ext_h[i], ext_w[j]),
                         f"tile_stitch.tiles[{n}][{i}][{j}]: expected {(C, ext_h[i], ext_w[j])} on {dev}, got {tuple(t.shape)} "
                         f"on {t.device}")
                table.append([t.data_ptr(), *t.stride()])
    if out is None:
        out = torch.empty(N, H, W, C, device=dev, dtype=torch.float16).permute(0, 3, 1, 2)
    _f16_cuda(out, "tile_stitch.out")
    _require(out.device == dev and tuple(out.shape) == (N, C, H, W),
             f"tile_stitch.out: expected {(N, C, H, W)} on {dev}, got {tuple(out.shape)} on {out.device}")
    desc = torch.tensor(table, dtype=torch.int64).to(dev)  # [N * rows * cols] av2v_tile_desc
    a = L.TileStitchArgs(desc.data_ptr(), _p(out), *out.stride(), N, C, H, W, rows, cols, tile, step, blend, row_limit)
    with _timed(f"tile_stitch N={N} C={C} {H}x{W} tiles={rows}x{cols}"):
        L.check(L.lib().av2v_tile_stitch_f16(ctypes.byref(a), _stream()), "av2v_tile_stitch_f16")
    _launches += 1
    return out


# ----------------------------------------------------------------------------------------------------------- attention
def _reach(t: torch.Tensor, name: str, rows: int, cols: int, offset: int = 0) -> None:
    """a 2-D token matrix must hold columns [0, cols) and reach element offset + (rows - 1) * ld + cols - 1 of its storage"""
    ld = t.stride(0)
    _require(t.shape[1] >= cols and (t.shape[0] - 1) * ld + t.shape[1] >= offset + (rows - 1) * ld + cols,
             f"{name}: shape {tuple(t.shape)} (row stride {ld}) does not cover {rows} rows x {cols} columns at offset {offset}")


def attention(q, k, v, heads: int, seq: int, batch: int, out, scale: float = 0.125, n_v: int = 1,
              v_branch_stride: int = 0, o_branch_stride: int = 0, frames_mode: bool = False, HW: int = 0,
              seq_kv: int = 0, kv_batch_div: int = 0):
    """PnP self-attention core (pnp_utils.py:189-210 / 295-316). q,k,v,out: 2-D token matrices (row-strided views ok).
    frames_mode: temporal attention over frame-major tokens [batch / HW clips][seq = F frames][HW][*]; any F >= 1.
    n_v = 3: q, k of the source branch, V / out of [source, uncond, cond] at v / out + b * branch stride; n_v = 2: the same
    with the two edit branches only (each bit-identical to the same branch at n_v = 3)."""
    global _launches
    for name, t in (("q", q), ("k", k), ("v", v), ("o", out)):
        _f16_cuda(t, "attention." + name)
        assert t.dim() == 2 and t.stride(1) == 1
    _require(n_v in (1, 2, 3), f"attention: n_v must be 1, 2 or 3, got {n_v}")
    C, extra = heads * 64, n_v - 1
    kv_rows = batch * seq if frames_mode else batch // max(kv_batch_div, 1) * (seq_kv if seq_kv > 0 else seq)
    _reach(q, "attention.q", batch * seq, C)
    _reach(k, "attention.k", kv_rows, C)
    _reach(v, "attention.v", kv_rows, C, extra * v_branch_stride)
    _reach(out, "attention.o", batch * seq, C, extra * o_branch_stride)
    a = L.AttnArgs()
    a.seq_mode = L.SEQ_FRAMES if frames_mode else L.SEQ_ROWS
    a.q, a.k, a.v, a.o = _p(q), _p(k), _p(v), _p(out)
    a.ldq, a.ldk, a.ldv, a.ldo = q.stride(0), k.stride(0), v.stride(0), out.stride(0)
    a.batch, a.seq, a.heads, a.HW, a.n_v = batch, seq, heads, HW, n_v
    a.v_branch_stride, a.o_branch_stride, a.scale = v_branch_stride, o_branch_stride, scale
    a.seq_kv, a.kv_batch_div = seq_kv, kv_batch_div
    with _timed(f"attention {'frames' if frames_mode else 'rows'} nv={n_v} batch={batch} seq={seq} heads={heads}"):
        L.check(L.lib().av2v_attn_pnp_f16(ctypes.byref(a), _stream()), "av2v_attn_pnp_f16")
    _launches += 1
    return out


def temporal_attention_fused(x, wqkv, heads: int, F: int, HW: int, clips: int, out, scale: float = 0.125, n_v: int = 1):
    """Temporal self-attention with the Q/K/V projection fused in (csrc/attention_wgmma.cu; pnp_utils.py:247-334).
    x: frame-major tokens [clips*F*HW, Cx]; wqkv: [3*heads*64, Cx]; out: [clips*F*HW, heads*64]; 1 <= F <= 128 (longer clips
    take ops.linear + ops.attention).  n_v = 3: PnP-injected step,
    clips ordered [source | uncond | cond]; Q, K of every clip come from the source clip of the same index (pnp_utils.py:295-302)."""
    global _launches
    for name, t in (("x", x), ("wqkv", wqkv), ("o", out)):
        _f16_cuda(t, "temporal_attention_fused." + name)
        assert t.dim() == 2 and t.stride(1) == 1
    assert wqkv.is_contiguous() and wqkv.shape[0] == 3 * heads * 64 and wqkv.shape[1] == x.shape[1]
    assert x.shape[0] == clips * F * HW == out.shape[0]
    _require(out.shape[1] >= heads * 64, f"temporal_attention_fused.o: {out.shape[1]} columns, the heads need {heads * 64}")
    a = L.TAttnFusedArgs(_p(x), _p(wqkv), _p(out), x.stride(0), out.stride(0), clips, F, HW, heads, x.shape[1], scale, n_v)
    with _timed(f"temporal attention fused nv={n_v} clips={clips} F={F} HW={HW} heads={heads} Cx={x.shape[1]}"):
        L.check(L.lib().av2v_tattn_fused_f16(ctypes.byref(a), _stream()), "av2v_tattn_fused_f16")
    _launches += 1
    return out


def temporal_attention_fused_qksrc(x, qk_src, wqkv, heads: int, F: int, HW: int, clips: int, out, scale: float = 0.125):
    """``temporal_attention_fused`` of a PnP-injected step with Q and K projected from ``qk_src`` (the source branch's tokens
    cached by an earlier edit of the clip): x: the edit clips [uncond | cond], frame-major [clips*F*HW, Cx]; qk_src: the
    clips / 2 source clips [clips/2*F*HW, Cx] (its own row stride); out: [clips*F*HW, heads*64].  Clip c + b * clips / 2
    attends with the Q, K of source clip c; each clip's output is bit-identical to the same clip at n_v = 3."""
    global _launches
    for name, t in (("x", x), ("qk_src", qk_src), ("wqkv", wqkv), ("o", out)):
        _f16_cuda(t, "temporal_attention_fused_qksrc." + name)
        _require(t.dim() == 2 and t.stride(1) == 1, f"temporal_attention_fused_qksrc.{name}: expected a 2-D row-major matrix")
    _require(wqkv.is_contiguous() and wqkv.shape[0] == 3 * heads * 64 and wqkv.shape[1] == x.shape[1] == qk_src.shape[1],
             "temporal_attention_fused_qksrc: wqkv must be a contiguous [3*heads*64, Cx] matching x and qk_src")
    _require(clips % 2 == 0 and x.shape[0] == clips * F * HW == out.shape[0] and qk_src.shape[0] == clips // 2 * F * HW,
             f"temporal_attention_fused_qksrc: x / out need {clips} clips and qk_src {clips // 2} of {F} x {HW} tokens")
    _require(out.shape[1] >= heads * 64, f"temporal_attention_fused_qksrc.o: {out.shape[1]} columns, the heads need {heads * 64}")
    _require(x.device == qk_src.device == wqkv.device == out.device, "temporal_attention_fused_qksrc: tensors on different devices")
    a = L.TAttnFusedQkSrcArgs(_p(x), _p(qk_src), _p(wqkv), _p(out), x.stride(0), qk_src.stride(0), out.stride(0), clips, F, HW,
                              heads, x.shape[1], scale)
    with _timed(f"temporal attention fused qksrc clips={clips} F={F} HW={HW} heads={heads} Cx={x.shape[1]}"):
        L.check(L.lib().av2v_tattn_fused_qksrc_f16(ctypes.byref(a), _stream()), "av2v_tattn_fused_qksrc_f16")
    _launches += 1
    return out
