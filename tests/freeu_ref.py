"""TEST INFRASTRUCTURE — FreeU (arXiv:2309.11497) for the tests of anyv2v_b200's FreeU path; nothing outside tests/ imports it.

1. Oracle: diffusers 0.26.3 `fourier_filter` (torch.fft) and `apply_freeu` [recalled: diffusers is not vendored], reached from
   the reference through pipeline_i2vgen_xl.py:623-650 (`enable_freeu` -> `unet.enable_freeu`), and FreeU for the oracle UNet
   of oracle/unet_ref.py: ``enable_freeu(net, ...)`` / ``disable_freeu(net)`` set the diffusers attributes on its up blocks and
   give them the FreeU step of diffusers' `UpBlock3D.forward` / `CrossAttnUpBlock3D.forward`.
2. Contract of `ops.freeu` (csrc/freeu.cu) in the style of tests/kernel_contracts.py: float64 closed form, one rounding to
   fp16; ``patch_ops`` swaps it in next to the ``emulated_ops`` fixture.
"""
from __future__ import annotations

import math

import torch

import kernel_contracts
from oracle import unet_ref


# ------------------------------------------------------------------------------------------------------------- oracle
def fourier_filter(x_in: torch.Tensor, threshold: int, scale: float) -> torch.Tensor:
    x = x_in
    B, C, H, W = x.shape
    # non-power-of-2 planes: cuFFT half does not take them.  diffusers casts to float32 unconditionally; here float64 is
    # kept, so that the tests can evaluate this restatement exactly (the reference only runs fp16 and fp32, which match)
    if ((W & (W - 1)) != 0 or (H & (H - 1)) != 0) and x.dtype != torch.float64:
        x = x.to(dtype=torch.float32)
    x_freq = torch.fft.fftn(x, dim=(-2, -1))
    x_freq = torch.fft.fftshift(x_freq, dim=(-2, -1))
    B, C, H, W = x_freq.shape
    mask = torch.ones((B, C, H, W), device=x.device)
    crow, ccol = H // 2, W // 2
    mask[..., crow - threshold:crow + threshold, ccol - threshold:ccol + threshold] = scale
    x_freq = x_freq * mask
    x_freq = torch.fft.ifftshift(x_freq, dim=(-2, -1))
    x_filtered = torch.fft.ifftn(x_freq, dim=(-2, -1)).real
    return x_filtered.to(dtype=x_in.dtype)


def apply_freeu(resolution_idx, hidden_states, res_hidden_states, **freeu_kwargs):
    """FreeU at one skip connection of up block `resolution_idx` (only 0 and 1 change anything); hidden_states is scaled in place"""
    if resolution_idx == 0:
        num_half_channels = hidden_states.shape[1] // 2
        hidden_states[:, :num_half_channels] = hidden_states[:, :num_half_channels] * freeu_kwargs["b1"]
        res_hidden_states = fourier_filter(res_hidden_states, threshold=1, scale=freeu_kwargs["s1"])
    if resolution_idx == 1:
        num_half_channels = hidden_states.shape[1] // 2
        hidden_states[:, :num_half_channels] = hidden_states[:, :num_half_channels] * freeu_kwargs["b2"]
        res_hidden_states = fourier_filter(res_hidden_states, threshold=1, scale=freeu_kwargs["s2"])
    return hidden_states, res_hidden_states


class FreeUUpBlock3D(unet_ref.UpBlock3D):
    """oracle/unet_ref.UpBlock3D with the FreeU step of diffusers' up blocks before each skip concat"""

    def forward(self, x, skips, temb, ctx, num_frames):
        is_freeu_enabled = (getattr(self, "s1", None) and getattr(self, "s2", None) and getattr(self, "b1", None)
                            and getattr(self, "b2", None))
        for i in range(len(self.resnets)):
            res_hidden = skips[-1]
            skips = skips[:-1]
            if is_freeu_enabled:
                x, res_hidden = apply_freeu(self.resolution_idx, x, res_hidden, s1=self.s1, s2=self.s2, b1=self.b1, b2=self.b2)
            x = torch.cat([x, res_hidden], dim=1)
            x = self._layer(i, x, temb, ctx, num_frames)
        if self.upsamplers is not None:
            x = self.upsamplers[0](x)
        return x


def enable_freeu(net: unet_ref.I2VGenXLUNet, s1, s2, b1, b2):
    """diffusers I2VGenXLUNet.enable_freeu on the oracle UNet (up block i has resolution_idx = i)"""
    for i, upsample_block in enumerate(net.up_blocks):
        upsample_block.__class__ = FreeUUpBlock3D
        upsample_block.resolution_idx = i
        setattr(upsample_block, "s1", s1)
        setattr(upsample_block, "s2", s2)
        setattr(upsample_block, "b1", b1)
        setattr(upsample_block, "b2", b2)


def disable_freeu(net: unet_ref.I2VGenXLUNet):
    freeu_keys = {"s1", "s2", "b1", "b2"}
    for upsample_block in net.up_blocks:
        for k in freeu_keys:
            if hasattr(upsample_block, k) or getattr(upsample_block, k, None) is not None:
                setattr(upsample_block, k, None)


# ------------------------------------------------------------------------------------------------------------- contract
def fourier_filter_closed_form(x, s):
    """fourier_filter(x, threshold=1, scale=s) of channels-last planes x[..., H, W, C] without an FFT: the shifted window
    [H//2-1 : H//2+1]^2 holds the modes {0, -1} of each axis (only {0} on a size-1 axis), so y = x + (s - 1) / (H W) * the sum
    over those modes of Re(X[mode] e^{-i angle}).  Evaluated in x's dtype (float64 in the contract)."""
    H, W = x.shape[-3], x.shape[-2]
    th = (2 * math.pi / H) * torch.arange(H, dtype=x.dtype, device=x.device)[:, None].expand(H, W)
    ph = (2 * math.pi / W) * torch.arange(W, dtype=x.dtype, device=x.device)[None, :].expand(H, W)
    angles = [torch.zeros(H, W, dtype=x.dtype, device=x.device)]
    if H > 1:
        angles.append(th)
    if W > 1:
        angles.append(ph)
    if H > 1 and W > 1:
        angles.append(th + ph)
    corr = torch.zeros_like(x)
    for ang in angles:
        c, sn = torch.cos(ang)[..., None], torch.sin(ang)[..., None]
        corr += (x * c).sum(dim=(-3, -2), keepdim=True) * c + (x * sn).sum(dim=(-3, -2), keepdim=True) * sn
    return x + (s - 1.0) / (H * W) * corr


def freeu(hidden, skip, b, s, out=None):
    """csrc/freeu.cu: hidden[..., :Ch/2] = fp16(fp32(x) * fp32(b)) in place; out = fourier_filter(skip, threshold=1, scale=s) in
    float64 (closed form above) with s the fp32 value the kernel receives, one rounding to fp16"""
    assert hidden.dtype == skip.dtype == torch.float16, "freeu: the C ABI takes fp16 tensors"
    half = hidden.shape[-1] // 2
    hidden[..., :half] = (hidden[..., :half].float() * torch.tensor(b, dtype=torch.float32)).to(torch.float16)
    y = fourier_filter_closed_form(skip.double(), float(torch.tensor(s, dtype=torch.float32)))
    kernel_contracts._count()
    return kernel_contracts._store(out, y, skip.shape)


def patch_ops(monkeypatch):
    """ops.freeu -> the contract for one test (use together with the emulated_ops fixture, which patches the other ops)"""
    from anyv2v_b200 import ops
    monkeypatch.setattr(ops, "freeu", freeu)
