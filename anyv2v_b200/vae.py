"""AutoencoderKL (the KL-f8 VAE of `ali-vilab/i2vgen-xl`) on the hand-written sm_90a kernels — SURVEY §8f row 4: the
steps either side of the sampling loops, `encode_vae_video` (i2vgen-xl/pipelines/pipeline_i2vgen_xl.py:565-592) and
`decode_latents` (:443-463).

Module / parameter names are diffusers' (`encoder.down_blocks.0.resnets.0.norm1.weight`, `decoder.mid_block.attentions.0.to_q…`,
`quant_conv`, `post_quant_conv`), so a real `diffusion_pytorch_model` state_dict loads unchanged.  Activations are
channels-last fp16 end to end; every 3x3 convolution with Cin % 64 == 0 (all but `conv_in`), every GroupNorm(+SiLU),
the 1x1 shortcuts and the attention projections run on `anyv2v_b200.ops` (wgmma implicit GEMM, fused bias/residual
epilogue).  Left on library calls for now
(`next_rows`): `conv_in` (3 -> 128), the convolutions that end in 3 / 8 / 4 channels, the stride-2 down-sampling
convolutions, and the single-head 512-wide mid-block attention core (head_dim 512 is outside the d = 64 kernel).
There is no CPU path.

Unlike the reference, which encodes and decodes one frame per VAE call (`decode_chunk_size=1`, one `vae.encode` per
frame), all frames go through in one batch — the per-frame results are identical (every op is per-sample).

Memory knobs (diffusers 0.26.3 `AutoencoderKL`, reached through pipeline_i2vgen_xl.py:191-222): `enable_slicing` runs the
encoder / decoder one sample at a time; `enable_tiling` splits images larger than `tile_sample_min_size` into overlapping
tiles and blends the seams.  Tiles of one shape, from all images of the call, go through the VAE together (`tile_batch`
per pass); the seams are blended by one kernel (`ops.tile_stitch`) instead of diffusers' row-by-row loop.
"""
from __future__ import annotations

from dataclasses import dataclass
from types import SimpleNamespace
from typing import List, Sequence, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import next_rows as nr
from . import ops
from .unet_i2vgen_xl import Conv3x3, GroupNorm, Linear, to_nchw_view, to_nhwc

SD_VAE_CONFIG = dict(in_channels=3, out_channels=3, latent_channels=4, block_out_channels=(128, 256, 512, 512),
                     layers_per_block=2, norm_num_groups=32, scaling_factor=0.18215)


class LibConv2d(nn.Conv2d):
    """The VAE's stem / head convolutions (3 -> 128, 128 -> 3 / 8, 4 -> 512 channels) stay on cuDNN: they run once per clip,
    outside the denoising loops, and their channel counts (3) are below the 16-byte granularity of the cp.async taps."""

    def forward_nhwc(self, x):
        return nr.conv2d_nhwc(x, self.weight, self.bias, stride=self.stride[0], padding=self.padding[0])

    def forward(self, x):
        return to_nchw_view(self.forward_nhwc(to_nhwc(x)))


class VaeResnetBlock2D(nn.Module):
    """GN -> SiLU -> conv1 -> GN -> SiLU -> conv2 (+ shortcut in the epilogue); no time embedding."""

    def __init__(self, in_channels, out_channels, groups=32, eps=1e-6):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.norm1 = GroupNorm(groups, in_channels, eps=eps)
        self.conv1 = Conv3x3(in_channels, out_channels)
        self.norm2 = GroupNorm(groups, out_channels, eps=eps)
        self.conv2 = Conv3x3(out_channels, out_channels)
        self.conv_shortcut = nn.Conv2d(in_channels, out_channels, 1) if in_channels != out_channels else None

    def forward_nhwc(self, x):
        n, h, w, cin = x.shape
        short = x
        if self.conv_shortcut is not None:
            short = ops.linear(x.view(-1, cin), self.conv_shortcut.weight.view(self.out_channels, cin),
                               bias=self.conv_shortcut.bias).view(n, h, w, self.out_channels)
        y = self.norm1.forward_rows(x.view(n, h * w, cin), silu=True).view(n, h, w, cin)
        y = self.conv1.forward_nhwc(y)
        y = self.norm2.forward_rows(y.view(n, h * w, -1), silu=True).view(n, h, w, -1)
        return self.conv2.forward_nhwc(y, residual=short)


class VaeAttention(nn.Module):
    """GroupNorm -> fused q,k,v projection -> one 512-wide head -> out projection with the residual in its epilogue."""

    def __init__(self, channels, groups=32, eps=1e-6):
        super().__init__()
        self.group_norm = GroupNorm(groups, channels, eps=eps)
        self.to_q = Linear(channels, channels)
        self.to_k = Linear(channels, channels)
        self.to_v = Linear(channels, channels)
        self.to_out = nn.ModuleList([Linear(channels, channels), nn.Dropout(0.0)])
        self.heads = 1

    def forward_nhwc(self, x):
        n, h, w, c = x.shape
        rows = x.view(n, h * w, c)
        y = self.group_norm.forward_rows(rows, silu=False)
        wqkv = torch.cat([self.to_q.weight, self.to_k.weight, self.to_v.weight], dim=0)
        bqkv = torch.cat([self.to_q.bias, self.to_k.bias, self.to_v.bias], dim=0)
        qkv = ops.linear(y.view(-1, c), wqkv, bias=bqkv).view(n, h * w, 3 * c)
        o = nr.cross_attention(qkv[..., :c], qkv[..., c:2 * c], qkv[..., 2 * c:], heads=1)  # library SDPA, head_dim = C
        o = ops.linear(o.reshape(-1, c), self.to_out[0].weight, bias=self.to_out[0].bias, residual=rows.reshape(-1, c))
        return o.view(n, h, w, c)


class _Down(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, stride=2, padding=0)

    def forward_nhwc(self, x):  # diffusers Downsample2D(padding=0): zero pad right / bottom, then stride 2
        return nr.conv2d_nhwc(F.pad(x, (0, 0, 0, 1, 0, 1)), self.conv.weight, self.conv.bias, stride=2, padding=0)


class _Up(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.conv = Conv3x3(channels, channels)

    def forward_nhwc(self, x):
        return self.conv.forward_nhwc(nr.nearest_up2_nhwc(x))


class DownEncoderBlock2D(nn.Module):
    def __init__(self, cin, cout, layers, groups, add_downsample):
        super().__init__()
        self.resnets = nn.ModuleList([VaeResnetBlock2D(cin if i == 0 else cout, cout, groups) for i in range(layers)])
        self.downsamplers = nn.ModuleList([_Down(cout)]) if add_downsample else None

    def forward_nhwc(self, x):
        for r in self.resnets:
            x = r.forward_nhwc(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0].forward_nhwc(x)
        return x


class UpDecoderBlock2D(nn.Module):
    def __init__(self, cin, cout, layers, groups, add_upsample):
        super().__init__()
        self.resnets = nn.ModuleList([VaeResnetBlock2D(cin if i == 0 else cout, cout, groups) for i in range(layers)])
        self.upsamplers = nn.ModuleList([_Up(cout)]) if add_upsample else None

    def forward_nhwc(self, x):
        for r in self.resnets:
            x = r.forward_nhwc(x)
        if self.upsamplers is not None:
            x = self.upsamplers[0].forward_nhwc(x)
        return x


class UNetMidBlock2D(nn.Module):
    def __init__(self, channels, groups):
        super().__init__()
        self.resnets = nn.ModuleList([VaeResnetBlock2D(channels, channels, groups), VaeResnetBlock2D(channels, channels, groups)])
        self.attentions = nn.ModuleList([VaeAttention(channels, groups)])

    def forward_nhwc(self, x):
        return self.resnets[1].forward_nhwc(self.attentions[0].forward_nhwc(self.resnets[0].forward_nhwc(x)))


class Encoder(nn.Module):
    def __init__(self, in_channels, latent_channels, chans: Sequence[int], layers, groups):
        super().__init__()
        self.conv_in = LibConv2d(in_channels, chans[0], 3, padding=1)
        self.down_blocks = nn.ModuleList()
        c = chans[0]
        for i, co in enumerate(chans):
            self.down_blocks.append(DownEncoderBlock2D(c, co, layers, groups, add_downsample=i < len(chans) - 1))
            c = co
        self.mid_block = UNetMidBlock2D(c, groups)
        self.conv_norm_out = GroupNorm(groups, c, eps=1e-6)
        self.conv_act = nn.SiLU()
        self.conv_out = LibConv2d(c, 2 * latent_channels, 3, padding=1)

    def forward_nhwc(self, x):
        x = self.conv_in.forward_nhwc(x)
        for blk in self.down_blocks:
            x = blk.forward_nhwc(x)
        x = self.mid_block.forward_nhwc(x)
        n, h, w, c = x.shape
        x = self.conv_norm_out.forward_rows(x.view(n, h * w, c), silu=True).view(n, h, w, c)
        return self.conv_out.forward_nhwc(x)


class Decoder(nn.Module):
    def __init__(self, latent_channels, out_channels, chans: Sequence[int], layers, groups):
        super().__init__()
        rev = list(reversed(chans))
        self.conv_in = LibConv2d(latent_channels, rev[0], 3, padding=1)
        self.mid_block = UNetMidBlock2D(rev[0], groups)
        self.up_blocks = nn.ModuleList()
        c = rev[0]
        for i, co in enumerate(rev):
            self.up_blocks.append(UpDecoderBlock2D(c, co, layers + 1, groups, add_upsample=i < len(rev) - 1))
            c = co
        self.conv_norm_out = GroupNorm(groups, c, eps=1e-6)
        self.conv_act = nn.SiLU()
        self.conv_out = LibConv2d(c, out_channels, 3, padding=1)

    def forward_nhwc(self, z):
        x = self.mid_block.forward_nhwc(self.conv_in.forward_nhwc(z))
        for blk in self.up_blocks:
            x = blk.forward_nhwc(x)
        n, h, w, c = x.shape
        x = self.conv_norm_out.forward_rows(x.view(n, h * w, c), silu=True).view(n, h, w, c)
        return self.conv_out.forward_nhwc(x)


class DiagonalGaussianDistribution:
    """diffusers' posterior object: parameters = cat(mean, logvar) on dim 1, logvar clamped to [-30, 20]."""

    def __init__(self, parameters: torch.Tensor):
        self.mean, logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)

    def sample(self, generator=None) -> torch.Tensor:
        noise = torch.randn(self.mean.shape, generator=generator, device=self.mean.device, dtype=self.mean.dtype)
        return self.mean + self.std * noise

    def mode(self) -> torch.Tensor:
        return self.mean


@dataclass(frozen=True)
class TileGrid:
    """diffusers' tile grid of one tiled encode / decode.  Input tile (i, j) is ``x[..., ys[i]:ys[i]+in_h[i], xs[j]:xs[j]+in_w[j]]``;
    its output is ``out_h[i] x out_w[j]``.  The stitch (``ops.tile_stitch``) works in output pixels: tiles start every ``step``
    pixels and are at most ``tile`` long, seams blend over ``blend`` pixels, and each tile keeps its first ``row_limit``."""
    ys: Tuple[int, ...]
    xs: Tuple[int, ...]
    in_h: Tuple[int, ...]
    in_w: Tuple[int, ...]
    out_h: Tuple[int, ...]
    out_w: Tuple[int, ...]
    H: int
    W: int
    tile: int
    step: int
    blend: int
    row_limit: int

    def shapes(self) -> List[Tuple[int, int]]:
        """the distinct input tile shapes, in order of first appearance"""
        return list(dict.fromkeys((h, w) for h in self.in_h for w in self.in_w))

    def members(self, shape) -> List[Tuple[int, int]]:
        """the (i, j) of the tiles of one input shape"""
        return [(i, j) for i, h in enumerate(self.in_h) for j, w in enumerate(self.in_w) if (h, w) == shape]


def tile_grid(h: int, w: int, tile_in: int, overlap_in: int, blend: int, row_limit: int, up: int = 1, down: int = 1) -> TileGrid:
    """The tiles diffusers' ``tiled_encode`` (pixels -> latents: up 1, down 8) or ``tiled_decode`` (latents -> pixels: up 8,
    down 1) cut from an ``h x w`` input: starts ``range(0, h|w, overlap_in)``, ``tile_in`` long, outputs ``up / down`` times
    their input.  Raises ValueError unless the kept parts (``row_limit``) tile the output exactly and every tile but the last
    is at least ``max(row_limit, 2 * blend)`` long in the output, the conditions of the stitch's closed form (for diffusers'
    own settings they hold whenever ``tile_sample_min_size`` and ``tile_latent_min_size`` agree)."""
    if tile_in < 1 or overlap_in < 1:
        raise ValueError(f"tile_grid: tile {tile_in} and step {overlap_in} must be positive")
    ys, xs = tuple(range(0, h, overlap_in)), tuple(range(0, w, overlap_in))
    in_h, in_w = tuple(min(tile_in, h - y) for y in ys), tuple(min(tile_in, w - x) for x in xs)
    for e in in_h + in_w + (h, w):
        if e * up % down:
            raise ValueError(f"tile_grid: an input extent of {e} does not map to whole output pixels ({up}/{down})")
    g = TileGrid(ys, xs, in_h, in_w, tuple(e * up // down for e in in_h), tuple(e * up // down for e in in_w), h * up // down,
                 w * up // down, tile_in * up // down, overlap_in * up // down, blend, row_limit)
    for axis, ext, L in (("H", g.out_h, g.H), ("W", g.out_w, g.W)):
        if any(t < max(row_limit, 2 * blend) for t in ext[:-1]) or (len(ext) - 1) * row_limit + min(row_limit, ext[-1]) != L:
            raise ValueError(f"tile_grid: output tiles {ext} along {axis} (row_limit {row_limit}, blend {blend}) do not tile "
                             f"{L} pixels: do tile_sample_min_size and tile_latent_min_size disagree?")
    return g


class AutoencoderKL(nn.Module):
    def __init__(self, in_channels=3, out_channels=3, latent_channels=4, block_out_channels=(128, 256, 512, 512),
                 layers_per_block=2, norm_num_groups=32, scaling_factor=0.18215, sample_size=768):
        super().__init__()
        self.encoder = Encoder(in_channels, latent_channels, block_out_channels, layers_per_block, norm_num_groups)
        self.decoder = Decoder(latent_channels, out_channels, block_out_channels, layers_per_block, norm_num_groups)
        self.quant_conv = nn.Conv2d(2 * latent_channels, 2 * latent_channels, 1)
        self.post_quant_conv = nn.Conv2d(latent_channels, latent_channels, 1)
        self.config = SimpleNamespace(scaling_factor=scaling_factor, latent_channels=latent_channels,
                                      block_out_channels=tuple(block_out_channels), sample_size=sample_size)
        # diffusers' memory knobs (off by default); sample_size is the checkpoint's vae/config.json value
        self.use_slicing = False
        self.use_tiling = False
        self.tile_sample_min_size = sample_size[0] if isinstance(sample_size, (list, tuple)) else sample_size
        self.tile_latent_min_size = int(self.tile_sample_min_size / 2 ** (len(block_out_channels) - 1))
        self.tile_overlap_factor = 0.25
        #: tiles of one shape that go through the encoder / decoder together (from any images of the call)
        self.tile_batch = 16

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    def enable_tiling(self, use_tiling: bool = True):
        """Split images larger than ``tile_sample_min_size`` into overlapping tiles for encode and decode, so that the
        memory of one VAE pass is that of ``tile_batch`` tiles whatever the image size.  The seams are blended."""
        self.use_tiling = use_tiling

    def disable_tiling(self):
        self.enable_tiling(False)

    def enable_slicing(self):
        """Run the encoder and the decoder one sample at a time (same result, memory of one sample)."""
        self.use_slicing = True

    def disable_slicing(self):
        self.use_slicing = False

    def _scale(self) -> int:
        return 2 ** (len(self.config.block_out_channels) - 1)

    def encode_grid(self, h: int, w: int) -> TileGrid:
        """the tiles of ``tiled_encode`` for an h x w image"""
        blend = int(self.tile_latent_min_size * self.tile_overlap_factor)
        return tile_grid(h, w, self.tile_sample_min_size, int(self.tile_sample_min_size * (1 - self.tile_overlap_factor)),
                         blend, self.tile_latent_min_size - blend, down=self._scale())

    def decode_grid(self, h: int, w: int) -> TileGrid:
        """the tiles of ``tiled_decode`` for an h x w latent"""
        blend = int(self.tile_sample_min_size * self.tile_overlap_factor)
        return tile_grid(h, w, self.tile_latent_min_size, int(self.tile_latent_min_size * (1 - self.tile_overlap_factor)),
                         blend, self.tile_sample_min_size - blend, up=self._scale())

    def encode(self, x: torch.Tensor):
        """x: [n, 3, H, W] in [-1, 1] -> `.latent_dist` (NCHW tensors, like diffusers)."""
        if self.use_tiling and (x.shape[-1] > self.tile_sample_min_size or x.shape[-2] > self.tile_sample_min_size):
            return self.tiled_encode(x)
        if self.use_slicing and x.shape[0] > 1:
            h = torch.cat([self.encoder.forward_nhwc(to_nhwc(s.to(self.dtype))) for s in x.split(1)])
        else:
            h = self.encoder.forward_nhwc(to_nhwc(x.to(self.dtype)))
        moments = F.conv2d(to_nchw_view(h), self.quant_conv.weight, self.quant_conv.bias)
        return SimpleNamespace(latent_dist=DiagonalGaussianDistribution(moments))

    def decode(self, z: torch.Tensor):
        """z: [n, 4, h, w] -> `.sample` [n, 3, 8h, 8w]."""
        if self.use_slicing and z.shape[0] > 1:
            n, _, h, w = z.shape
            s = self._scale()
            out = to_nchw_view(torch.empty(n, h * s, w * s, self.decoder.conv_out.out_channels, device=z.device, dtype=self.dtype))
            for i in range(n):  # written in place: peak memory is the output plus one sample's decode
                out[i:i + 1] = self._decode(z[i:i + 1])
            return SimpleNamespace(sample=out)
        return SimpleNamespace(sample=self._decode(z))

    def _decode(self, z: torch.Tensor) -> torch.Tensor:
        if self.use_tiling and (z.shape[-1] > self.tile_latent_min_size or z.shape[-2] > self.tile_latent_min_size):
            return self.tiled_decode(z)
        z = F.conv2d(z.to(self.dtype), self.post_quant_conv.weight, self.post_quant_conv.bias)
        return to_nchw_view(self.decoder.forward_nhwc(to_nhwc(z)))

    def _tiled(self, x: torch.Tensor, g: TileGrid, run) -> torch.Tensor:
        """``run([b, c, h, w] tiles) -> [b, C, h', w']`` on every tile of every image, gathered by shape, ``tile_batch`` per
        pass; then one stitch of the raw outputs"""
        n = x.shape[0]
        raw = [[[None] * len(g.xs) for _ in g.ys] for _ in range(n)]
        for shape in g.shapes():
            jobs = [(b, i, j) for b in range(n) for i, j in g.members(shape)]
            per_pass = max(1, int(self.tile_batch))
            for k in range(0, len(jobs), per_pass):
                chunk = jobs[k:k + per_pass]
                batch = torch.stack([x[b, :, g.ys[i]:g.ys[i] + shape[0], g.xs[j]:g.xs[j] + shape[1]] for b, i, j in chunk])
                y = run(batch)
                for m, (b, i, j) in enumerate(chunk):
                    raw[b][i][j] = y[m]
        return ops.tile_stitch(raw, g.H, g.W, g.tile, g.step, g.blend, g.row_limit)

    def tiled_encode(self, x: torch.Tensor):
        """diffusers `AutoencoderKL.tiled_encode`: every tile through the encoder and quant_conv, the seams blended over
        int(tile_latent_min_size / 4) latent pixels -> `.latent_dist`."""
        def run(t):
            h = self.encoder.forward_nhwc(to_nhwc(t.to(self.dtype)))
            return F.conv2d(to_nchw_view(h), self.quant_conv.weight, self.quant_conv.bias)
        moments = self._tiled(x, self.encode_grid(x.shape[-2], x.shape[-1]), run)
        return SimpleNamespace(latent_dist=DiagonalGaussianDistribution(moments))

    def tiled_decode(self, z: torch.Tensor) -> torch.Tensor:
        """diffusers `AutoencoderKL.tiled_decode`: every tile through post_quant_conv and the decoder, the seams blended over
        int(tile_sample_min_size / 4) pixels -> [n, 3, 8h, 8w]."""
        def run(t):
            t = F.conv2d(t.to(self.dtype), self.post_quant_conv.weight, self.post_quant_conv.bias)
            return to_nchw_view(self.decoder.forward_nhwc(to_nhwc(t)))
        return self._tiled(z, self.decode_grid(z.shape[-2], z.shape[-1]), run)


def decode_latents(vae: AutoencoderKL, latents: torch.Tensor, decode_chunk_size=None) -> torch.Tensor:
    """pipeline_i2vgen_xl.py:443-463 — latents [b, c, f, h, w] -> video [b, 3, f, 8h, 8w] float32.  `decode_chunk_size`
    keeps its meaning (frames per VAE call; None = all at once); the per-frame result does not depend on it."""
    latents = 1 / vae.config.scaling_factor * latents
    b, c, f, h, w = latents.shape
    latents = latents.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w)
    if decode_chunk_size is not None:
        image = torch.cat([vae.decode(latents[i:i + decode_chunk_size]).sample
                           for i in range(0, latents.shape[0], decode_chunk_size)], dim=0)
    else:
        image = vae.decode(latents).sample
    video = image[None, :].reshape((b, f, -1) + image.shape[2:]).permute(0, 2, 1, 3, 4)
    return video.float()


def encode_vae_video(vae: AutoencoderKL, frames: torch.Tensor, generator=None) -> torch.Tensor:
    """pipeline_i2vgen_xl.py:565-592 after the image pre-processing: frames [f, 3, H, W] in [-1, 1] -> video latents
    [1, c, f, H/8, W/8] (posterior SAMPLE x scaling_factor).  One batched encoder pass, or with `vae.use_slicing` one
    `vae.encode` per frame as the reference does; the posterior noise is drawn frame by frame in the reference's order so a
    seeded generator gives the same draws."""
    if getattr(vae, "use_slicing", False):
        dists = [vae.encode(frames[i:i + 1]).latent_dist for i in range(frames.shape[0])]
        mean, std = torch.cat([d.mean for d in dists]), torch.cat([d.std for d in dists])
    else:
        dist = vae.encode(frames).latent_dist
        mean, std = dist.mean, dist.std
    lat = []
    for i in range(frames.shape[0]):
        noise = torch.randn(mean[i:i + 1].shape, generator=generator, device=mean.device, dtype=mean.dtype)
        lat.append(((mean[i:i + 1] + std[i:i + 1] * noise) * vae.config.scaling_factor).squeeze(0))
    lat = torch.stack(lat)
    return lat.reshape(1, frames.shape[0], *lat.shape[1:]).permute(0, 2, 1, 3, 4)
