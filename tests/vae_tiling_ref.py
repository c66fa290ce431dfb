"""TEST INFRASTRUCTURE — diffusers' tiled / sliced VAE for the tests of anyv2v_b200's VAE tiling; nothing outside tests/ imports it.

1. Oracle: diffusers 0.26.3 `AutoencoderKL` memory knobs [recalled: diffusers is not vendored], reached from the reference
   through pipeline_i2vgen_xl.py:191-222 (`enable_vae_slicing` / `enable_vae_tiling` -> `vae.enable_slicing` / `enable_tiling`).
   ``DiffusersTiling(vae)`` wraps an oracle/vae_ref.py AutoencoderKL with diffusers' attributes, `encode` / `decode` dispatch,
   `tiled_encode`, `tiled_decode`, and the in-place `blend_v` / `blend_h` loop (``blend_loop``).
2. Contract of `ops.tile_stitch` (csrc/vae_tiles.cu): ``stitch_closed_form``, each output element from at most four raw tiles,
   evaluated with the same torch fp16 rounding sequence as the loop, on the tiles' device; ``tile_stitch`` stands in for the
   kernel under ``patch_ops``.
3. Geometry: ``geometry``, the tile starts / extents, blend extent and row limit of the loop, stated from diffusers' formulas.
"""
from __future__ import annotations

from types import SimpleNamespace

import torch

import kernel_contracts
from oracle.vae_ref import DiagonalGaussianDistribution


# ------------------------------------------------------------------------------------------------------------- oracle
def blend_v(a, b, blend_extent):
    blend_extent = min(a.shape[2], b.shape[2], blend_extent)
    for y in range(blend_extent):
        b[:, :, y, :] = a[:, :, -blend_extent + y, :] * (1 - y / blend_extent) + b[:, :, y, :] * (y / blend_extent)
    return b


def blend_h(a, b, blend_extent):
    blend_extent = min(a.shape[3], b.shape[3], blend_extent)
    for x in range(blend_extent):
        b[:, :, :, x] = a[:, :, :, -blend_extent + x] * (1 - x / blend_extent) + b[:, :, :, x] * (x / blend_extent)
    return b


def blend_loop(rows, blend_extent, row_limit, h_first=False, raw_neighbours=False):
    """diffusers' seam loop over the raw tile outputs ``rows[i][j]`` ([N, C, h, w]; blended IN PLACE) -> the stitched output.
    ``h_first`` / ``raw_neighbours`` are the negative controls: blend_h before blend_v, or read the neighbours unblended."""
    raw = [[t.clone() for t in row] for row in rows] if raw_neighbours else rows
    result_rows = []
    for i, row in enumerate(rows):
        result_row = []
        for j, tile in enumerate(row):
            steps = [("v", i > 0), ("h", j > 0)]
            for axis, on in (steps[::-1] if h_first else steps):
                if on and axis == "v":
                    tile = blend_v(raw[i - 1][j], tile, blend_extent)
                elif on and axis == "h":
                    tile = blend_h(raw[i][j - 1], tile, blend_extent)
            result_row.append(tile[:, :, :row_limit, :row_limit])
        result_rows.append(torch.cat(result_row, dim=3))
    return torch.cat(result_rows, dim=2)


class DiffusersTiling:
    """diffusers' AutoencoderKL encode / decode with its slicing and tiling knobs, over the modules of an oracle VAE.
    ``trace`` records the path each call took ("tiled_encode", "sliced_encode", "encode", "tiled_decode", "decode")."""

    def __init__(self, vae, sample_size=768):
        self.vae = vae
        self.config = vae.config
        self.use_slicing = False
        self.use_tiling = False
        self.tile_sample_min_size = sample_size[0] if isinstance(sample_size, (list, tuple)) else sample_size
        self.tile_latent_min_size = int(self.tile_sample_min_size / (2 ** (len(vae.config.block_out_channels) - 1)))
        self.tile_overlap_factor = 0.25
        self.trace = []

    def enable_tiling(self, use_tiling: bool = True):
        self.use_tiling = use_tiling

    def disable_tiling(self):
        self.enable_tiling(False)

    def enable_slicing(self):
        self.use_slicing = True

    def disable_slicing(self):
        self.use_slicing = False

    def encode(self, x):
        if self.use_tiling and (x.shape[-1] > self.tile_sample_min_size or x.shape[-2] > self.tile_sample_min_size):
            return self.tiled_encode(x)
        if self.use_slicing and x.shape[0] > 1:
            self.trace.append("sliced_encode")
            h = torch.cat([self.vae.encoder(x_slice) for x_slice in x.split(1)])
        else:
            self.trace.append("encode")
            h = self.vae.encoder(x)
        return SimpleNamespace(latent_dist=DiagonalGaussianDistribution(self.vae.quant_conv(h)))

    def _decode(self, z):
        if self.use_tiling and (z.shape[-1] > self.tile_latent_min_size or z.shape[-2] > self.tile_latent_min_size):
            return self.tiled_decode(z)
        self.trace.append("decode")
        return self.vae.decoder(self.vae.post_quant_conv(z))

    def decode(self, z):
        if self.use_slicing and z.shape[0] > 1:
            return SimpleNamespace(sample=torch.cat([self._decode(z_slice) for z_slice in z.split(1)]))
        return SimpleNamespace(sample=self._decode(z))

    def tiled_encode(self, x):
        self.trace.append("tiled_encode")
        overlap_size = int(self.tile_sample_min_size * (1 - self.tile_overlap_factor))
        blend_extent = int(self.tile_latent_min_size * self.tile_overlap_factor)
        row_limit = self.tile_latent_min_size - blend_extent
        rows = []
        for i in range(0, x.shape[2], overlap_size):
            row = []
            for j in range(0, x.shape[3], overlap_size):
                tile = x[:, :, i:i + self.tile_sample_min_size, j:j + self.tile_sample_min_size]
                row.append(self.vae.quant_conv(self.vae.encoder(tile)))
            rows.append(row)
        return SimpleNamespace(latent_dist=DiagonalGaussianDistribution(blend_loop(rows, blend_extent, row_limit)))

    def tiled_decode(self, z):
        self.trace.append("tiled_decode")
        overlap_size = int(self.tile_latent_min_size * (1 - self.tile_overlap_factor))
        blend_extent = int(self.tile_sample_min_size * self.tile_overlap_factor)
        row_limit = self.tile_sample_min_size - blend_extent
        rows = []
        for i in range(0, z.shape[2], overlap_size):
            row = []
            for j in range(0, z.shape[3], overlap_size):
                tile = z[:, :, i:i + self.tile_latent_min_size, j:j + self.tile_latent_min_size]
                row.append(self.vae.decoder(self.vae.post_quant_conv(tile)))
            rows.append(row)
        return blend_loop(rows, blend_extent, row_limit)


# ----------------------------------------------------------------------------------------------------------- geometry
def geometry(h, w, sample_size, levels=4, decode=True):
    """the loop's tiles for an h x w input (latents when ``decode``, pixels otherwise): starts, input extents, and the blend
    extent / row limit in output pixels"""
    t_sample = sample_size
    t_latent = int(sample_size / 2 ** (levels - 1))
    tile, blend_src = (t_latent, t_sample) if decode else (t_sample, t_latent)
    step = int(tile * 0.75)
    blend = int(blend_src * 0.25)
    ys, xs = list(range(0, h, step)), list(range(0, w, step))
    return SimpleNamespace(ys=ys, xs=xs, in_h=[min(tile, h - y) for y in ys], in_w=[min(tile, w - x) for x in xs],
                           blend=blend, row_limit=blend_src - blend)


# ---------------------------------------------------------------------------------------------------------- contract
def _blend(a, b, pos, e, dim):
    """``a * (1 - pos/e) + b * (pos/e)`` with pos running along ``dim`` of fp16 tensors, as torch rounds the loop's ops:
    weights from double to fp32, each product and the sum in fp32 rounded to fp16"""
    shape = [1] * a.dim()
    shape[dim] = len(pos)
    r = torch.tensor([p / e for p in pos], dtype=torch.float64)
    wa, wb = (1 - r).float().view(shape).to(a.device), r.float().view(shape).to(a.device)
    return ((a.float() * wa).half().float() + (b.float() * wb).half().float()).half()


def stitch_closed_form(tiles, H, W, tile, step, blend, row_limit):
    """ops.tile_stitch: tiles[n][i][j] = raw [C, t_i, t_j] fp16 -> [N, C, H, W] fp16, from the four-tile closed form"""
    rows, cols = len(tiles[0]), len(tiles[0][0])
    ext_h = [min(tile, H - i * step) for i in range(rows)]
    ext_w = [min(tile, W - j * step) for j in range(cols)]
    out = []
    for img in tiles:
        out_rows = []
        for i in range(rows):
            out_row = []
            for j in range(cols):
                kh, kw = min(row_limit, ext_h[i]), min(row_limit, ext_w[j])
                v = img[i][j][:, :kh, :kw].clone()
                ev = min(ext_h[i - 1], ext_h[i], blend) if i > 0 else 0
                eh = min(ext_w[j - 1], ext_w[j], blend) if j > 0 else 0
                tu = ext_h[i - 1] if i > 0 else 0
                tl = ext_w[j - 1] if j > 0 else 0
                if ev > 0:
                    u = img[i - 1][j][:, tu - ev:tu, :kw].clone()                          # upper neighbour, rows it is read at
                    if eh > 0:
                        ul = img[i - 1][j - 1][:, tu - ev:tu, tl - eh:tl]
                        u[:, :, :eh] = _blend(ul, u[:, :, :eh], range(eh), eh, 2)          # ... after its own blend_h
                    v[:, :ev] = _blend(u, v[:, :ev], range(ev), ev, 1)
                if eh > 0:
                    lt = img[i][j - 1][:, :kh, tl - eh:tl].clone()                         # left neighbour, columns it is read at
                    if ev > 0:
                        ul = img[i - 1][j - 1][:, tu - ev:tu, tl - eh:tl]
                        lt[:, :ev] = _blend(ul, lt[:, :ev], range(ev), ev, 1)              # ... after its own blend_v
                    v[:, :, :eh] = _blend(lt, v[:, :, :eh], range(eh), eh, 2)
                out_row.append(v)
            out_rows.append(torch.cat(out_row, dim=2))
        out.append(torch.cat(out_rows, dim=1))
    return torch.stack(out)


def tile_stitch(tiles, H, W, tile, step, blend, row_limit, out=None):
    """ops.tile_stitch as one counted launch of the closed form (into ``out`` when it is given)"""
    y = stitch_closed_form(tiles, H, W, tile, step, blend, row_limit)
    kernel_contracts._count()
    if out is None:
        return y
    out.copy_(y)
    return out


def patch_ops(monkeypatch):
    """ops.tile_stitch -> the contract for one test (use together with the emulated_ops fixture, which patches the other ops)"""
    from anyv2v_b200 import ops
    monkeypatch.setattr(ops, "tile_stitch", tile_stitch)
