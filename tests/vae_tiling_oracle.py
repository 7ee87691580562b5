"""Restatement of diffusers' tiled VAE encode / decode (`AutoencoderKLWan.enable_tiling`) on top of oracle/vae_oracle.py.

TEST INFRASTRUCTURE ONLY, as the oracle package.  diffusers is not vendored, so the rule below is restated from diffusers 0.35.2
(the version requirements.txt pins) from memory [diffusers-mem]:

  state       use_tiling = use_slicing = False; tile_sample_min_{height,width} = 256, tile_sample_stride_{height,width} = 192
              pixels; enable_tiling(...) sets use_tiling and overrides the sizes it is given (`size or current`).
  trigger     encode tiles when W > min_w or H > min_h (pixels); decode when w > min_w // 8 or h > min_h // 8 (latents).
  encode      tiles x[..., i:i+min_h, j:j+min_w] for i in range(0, H, stride_h), j in range(0, W, stride_w); each a fresh causal
              encode (frame 0, then 4-frame chunks) + quant_conv; blend extents min//8 - stride//8 latents, crop stride//8, then
              the result to [h, w].
  decode      latent tiles from range(0, h, stride_h // 8) covering min // 8 latents; each post_quant_conv + a fresh decode one
              latent frame at a time; blend extents min - stride pixels, crop stride pixels, then the result to [8h, 8w].
  blend       row-major over the grid, in place: blend_v(rows[i-1][j], tile) then blend_h(row[j-1], tile), so a neighbour is
              read after its own blends.
  clamp       the untiled decode clamps to [-1, 1]; the tiled one, as recalled, does not (TILED_DECODE_CLAMPS).

Restated differently from the issue that asked for it: the functions live here, beside the tests, and not in oracle/vae_oracle.py,
which stays as it is; and the encode blends the posterior mean that oracle.vae_encode returns, not the full moments -- the blend
acts on every channel alone, so the mean of the blended moments is the blended mean.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import torch

from oracle import pipeline_oracle as P
from oracle import vae_oracle as V

Tensor = torch.Tensor
Tiles = Tuple[int, int, int, int]   # (min_h, min_w, stride_h, stride_w), pixels

DEFAULT_TILES: Tiles = (256, 256, 192, 192)
TILED_DECODE_CLAMPS = False


def blend_v(a: Tensor, b: Tensor, blend_extent: int) -> Tensor:
    """diffusers AutoencoderKLWan.blend_v: overwrites the first rows of b with a's last rows faded in, in b's dtype."""
    blend_extent = min(a.shape[-2], b.shape[-2], blend_extent)
    for y in range(blend_extent):
        b[:, :, :, y, :] = a[:, :, :, -blend_extent + y, :] * (1 - y / blend_extent) + b[:, :, :, y, :] * (y / blend_extent)
    return b


def blend_h(a: Tensor, b: Tensor, blend_extent: int) -> Tensor:
    """diffusers AutoencoderKLWan.blend_h: the same along the last (width) axis."""
    blend_extent = min(a.shape[-1], b.shape[-1], blend_extent)
    for x in range(blend_extent):
        b[:, :, :, :, x] = a[:, :, :, :, -blend_extent + x] * (1 - x / blend_extent) + b[:, :, :, :, x] * (x / blend_extent)
    return b


def blend_grid(rows: List[List[Tensor]], blend_h_extent: int, blend_w_extent: int, crop_h: int, crop_w: int, out_h: int,
               out_w: int) -> Tensor:
    """The blend-and-crop loop shared by tiled_encode and tiled_decode."""
    result_rows = []
    for i, row in enumerate(rows):
        result_row = []
        for j, tile in enumerate(row):
            if i > 0:
                tile = blend_v(rows[i - 1][j], tile, blend_h_extent)
            if j > 0:
                tile = blend_h(row[j - 1], tile, blend_w_extent)
            result_row.append(tile[:, :, :, :crop_h, :crop_w])
        result_rows.append(torch.cat(result_row, dim=-1))
    return torch.cat(result_rows, dim=3)[:, :, :, :out_h, :out_w]


@torch.no_grad()
def vae_encode_tiled(sd: Dict[str, Tensor], cfg: V.VAEConfig, x: Tensor, tiles: Tiles = DEFAULT_TILES) -> Tensor:
    """x [B,3,T,H,W] -> posterior mean [B,z,1+k,H/8,W/8], tile by tile (diffusers' tiled_encode)."""
    min_h, min_w, stride_h, stride_w = tiles
    H, W = x.shape[-2:]
    rows = []
    for i in range(0, H, stride_h):
        row = []
        for j in range(0, W, stride_w):
            row.append(V.vae_encode(sd, cfg, x[:, :, :, i: i + min_h, j: j + min_w]))
        rows.append(row)
    return blend_grid(rows, min_h // 8 - stride_h // 8, min_w // 8 - stride_w // 8, stride_h // 8, stride_w // 8, H // 8, W // 8)


@torch.no_grad()
def vae_decode_tiled(sd: Dict[str, Tensor], cfg: V.VAEConfig, z: Tensor, tiles: Tiles = DEFAULT_TILES) -> Tensor:
    """z [B,z,Tl,h,w] -> video [B,3,1+4(Tl-1),8h,8w], tile by tile (diffusers' tiled_decode)."""
    min_h, min_w, stride_h, stride_w = tiles
    h, w = z.shape[-2:]
    rows = []
    for i in range(0, h, stride_h // 8):
        row = []
        for j in range(0, w, stride_w // 8):
            row.append(V.vae_decode(sd, cfg, z[:, :, :, i: i + min_h // 8, j: j + min_w // 8], clamp=False))
        rows.append(row)
    out = blend_grid(rows, min_h - stride_h, min_w - stride_w, stride_h, stride_w, 8 * h, 8 * w)
    return out.clamp(-1.0, 1.0) if TILED_DECODE_CLAMPS else out


def tiles_encode(tiles: Tiles, H: int, W: int) -> bool:
    return W > tiles[1] or H > tiles[0]


def tiles_decode(tiles: Tiles, h: int, w: int) -> bool:
    return w > tiles[1] // 8 or h > tiles[0] // 8


class TiledOracleVAE(P.OracleVAE):
    """pipeline_oracle.OracleVAE with enable_tiling(): frames larger than one tile go through the tiled rule above."""

    def __init__(self, sd, cfg, dtype, tiles: Tiles = DEFAULT_TILES, clamp: bool = True):
        super().__init__(sd, cfg, dtype, clamp=clamp)
        self.tiles = tiles
        self.tiled_calls = 0

    def encode(self, x):
        if not tiles_encode(self.tiles, *x.shape[-2:]):
            return super().encode(x)
        self.tiled_calls += 1
        mean = vae_encode_tiled(self.sd, self.cfg, x.to(self.dtype), self.tiles)
        return P.SimpleNamespace(latent_dist=P._Posterior(mean))

    def decode(self, z, return_dict=True):
        if not tiles_decode(self.tiles, *z.shape[-2:]):
            return super().decode(z, return_dict=return_dict)
        self.tiled_calls += 1
        out = vae_decode_tiled(self.sd, self.cfg, z.to(self.dtype), self.tiles)
        return (out,) if not return_dict else P.SimpleNamespace(sample=out)
