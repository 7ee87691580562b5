// Interface of the HBM-bound VAE kernels (vae_kernels.cu).
#pragma once
#include "host_common.h"
#include "ptx.cuh"

namespace ce {

int launch_rms_silu_cl(const bf16* x, const bf16* gamma, bf16* y, size_t pixels, int C, int apply_silu, cudaStream_t stream);
int launch_upsample2x_cl(const bf16* in, bf16* out, int T, int H, int W, int C, cudaStream_t stream);
int launch_im2row(const bf16* x, size_t sc, size_t st, size_t sh, size_t sw, int Tin, int Hin, int Win, int Cin, bf16* A, int Kpad,
                  int Tout, int Hout, int Wout, int kt, int kh, int kw, int ph, int pw, int t_base, cudaStream_t stream);
int launch_cl_to_planar(const bf16* cl, int C, bf16* planar, size_t pixels, int Cout, cudaStream_t stream);

// The fp32 VAE's row kernels.  A "pair" is the split a convolution reads (conv.cuh, launch_conv3d_cl_f32): [pixels, 2, C] bf16, hi then lo.
// RMS_norm (+ SiLU) in fp32 of x [pixels, C] into y (fp32 [pixels, C]) or y_pair (exactly one of them)
int launch_rms_silu_cl_f32(const float* x, const float* gamma, float* y, bf16* y_pair, size_t pixels, int C, int apply_silu,
                           cudaStream_t stream);
// nearest 2x spatial upsample of x [T, H, W, C] fp32 into the pair of [T, 2H, 2W, C]
int launch_upsample2x_cl_f32(const float* in, bf16* out_pair, int T, int H, int W, int C, cudaStream_t stream);
// planar fp32 [C, pixels] -> the pair [pixels, 2, Cp] with channels C .. Cp-1 zero
int launch_planar_to_pair(const float* planar, int C, size_t pixels, bf16* pair, int Cp, cudaStream_t stream);
// planar[c, p] = cl[p, c] for c < Cout, fp32
int launch_cl_to_planar_f32(const float* cl, int C, float* planar, size_t pixels, int Cout, cudaStream_t stream);

// One tile of a tiled encode or decode (diffusers' blend_v then blend_h, in place, then the crop).  Every tensor is planar
// [C, T, rows, cols] in the tile's dtype (bf16 or fp32, `fp32`).  The tile [C, T, th, tw] is blended with the last `above_h` rows
// of the blended tile above (`above` [C, T, above_h, tw], extent min(above_h, th)) and then with the last `left_w` columns of the
// blended tile to its left (`left` [C, T, th, left_w], extent min(left_w, tw)); a null neighbour is no blend.  The blended values go
// to: out [C, T, out_h, out_w] at (oy, ox) for tile rows < crop_h and columns < crop_w, clipped to out (clamped to [-1, 1] if
// clamp); strip [C, T, strip_h, tw] = the last strip_h rows; tail [C, T, th, tail_w] = the last tail_w columns (null: not kept).
struct TileBlend {
  const void* tile = nullptr;
  int C = 0, T = 0, th = 0, tw = 0;
  const void* above = nullptr;
  int above_h = 0;
  const void* left = nullptr;
  int left_w = 0;
  void* out = nullptr;
  int out_h = 0, out_w = 0, oy = 0, ox = 0, crop_h = 0, crop_w = 0, clamp = 0;
  void* strip = nullptr;
  int strip_h = 0;
  void* tail = nullptr;
  int tail_w = 0;
  int fp32 = 0;
};
int launch_tile_blend(const TileBlend& b, cudaStream_t stream);
// elements per 16-byte access the launch uses for these extents (8 / 4 / 2 / 1 bf16, 4 / 2 / 1 fp32)
int tile_blend_vector(const TileBlend& b);

}  // namespace ce
