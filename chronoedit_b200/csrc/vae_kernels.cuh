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

}  // namespace ce
