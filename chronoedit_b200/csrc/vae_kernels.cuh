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

}  // namespace ce
