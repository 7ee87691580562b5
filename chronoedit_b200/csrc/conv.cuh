// Interface of the wgmma implicit-GEMM convolution used by the Wan VAE path (conv.cu).
#pragma once
#include "host_common.h"
#include "ptx.cuh"

namespace ce {

// Channels-last ("T,H,W,C") bf16 activations.  One launch computes, for every output voxel (to, oh, ow) and channel n:
//   y = bias[n] + sum_{dt,dh,dw,c} W[n, (dt,dh,dw), c] * X[t_base + to*st + dt, oh*sh + dh - ph, ow*sw + dw - pw, c]
// with zero for spatial coordinates outside X (conv padding) — the temporal halo comes from the history frames the
// caller keeps in front of the chunk inside X (causal padding, wan2pt1.py:49-60).
struct ConvArgs {
  // input tensor X [Tin, Hin, Win, Cin]
  const bf16* x = nullptr;
  int Tin = 0, Hin = 0, Win = 0, Cin = 0;
  // weights [Cout, kt*kh*kw, Cin_pad] (Cin_pad = Cin rounded up to 64, zero filled) and bias [Cout]
  const bf16* w = nullptr;
  const bf16* bias = nullptr;
  int Cout = 0, Cin_pad = 0;
  int kt = 1, kh = 1, kw = 1;
  int st = 1, sh = 1, sw = 1;
  int ph = 0, pw = 0;
  int t_base = 0;
  // output [Tout, Hout, Wout, Cout_store]
  bf16* y = nullptr;
  int Tout = 0, Hout = 0, Wout = 0;
  // epilogue
  const bf16* resid = nullptr;   // optional, same geometry as y: y = bf16(float(bf16(conv)) + float(resid))   (ResidualBlock x + h)
  int split_time = 0;            // 1: Cout = 2*C; channel n goes to frame 2*to + n / C, channel n % C (upsample3d interleave, wan2pt1.py:137-139)
  int planar_out = 0;            // 1: y is planar [Cout, planar_T, Hout, Wout] (NCTHW), frame `to` stored at planar_t0 + to; values
  int clamp = 0;                 //    are clamped to [-1, 1] when clamp != 0
  int planar_T = 0, planar_t0 = 0;
};

int launch_conv3d_cl(const ConvArgs& a, cudaStream_t stream);

// The same convolution in fp32 (the fp32 VAE).  The activation arrives as its split pair: x [Tin, Hin, Win, 2, Cin] bf16 holds
// hi = bf16(v) then lo = bf16(v - hi) of every pixel's channels, and the weight is packed [Cout, taps, Cin_pad / 64, 3, 64] bf16 as
// W_hi | W_hi | W_lo per 64-channel block, so that the K loop sums A_hi.W_hi + A_lo.W_hi + A_hi.W_lo (fp32_chain.cuh's rule) in
// fp32.  ConvArgs supplies the geometry, x and w; its bias, y and resid are not read.  The epilogue adds bias (fp32) and resid (fp32,
// y's layout) and stores y (fp32: channels-last, split_time interleave, or planar with the optional clamp) and / or the split pair
// of y, [frame, oh, ow, 2, C], for a convolution that reads it next.
struct ConvF32 {
  const float* bias = nullptr;
  const float* resid = nullptr;
  float* y = nullptr;
  bf16* y_pair = nullptr;
};
int launch_conv3d_cl_f32(const ConvArgs& a, const ConvF32& f, cudaStream_t stream);

}  // namespace ce
