// Implicit-GEMM convolution for the Wan 3D causal VAE on sm_90a (wgmma + TMA), channels-last activations.
//
// GEMM view: M = output voxels (tiles of 8 x 16 pixels of one frame = 128 rows), N = output channels, K = taps x Cin.
// For every tap (dt,dh,dw) and 64-channel block the producer issues ONE 4-D TMA box load {64 ch, 16 w, 8 h, 1 t} at the
// tap-shifted coordinate: it lands in shared memory as a 128-row x 128-byte K-major, 128B-swizzled A tile, and TMA's
// out-of-bounds zero fill IS the convolution's spatial zero padding (negative / overflowing coordinates) and the channel
// padding of Cin up to 64.  Stride-2 convolutions use the tensor map's element strides.  The temporal halo is real data:
// the caller keeps the causal history frames in front of the chunk (wan2pt1.py:49-60, CACHE_T = 2).
// Weights are pre-packed [Cout, taps, Cin_pad] so the B tile is a plain 2-D box.  Pipeline and warpgroup roles are those of
// the GEMM (ring_gemm.cuh: one TMA producer warpgroup, two wgmma consumer warpgroups of 64 rows each); the epilogue adds bias,
// optional residual, the upsample3d frame interleave and an optional planar (NCTHW) clamped store for the decoder head.
//
// Replaces cuDNN's conv3d/conv2d behind CausalConv3d / nn.Conv2d of the reference's chronoedit/_src/tokenizers/wan2pt1.py
// (:42-60, :98-110, :186-220) plus F.pad / torch.cat cache handling and the residual add (:220).
#include "conv.cuh"
#include "ring_gemm.cuh"

namespace ce {

namespace {

constexpr int TILE_H = 8, TILE_W = 16;
static_assert(TILE_H * TILE_W == BM, "a tile of output pixels is one BM-row GEMM tile");

struct ConvGeom {
  int tiles_w, tiles_h, tiles_n, num_tiles;
  int cblocks, kblocks, taps;
};

__device__ __forceinline__ void conv_tile_coords(int t, const ConvGeom& g, int& to, int& th, int& tw, int& nb) {
  nb = t % g.tiles_n;
  t /= g.tiles_n;
  tw = t % g.tiles_w;
  t /= g.tiles_w;
  th = t % g.tiles_h;
  to = t / g.tiles_h;
}

// K-blocks of one fp32 accumulation chunk: the wgmma accumulator loses low bits at every k-step relative to the sum so far, so the
// TERMS = 3 kernel sums chunks of A_hi.W_hi over 256 channels (with their two small products) and adds the chunks in fp32
// (fp32_chain.cuh, kHiChunk)
constexpr int kFlushKBlocks = 3 * 256 / BK;

// TERMS = 1: bf16 activations and weights, bf16 epilogue.  TERMS = 3: the fp32 convolution of launch_conv3d_cl_f32 (conv.cuh); the
// producer loads, per tap and 64-channel block, the (A_hi, W_hi), (A_lo, W_hi), (A_hi, W_lo) k-blocks.
template <int BN, int STAGES, int TERMS>
__global__ void __launch_bounds__(RING_THREADS, 1)
conv3d_cl_kernel(const __grid_constant__ CUtensorMap tma_x, const __grid_constant__ CUtensorMap tma_w, ConvArgs a, ConvGeom g, ConvF32 f) {
  static_assert(TERMS == 1 || TERMS == 3, "bf16 or the 3-term split");
  Ring<BN, STAGES> ring;
  if (!ring.start(&tma_x, &tma_w, g.num_tiles, [&](int t) {
        int to, th, tw, nb;
        conv_tile_coords(t, g, to, th, tw, nb);
        const int w_in0 = tw * TILE_W * a.sw - a.pw;
        const int h_in0 = th * TILE_H * a.sh - a.ph;
        const int t_in0 = a.t_base + to * a.st;
        int tap = 0;
        for (int dt = 0; dt < a.kt; ++dt)
          for (int dh = 0; dh < a.kh; ++dh)
            for (int dw = 0; dw < a.kw; ++dw, ++tap)
              for (int cb = 0; cb < g.cblocks; ++cb) {
                if constexpr (TERMS == 1) {
                  const auto s = ring.acquire();
                  tma_load_4d(s.a, &tma_x, s.bar, cb * BK, w_in0 + dw, h_in0 + dh, t_in0 + dt);
                  tma_load_2d(s.b, &tma_w, s.bar, tap * a.Cin_pad + cb * BK, nb * BN);
                } else {
                  for (int term = 0; term < 3; ++term) {
                    const auto s = ring.acquire();
                    tma_load_5d(s.a, &tma_x, s.bar, cb * BK, term == 1 ? 1 : 0, w_in0 + dw, h_in0 + dh, t_in0 + dt);
                    tma_load_2d(s.b, &tma_w, s.bar, ((tap * g.cblocks + cb) * 3 + term) * BK, nb * BN);
                  }
                }
              }
      }))
    return;
  const int r0 = ring_row();   // the thread's rows of the tile: r0 and r0 + 8
  const int c_in_group = ring_col();
  const int c_half = a.split_time ? a.Cout / 2 : a.Cout;  // channels per stored voxel
  float acc[BN / 2];
  for (int t : RingTiles{g.num_tiles}) {
    int to, th, tw, nb;
    conv_tile_coords(t, g, to, th, tw, nb);
    if constexpr (TERMS == 3) {
      float sum[BN / 2];
      for (int k0 = 0; k0 < g.kblocks; k0 += kFlushKBlocks) {
        ring.mma_tile(acc, g.kblocks - k0 < kFlushKBlocks ? g.kblocks - k0 : kFlushKBlocks);
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) sum[i] = k0 ? sum[i] + acc[i] : acc[i];
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r0 + 8 * h;
        const int oh = th * TILE_H + (r >> 4), ow = tw * TILE_W + (r & 15);
        if (oh >= a.Hout || ow >= a.Wout) continue;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int n = nb * BN + j * 8 + c_in_group + e;
            if (n >= a.Cout) continue;
            float y = sum[4 * j + 2 * h + e];
            if (f.bias) y += f.bias[n];
            if (a.planar_out) {
              if (a.clamp) y = fminf(fmaxf(y, -1.0f), 1.0f);
              f.y[(((size_t)n * a.planar_T + a.planar_t0 + to) * a.Hout + oh) * a.Wout + ow] = y;
              continue;
            }
            const int frame = a.split_time ? 2 * to + (n >= c_half ? 1 : 0) : to;
            const int ch = n >= c_half ? n - c_half : n;
            const size_t pix = ((size_t)frame * a.Hout + oh) * a.Wout + ow;
            if (f.resid) y += f.resid[pix * c_half + ch];
            if (f.y) f.y[pix * c_half + ch] = y;
            if (f.y_pair) {
              const bf16 hi = __float2bfloat16_rn(y);
              f.y_pair[pix * 2 * c_half + ch] = hi;
              f.y_pair[pix * 2 * c_half + c_half + ch] = __float2bfloat16_rn(y - __bfloat162float(hi));
            }
          }
        }
      }
      continue;
    }
    ring.mma_tile(acc, g.kblocks);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r0 + 8 * h;
      const int oh = th * TILE_H + (r >> 4), ow = tw * TILE_W + (r & 15);
      if (oh >= a.Hout || ow >= a.Wout) continue;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {   // 8-channel groups, two channels per lane
        const int n = nb * BN + j * 8 + c_in_group;
        if (n >= a.Cout) continue;
        float y[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          y[e] = acc[4 * j + 2 * h + e];
          if (a.bias && n + e < a.Cout) y[e] += __bfloat162float(a.bias[n + e]);
          y[e] = bf16_round(y[e]);  // the convolution returns a bf16 tensor
        }
        if (a.planar_out) {
          // decoder head: [Cout, Tout, Hout, Wout], optional clamp (diffusers AutoencoderKLWan.decode)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            if (n + e < a.Cout) {
              float o = y[e];
              if (a.clamp) o = fminf(fmaxf(o, -1.0f), 1.0f);
              a.y[(((size_t)(n + e) * a.planar_T + a.planar_t0 + to) * a.Hout + oh) * a.Wout + ow] = __float2bfloat16_rn(o);
            }
          }
          continue;
        }
        int frame = to, ch = n;
        if (a.split_time) {
          frame = 2 * to + (n >= c_half ? 1 : 0);
          ch = n >= c_half ? n - c_half : n;
        }
        const size_t off = (((size_t)frame * a.Hout + oh) * a.Wout + ow) * c_half + ch;
        if ((c_half & 1) == 0 && n + 2 <= a.Cout) {
          if (a.resid) {
            const float2 x = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(a.resid + off));
            y[0] += x.x;
            y[1] += x.y;
          }
          *reinterpret_cast<uint32_t*>(a.y + off) = pack_bf16x2(y[0], y[1]);
        } else {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            if (n + e < a.Cout) {
              float o = y[e];
              if (a.resid) o += __bfloat162float(a.resid[off + e]);
              a.y[off + e] = __float2bfloat16_rn(o);
            }
          }
        }
      }
    }
  }
}

template <int TERMS>
int launch_conv(const ConvArgs& a, const ConvF32& f, cudaStream_t stream) {
  if constexpr (TERMS == 1) {
    CE_REQUIRE(a.x && a.w && a.y, "conv: null pointer");
  } else {
    CE_REQUIRE(a.x && a.w && (f.y || (f.y_pair && !a.planar_out)), "conv fp32: null pointer");
  }
  CE_REQUIRE(a.Cin % 8 == 0 && a.Cin_pad % 64 == 0 && a.Cin_pad >= a.Cin, "conv: Cin % 8, Cin_pad % 64");
  CE_REQUIRE(a.Tout > 0 && a.Hout > 0 && a.Wout > 0 && a.Cout > 0, "conv: empty output");
  CE_REQUIRE(a.sw >= 1 && a.sw <= 2 && a.sh >= 1 && a.sh <= 2, "conv: spatial stride 1 or 2");
  CE_REQUIRE(!a.split_time || a.Cout % 16 == 0, "conv: split_time needs Cout % 16 == 0");
  CE_REQUIRE(a.t_base + (a.Tout - 1) * a.st + a.kt <= a.Tin, "conv: temporal extent exceeds the input buffer");
  CE_REQUIRE(!a.planar_out || (a.planar_t0 >= 0 && a.planar_t0 + a.Tout <= a.planar_T && !a.resid && !f.resid && !a.split_time),
             "conv: planar output frames must lie inside the video, without resid or split_time");
  ConvGeom g;
  g.tiles_w = (a.Wout + TILE_W - 1) / TILE_W;
  g.tiles_h = (a.Hout + TILE_H - 1) / TILE_H;
  g.taps = a.kt * a.kh * a.kw;
  g.cblocks = a.Cin_pad / 64;
  g.kblocks = g.taps * g.cblocks * TERMS;
  CUtensorMap tx, tw;
  if constexpr (TERMS == 1) {
    uint64_t dims[4] = {(uint64_t)a.Cin, (uint64_t)a.Win, (uint64_t)a.Hin, (uint64_t)a.Tin};
    uint64_t strides[3] = {(uint64_t)a.Cin * 2, (uint64_t)a.Win * a.Cin * 2, (uint64_t)a.Hin * a.Win * a.Cin * 2};
    uint32_t box[4] = {64, (uint32_t)(TILE_W * a.sw), (uint32_t)(TILE_H * a.sh), 1};
    uint32_t es[4] = {1, (uint32_t)a.sw, (uint32_t)a.sh, 1};
    int rc = make_tmap_bf16(&tx, a.x, 4, dims, strides, box, es);
    if (rc) return rc;
  } else {   // [Tin, Hin, Win, 2, Cin]: one box per (tap, channel block, term)
    const uint64_t pix = (uint64_t)a.Cin * 4;
    uint64_t dims[5] = {(uint64_t)a.Cin, 2, (uint64_t)a.Win, (uint64_t)a.Hin, (uint64_t)a.Tin};
    uint64_t strides[4] = {(uint64_t)a.Cin * 2, pix, a.Win * pix, (uint64_t)a.Hin * a.Win * pix};
    uint32_t box[5] = {64, 1, (uint32_t)(TILE_W * a.sw), (uint32_t)(TILE_H * a.sh), 1};
    uint32_t es[5] = {1, 1, (uint32_t)a.sw, (uint32_t)a.sh, 1};
    int rc = make_tmap_bf16(&tx, a.x, 5, dims, strides, box, es);
    if (rc) return rc;
  }
  const int bn = TERMS == 3 ? (a.Cout <= 32 ? 32 : 96)
                            : a.Cout <= 32 ? 32 : (a.Cout % 192 == 0 ? 192 : (a.Cout % 96 == 0 ? 96 : (a.Cout > 96 ? 192 : 96)));
  {
    uint64_t dims[2] = {(uint64_t)g.taps * a.Cin_pad * TERMS, (uint64_t)a.Cout};
    uint64_t strides[1] = {(uint64_t)g.taps * a.Cin_pad * TERMS * 2};
    uint32_t box[2] = {64, (uint32_t)bn};
    int rc = make_tmap_bf16(&tw, a.w, 2, dims, strides, box);
    if (rc) return rc;
  }
  g.tiles_n = (a.Cout + bn - 1) / bn;
  g.num_tiles = a.Tout * g.tiles_h * g.tiles_w * g.tiles_n;
  if (bn == 32) return launch_ring_gemm<32, 8>(conv3d_cl_kernel<32, 8, TERMS>, g.num_tiles, stream, tx, tw, a, g, f);
  if (bn == 96) return launch_ring_gemm<96, 6>(conv3d_cl_kernel<96, 6, TERMS>, g.num_tiles, stream, tx, tw, a, g, f);
  if constexpr (TERMS == 1) return launch_ring_gemm<192, 5>(conv3d_cl_kernel<192, 5, 1>, g.num_tiles, stream, tx, tw, a, g, f);
  return fail(CE_ERR_INVALID, "conv fp32: no BN = 192 kernel");
}

}  // namespace

int launch_conv3d_cl(const ConvArgs& a, cudaStream_t stream) { return launch_conv<1>(a, ConvF32(), stream); }

int launch_conv3d_cl_f32(const ConvArgs& a, const ConvF32& f, cudaStream_t stream) { return launch_conv<3>(a, f, stream); }

}  // namespace ce
