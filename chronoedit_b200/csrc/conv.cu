// Implicit-GEMM convolution for the Wan 3D causal VAE on sm_90a (wgmma + TMA), channels-last activations.
//
// GEMM view: M = output voxels (tiles of 8 x 16 pixels of one frame = 128 rows), N = output channels, K = taps x Cin.
// For every tap (dt,dh,dw) and 64-channel block the producer issues ONE 4-D TMA box load {64 ch, 16 w, 8 h, 1 t} at the
// tap-shifted coordinate: it lands in shared memory as a 128-row x 128-byte K-major, 128B-swizzled A tile, and TMA's
// out-of-bounds zero fill IS the convolution's spatial zero padding (negative / overflowing coordinates) and the channel
// padding of Cin up to 64.  Stride-2 convolutions use the tensor map's element strides.  The temporal halo is real data:
// the caller keeps the causal history frames in front of the chunk (wan2pt1.py:49-60, CACHE_T = 2).
// Weights are pre-packed [Cout, taps, Cin_pad] so the B tile is a plain 2-D box.  Pipeline and warpgroup roles are those of
// gemm.cu (one TMA producer warpgroup, two wgmma consumer warpgroups of 64 rows each); the epilogue adds bias, optional
// residual, the upsample3d frame interleave and an optional planar (NCTHW) clamped store for the decoder head.
//
// Replaces cuDNN's conv3d/conv2d behind CausalConv3d / nn.Conv2d of the reference's chronoedit/_src/tokenizers/wan2pt1.py
// (:42-60, :98-110, :186-220) plus F.pad / torch.cat cache handling and the residual add (:220).
#include "conv.cuh"
#include "wgmma.cuh"

namespace ce {

namespace {

constexpr int TILE_H = 8, TILE_W = 16, BM = 128, BK = 64;
constexpr int CONV_THREADS = 384;

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

template <int BN, int STAGES>
__global__ void __launch_bounds__(CONV_THREADS, 1)
conv3d_cl_kernel(const __grid_constant__ CUtensorMap tma_x, const __grid_constant__ CUtensorMap tma_w, ConvArgs a, ConvGeom g) {
  constexpr uint32_t A_BYTES = BM * BK * 2;
  constexpr uint32_t B_BYTES = BN * BK * 2;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * (A_BYTES + B_BYTES));
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);  // one arrive per consumer warpgroup
    }
    fence_mbar_init();
    tma_prefetch_desc(&tma_x);
    tma_prefetch_desc(&tma_w);
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one_sync()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < g.num_tiles; t += gridDim.x) {
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
                mbar_wait(&empty[stage], phase ^ 1);
                mbar_arrive_expect_tx(&full[stage], A_BYTES + B_BYTES);
                tma_load_4d(sA + stage * A_BYTES, &tma_x, &full[stage], cb * BK, w_in0 + dw, h_in0 + dh, t_in0 + dt);
                tma_load_2d(sB + stage * B_BYTES, &tma_w, &full[stage], tap * a.Cin_pad + cb * BK, nb * BN);
                if (++stage == STAGES) {
                  stage = 0;
                  phase ^= 1;
                }
              }
      }
    }
    return;
  }

  setmaxnreg_inc<232>();
  const int wg = (warp >> 2) - 1;
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // the thread's rows of the tile: r0 and r0 + 8
  const int c_in_group = 2 * (lane & 3);
  const int c_half = a.split_time ? a.Cout / 2 : a.Cout;  // channels per stored voxel
  int stage = 0;
  uint32_t phase = 0;
  float acc[BN / 2];
  for (int t = blockIdx.x; t < g.num_tiles; t += gridDim.x) {
    int to, th, tw, nb;
    conv_tile_coords(t, g, to, th, tw, nb);
    wgmma_ring_tile<BN, STAGES>(acc, smem_u32(sA) + wg * 64 * 128, smem_u32(sB), A_BYTES, B_BYTES, full, empty, g.kblocks, stage, phase);
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

template <int BN, int STAGES>
int launch_conv_variant(const CUtensorMap& tx, const CUtensorMap& tw, const ConvArgs& a, ConvGeom g, cudaStream_t stream) {
  constexpr size_t smem = (size_t)STAGES * (BM * BK * 2 + BN * BK * 2) + 1024 + 256;
  CE_ENSURE_SMEM((conv3d_cl_kernel<BN, STAGES>), smem);
  g.tiles_n = (a.Cout + BN - 1) / BN;
  g.num_tiles = a.Tout * g.tiles_h * g.tiles_w * g.tiles_n;
  const int grid = g.num_tiles < device_sm_count() ? g.num_tiles : device_sm_count();
  conv3d_cl_kernel<BN, STAGES><<<grid, CONV_THREADS, smem, stream>>>(tx, tw, a, g);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

}  // namespace

int launch_conv3d_cl(const ConvArgs& a, cudaStream_t stream) {
  CE_REQUIRE(a.x && a.w && a.y, "conv: null pointer");
  CE_REQUIRE(a.Cin % 8 == 0 && a.Cin_pad % 64 == 0 && a.Cin_pad >= a.Cin, "conv: Cin % 8, Cin_pad % 64");
  CE_REQUIRE(a.Tout > 0 && a.Hout > 0 && a.Wout > 0 && a.Cout > 0, "conv: empty output");
  CE_REQUIRE(a.sw >= 1 && a.sw <= 2 && a.sh >= 1 && a.sh <= 2, "conv: spatial stride 1 or 2");
  CE_REQUIRE(!a.split_time || a.Cout % 16 == 0, "conv: split_time needs Cout % 16 == 0");
  CE_REQUIRE(a.t_base + (a.Tout - 1) * a.st + a.kt <= a.Tin, "conv: temporal extent exceeds the input buffer");
  ConvGeom g;
  g.tiles_w = (a.Wout + TILE_W - 1) / TILE_W;
  g.tiles_h = (a.Hout + TILE_H - 1) / TILE_H;
  g.taps = a.kt * a.kh * a.kw;
  g.cblocks = a.Cin_pad / 64;
  g.kblocks = g.taps * g.cblocks;
  g.tiles_n = 0;
  g.num_tiles = 0;
  CUtensorMap tx, tw;
  {
    uint64_t dims[4] = {(uint64_t)a.Cin, (uint64_t)a.Win, (uint64_t)a.Hin, (uint64_t)a.Tin};
    uint64_t strides[3] = {(uint64_t)a.Cin * 2, (uint64_t)a.Win * a.Cin * 2, (uint64_t)a.Hin * a.Win * a.Cin * 2};
    uint32_t box[4] = {64, (uint32_t)(TILE_W * a.sw), (uint32_t)(TILE_H * a.sh), 1};
    uint32_t es[4] = {1, (uint32_t)a.sw, (uint32_t)a.sh, 1};
    int rc = make_tmap_bf16(&tx, a.x, 4, dims, strides, box, es);
    if (rc) return rc;
  }
  const int bn = a.Cout <= 32 ? 32 : (a.Cout % 192 == 0 ? 192 : (a.Cout % 96 == 0 ? 96 : (a.Cout > 96 ? 192 : 96)));
  {
    uint64_t dims[2] = {(uint64_t)g.taps * a.Cin_pad, (uint64_t)a.Cout};
    uint64_t strides[1] = {(uint64_t)g.taps * a.Cin_pad * 2};
    uint32_t box[2] = {64, (uint32_t)bn};
    int rc = make_tmap_bf16(&tw, a.w, 2, dims, strides, box);
    if (rc) return rc;
  }
  if (bn == 32) return launch_conv_variant<32, 8>(tx, tw, a, g, stream);
  if (bn == 96) return launch_conv_variant<96, 6>(tx, tw, a, g, stream);
  return launch_conv_variant<192, 5>(tx, tw, a, g, stream);
}

}  // namespace ce
