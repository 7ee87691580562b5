// HBM-bound kernels of the Wan VAE path (channels-last bf16): RMS_norm(+SiLU), nearest 2x upsample, im2row for the
// few small-Cin convolutions, layout conversion; the fp32 VAE's RMS_norm(+SiLU), upsample and layout conversions, which write
// the split pair its convolutions read; and the tiled VAE's blend of one tile with its neighbours (bf16 and fp32).
#include "vae_kernels.cuh"

#include <algorithm>

namespace ce {

namespace {

__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + __expf(-x)); }

// RMS_norm.forward (wan2pt1.py:74-75) evaluated with the reference's bf16 rounding points:
//   n = bf16(||x||_2) ; y = bf16(x / max(n, 1e-12)) ; y = bf16(y * sqrt(C)) ; y = bf16(y * gamma) ; [y = bf16(silu(y))]
// One pixel per group of G lanes (G = 16 for C <= 128, else 32); 16-byte accesses.
template <int G>
__global__ void __launch_bounds__(256)
rms_silu_cl_kernel(const bf16* __restrict__ x, const bf16* __restrict__ gamma, bf16* __restrict__ y, size_t pixels, int C,
                   int apply_silu) {
  const int lane_in_group = threadIdx.x % G;
  const size_t group = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) / G;
  const size_t ngroups = ((size_t)gridDim.x * blockDim.x) / G;
  const int nvec = C >> 3;
  const float sqrt_c = sqrtf((float)C);
  for (size_t p = group; p < pixels; p += ngroups) {
    const uint4* xr = reinterpret_cast<const uint4*>(x + p * C);
    uint4 v[2];
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int idx = lane_in_group + i * G;
      if (idx < nvec) {
        v[i] = xr[idx];
        const float2 a = unpack_bf16x2(v[i].x), b = unpack_bf16x2(v[i].y), c = unpack_bf16x2(v[i].z), d = unpack_bf16x2(v[i].w);
        ss += a.x * a.x + a.y * a.y + b.x * b.x + b.y * b.y + c.x * c.x + c.y * c.y + d.x * d.x + d.y * d.y;
      }
    }
    const uint32_t gmask = (G == 32) ? 0xffffffffu : (0xFFFFu << ((threadIdx.x & 31) & 16));
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) ss += __shfl_xor_sync(gmask, ss, o, G);
    const float n = fmaxf(bf16_round(sqrtf(ss)), 1e-12f);
    uint4* yr = reinterpret_cast<uint4*>(y + p * C);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int idx = lane_in_group + i * G;
      if (idx < nvec) {
        const uint4 gv = reinterpret_cast<const uint4*>(gamma)[idx];
        const uint32_t xin[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
        const uint32_t gin[4] = {gv.x, gv.y, gv.z, gv.w};
        uint32_t out[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 xv = unpack_bf16x2(xin[k]);
          const float2 gg = unpack_bf16x2(gin[k]);
          float a = bf16_round(bf16_round(bf16_round(xv.x / n) * sqrt_c) * gg.x);
          float b = bf16_round(bf16_round(bf16_round(xv.y / n) * sqrt_c) * gg.y);
          if (apply_silu) {
            a = silu_f(a);
            b = silu_f(b);
          }
          out[k] = pack_bf16x2(a, b);
        }
        yr[idx] = make_uint4(out[0], out[1], out[2], out[3]);
      }
    }
  }
}

// out[t, 2h+a, 2w+b, :] = in[t, h, w, :]   (nn.Upsample(scale 2, nearest-exact), wan2pt1.py:78-83, 98-104)
__global__ void upsample2x_cl_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, int T, int H, int W, int cvec) {
  const size_t total = (size_t)T * (2 * H) * (2 * W) * cvec;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % cvec);
    size_t r = i / cvec;
    const int ow = (int)(r % (2 * W)); r /= (2 * W);
    const int oh = (int)(r % (2 * H));
    const int t = (int)(r / (2 * H));
    out[i] = in[(((size_t)t * H + (oh >> 1)) * W + (ow >> 1)) * cvec + c];
  }
}

// A[(to,oh,ow), tap*Cin + c] = X[t_base + to + dt, oh + dh - ph, ow + dw - pw, c]  (0 outside / in the K padding).
// X is addressed through explicit strides so planar (NCTHW) and channels-last inputs both work.
// One thread = one output pixel x eight consecutive k: a single 16-byte store (the matrix is 236 MB per 720p frame and this kernel is
// pure HBM write traffic), 32-bit index arithmetic, the (at most 81) scattered input reads hit L1/L2.
__global__ void __launch_bounds__(256)
im2row_kernel(const bf16* __restrict__ x, size_t sc, size_t st, size_t sh, size_t sw, int Tin, int Hin, int Win, int Cin,
              bf16* __restrict__ A, int Kpad, int Tout, int Hout, int Wout, int kt, int kh, int kw, int ph, int pw, int t_base) {
  const int groups = Kpad >> 3;
  const size_t total = (size_t)Tout * Hout * Wout * groups;
  const int K = kt * kh * kw * Cin;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    uint32_t r = (uint32_t)(i / groups);   // pixel index < 2^31 (checked by the launcher)
    const int ow = (int)(r % (uint32_t)Wout);
    r /= (uint32_t)Wout;
    const int oh = (int)(r % (uint32_t)Hout);
    const int to = (int)(r / (uint32_t)Hout);
    uint32_t w[4];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = g * 8 + e;
      unsigned short bits = 0;
      if (k < K) {
        const int c = k % Cin;
        int tap = k / Cin;
        const int dw = tap % kw;
        tap /= kw;
        const int dh = tap % kh;
        const int dt = tap / kh;
        const int ti = t_base + to + dt, hi = oh + dh - ph, wi = ow + dw - pw;
        if (ti >= 0 && ti < Tin && hi >= 0 && hi < Hin && wi >= 0 && wi < Win)
          bits = __bfloat16_as_ushort(x[c * sc + ti * st + hi * sh + wi * sw]);
      }
      if (e & 1) w[e >> 1] |= (uint32_t)bits << 16;
      else w[e >> 1] = bits;
    }
    *reinterpret_cast<uint4*>(A + i * 8) = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

// planar[c, p] = cl[p, c] for c < Cout (posterior mean = first z_dim channels of conv1's output)
__global__ void cl_to_planar_kernel(const bf16* __restrict__ cl, int C, bf16* __restrict__ planar, size_t pixels, int Cout) {
  const size_t total = pixels * Cout;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t p = i % pixels;
    const int c = (int)(i / pixels);
    planar[i] = cl[p * C + c];
  }
}

// ---- fp32 (the fp32 VAE)
__device__ __forceinline__ void store_pair(bf16* p, int C, float v) {   // p = &pair[pixel][0][c]
  const bf16 hi = __float2bfloat16_rn(v);
  p[0] = hi;
  p[C] = __float2bfloat16_rn(v - __bfloat162float(hi));
}

// RMS_norm.forward (wan2pt1.py:74-75) in fp32: F.normalize (x / max(||x||, 1e-12)) * sqrt(C) * gamma, then SiLU.  One warp per pixel.
__global__ void __launch_bounds__(256)
rms_silu_cl_f32_kernel(const float* __restrict__ x, const float* __restrict__ gamma, float* __restrict__ y, bf16* __restrict__ y_pair,
                       size_t pixels, int C, int apply_silu) {
  const int lane = threadIdx.x & 31;
  const float sqrt_c = sqrtf((float)C);
  for (size_t p = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < pixels; p += ((size_t)gridDim.x * blockDim.x) >> 5) {
    const float* xr = x + p * C;
    float ss = 0.f;
    for (int c = lane; c < C; c += 32) ss += xr[c] * xr[c];
    const float n = fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
    for (int c = lane; c < C; c += 32) {
      float v = xr[c] / n * sqrt_c * gamma[c];
      if (apply_silu) v = v / (1.0f + expf(-v));
      if (y_pair) store_pair(y_pair + p * 2 * C + c, C, v);
      else y[p * C + c] = v;
    }
  }
}

// out[t, 2h+a, 2w+b, :] = in[t, h, w, :] (nearest-exact), stored as the pair
__global__ void upsample2x_cl_f32_kernel(const float* __restrict__ in, bf16* __restrict__ out, int T, int H, int W, int C) {
  const size_t total = (size_t)T * (2 * H) * (2 * W) * C;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    size_t r = i / C;
    const int ow = (int)(r % (2 * W)); r /= (2 * W);
    const int oh = (int)(r % (2 * H));
    const int t = (int)(r / (2 * H));
    store_pair(out + (i / C) * 2 * C + c, C, in[(((size_t)t * H + (oh >> 1)) * W + (ow >> 1)) * C + c]);
  }
}

__global__ void planar_to_pair_kernel(const float* __restrict__ planar, int C, size_t pixels, bf16* __restrict__ pair, int Cp) {
  const size_t total = pixels * Cp;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % Cp);
    const size_t p = i / Cp;
    store_pair(pair + p * 2 * Cp + c, Cp, c < C ? planar[(size_t)c * pixels + p] : 0.f);
  }
}

__global__ void cl_to_planar_f32_kernel(const float* __restrict__ cl, int C, float* __restrict__ planar, size_t pixels, int Cout) {
  const size_t total = pixels * Cout;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
    planar[i] = cl[(i % pixels) * C + i / pixels];
}

// ---- tiled encode / decode: the blend of one tile with its blended neighbours, and its crop
template <class E, int V>
struct alignas(sizeof(E) * V) Vec {
  E v[V];
};
__device__ __forceinline__ float to_f(bf16 x) { return __bfloat162float(x); }
__device__ __forceinline__ float to_f(float x) { return x; }
template <class E>
__device__ __forceinline__ E from_f(float x);
template <>
__device__ __forceinline__ bf16 from_f<bf16>(float x) { return __float2bfloat16_rn(x); }
template <>
__device__ __forceinline__ float from_f<float>(float x) { return x; }

// diffusers' blend step  b[k] = a[-e + k] * (1 - k / e) + b[k] * (k / e)  as torch evaluates it on a tensor of type E: the weights are
// Python floats (double) converted to fp32, each product is rounded to E, then the sum is (no fused multiply-add anywhere).
template <class E>
__device__ __forceinline__ float blend_step(float a, float b, int k, int e) {
  const double r = (double)k / (double)e;
  const float wa = (float)(1.0 - r), wb = (float)r;
  const float pa = to_f(from_f<E>(__fmul_rn(a, wa))), pb = to_f(from_f<E>(__fmul_rn(b, wb)));
  return to_f(from_f<E>(__fadd_rn(pa, pb)));
}

// One thread per V consecutive columns of a tile row: the tile's value, blended vertically with the stored rows of the tile above and
// then horizontally with the stored columns of the tile to its left, stored to the output crop, the strip and the tail (TileBlend).
template <class E, int V>
__global__ void __launch_bounds__(256) tile_blend_kernel(TileBlend b) {
  using Vt = Vec<E, V>;
  const int nv = b.tw / V;
  const int ev = b.above ? min(b.above_h, b.th) : 0, eh = b.left ? min(b.left_w, b.tw) : 0;
  const size_t total = (size_t)b.C * b.T * b.th * nv;
  const E* tile = static_cast<const E*>(b.tile);
  const E* above = static_cast<const E*>(b.above);
  const E* left = static_cast<const E*>(b.left);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int x0 = (int)(i % nv) * V;
    const size_t r = i / nv;
    const int y = (int)(r % b.th);
    const size_t plane = r / b.th;
    Vt t = *reinterpret_cast<const Vt*>(tile + r * b.tw + x0);
    float v[V];
#pragma unroll
    for (int k = 0; k < V; ++k) v[k] = to_f(t.v[k]);
    if (y < ev) {
      const Vt a = *reinterpret_cast<const Vt*>(above + (plane * b.above_h + b.above_h - ev + y) * b.tw + x0);
#pragma unroll
      for (int k = 0; k < V; ++k) v[k] = blend_step<E>(to_f(a.v[k]), v[k], y, ev);
    }
    if (x0 < eh) {   // V divides eh: the whole vector is inside the extent
      const Vt a = *reinterpret_cast<const Vt*>(left + r * b.left_w + b.left_w - eh + x0);
#pragma unroll
      for (int k = 0; k < V; ++k) v[k] = blend_step<E>(to_f(a.v[k]), v[k], x0 + k, eh);
    }
#pragma unroll
    for (int k = 0; k < V; ++k) t.v[k] = from_f<E>(v[k]);
    if (b.strip && y >= b.th - b.strip_h)
      *reinterpret_cast<Vt*>(static_cast<E*>(b.strip) + (plane * b.strip_h + y - (b.th - b.strip_h)) * b.tw + x0) = t;
    if (b.tail && x0 >= b.tw - b.tail_w)
      *reinterpret_cast<Vt*>(static_cast<E*>(b.tail) + r * b.tail_w + x0 - (b.tw - b.tail_w)) = t;
    const int oy = b.oy + y, ox = b.ox + x0;
    if (y < b.crop_h && x0 < b.crop_w && oy < b.out_h && ox < b.out_w) {
      if (b.clamp) {
#pragma unroll
        for (int k = 0; k < V; ++k) t.v[k] = from_f<E>(fminf(fmaxf(v[k], -1.0f), 1.0f));
      }
      *reinterpret_cast<Vt*>(static_cast<E*>(b.out) + (plane * b.out_h + oy) * b.out_w + ox) = t;
    }
  }
}

int gcd_int(int a, int b) {
  while (b) {
    const int t = a % b;
    a = b;
    b = t;
  }
  return a;
}

}  // namespace

int tile_blend_vector(const TileBlend& b) {
  int g = b.tw;
  const int eh = b.left ? std::min(b.left_w, b.tw) : 0;
  for (int v : {b.left ? b.left_w : 0, eh, b.out_w, b.ox, b.crop_w < b.tw ? b.crop_w : 0, b.tail ? b.tail_w : 0}) g = gcd_int(g, v);
  for (const void* p : {b.tile, b.above, b.left, (const void*)b.out, (const void*)b.strip, (const void*)b.tail}) {
    const int misaligned = (int)(reinterpret_cast<uintptr_t>(p) & 15) / (b.fp32 ? 4 : 2);   // elements past a 16-byte boundary
    if (misaligned) g = gcd_int(g, misaligned);
  }
  const int vmax = b.fp32 ? 4 : 8;
  int v = 1;
  while (v < vmax && g % (2 * v) == 0) v *= 2;
  return v;
}

int launch_tile_blend(const TileBlend& b, cudaStream_t stream) {
  CE_REQUIRE(b.tile && b.out && b.C > 0 && b.T > 0 && b.th > 0 && b.tw > 0 && b.out_h > 0 && b.out_w > 0 && b.oy >= 0 && b.ox >= 0,
             "tile blend: null tile / output or empty extents");
  CE_REQUIRE(!b.above || b.above_h > 0, "tile blend: above rows");
  CE_REQUIRE(!b.left || b.left_w > 0, "tile blend: left columns");
  CE_REQUIRE(!b.strip || (b.strip_h > 0 && b.strip_h <= b.th), "tile blend: strip rows must be 1 .. th");
  CE_REQUIRE(!b.tail || (b.tail_w > 0 && b.tail_w <= b.tw), "tile blend: tail columns must be 1 .. tw");
  const int v = tile_blend_vector(b);
  const size_t n = (size_t)b.C * b.T * b.th * (b.tw / v);
  const int grid = grid_for(n);
#define CE_TILE_BLEND(E, V) tile_blend_kernel<E, V><<<grid, TPB, 0, stream>>>(b)
  if (b.fp32) {
    if (v == 4) CE_TILE_BLEND(float, 4);
    else if (v == 2) CE_TILE_BLEND(float, 2);
    else CE_TILE_BLEND(float, 1);
  } else {
    if (v == 8) CE_TILE_BLEND(bf16, 8);
    else if (v == 4) CE_TILE_BLEND(bf16, 4);
    else if (v == 2) CE_TILE_BLEND(bf16, 2);
    else CE_TILE_BLEND(bf16, 1);
  }
#undef CE_TILE_BLEND
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_rms_silu_cl_f32(const float* x, const float* gamma, float* y, bf16* y_pair, size_t pixels, int C, int apply_silu,
                           cudaStream_t stream) {
  CE_REQUIRE(x && gamma && (y == nullptr) != (y_pair == nullptr) && C > 0, "rms_silu fp32: null pointer, or not exactly one output");
  rms_silu_cl_f32_kernel<<<grid_for(pixels * 32), TPB, 0, stream>>>(x, gamma, y, y_pair, pixels, C, apply_silu);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_upsample2x_cl_f32(const float* in, bf16* out_pair, int T, int H, int W, int C, cudaStream_t stream) {
  upsample2x_cl_f32_kernel<<<grid_for((size_t)T * 4 * H * W * C), TPB, 0, stream>>>(in, out_pair, T, H, W, C);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_planar_to_pair(const float* planar, int C, size_t pixels, bf16* pair, int Cp, cudaStream_t stream) {
  CE_REQUIRE(Cp >= C, "planar_to_pair: Cp >= C");
  planar_to_pair_kernel<<<grid_for(pixels * Cp), TPB, 0, stream>>>(planar, C, pixels, pair, Cp);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_cl_to_planar_f32(const float* cl, int C, float* planar, size_t pixels, int Cout, cudaStream_t stream) {
  cl_to_planar_f32_kernel<<<grid_for(pixels * Cout), TPB, 0, stream>>>(cl, C, planar, pixels, Cout);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_rms_silu_cl(const bf16* x, const bf16* gamma, bf16* y, size_t pixels, int C, int apply_silu, cudaStream_t stream) {
  CE_REQUIRE(C % 8 == 0 && C <= 512, "rms_silu: C % 8, C <= 512");
  if (C <= 256 / 2) {
    const size_t threads = pixels * 16;
    rms_silu_cl_kernel<16><<<grid_for(threads), TPB, 0, stream>>>(x, gamma, y, pixels, C, apply_silu);
  } else {
    const size_t threads = pixels * 32;
    rms_silu_cl_kernel<32><<<grid_for(threads), TPB, 0, stream>>>(x, gamma, y, pixels, C, apply_silu);
  }
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_upsample2x_cl(const bf16* in, bf16* out, int T, int H, int W, int C, cudaStream_t stream) {
  CE_REQUIRE(C % 8 == 0, "upsample: C % 8");
  const size_t total = (size_t)T * 4 * H * W * (C / 8);
  upsample2x_cl_kernel<<<grid_for(total), TPB, 0, stream>>>(reinterpret_cast<const uint4*>(in), reinterpret_cast<uint4*>(out), T, H, W, C / 8);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_im2row(const bf16* x, size_t sc, size_t st, size_t sh, size_t sw, int Tin, int Hin, int Win, int Cin, bf16* A, int Kpad,
                  int Tout, int Hout, int Wout, int kt, int kh, int kw, int ph, int pw, int t_base, cudaStream_t stream) {
  CE_REQUIRE(Kpad % 8 == 0 && Kpad >= kt * kh * kw * Cin, "im2row: Kpad");
  CE_REQUIRE((size_t)Tout * Hout * Wout < (size_t(1) << 31) && (reinterpret_cast<uintptr_t>(A) & 15) == 0, "im2row: pixel count / alignment");
  const size_t total = (size_t)Tout * Hout * Wout * (Kpad / 8);
  im2row_kernel<<<grid_for(total), TPB, 0, stream>>>(x, sc, st, sh, sw, Tin, Hin, Win, Cin, A, Kpad, Tout, Hout, Wout, kt, kh, kw, ph, pw, t_base);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_cl_to_planar(const bf16* cl, int C, bf16* planar, size_t pixels, int Cout, cudaStream_t stream) {
  cl_to_planar_kernel<<<grid_for(pixels * Cout), TPB, 0, stream>>>(cl, C, planar, pixels, Cout);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

}  // namespace ce
