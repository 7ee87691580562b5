// HBM-bound row kernels of the DiT path: fp32 LayerNorm + adaLN modulate, RMSNorm-across-heads + 3D RoPE,
// patchify / unpatchify, the tiny-M Linear layers of the time embedder, the FP8 mode's row quantisation and the FP8
// self-attention's q | k and v quantisation.  All are coalesced 16-byte
// accesses with one CTA per token row (rows >> SM count), statistics in fp32 via warp shuffles.
#include "elementwise.cuh"

#include <cuda_fp8.h>

#include <type_traits>

namespace ce {

namespace {

constexpr int ROW_THREADS = 256;
constexpr int MAX_D = 8192;                // 64 lanes x 16 vectors x 8 bf16

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}

// ---------------------------------------------------------------------------------------------
// LayerNorm and RMSNorm: one WARP PAIR per token row (4 rows per 256-thread CTA), 16-byte vectors.  The row statistics come from
// one of two sources, chosen at compile time (FromPartials); the rest of each kernel is the same for both:
//   - reduced in the kernel: each lane keeps HV 16-byte vectors of the row in registers, all of them loaded before anything consumes
//     them; statistics = warp shuffles + one 64-thread named barrier.  ~100 registers/thread -> 16+ resident warps per SM, so one
//     row's arithmetic overlaps other rows' loads.
//   - per-(row, N tile) partials from the epilogue of the GEMM that produced the row (GemmArgs::stats_out): each warp merges them with
//     shuffles and the row kernel becomes a pure streaming pass: no reduction over the data, no barrier, loads and stores of different
//     vectors independent of each other.  The row is read from global memory where it is consumed, not held in registers.
__device__ __forceinline__ float2 pair_sum(float a, float b, float2* part) {
  a = warp_sum(a);
  b = warp_sum(b);
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) part[warp] = make_float2(a, b);
  named_bar_sync(1 + (warp >> 1), 64);
  const float2 o = part[warp ^ 1];
  return make_float2(a + o.x, b + o.y);
}

// Merge of the LayerNorm partials: Chan's pairwise update for (mean, M2), always (lower lane, higher lane) so that every lane ends with
// bit-identical values.
struct RowStat {
  float n, mean, m2;
};
__device__ __forceinline__ RowStat chan_merge(const RowStat& a, const RowStat& b) {
  const float tot = a.n + b.n;
  if (tot == 0.f) return a;
  const float delta = b.mean - a.mean, w = b.n / tot;
  RowStat r;
  r.n = tot;
  r.mean = fmaf(delta, w, a.mean);
  r.m2 = a.m2 + b.m2 + delta * delta * a.n * w;
  return r;
}
__device__ __forceinline__ RowStat warp_merge_stats(const float2* __restrict__ partial, int tiles, int tile_n, int D) {
  const int lane = threadIdx.x & 31;
  RowStat s{0.f, 0.f, 0.f};
  if (lane < tiles) {
    const float2 p = partial[lane];
    const int n = D - lane * tile_n;
    s.n = (float)(n < tile_n ? n : tile_n);
    s.mean = p.x;
    s.m2 = p.y;
  }
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    RowStat t;
    t.n = __shfl_xor_sync(0xffffffffu, s.n, o);
    t.mean = __shfl_xor_sync(0xffffffffu, s.mean, o);
    t.m2 = __shfl_xor_sync(0xffffffffu, s.m2, o);
    s = (lane & o) ? chan_merge(t, s) : chan_merge(s, t);
  }
  return s;
}

// This lane's vector lane64 + i * 64 (i < HV) of a row: from registers filled up front (zero past the row's end) when the kernel
// reduces over the row, from global memory where it is consumed when the statistics come from partials.
template <int HV, bool FromPartials>
struct RowVecs {
  const uint4* xr;
  int lane64;
  uint4 v[FromPartials ? 1 : HV];
  __device__ __forceinline__ RowVecs(const uint4* xr_, int lane64_, int nvec) : xr(xr_), lane64(lane64_) {
    if constexpr (!FromPartials) {
#pragma unroll
      for (int i = 0; i < HV; ++i) v[i] = lane64 + i * 64 < nvec ? xr[lane64 + i * 64] : make_uint4(0u, 0u, 0u, 0u);
    }
  }
  __device__ __forceinline__ uint4 operator[](int i) const { return FromPartials ? xr[lane64 + i * 64] : v[i]; }
};

template <int HV, bool FromPartials>
__global__ void __launch_bounds__(ROW_THREADS, 2)
layernorm_kernel(const bf16* __restrict__ x, int ldx, bf16* __restrict__ y, int ldy, int rows, int D, float eps,
                 const float* __restrict__ scale, const float* __restrict__ shift, int mod_stride, int rows_per_batch,
                 const float* __restrict__ weight, const float* __restrict__ bias, int scale_is_1p, RowPartials ps) {
  const int lane64 = threadIdx.x & 63;
  const int row0 = blockIdx.x * (ROW_THREADS / 64) + (threadIdx.x >> 6);
  const int row = min(row0, rows - 1);  // a pair past the last row joins the pair barrier, then leaves without storing
  const int nvec = D >> 3;
  const RowVecs<HV, FromPartials> v(reinterpret_cast<const uint4*>(x + (size_t)row * ldx), lane64, nvec);
  float mean, rstd;
  if constexpr (FromPartials) {
    const RowStat st = warp_merge_stats(ps.p + (size_t)row * ps.ld, ps.tiles, ps.tile_n, D);
    mean = st.mean;
    rstd = rsqrtf(st.m2 / (float)D + eps);
  } else {
    __shared__ float2 part[ROW_THREADS / 32];
    // single statistics pass on pivot-shifted data d = x - x[row, 0]:  mean = pivot + E[d],  var = E[d^2] - E[d]^2
    const float pivot = __bfloat162float(x[(size_t)row * ldx]);
    float s = 0.f, ss = 0.f;
#pragma unroll
    for (int i = 0; i < HV; ++i) {
      if (lane64 + i * 64 < nvec) {
        float f[8];
        unpack8(v[i], f);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = f[j] - pivot;
          s += d;
          ss = fmaf(d, d, ss);
        }
      }
    }
    const float2 tot = pair_sum(s, ss, part);
    const float md = tot.x / (float)D;
    mean = pivot + md;
    rstd = rsqrtf(fmaxf(tot.y / (float)D - md * md, 0.f) + eps);
  }
  if (row0 >= rows) return;
  const float nmr = -mean * rstd;
  const int b = row / rows_per_batch;
  uint4* yr = reinterpret_cast<uint4*>(y + (size_t)row * ldy);
  const float* pa = scale ? scale + (size_t)b * mod_stride : weight;  // multiplier: (1 + scale) / scale / affine weight
  const float* pb = scale ? shift + (size_t)b * mod_stride : bias;
  // vectors per batch: their parameter loads are in flight together.  Batching pays when the row is already in registers; when it is
  // streamed, a batch of one is faster (M = 14400, D = 5120 on an H100 80GB HBM3 at 700 W: 0.116 ms against 0.123 ms with 2).
  constexpr int G = FromPartials ? 1 : 2;
#pragma unroll
  for (int i0 = 0; i0 < HV; i0 += G) {
    float4 ta[G][2], tb[G][2];
    if (pa) {
#pragma unroll
      for (int k = 0; k < G; ++k) {
        const int idx = lane64 + (i0 + k) * 64;
        if (i0 + k < HV && idx < nvec) {
          const float4* qa = reinterpret_cast<const float4*>(pa + idx * 8);
          const float4* qb = reinterpret_cast<const float4*>(pb + idx * 8);
          ta[k][0] = qa[0]; ta[k][1] = qa[1];
          tb[k][0] = qb[0]; tb[k][1] = qb[1];
        }
      }
    }
#pragma unroll
    for (int k = 0; k < G; ++k) {
      const int idx = lane64 + (i0 + k) * 64;
      if (i0 + k < HV && idx < nvec) {
        float f[8], o[8];
        unpack8(v[i0 + k], f);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = fmaf(f[j], rstd, nmr);  // (x - mean) * rstd
        if (pa) {
          const float av[8] = {ta[k][0].x, ta[k][0].y, ta[k][0].z, ta[k][0].w, ta[k][1].x, ta[k][1].y, ta[k][1].z, ta[k][1].w};
          const float bv[8] = {tb[k][0].x, tb[k][0].y, tb[k][0].z, tb[k][0].w, tb[k][1].x, tb[k][1].y, tb[k][1].z, tb[k][1].w};
          if (scale && !scale_is_1p) {
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] = fmaf(o[j], 1.0f + av[j], bv[j]);
          } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] = fmaf(o[j], av[j], bv[j]);
          }
        }
        yr[idx] = pack8(o);
      }
    }
  }
}

// RMSNorm across heads (+ RoPE) on `nmat` matrices side by side in one row (q | k of the fused QKV output): blockIdx.y selects the
// matrix (column offset y * D, its own weight and, from partials, its own tile range)
template <int HV, bool FromPartials>
__global__ void __launch_bounds__(ROW_THREADS, 2)
rmsnorm_rope_kernel(bf16* __restrict__ x, int ldx, int rows, int D, float eps, const bf16* __restrict__ weight0,
                    const bf16* __restrict__ weight1, const float* __restrict__ rope_cos, const float* __restrict__ rope_sin, int L,
                    int head_dim, RowPartials ps, SpScatter sp) {
  const int lane64 = threadIdx.x & 63;
  const int row0 = blockIdx.x * (ROW_THREADS / 64) + (threadIdx.x >> 6);
  const int row = min(row0, rows - 1);  // a pair past the last row joins the pair barrier, then leaves without storing
  const int mat = blockIdx.y;
  const int nvec = D >> 3;
  uint4* xr = reinterpret_cast<uint4*>(x + (size_t)row * ldx + (size_t)mat * D);
  const RowVecs<HV, FromPartials> v(xr, lane64, nvec);
  float rstd;
  if constexpr (FromPartials) {
    const int lane = threadIdx.x & 31;
    float ss = lane < ps.tiles ? ps.p[(size_t)row * ps.ld + mat * ps.tiles + lane].x : 0.f;
    ss = warp_sum(ss);   // butterfly of commutative adds: identical in every lane
    rstd = rsqrtf(ss / (float)D + eps);
  } else {
    __shared__ float2 part[ROW_THREADS / 32];
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < HV; ++i) {
      float f[8];
      unpack8(v[i], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) ss = fmaf(f[j], f[j], ss);
    }
    const float2 tot = pair_sum(ss, 0.f, part);
    rstd = rsqrtf(tot.x / (float)D + eps);
  }
  if (row0 >= rows) return;
  const uint4* wr = reinterpret_cast<const uint4*>(mat ? weight1 : weight0);
  // the sequence-parallel scatter runs only with partials: it requires D % 256 == 0, where the GEMM writes them (launcher check)
  const bool scatter = FromPartials && sp.world;
  const int tok = scatter ? sp.tok0 + row % sp.rows_per_batch : (rope_cos ? row % L : 0);   // global token (RoPE position)
  const int half = head_dim >> 1;
  // One body, instantiated for each store: neither copy branches between vectors, so loads can move ahead of earlier stores.
  auto normalise = [&](auto store) {
#pragma unroll
    for (int i = 0; i < HV; ++i) {
      const int idx = lane64 + i * 64;
      if (idx < nvec) {
        float f[8], w[8], o[8];
        unpack8(v[i], f);
        unpack8(wr[idx], w);
        // diffusers RMSNorm with a bf16 weight: (x * rstd) rounded to bf16, then * weight (bf16 multiply)
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = bf16_round(bf16_round(f[j] * rstd) * w[j]);
        if (rope_cos) {
          const int pair0 = (idx * 8 % head_dim) >> 1;  // 4 consecutive (even, odd) pairs of one head
          const float4 cs = *reinterpret_cast<const float4*>(rope_cos + (size_t)tok * half + pair0);
          const float4 sn = *reinterpret_cast<const float4*>(rope_sin + (size_t)tok * half + pair0);
          const float cv[4] = {cs.x, cs.y, cs.z, cs.w};
          const float sv[4] = {sn.x, sn.y, sn.z, sn.w};
#pragma unroll
          for (int p = 0; p < 4; ++p) {
            const float re = o[2 * p], im = o[2 * p + 1];
            o[2 * p] = re * cv[p] - im * sv[p];
            o[2 * p + 1] = re * sv[p] + im * cv[p];
          }
        }
        store(idx, pack8(o));
      }
    }
  };
  if (scatter) {
    normalise([&](int idx, uint4 o) {   // to the rank that owns this head (peer store)
      const int c = idx * 8, head = c / head_dim, dr = head / sp.heads_per_rank, bi = row / sp.rows_per_batch;
      bf16* d = sp.dst[mat][dr] + ((size_t)bi * sp.L_total + tok) * ((size_t)sp.heads_per_rank * head_dim) +
                (size_t)(head % sp.heads_per_rank) * head_dim + c % head_dim;
      *reinterpret_cast<uint4*>(d) = o;
    });
  } else {
    normalise([&](int idx, uint4 o) { xr[idx] = o; });
  }
}

// Launches kernel<HV, FromPartials> (through `launch`, given both as integral constants) with the smallest HV -- 16-byte vectors
// per lane, 64 lanes per row -- that covers D.
template <class Launch>
void dispatch_row_kernel(int D, bool from_partials, Launch&& launch) {
  const int nvec = D / 8;
  auto by_hv = [&](auto from_partials_c) {
    if (nvec <= 128) launch(std::integral_constant<int, 2>(), from_partials_c);
    else if (nvec <= 256) launch(std::integral_constant<int, 4>(), from_partials_c);
    else if (nvec <= 640) launch(std::integral_constant<int, 10>(), from_partials_c);
    else launch(std::integral_constant<int, 16>(), from_partials_c);
  };
  if (from_partials) by_hv(std::true_type());
  else by_hv(std::false_type());
}

// ---------------------------------------------------------------------------------------------
__global__ void patchify_kernel(const bf16* __restrict__ x, bf16* __restrict__ patches, int B, int C, int T, int H, int W, int tok0, int ntok) {
  const int hp = H >> 1, wp = W >> 1;
  const int K = C * 4;
  const size_t total = (size_t)B * ntok * K;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % K);
    const size_t r = i / K;
    const int tok = tok0 + (int)(r % ntok);
    const int b = (int)(r / ntok);
    const int j = tok % wp, ii = (tok / wp) % hp, f = tok / (wp * hp);
    const int c = k >> 2, dh = (k >> 1) & 1, dw = k & 1;
    patches[i] = x[((((size_t)b * C + c) * T + f) * H + (2 * ii + dh)) * W + (2 * j + dw)];
  }
}

__global__ void unpatchify_kernel(const bf16* __restrict__ y, int ldy, bf16* __restrict__ out, int B, int C, int T, int H, int W) {
  const int hp = H >> 1, wp = W >> 1;
  const size_t total = (size_t)B * C * T * H * W;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    size_t r = i;
    const int w = (int)(r % W); r /= W;
    const int hh = (int)(r % H); r /= H;
    const int f = (int)(r % T); r /= T;
    const int c = (int)(r % C);
    const int b = (int)(r / C);
    const size_t row = (((size_t)b * T + f) * hp + (hh >> 1)) * wp + (w >> 1);
    out[i] = y[row * ldy + ((hh & 1) * 2 + (w & 1)) * C + c];
  }
}

// ---------------------------------------------------------------------------------------------
constexpr int SL_MAX_B = 8;
__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + __expf(-x)); }

template <bool W_BF16>
__global__ void __launch_bounds__(256)
small_linear_kernel(const float* __restrict__ x, int K, const void* __restrict__ Wv, const void* __restrict__ biasv, int N,
                    int B, int act, int in_silu_bf16, float* __restrict__ out_f32, bf16* __restrict__ out_bf16) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= N) return;
  float acc[SL_MAX_B];
#pragma unroll
  for (int b = 0; b < SL_MAX_B; ++b) acc[b] = 0.f;
  for (int k = lane * 4; k < K; k += 128) {
    float w[4];
    if (W_BF16) {
      const uint2 u = *reinterpret_cast<const uint2*>(reinterpret_cast<const bf16*>(Wv) + (size_t)warp * K + k);
      const float2 a = unpack_bf16x2(u.x), c = unpack_bf16x2(u.y);
      w[0] = a.x; w[1] = a.y; w[2] = c.x; w[3] = c.y;
    } else {
      const float4 u = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(Wv) + (size_t)warp * K + k);
      w[0] = u.x; w[1] = u.y; w[2] = u.z; w[3] = u.w;
    }
#pragma unroll
    for (int b = 0; b < SL_MAX_B; ++b) {
      if (b < B) {
        float4 xv = *reinterpret_cast<const float4*>(x + (size_t)b * K + k);
        if (in_silu_bf16) {  // act_fn(temb) evaluated on the bf16 tensor: SiLU in fp32, rounded to bf16
          xv.x = bf16_round(silu_f(xv.x)); xv.y = bf16_round(silu_f(xv.y));
          xv.z = bf16_round(silu_f(xv.z)); xv.w = bf16_round(silu_f(xv.w));
        }
        acc[b] += xv.x * w[0] + xv.y * w[1] + xv.z * w[2] + xv.w * w[3];
      }
    }
  }
#pragma unroll
  for (int b = 0; b < SL_MAX_B; ++b) acc[b] = warp_sum(acc[b]);
  if (lane == 0) {
    float bias = 0.f;
    if (biasv) bias = W_BF16 ? __bfloat162float(reinterpret_cast<const bf16*>(biasv)[warp]) : reinterpret_cast<const float*>(biasv)[warp];
    for (int b = 0; b < B; ++b) {
      float y = acc[b] + bias;
      if (out_bf16) y = bf16_round(y);  // the Linear output is a bf16 tensor in the reference
      if (act == 1) y = silu_f(y);
      if (out_f32) out_f32[(size_t)b * N + warp] = y;
      if (out_bf16) out_bf16[(size_t)b * N + warp] = __float2bfloat16_rn(y);
    }
  }
}

__global__ void timestep_sinusoid_kernel(const float* __restrict__ t, float* __restrict__ emb, int B, int dim) {
  const int half = dim >> 1;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * half) return;
  const int b = i / half, k = i % half;
  // exponent = -ln(10000) * k / half (fp32, as torch.arange(float32) * scalar / half), freq = exp(exponent)
  const float exponent = (-9.210340371976184f * (float)k) / (float)half;
  const float arg = t[b] * expf(exponent);
  emb[(size_t)b * dim + k] = cosf(arg);
  emb[(size_t)b * dim + half + k] = sinf(arg);
}

__global__ void add_table_kernel(const float* __restrict__ table, int table_rows, const bf16* __restrict__ src, int src_ld,
                                 int src_per_chunk, float* __restrict__ dst, int B, int n, int chunks, unsigned plus_one_mask) {
  // dst[l, b, c, d] = table[l, c, d] + float(src[b, (src_per_chunk ? c*n : 0) + d])
  const size_t total = (size_t)table_rows * B * chunks * n;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int d = (int)(i % n);
    size_t r = i / n;
    const int c = (int)(r % chunks); r /= chunks;
    const int b = (int)(r % B);
    const int l = (int)(r / B);
    const float v = table[((size_t)l * chunks + c) * n + d] + __bfloat162float(src[(size_t)b * src_ld + (src_per_chunk ? c * n : 0) + d]);
    dst[i] = ((plus_one_mask >> c) & 1u) ? 1.0f + v : v;  // "scale" chunks are stored as (1 + scale)
  }
}

// One CTA per row: the row's absolute maximum (exact in fp32), then q = e4m3_satfinite(x / s) with s = amax / 448 (1 for a zero
// row) as IEEE divisions, the same operations as the torch expression of the rule (DESIGN.md, "FP8 mode").  The second read of
// the row comes from L1 / L2.
__global__ void __launch_bounds__(ROW_THREADS)
quantize_rows_fp8_kernel(const bf16* __restrict__ x, int ldx, int K, uint8_t* __restrict__ q, int ldq, float* __restrict__ scale) {
  __shared__ float part[ROW_THREADS / 32];
  const bf16* xr = x + (size_t)blockIdx.x * ldx;
  float m = 0.f;
  for (int c = threadIdx.x * 8; c < K; c += ROW_THREADS * 8) {
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(xr + c), f);
#pragma unroll
    for (int e = 0; e < 8; ++e) m = fmaxf(m, fabsf(f[e]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = m;
  __syncthreads();
  m = part[0];
#pragma unroll
  for (int w = 1; w < ROW_THREADS / 32; ++w) m = fmaxf(m, part[w]);
  const float s = m == 0.f ? 1.f : __fdiv_rn(m, 448.f);
  if (threadIdx.x == 0) scale[blockIdx.x] = s;
  uint8_t* qr = q + (size_t)blockIdx.x * ldq;
  for (int c = threadIdx.x * 8; c < K; c += ROW_THREADS * 8) {
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(xr + c), f);
    uint32_t w[4];
#pragma unroll
    for (int e = 0; e < 4; ++e)
      w[e] = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(f[2 * e], s), __fdiv_rn(f[2 * e + 1], s)), __NV_SATFINITE, __NV_E4M3);
    *reinterpret_cast<uint2*>(qr + c) = make_uint2(w[0] | (w[1] << 16), w[2] | (w[3] << 16));
  }
}

// FP8 self-attention, q | k: one warp per (row, head); lane l holds values 4l .. 4l+3 of the head's 128.  Same operations as
// quantize_rows_fp8_kernel.
__global__ void __launch_bounds__(ROW_THREADS)
quantize_heads_fp8_kernel(const bf16* __restrict__ x, int ldx, int rows, int nh, uint8_t* __restrict__ q, int ldq, float* __restrict__ scale) {
  const int gw = blockIdx.x * (ROW_THREADS / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (gw >= rows * nh) return;
  const int row = gw / nh, hd = gw - row * nh;
  const uint2 u = *reinterpret_cast<const uint2*>(x + (size_t)row * ldx + hd * 128 + lane * 4);
  const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y);
  const float m = warp_max(fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(b.x), fabsf(b.y))));
  const float s = m == 0.f ? 1.f : __fdiv_rn(m, 448.f);
  if (lane == 0) scale[(size_t)row * nh + hd] = s;
  const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(a.x, s), __fdiv_rn(a.y, s)), __NV_SATFINITE, __NV_E4M3);
  const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(b.x, s), __fdiv_rn(b.y, s)), __NV_SATFINITE, __NV_E4M3);
  *reinterpret_cast<uint32_t*>(q + (size_t)row * ldq + hd * 128 + lane * 4) = lo | (hi << 16);
}

// FP8 self-attention, v pass 1: the channel maxima over a sample's tokens.  CTA (32 channels, sample b): 64 row groups x 4 lanes of
// 8 channels (16-byte loads) walk the tokens, then one smem reduction per channel.
constexpr int VMAX_COLS = 32;
__global__ void __launch_bounds__(ROW_THREADS)
v_channel_scale_kernel(const bf16* __restrict__ v, int ldv, int L, int D, float* __restrict__ scale) {
  __shared__ float part[ROW_THREADS / 4][VMAX_COLS + 1];
  const int b = blockIdx.y;
  const int sub = threadIdx.x & 3, rg = threadIdx.x >> 2;
  const int c0 = blockIdx.x * VMAX_COLS + sub * 8;
  float m[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const bf16* base = v + (size_t)b * L * ldv + c0;
#pragma unroll 4
  for (int r = rg; r < L; r += ROW_THREADS / 4) {
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(base + (size_t)r * ldv), f);
#pragma unroll
    for (int e = 0; e < 8; ++e) m[e] = fmaxf(m[e], fabsf(f[e]));
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) part[rg][sub * 8 + e] = m[e];
  __syncthreads();
  if (threadIdx.x < VMAX_COLS) {
    float mx = 0.f;
    for (int r = 0; r < ROW_THREADS / 4; ++r) mx = fmaxf(mx, part[r][threadIdx.x]);
    scale[(size_t)b * D + blockIdx.x * VMAX_COLS + threadIdx.x] = mx == 0.f ? 1.f : __fdiv_rn(mx, 448.f);
  }
}

// Key at stored position p of a 32-key group of V^T.  The S accumulator gives a thread keys 8c + 2 (lane % 4) + {0, 1}; the 8-bit
// A fragment of a K32 step wants keys 4 (lane % 4) + {0..3} (+ 16) in one register: packing the accumulator pairs c = 2j, 2j + 1
// into register j of the fragment makes fragment position p hold this key, so V^T is stored in the same order.
__device__ __forceinline__ int vt_key_of(int p) { return 16 * (p >> 4) + 8 * ((p & 3) >> 1) + 2 * ((p & 15) >> 2) + (p & 1); }

// FP8 self-attention, v pass 2: CTA (32-key group g, head h, sample b) stages the [32 keys x 128 channels] bf16 block in shared
// memory, then thread (channel c, half) writes stored positions 16 half .. 16 half + 15 of channel c's row (16 bytes).
__global__ void __launch_bounds__(ROW_THREADS)
quantize_vt_fp8_kernel(const bf16* __restrict__ v, int ldv, int L, int H, const float* __restrict__ scale, uint8_t* __restrict__ vt,
                       int Lpad) {
  __shared__ __align__(16) bf16 tile[32][128];
  const int g = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  for (int i = threadIdx.x; i < 32 * 16; i += ROW_THREADS) {
    const int r = i >> 4, ch = (i & 15) * 8, key = g * 32 + r;
    uint4 u = make_uint4(0, 0, 0, 0);
    if (key < L) u = *reinterpret_cast<const uint4*>(v + ((size_t)b * L + key) * ldv + h * 128 + ch);
    *reinterpret_cast<uint4*>(&tile[r][ch]) = u;
  }
  __syncthreads();
  const int c = threadIdx.x >> 1, half = threadIdx.x & 1;
  const float s = scale[(size_t)b * H * 128 + h * 128 + c];
  uint32_t w[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    uint32_t word = 0;
#pragma unroll
    for (int e = 0; e < 4; e += 2) {
      const int p = 16 * half + 4 * j + e;
      const float x0 = __bfloat162float(tile[vt_key_of(p)][c]), x1 = __bfloat162float(tile[vt_key_of(p + 1)][c]);
      const uint32_t pair = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(x0, s), __fdiv_rn(x1, s)), __NV_SATFINITE, __NV_E4M3);
      word |= pair << (8 * e);
    }
    w[j] = word;
  }
  *reinterpret_cast<uint4*>(vt + (((size_t)b * H + h) * 128 + c) * Lpad + g * 32 + 16 * half) = make_uint4(w[0], w[1], w[2], w[3]);
}

// Score rules of softmax_rows_kernel: which keys of a row count, the score of key j from the GEMM accumulators s, and the
// exponential of (score - row max).
template <bool FAST>
struct ScaledScore {
  float scale;
  __device__ int keys(int cols) const { return cols; }
  __device__ float operator()(const float* s, int, int j) const { return s[j]; }
  __device__ float exp(float d) const { return FAST ? __expf(d * scale) : expf(d * scale); }
};
struct T5Score {
  const bf16* bias;
  int bias_ld, Lq, valid;
  __device__ int keys(int cols) const { return valid < cols ? valid : cols; }
  __device__ float operator()(const float* s, int row, int j) const {
    const bf16* bh = bias + (size_t)(row / Lq) * bias_ld + (Lq - 1 - row % Lq);
    return bf16_round(bf16_round(s[j]) + __bfloat162float(bh[j]));
  }
  __device__ float exp(float d) const { return expf(d); }
};
struct ClipScore {
  float scale;
  __device__ int keys(int cols) const { return cols; }
  __device__ float operator()(const float* s, int, int j) const { return bf16_round(bf16_round(s[j]) * scale); }
  __device__ float exp(float d) const { return expf(d); }
};

__device__ __forceinline__ void store_prob(float* p, float v) { *p = v; }
__device__ __forceinline__ void store_prob(bf16* p, float v) { *p = __float2bfloat16_rn(v); }

// One block per row: two-pass block reduction (max, then sum of exponentials), then p = exp(score - max) / sum.
template <class Score, class Out>
__global__ void __launch_bounds__(256)
softmax_rows_kernel(const float* __restrict__ S, int lds, Out* __restrict__ P, int ldp, int cols, Score score) {
  __shared__ float red[32];
  const int row = blockIdx.x;
  const float* s = S + (size_t)row * lds;
  Out* p = P + (size_t)row * ldp;
  const int nk = score.keys(cols);
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < nk; j += blockDim.x) mx = fmaxf(mx, score(s, row, j));
  mx = warp_max(mx);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = warp_max((threadIdx.x & 31) < (blockDim.x >> 5) ? red[threadIdx.x & 31] : -INFINITY);
  __syncthreads();
  float sum = 0.f;
  for (int j = threadIdx.x; j < nk; j += blockDim.x) sum += score.exp(score(s, row, j) - mx);
  sum = warp_sum(sum);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = warp_sum((threadIdx.x & 31) < (blockDim.x >> 5) ? red[threadIdx.x & 31] : 0.f);
  const float inv = 1.0f / sum;
  for (int j = threadIdx.x; j < ldp; j += blockDim.x) store_prob(p + j, j < nk ? score.exp(score(s, row, j) - mx) * inv : 0.f);
}

}  // namespace

int launch_softmax_rows(const float* S, int lds, bf16* P, int ldp, int rows, int cols, const SoftmaxScores& sc, cudaStream_t stream) {
  switch (sc.rule) {
    case SOFTMAX_SCALED:
      softmax_rows_kernel<<<rows, 256, 0, stream>>>(S, lds, P, ldp, cols, ScaledScore<true>{sc.scale});
      break;
    case SOFTMAX_T5:
      softmax_rows_kernel<<<rows, 256, 0, stream>>>(S, lds, P, ldp, cols, T5Score{sc.bias, sc.bias_ld, sc.Lq, sc.valid});
      break;
    case SOFTMAX_CLIP:
      softmax_rows_kernel<<<rows, 256, 0, stream>>>(S, lds, P, ldp, cols, ClipScore{sc.scale});
      break;
  }
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_softmax_rows_f32(const float* S, int lds, float* P, int ldp, int rows, int cols, float scale, cudaStream_t stream) {
  softmax_rows_kernel<<<rows, 256, 0, stream>>>(S, lds, P, ldp, cols, ScaledScore<false>{scale});
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_quantize_rows_fp8(const bf16* x, int ldx, int rows, int K, uint8_t* q, int ldq, float* scale, cudaStream_t stream) {
  CE_REQUIRE(rows > 0 && K > 0 && K % 16 == 0, "quantize_rows_fp8: rows > 0 and a width that is a multiple of 16");
  CE_REQUIRE(ldx % 8 == 0 && ldx >= K && ldq % 16 == 0 && ldq >= K, "quantize_rows_fp8: ldx % 8, ldq % 16, both >= K");
  CE_REQUIRE(x && q && scale && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(q) & 15) == 0,
             "quantize_rows_fp8: x and q must be 16-byte aligned");
  quantize_rows_fp8_kernel<<<rows, ROW_THREADS, 0, stream>>>(x, ldx, K, q, ldq, scale);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_quantize_heads_fp8(const bf16* x, int ldx, int rows, int nh, uint8_t* q, int ldq, float* scale, cudaStream_t stream) {
  CE_REQUIRE(rows > 0 && nh > 0, "quantize_heads_fp8: rows > 0 and at least one head");
  CE_REQUIRE(ldx % 8 == 0 && ldx >= nh * 128 && ldq % 16 == 0 && ldq >= nh * 128, "quantize_heads_fp8: ldx % 8, ldq % 16, both >= nh * 128");
  CE_REQUIRE(x && q && scale && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(q) & 15) == 0,
             "quantize_heads_fp8: x and q must be 16-byte aligned");
  const int64_t warps = (int64_t)rows * nh;
  quantize_heads_fp8_kernel<<<(unsigned)((warps + ROW_THREADS / 32 - 1) / (ROW_THREADS / 32)), ROW_THREADS, 0, stream>>>(x, ldx, rows, nh, q,
                                                                                                                        ldq, scale);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_quantize_v_fp8(const bf16* v, int ldv, int B, int L, int H, uint8_t* vt, int Lpad, float* scale, cudaStream_t stream) {
  CE_REQUIRE(B > 0 && L > 0 && H > 0 && Lpad >= L && Lpad % 32 == 0, "quantize_v_fp8: B, L, H > 0 and Lpad >= L a multiple of 32");
  CE_REQUIRE(ldv % 8 == 0 && ldv >= H * 128, "quantize_v_fp8: ldv % 8 and >= H * 128");
  CE_REQUIRE(v && vt && scale && (reinterpret_cast<uintptr_t>(v) & 15) == 0 && (reinterpret_cast<uintptr_t>(vt) & 15) == 0,
             "quantize_v_fp8: v and vt must be 16-byte aligned");
  v_channel_scale_kernel<<<dim3(H * 128 / VMAX_COLS, B), ROW_THREADS, 0, stream>>>(v, ldv, L, H * 128, scale);
  CE_CHECK_CUDA(cudaGetLastError());
  quantize_vt_fp8_kernel<<<dim3(Lpad / 32, H, B), ROW_THREADS, 0, stream>>>(v, ldv, L, H, scale, vt, Lpad);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_layernorm(const bf16* x, int ldx, bf16* y, int ldy, int rows, int D, float eps, const float* scale, const float* shift,
                     int mod_stride, int rows_per_batch, const float* weight, const float* bias, int scale_is_1p, const RowPartials& ps,
                     cudaStream_t stream) {
  CE_REQUIRE(rows > 0 && D % 8 == 0 && D <= MAX_D, "layernorm: D must be a multiple of 8 and <= 8192");
  CE_REQUIRE(ldx % 8 == 0 && ldy % 8 == 0, "layernorm: leading dims % 8");
  CE_REQUIRE((scale == nullptr) == (shift == nullptr), "layernorm: scale and shift come together");
  CE_REQUIRE((weight == nullptr) == (bias == nullptr), "layernorm: weight and bias come together");
  if (ps.p)
    CE_REQUIRE(ps.tiles >= 1 && ps.tiles <= 32 && ps.ld >= ps.tiles && ps.tile_n > 0 && (ps.tiles - 1) * ps.tile_n < D && ps.tiles * ps.tile_n >= D,
               "layernorm(stats): the tile partials must cover exactly [0, D) in at most 32 tiles");
  if (rows_per_batch <= 0) rows_per_batch = rows;
  const int grid = (rows + ROW_THREADS / 64 - 1) / (ROW_THREADS / 64);
  dispatch_row_kernel(D, ps.p != nullptr, [&](auto hv, auto from_partials) {
    layernorm_kernel<hv, from_partials><<<grid, ROW_THREADS, 0, stream>>>(x, ldx, y, ldy, rows, D, eps, scale, shift, mod_stride,
                                                                          rows_per_batch, weight, bias, scale_is_1p, ps);
  });
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_rmsnorm_rope(bf16* x, int ldx, int rows, int D, float eps, const bf16* weight0, const bf16* weight1, int nmat,
                        const float* rope_cos, const float* rope_sin, int L, int head_dim, const RowPartials& ps, cudaStream_t stream,
                        const SpScatter* sp) {
  CE_REQUIRE(rows > 0 && D % 8 == 0 && D <= MAX_D, "rmsnorm: D must be a multiple of 8 and <= 8192");
  CE_REQUIRE(ldx % 8 == 0 && weight0 != nullptr, "rmsnorm: ldx % 8, weight");
  CE_REQUIRE(nmat == 1 || (nmat == 2 && weight1 != nullptr), "rmsnorm: one or two matrices");
  if (ps.p) CE_REQUIRE(ps.tiles >= 1 && ps.tiles <= 32 && ps.ld >= nmat * ps.tiles, "rmsnorm(stats): tile partials");
  if (rope_cos) CE_REQUIRE(rope_sin && L > 0 && head_dim % 8 == 0 && D % head_dim == 0, "rmsnorm: rope table / head_dim");
  SpScatter spv;
  if (sp) spv = *sp;
  if (spv.world)
    CE_REQUIRE(ps.p && spv.world <= 8 && spv.heads_per_rank > 0 && spv.rows_per_batch > 0 && rows % spv.rows_per_batch == 0,
               "rmsnorm: scatter (with partials only)");
  const dim3 grid((rows + ROW_THREADS / 64 - 1) / (ROW_THREADS / 64), nmat);
  dispatch_row_kernel(D, ps.p != nullptr, [&](auto hv, auto from_partials) {
    rmsnorm_rope_kernel<hv, from_partials><<<grid, ROW_THREADS, 0, stream>>>(x, ldx, rows, D, eps, weight0, weight1, rope_cos, rope_sin,
                                                                             L, head_dim, ps, spv);
  });
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_patchify(const bf16* x, bf16* patches, int B, int C, int T, int H, int W, int tok0, int ntok, cudaStream_t stream) {
  CE_REQUIRE(H % 2 == 0 && W % 2 == 0, "patchify: H, W must be even");
  CE_REQUIRE(tok0 >= 0 && ntok > 0 && tok0 + ntok <= T * (H / 2) * (W / 2), "patchify: token range");
  const size_t total = (size_t)B * ntok * C * 4;
  const int grid = (int)((total + 255) / 256 < device_sm_count() * 16 ? (total + 255) / 256 : device_sm_count() * 16);
  patchify_kernel<<<grid, 256, 0, stream>>>(x, patches, B, C, T, H, W, tok0, ntok);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_unpatchify(const bf16* y, int ldy, bf16* out, int B, int C, int T, int H, int W, cudaStream_t stream) {
  const size_t total = (size_t)B * C * T * H * W;
  const int grid = (int)((total + 255) / 256 < device_sm_count() * 16 ? (total + 255) / 256 : device_sm_count() * 16);
  unpatchify_kernel<<<grid, 256, 0, stream>>>(y, ldy, out, B, C, T, H, W);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_small_linear(const float* x, int K, const void* W, const void* bias, int w_is_bf16, int N, int B, int act,
                        int in_silu_bf16, float* out_f32, bf16* out_bf16, cudaStream_t stream) {
  CE_REQUIRE(B >= 1 && B <= SL_MAX_B, "small_linear: batch must be 1..8");
  CE_REQUIRE(K % 4 == 0, "small_linear: K % 4");
  const int blocks = (N * 32 + 255) / 256;
  if (w_is_bf16)
    small_linear_kernel<true><<<blocks, 256, 0, stream>>>(x, K, W, bias, N, B, act, in_silu_bf16, out_f32, out_bf16);
  else
    small_linear_kernel<false><<<blocks, 256, 0, stream>>>(x, K, W, bias, N, B, act, in_silu_bf16, out_f32, out_bf16);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_timestep_sinusoid(const float* t, float* emb, int B, int dim, cudaStream_t stream) {
  const int n = B * (dim / 2);
  timestep_sinusoid_kernel<<<(n + 127) / 128, 128, 0, stream>>>(t, emb, B, dim);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_add_table(const float* table, int table_rows, const bf16* src, int src_ld, float* dst, int B, int n,
                     int chunks, cudaStream_t stream, unsigned plus_one_mask) {
  const size_t total = (size_t)table_rows * B * chunks * n;
  const int grid = (int)((total + 255) / 256 < device_sm_count() * 8 ? (total + 255) / 256 : device_sm_count() * 8);
  const int src_per_chunk = src_ld >= chunks * n ? 1 : 0;
  add_table_kernel<<<grid, 256, 0, stream>>>(table, table_rows, src, src_ld, src_per_chunk, dst, B, n, chunks, plus_one_mask);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

}  // namespace ce
