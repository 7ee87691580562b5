// FP8 self-attention forward for sm_90a (head_dim 128), flash-style, on e4m3 wgmma (DESIGN.md, "FP8 attention").
//
//   S = (q^ k^T) s_q[i] s_k[j],   P^ = e4m3(256 exp2(S scale log2e - m)),   out = bf16((sum_j P^ V^) s_v[c] / sum_j P^)
//
// q^, k^: e4m3 with one scale per (token, head); V^: e4m3 with one scale per (sample, channel), stored transposed (V^T, keys
// contiguous, launch_quantize_v_fp8) because FP8 wgmma takes B K-major only.  The online softmax runs over 128-key tiles in key
// order as in attention_fwd_kernel; a quarter of the exponentials are evaluated on the FMA pipe (exp2_fma) so that MUFU does not
// set the pace.  The row sum of the quantized P^ comes from the tensor cores: the same A fragment times a tile of ones (m64n8k32), so the softmax does no per-score
// work for it and the normalisation matches what was multiplied.  Each key tile's P^ V^ and row sum go into fresh accumulators
// and are added with o = o * alpha + o_tile in fp32, so no FP8 wgmma accumulates over more than 128 keys.
//
// One CTA per (128-query tile, head, batch); 384 threads = 3 warpgroups:
//   warpgroup 0     warp 0 (one lane): TMA of the Q tile once, then K_j / V^T_j tiles through NS-deep rings;
//                   warp 1: the 128 key scales of tile j into shared memory (a strided gather TMA cannot do)
//   warpgroups 1,2  one 64-query half of the tile each: S_j = Q K_j^T (4 x K32, both from shared memory), online softmax,
//                   O_j = P^_j V^_j (4 x K32, P^_j from registers as the A operand)
// Every tile is one 128-byte swizzled box (16 KB), half the bf16 kernel's, so the rings are twice as deep.
#include "attention.cuh"
#include "wgmma.cuh"

#include <cuda_fp8.h>

namespace ce {

namespace {

constexpr int HD = 128;
constexpr int BQ = 128;
constexpr int BKV = 128;
constexpr int NS = 4;   // ring depth
constexpr int ATTN_THREADS = 384;
constexpr uint32_t TILE_BYTES = 128 * 128;   // 16 KB: [128 rows x 128 e4m3]

struct SmemLayout {
  static constexpr uint32_t q = 0;
  static constexpr uint32_t k = q + TILE_BYTES;
  static constexpr uint32_t v = k + NS * TILE_BYTES;
  static constexpr uint32_t ones = v + NS * TILE_BYTES;   // [8 x 128] e4m3 ones: the B operand of the row sums
  static constexpr uint32_t ks = ones + 1024;            // NS x 128 key scales
  static constexpr uint32_t bars = ks + NS * BKV * 4;
  static constexpr uint32_t total = bars + 256;
};

// barrier indices
enum { Q_FULL = 0, K_FULL = 1, K_EMPTY = K_FULL + NS, V_FULL = K_EMPTY + NS, V_EMPTY = V_FULL + NS, NUM_BARS = V_EMPTY + NS };

// 2^x on the FMA pipe, for the share of the exponentials that would otherwise queue on MUFU: x = n + f with n = rint(x) by the
// 1.5 * 2^23 trick and |f| <= 1/2, 2^f by its degree-3 Taylor polynomial (relative error < 8e-4 in fp32, far below e4m3's 2^-4), n
// added to the exponent field.  x is clamped to -126 so that the result stays a normal number (it rounds to e4m3 0 there); -inf
// gives 2^-126.
__device__ __forceinline__ float exp2_fma(float x) {
  x = fmaxf(x, -126.f);
  const float t = x + 12582912.f;
  const float f = x - (t - 12582912.f);
  const float p = fmaf(fmaf(fmaf(0.0555041087f, f, 0.240226507f), f, 0.693147181f), f, 1.f);
  return __int_as_float(__float_as_int(p) + (__float_as_int(t) << 23));
}

// e4m3(exp2(a0)) | e4m3(exp2(a1)) << 8, nearest-even, satfinite; exp2 on MUFU or (FMA) on the FMA pipe.
template <bool FMA>
__device__ __forceinline__ uint32_t exp2_e4m3x2(float a0, float a1) {
  const float2 e = FMA ? make_float2(exp2_fma(a0), exp2_fma(a1)) : make_float2(fast_exp2(a0), fast_exp2(a1));
  return __nv_cvt_float2_to_fp8x2(e, __NV_SATFINITE, __NV_E4M3);
}

__global__ void __launch_bounds__(ATTN_THREADS, 1)
attention_fp8_kernel(const __grid_constant__ CUtensorMap tma_q, const __grid_constant__ CUtensorMap tma_k,
                     const __grid_constant__ CUtensorMap tma_vt, AttnFp8Args a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SmemLayout::bars);
  float* kscale = reinterpret_cast<float*>(smem + SmemLayout::ks);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * BQ;
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  const int T = (a.L + BKV - 1) / BKV;

  for (int i = threadIdx.x; i < 256; i += ATTN_THREADS) reinterpret_cast<uint32_t*>(smem + SmemLayout::ones)[i] = 0x38383838u;  // 1.0
  fence_proxy_async_smem();   // read by wgmma (async proxy)
  if (threadIdx.x == 0) {
    if ((smem_u32(smem) & 1023u) != 0) __trap();  // the swizzled tiles need 1024-byte alignment
    mbar_init(&bars[Q_FULL], 1);
    for (int i = 0; i < NS; ++i) {
      mbar_init(&bars[K_FULL + i], 1 + 32);   // the TMA's expect_tx, and every lane of the key-scale warp
      mbar_init(&bars[K_EMPTY + i], 8);       // every consumer warp (each has read its key scales)
      mbar_init(&bars[V_FULL + i], 1);
      mbar_init(&bars[V_EMPTY + i], 2);       // one per consumer warpgroup
    }
    fence_mbar_init();
    tma_prefetch_desc(&tma_q);
    tma_prefetch_desc(&tma_k);
    tma_prefetch_desc(&tma_vt);
  }
  __syncthreads();

  if (warp < 4) {
    // ---------------------------------------------------------------- producers
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one_sync()) {
      mbar_arrive_expect_tx(&bars[Q_FULL], TILE_BYTES);
      tma_load_3d(smem + SmemLayout::q, &tma_q, &bars[Q_FULL], h * HD, q0, b);
      for (int t = 0; t < T; ++t) {
        const int s = t % NS;
        const uint32_t free_parity = ((t / NS) & 1) ^ 1;
        mbar_wait(&bars[K_EMPTY + s], free_parity);
        mbar_arrive_expect_tx(&bars[K_FULL + s], TILE_BYTES);
        tma_load_3d(smem + SmemLayout::k + s * TILE_BYTES, &tma_k, &bars[K_FULL + s], h * HD, t * BKV, b);
        mbar_wait(&bars[V_EMPTY + s], free_parity);
        mbar_arrive_expect_tx(&bars[V_FULL + s], TILE_BYTES);
        tma_load_3d(smem + SmemLayout::v + s * TILE_BYTES, &tma_vt, &bars[V_FULL + s], t * BKV, h * HD, b);
      }
    } else if (warp == 1) {
      const float* ksrc = a.k_scale + (size_t)b * a.L * a.lds + h;
      for (int t = 0; t < T; ++t) {
        const int s = t % NS;
        mbar_wait(&bars[K_EMPTY + s], ((t / NS) & 1) ^ 1);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = t * BKV + lane * 4 + e;
          kscale[s * BKV + lane * 4 + e] = key < a.L ? ksrc[(size_t)key * a.lds] : 1.f;
        }
        mbar_arrive(&bars[K_FULL + s]);
      }
    }
    return;
  }

  // ------------------------------------------------------------------ consumers: 64 query rows per warpgroup
  setmaxnreg_inc<232>();
  const int wg = (warp >> 2) - 1;
  const bool signaller = (threadIdx.x & 127) == 0;
  const int quad = lane & 3;
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // the thread's rows of the query tile: r0 and r0 + 8
  const float sl2 = a.scale * 1.4426950408889634f;
  const uint32_t q_smem = smem_u32(smem + SmemLayout::q) + wg * 64 * 128;
  float rf[2];   // s_q * scale * log2(e) of the two rows
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int row = q0 + r0 + 8 * hh;
    rf[hh] = (row < a.L ? a.q_scale[((size_t)b * a.L + row) * a.lds + h] : 1.f) * sl2;   // rows >= L are zeros, not stored
  }

  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // per row: running max, row sum of P^ (every lane has the whole row)

  mbar_wait(&bars[Q_FULL], 0);
  for (int t = 0; t < T; ++t) {
    const int s = t % NS;
    const uint32_t parity = (t / NS) & 1;
    const int valid = a.L - t * BKV;   // >= 1; >= 128 means no masking
    // ---- S = Q K^T: 4 K32 steps over head_dim (one 128-byte swizzled row per query / key)
    float sc[64];
    mbar_wait(&bars[K_FULL + s], parity);
    {
      const uint32_t k_smem = smem_u32(smem + SmemLayout::k) + s * TILE_BYTES;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        wgmma_ss_e4m3<128>(sc, wgmma_desc_kmajor_sw128(q_smem + kk * 32), wgmma_desc_kmajor_sw128(k_smem + kk * 32), kk != 0);
      wgmma_commit();
      wgmma_wait<0>();
      // sc[4c + e + 2hh] is row r0 + 8hh, key 8c + 2quad + e: times the key's scale
      const float* kss = kscale + s * BKV;
#pragma unroll
      for (int c = 0; c < 16; ++c) {
        const float2 ks = *reinterpret_cast<const float2*>(kss + 8 * c + 2 * quad);
        sc[4 * c] *= ks.x;
        sc[4 * c + 2] *= ks.x;
        sc[4 * c + 1] *= ks.y;
        sc[4 * c + 3] *= ks.y;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars[K_EMPTY + s]);
    }
    // ---- online softmax
    if (valid < BKV) {  // last key tile only (warp-uniform): masked scores -> -inf -> p = 0
#pragma unroll
      for (int i = 0; i < 64; ++i)
        if (8 * (i >> 2) + 2 * quad + (i & 1) >= valid) sc[i] = -INFINITY;
    }
    // P^ as the 8-bit A fragment: pk[2j + hh] = e4m3 of keys 8c + 2quad + {0, 1} for c = 2j, 2j + 1 (4 bytes) of row r0 + 8hh
    uint32_t pk[16];
    float alpha[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float mx = -INFINITY;
#pragma unroll
      for (int c = 0; c < 16; ++c) mx = fmaxf(mx, fmaxf(sc[4 * c + 2 * hh], sc[4 * c + 2 * hh + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m[hh], mx * rf[hh]);   // finite: every tile has at least one valid key
      alpha[hh] = fast_exp2(m[hh] - m_new);             // 0 on the first tile (m = -inf)
      m[hh] = m_new;
      const float mb = 8.f - m_new;                     // 256 exp2(x - m) = exp2(x - m + 8)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = 2 * j;
        // keys 8c + 2quad + e with c % 4 == 3 (a quarter) take exp2 on the FMA pipe, the rest on MUFU
        const uint32_t lo = exp2_e4m3x2<false>(fmaf(sc[4 * c + 2 * hh], rf[hh], mb), fmaf(sc[4 * c + 2 * hh + 1], rf[hh], mb));
        const float b0 = fmaf(sc[4 * c + 4 + 2 * hh], rf[hh], mb), b1 = fmaf(sc[4 * c + 4 + 2 * hh + 1], rf[hh], mb);
        const uint32_t hi = (j & 1) ? exp2_e4m3x2<true>(b0, b1) : exp2_e4m3x2<false>(b0, b1);
        pk[2 * j + hh] = lo | (hi << 16);
      }
    }
    // ---- O_j = P^ V^ and the row sums P^ 1: 4 K32 steps over the keys into fresh accumulators; fragment of step kk =
    // {pk[4kk .. 4kk + 3]}.  lt[2hh] (= lt[2hh + 1], every column of the ones tile) is the row sum of row r0 + 8hh.
    float ot[64], lt[4];
    mbar_wait(&bars[V_FULL + s], parity);
    {
      const uint32_t v_smem = smem_u32(smem + SmemLayout::v) + s * TILE_BYTES;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint32_t frag[4] = {pk[4 * kk], pk[4 * kk + 1], pk[4 * kk + 2], pk[4 * kk + 3]};
        const uint32_t ones = smem_u32(smem + SmemLayout::ones) + kk * 32;
        if (kk == 0) {
          wgmma_rs_e4m3_overwrite<128>(ot, frag, wgmma_desc_kmajor_sw128(v_smem));
          wgmma_rs_e4m3_overwrite<8>(lt, frag, wgmma_desc_kmajor_sw128(ones));
        } else {
          wgmma_rs_e4m3<128>(ot, frag, wgmma_desc_kmajor_sw128(v_smem + kk * 32), 1);
          wgmma_rs_e4m3<8>(lt, frag, wgmma_desc_kmajor_sw128(ones), 1);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      if (signaller) mbar_arrive(&bars[V_EMPTY + s]);
    }
    l[0] = fmaf(l[0], alpha[0], lt[0]);
    l[1] = fmaf(l[1], alpha[1], lt[2]);
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      o[4 * c] = fmaf(o[4 * c], alpha[0], ot[4 * c]);
      o[4 * c + 1] = fmaf(o[4 * c + 1], alpha[0], ot[4 * c + 1]);
      o[4 * c + 2] = fmaf(o[4 * c + 2], alpha[1], ot[4 * c + 2]);
      o[4 * c + 3] = fmaf(o[4 * c + 3], alpha[1], ot[4 * c + 3]);
    }
  }

  // ---- out = bf16(o s_v / l)
  const float* vs = a.v_scale + (size_t)b * a.H * HD + h * HD + 2 * quad;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const float inv = 1.0f / l[hh];
    const int row = q0 + r0 + 8 * hh;
    if (row >= a.L) continue;
    bf16* orow = a.out + ((size_t)b * a.L + row) * a.ldo + h * HD;
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      const float2 sv = *reinterpret_cast<const float2*>(vs + 8 * c);
      *reinterpret_cast<uint32_t*>(orow + 8 * c + 2 * quad) =
          pack_bf16x2(o[4 * c + 2 * hh] * sv.x * inv, o[4 * c + 2 * hh + 1] * sv.y * inv);
    }
  }
}

}  // namespace

int launch_attention_fp8(const AttnFp8Args& a, cudaStream_t stream) {
  CE_REQUIRE(a.B > 0 && a.H > 0 && a.L > 0, "attention_fp8: empty problem");
  CE_REQUIRE(a.q && a.k && a.q_scale && a.k_scale && a.vt && a.v_scale && a.out, "attention_fp8: null pointer");
  CE_REQUIRE(a.ldqk % 16 == 0 && a.ldqk >= a.H * HD && a.lds >= a.H && a.ldo % 8 == 0 && a.ldo >= a.H * HD,
             "attention_fp8: ldqk % 16 and >= H * 128, lds >= H, ldo % 8 and >= H * 128");
  CE_REQUIRE(a.Lpad >= a.L && a.Lpad % 32 == 0, "attention_fp8: Lpad >= L, a multiple of 32");
  CUtensorMap tq, tk, tv;
  const uint32_t box[3] = {128, 128, 1};
  const uint64_t dqk[3] = {(uint64_t)a.H * HD, (uint64_t)a.L, (uint64_t)a.B};
  const uint64_t sqk[2] = {(uint64_t)a.ldqk, (uint64_t)a.L * a.ldqk};
  CE_TRY(make_tmap_u8(&tq, a.q, 3, dqk, sqk, box));
  CE_TRY(make_tmap_u8(&tk, a.k, 3, dqk, sqk, box));
  const uint64_t dv[3] = {(uint64_t)a.Lpad, (uint64_t)a.H * HD, (uint64_t)a.B};
  const uint64_t sv[2] = {(uint64_t)a.Lpad, (uint64_t)a.H * HD * a.Lpad};
  CE_TRY(make_tmap_u8(&tv, a.vt, 3, dv, sv, box));
  CE_ENSURE_SMEM(attention_fp8_kernel, SmemLayout::total);
  dim3 grid((a.L + BQ - 1) / BQ, a.H, a.B);
  attention_fp8_kernel<<<grid, ATTN_THREADS, SmemLayout::total, stream>>>(tq, tk, tv, a);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

}  // namespace ce
