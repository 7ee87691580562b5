// Non-causal multi-head attention forward for sm_90a (head_dim 128), flash-style, on wgmma, with bf16 or e4m3 operands.
//
//   bf16:  out[b, i, h*128:(h+1)*128] = softmax_j( q[b,i,h,:] . k[b,j,h,:] * scale ) @ v[b,j,h,:]
//   FP8 (DESIGN.md, "FP8 attention"):
//          S = (q^ k^T) s_q[i] s_k[j],   P^ = e4m3(256 exp2(S scale log2e - m)),   out = bf16((sum_j P^ V^) s_v[c] / sum_j P^)
//
// One CTA per (128-query tile, head, batch); 384 threads = 3 warpgroups (registers re-partitioned with setmaxnreg):
//   warpgroup 0     warp 0 (one lane): TMA of the Q tile once, then K_j / V_j tiles (128 keys) through NS-deep rings;
//                   FP8 only, warp 1: the 128 key scales of tile j into shared memory (a strided gather TMA cannot do)
//   warpgroups 1,2  one 64-query half of the tile each, everything in registers:
//                   S_j = Q K_j^T (wgmma, both operands from shared memory), online softmax (fp32: running max, exp2, row sum),
//                   O += P_j V_j (wgmma, P_j straight from the S accumulator registers as the A operand)
// A tile row is 128 bytes (one swizzled box) in e4m3 and two in bf16; the rings hold 64 KB each, 2 bf16 or 4 e4m3 tiles deep.
//
// Two schedules of the consumer loop (attention_tiles<T, PIPE>), with bit-identical results:
//   serial     (FP8, and bf16 as a reference: ce_debug_attention_kernel(1))  per key tile S_j, wait; softmax_j; P_j V_j, wait.
//              Registers 40 / 232 per thread (producer / consumers).
//   pipelined  (bf16, the default)  per key tile j >= 1: issue S_j, then P_{j-1} V_{j-1} (two commit groups, in that order),
//              wait_group 1 for S_j, softmax_j while P_{j-1} V_{j-1} runs, wait_group 0, o *= alpha_j; a prologue (S_0 and
//              its softmax) and a drain (the last P V) per key/value source.  o still sees ..., * alpha_j, + P_j V_j, and l and
//              every P are computed as in the serial loop.  P alternates between two register fragments.  The two warpgroups
//              take turns at issuing (named barriers 1 and 2), so that one's MMAs run while the other is in its softmax.
//              Registers 24 / 240 (o, S_j and two P fragments: 160 of them).
//
// Where the two operand types differ:
//   bf16  V_j is [keys, channels] (MN-major B).  o is rescaled by alpha before P V and accumulates in place; the row sum is
//         each lane's share of the fp32 P, reduced by shuffles at the end.  A second key/value source (text + image
//         cross-attention) is walked after the first, and its separately normalised, bf16-rounded result added to the first
//         one's.  Sequence-parallel output scatter, timing hooks (ce_debug_attention_timing).
//   FP8   V^ is stored transposed, V^T [channels, keys] (launch_quantize_v_fp8), because FP8 wgmma takes B K-major only.  A
//         quarter of the exponentials run on the FMA pipe (exp2_fma) so that MUFU does not set the pace.  The row sum of the
//         quantized P^ comes from the tensor cores: the same A fragment times a tile of ones (m64n8k32), so the softmax does no
//         per-score work for it and the normalisation matches what was multiplied.  Each key tile's P^ V^ and row sum go into
//         fresh accumulators, added as o = o * alpha + o_tile in fp32, so no FP8 wgmma accumulates over more than 128 keys.
//
// Shared memory: Q | K[NS] | V[NS] | (FP8: ones 1 KB | key scales NS x 512 B) | barriers.
//
// Replaces F.scaled_dot_product_attention at chronoedit_diffusers/transformer_chronoedit.py:91-99 of the reference
// (self-attention, text cross-attention and image cross-attention; the latter two are summed, :103-104).
#include "attention.cuh"
#include "wgmma.cuh"

#include <cuda_fp8.h>

namespace ce {

namespace {

constexpr int HD = 128;
constexpr int BQ = 128;
constexpr int BKV = 128;
constexpr int ATTN_THREADS = 384;
constexpr uint32_t BOX_BYTES = 128 * 128;   // one TMA box: 128 rows x 128 bytes, the 128-byte swizzle's row

template <class T>
struct SmemLayout {
  static constexpr uint32_t TILE_BYTES = 128 * 128 * sizeof(T);   // a Q, K or V tile: 128 rows x 128 elements
  static constexpr int NS = 65536 / TILE_BYTES;                   // ring depth
  static constexpr uint32_t q = 0;
  static constexpr uint32_t k = q + TILE_BYTES;
  static constexpr uint32_t v = k + NS * TILE_BYTES;
  static constexpr uint32_t ones = v + NS * TILE_BYTES;   // FP8: [8 x 128] e4m3 ones, the B operand of the row sums
  static constexpr uint32_t ks = ones + 1024;            // FP8: NS x 128 key scales
  static constexpr uint32_t bars = sizeof(T) == 1 ? ks + NS * BKV * 4 : ones;
  static constexpr uint32_t total = bars + 256;
};

// mbar_wait with its timed loop out of line, for the pipelined consumers, which keep most of their setmaxnreg budget live
// across the wait: ptxas caps the registers of code that can reach an inlined trap well below that budget (the loop spilled
// 200 bytes and had its wgmmas serialised).  The call costs nothing on the fast path.  Not for waits between
// wgmma.mma_async and its wait_group: a call there serialises the wgmmas (C7510).
__device__ __noinline__ void mbar_wait_slow(uint64_t* bar, uint32_t parity) { mbar_wait(bar, parity); }
__device__ __forceinline__ void mbar_wait_outlined(uint64_t* bar, uint32_t parity) {
  if (!mbar_try_wait(bar, parity)) mbar_wait_slow(bar, parity);
}

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

// A [128 x 128] tile of T at element coordinates (x, y) of sample b, as sizeof(T) boxes side by side.
template <class T>
__device__ __forceinline__ void tma_load_tile(uint8_t* dst, const CUtensorMap* m, uint64_t* bar, int x, int y, int b) {
#pragma unroll
  for (int i = 0; i < (int)sizeof(T); ++i) tma_load_3d(dst + i * BOX_BYTES, m, bar, x + i * (128 / (int)sizeof(T)), y, b);
}

// The kernel body for operands of type T: bf16 (Args = AttnArgs) or e4m3 (Args = AttnFp8Args, one key/value source: k2 / v2
// are not read).  PIPE selects the consumers' schedule: false, one serial chain per key tile (S_j, softmax_j, P_j V_j); true
// (bf16 only), S_j and P_{j-1} V_{j-1} issued together and softmax_j run while P_{j-1} V_{j-1} executes.  Both apply the same
// operations in the same order to o, l and every P, so their outputs are bit-identical.
template <class T, bool PIPE, class Args>
__device__ __forceinline__ void attention_tiles(const CUtensorMap* tma_q, const CUtensorMap* tma_k, const CUtensorMap* tma_v,
                                                const CUtensorMap* tma_k2, const CUtensorMap* tma_v2, const Args& a) {
  constexpr bool FP8 = sizeof(T) == 1;
  static_assert(!(FP8 && PIPE), "the FP8 kernel keeps the serial schedule: its ot / lt accumulators leave no room for a second S");
  using Smem = SmemLayout<T>;
  constexpr uint32_t TILE_BYTES = Smem::TILE_BYTES;
  constexpr int NS = Smem::NS;
  constexpr int KSTEPS = 4 * sizeof(T);   // 32-byte wgmma K steps over the 128 channels (S) or keys (P V): K16 bf16, K32 e4m3
  enum { Q_FULL = 0, K_FULL = 1, K_EMPTY = K_FULL + NS, V_FULL = K_EMPTY + NS, V_EMPTY = V_FULL + NS };

  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Smem::bars);
  float* kscale = reinterpret_cast<float*>(smem + Smem::ks);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * BQ;
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  int Lq, Lk, Lk2 = 0;
  if constexpr (FP8) {
    Lq = Lk = a.L;
  } else {
    Lq = a.Lq;
    Lk = a.Lk;
    Lk2 = a.Lk2;
  }
  // key tiles of source 0 (k / v, Lk keys), then of source 1 (k2 / v2, Lk2 keys; none for a single source), through one ring
  const int T0 = (Lk + BKV - 1) / BKV;
  const int T1 = (Lk2 + BKV - 1) / BKV;

  if constexpr (FP8) {
    for (int i = threadIdx.x; i < 256; i += ATTN_THREADS) reinterpret_cast<uint32_t*>(smem + Smem::ones)[i] = 0x38383838u;  // 1.0
    fence_proxy_async_smem();   // read by wgmma (async proxy)
  }
  if (threadIdx.x == 0) {
    if ((smem_u32(smem) & 1023u) != 0) __trap();  // the swizzled tiles need 1024-byte alignment
    mbar_init(&bars[Q_FULL], 1);
    for (int i = 0; i < NS; ++i) {
      mbar_init(&bars[K_FULL + i], FP8 ? 1 + 32 : 1);   // the TMA's expect_tx (FP8: and every lane of the key-scale warp)
      mbar_init(&bars[K_EMPTY + i], FP8 ? 8 : 2);       // every consumer warp in FP8, one per consumer warpgroup in bf16
      mbar_init(&bars[V_FULL + i], 1);
      mbar_init(&bars[V_EMPTY + i], 2);                 // one per consumer warpgroup
    }
    fence_mbar_init();
    tma_prefetch_desc(tma_q);
    tma_prefetch_desc(tma_k);
    tma_prefetch_desc(tma_v);
    if (!FP8) {
      tma_prefetch_desc(tma_k2);
      tma_prefetch_desc(tma_v2);
    }
  }
  __syncthreads();

  if (warp < 4) {
    // ---------------------------------------------------------------- producers
    setmaxnreg_dec<PIPE ? 24 : 40>();
    if (warp == 0 && elect_one_sync()) {
      mbar_arrive_expect_tx(&bars[Q_FULL], TILE_BYTES);
      tma_load_tile<T>(smem + Smem::q, tma_q, &bars[Q_FULL], h * HD, q0, b);
      for (int t = 0; t < T0 + T1; ++t) {
        const int s = t % NS;
        const uint32_t free_parity = ((t / NS) & 1) ^ 1;
        const CUtensorMap* mk = t < T0 ? tma_k : tma_k2;
        const CUtensorMap* mv = t < T0 ? tma_v : tma_v2;
        const int key0 = (t < T0 ? t : t - T0) * BKV;
        mbar_wait(&bars[K_EMPTY + s], free_parity);
        mbar_arrive_expect_tx(&bars[K_FULL + s], TILE_BYTES);
        tma_load_tile<T>(smem + Smem::k + s * TILE_BYTES, mk, &bars[K_FULL + s], h * HD, key0, b);
        mbar_wait(&bars[V_EMPTY + s], free_parity);
        mbar_arrive_expect_tx(&bars[V_FULL + s], TILE_BYTES);
        // bf16 V is [keys, channels]; the FP8 V^T is [channels, keys]
        tma_load_tile<T>(smem + Smem::v + s * TILE_BYTES, mv, &bars[V_FULL + s], FP8 ? key0 : h * HD, FP8 ? h * HD : key0, b);
      }
    } else if (warp == 1) {
      if constexpr (FP8) {
        const float* ksrc = a.k_scale + (size_t)b * a.L * a.lds + h;
        for (int t = 0; t < T0; ++t) {
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
    }
    return;
  }

  // ------------------------------------------------------------------ consumers: 64 query rows per warpgroup
  setmaxnreg_inc<PIPE ? 240 : 232>();
  const int wg = (warp >> 2) - 1;
  const bool signaller = (threadIdx.x & 127) == 0;
  const int quad = lane & 3;
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // the thread's rows of the query tile: r0 and r0 + 8
  const uint32_t q_smem = smem_u32(smem + Smem::q) + wg * 64 * 128;
  const float sl2 = a.scale * 1.4426950408889634f;
  float rf[2] = {sl2, sl2};   // the score factor of the two rows: scale * log2(e), times s_q in FP8
  if constexpr (FP8) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int row = q0 + r0 + 8 * hh;
      rf[hh] = (row < a.L ? a.q_scale[((size_t)b * a.L + row) * a.lds + h] : 1.f) * sl2;   // rows >= L are zeros, not stored
    }
  }
  // ---- S = Q K^T of the key tile in stage s: KSTEPS 32-byte steps over head_dim (two 64-wide swizzled boxes in bf16, one in
  // e4m3).  Issued and committed as one group; the caller fences and waits.
  auto issue_s = [&](float (&sc)[64], int s) {
    const uint32_t k_smem = smem_u32(smem + Smem::k) + s * TILE_BYTES;
#pragma unroll
    for (int kk = 0; kk < KSTEPS; ++kk) {
      const uint32_t off = (kk >> 2) * BOX_BYTES + (kk & 3) * 32;
      const uint64_t da = wgmma_desc_kmajor_sw128(q_smem + off), db = wgmma_desc_kmajor_sw128(k_smem + off);
      if constexpr (FP8) wgmma_ss_e4m3<128>(sc, da, db, kk != 0);
      else wgmma_ss<128, 0>(sc, da, db, kk != 0);
    }
    wgmma_commit();
  };
  // ---- P V of the value tile in stage s: KSTEPS steps over the keys; the A fragment of step kk is p[4kk .. 4kk + 3].
  // bf16: acc = o, O += P V.  FP8: fresh accumulators acc = P^ V^ and lt = P^ 1 (lt[2hh] = lt[2hh + 1], every column of the
  // ones tile, is the row sum of row r0 + 8hh).  One committed group.
  auto issue_pv = [&](float (&acc)[64], float (&lt)[4], const uint32_t (&p)[4 * KSTEPS], int s) {
    const uint32_t v_smem = smem_u32(smem + Smem::v) + s * TILE_BYTES;
#pragma unroll
    for (int kk = 0; kk < KSTEPS; ++kk) {
      const uint32_t frag[4] = {p[4 * kk], p[4 * kk + 1], p[4 * kk + 2], p[4 * kk + 3]};
      if constexpr (FP8) {
        const uint32_t ones = smem_u32(smem + Smem::ones) + kk * 32;
        if (kk == 0) {
          wgmma_rs_e4m3_overwrite<128>(acc, frag, wgmma_desc_kmajor_sw128(v_smem));
          wgmma_rs_e4m3_overwrite<8>(lt, frag, wgmma_desc_kmajor_sw128(ones));
        } else {
          wgmma_rs_e4m3<128>(acc, frag, wgmma_desc_kmajor_sw128(v_smem + kk * 32), 1);
          wgmma_rs_e4m3<8>(lt, frag, wgmma_desc_kmajor_sw128(ones), 1);
        }
      } else {
        wgmma_rs<128, 1>(acc, frag, wgmma_desc_mnmajor_sw128(v_smem + kk * 2048, BOX_BYTES), 1);
      }
    }
    wgmma_commit();
  };
  auto release_k = [&](int s) {
    if constexpr (FP8) {   // per warp: each has read its key scales from the stage
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars[K_EMPTY + s]);
    } else if (signaller) {
      mbar_arrive(&bars[K_EMPTY + s]);
    }
  };
  auto release_v = [&](int s) {
    if (signaller) mbar_arrive(&bars[V_EMPTY + s]);
  };
  // ---- online softmax on the accumulator registers of tile j (`valid` = keys left in the source, >= 1; >= 128: no masking):
  // sc[4 * c + e + 2 * hh] is row r0 + 8 * hh, key 8 * c + 2 * quad + e.  Updates m (and l in bf16) and gives alpha, the
  // factor of everything accumulated before this tile, and P as the A fragment of P V, for row r0 + 8hh:
  //   bf16  p[2c + hh] = keys 8c + 2quad + {0, 1} (two bf16)
  //   e4m3  p[2j + hh] = keys 8c + 2quad + {0, 1} for c = 2j, 2j + 1 (four e4m3)
  auto softmax = [&](float (&sc)[64], int valid, float (&m)[2], float (&l)[2], uint32_t (&p)[4 * KSTEPS], float (&alpha)[2]) {
    if (valid < BKV) {  // last key tile only (warp-uniform): masked scores -> -inf -> p = 0
#pragma unroll
      for (int i = 0; i < 64; ++i)
        if (8 * (i >> 2) + 2 * quad + (i & 1) >= valid) sc[i] = -INFINITY;
    }
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
      if constexpr (FP8) {
        const float mb = 8.f - m_new;   // 256 exp2(x - m) = exp2(x - m + 8)
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int c = 2 * jj;
          // keys 8c + 2quad + e with c % 4 == 3 (a quarter) take exp2 on the FMA pipe, the rest on MUFU
          const uint32_t lo = exp2_e4m3x2<false>(fmaf(sc[4 * c + 2 * hh], rf[hh], mb), fmaf(sc[4 * c + 2 * hh + 1], rf[hh], mb));
          const float b0 = fmaf(sc[4 * c + 4 + 2 * hh], rf[hh], mb), b1 = fmaf(sc[4 * c + 4 + 2 * hh + 1], rf[hh], mb);
          const uint32_t hi = (jj & 1) ? exp2_e4m3x2<true>(b0, b1) : exp2_e4m3x2<false>(b0, b1);
          p[2 * jj + hh] = lo | (hi << 16);
        }
      } else {
        float sum = 0.f;
#pragma unroll
        for (int c = 0; c < 16; ++c) {
          const float p0 = fast_exp2(fmaf(sc[4 * c + 2 * hh], rf[hh], -m_new));
          const float p1 = fast_exp2(fmaf(sc[4 * c + 2 * hh + 1], rf[hh], -m_new));
          sum += p0 + p1;
          p[2 * c + hh] = pack_bf16x2(p0, p1);
        }
        l[hh] = l[hh] * alpha[hh] + sum;
      }
    }
  };
  auto rescale = [&](float (&o)[64], const float (&alpha)[2]) {   // bf16: o *= alpha, before P_j V_j is added
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      o[4 * c] *= alpha[0];
      o[4 * c + 1] *= alpha[0];
      o[4 * c + 2] *= alpha[1];
      o[4 * c + 3] *= alpha[1];
    }
  };

  long long* timing = nullptr;   // phase hooks of the bf16 kernel (ce_debug_attention_timing); compiled out of FP8
  if constexpr (!FP8) timing = a.timing;
  const bool timed = timing != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && threadIdx.x == 128;
  // cycles of the three phases; serial schedule: S = Q K^T (incl. the wait for K), softmax, P V (incl. the wait for V);
  // pipelined: up to S_j's result (waits for K_j / V_{j-1} and the turn, issue of S_j and P_{j-1} V_{j-1}, wait for S_j),
  // softmax_j, wait for P_{j-1} V_{j-1} plus the rescale
  long long tacc[3] = {0, 0, 0};
  long long tc0 = timed ? clock64() : 0;
#define CE_TICK(slot)               \
  if (timed) {                      \
    const long long _t = clock64(); \
    tacc[slot] += _t - tc0;         \
    tc0 = _t;                       \
  }

  // Ping-pong (pipelined schedule): the two consumer warpgroups take turns at issuing their MMAs, so that the tensor cores run
  // one warpgroup's S and P V while the other one is in its softmax.  Named barrier 1 + w is warpgroup w's turn: it syncs there
  // before each issue point and hands the turn over (arrive at the other's barrier) after it.  Warpgroup 1 gives warpgroup 0
  // the first turn and does not hand over after its last issue point, so every barrier sees as many arrivals as syncs: both
  // walk T0 + T1 tiles and one drain per source, whatever Lq, Lk and Lk2 are.
  const int n_src = T1 > 0 ? 2 : 1;
  auto await_turn = [&]() {
    if constexpr (PIPE) named_bar_sync(1 + wg, 256);
  };
  auto pass_turn = [&](bool last) {
    if constexpr (PIPE) {
      if (!(last && wg == 1)) named_bar_arrive(2 - wg, 256);
    }
  };
  if constexpr (PIPE) {
    if (wg == 1) named_bar_arrive(1, 256);
  }

  // The pipelined loop holds o, S_j and two P fragments across its waits: their timed slow path goes out of line
  // (mbar_wait_outlined).
  auto wait_full = [&](int bar, uint32_t parity) {
    if constexpr (PIPE) mbar_wait_outlined(&bars[bar], parity);
    else mbar_wait(&bars[bar], parity);
  };
  wait_full(Q_FULL, 0);
  uint32_t t = 0;   // position in the ring, over both sources
  for (int src = 0; src < n_src; ++src) {
    const int my_tiles = src ? T1 : T0;
    const int my_len = src ? Lk2 : Lk;
    float o[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] = 0.f;
    // per row: running max, row sum (bf16: this lane's share of it; FP8: the whole row's, from the tensor cores)
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};

    if constexpr (PIPE) {
      // ---- pipelined: prologue S_0 -> softmax_0; per tile j >= 1: issue S_j and P_{j-1} V_{j-1}, softmax_j while
      // P_{j-1} V_{j-1} runs, then o *= alpha_j; drain P_{last} V_{last}.  o sees ..., * alpha_j, + P_j V_j as in the serial
      // schedule.  P alternates between two fragments, so that softmax_j never writes the registers P V reads in flight.
      float sc[64], alpha[2], lt_unused[4];
      uint32_t pa[4 * KSTEPS], pb[4 * KSTEPS];
      int s = t % NS;
      wait_full(K_FULL + s, (t / NS) & 1);
      await_turn();
      wgmma_fence();
      issue_s(sc, s);
      pass_turn(false);
      wgmma_wait<0>();
      wgmma_fence_operand(sc);
      release_k(s);
      CE_TICK(0)
      softmax(sc, my_len, m, l, pa, alpha);
      rescale(o, alpha);
      CE_TICK(1)
      // tile j: P_{j-1} V_{j-1} from pv, softmax_j into pn
      auto step = [&](uint32_t (&pv)[4 * KSTEPS], uint32_t (&pn)[4 * KSTEPS], int j) {
        const int sn = (t + 1) % NS;
        wait_full(K_FULL + sn, ((t + 1) / NS) & 1);
        wait_full(V_FULL + s, (t / NS) & 1);
        await_turn();
        wgmma_fence_operand(o);   // o *= alpha and P_{j-1} complete before the issue, not sunk between the wgmmas
        wgmma_fence_operand(pv);
        wgmma_fence();
        issue_s(sc, sn);   // committed first: wait_group 1 below retires it and leaves P V in flight
        issue_pv(o, lt_unused, pv, s);
        pass_turn(false);
        wgmma_wait<1>();
        wgmma_fence_operand(sc);
        release_k(sn);
        CE_TICK(0)
        softmax(sc, my_len - j * BKV, m, l, pn, alpha);
        CE_TICK(1)
        wgmma_wait<0>();
        wgmma_fence_operand(o);   // pv stays allocated up to here; rescale after the P V is done
        wgmma_fence_operand(pv);
        release_v(s);
        rescale(o, alpha);
        CE_TICK(2)
        ++t;
        s = sn;
      };
      auto drain = [&](uint32_t (&pv)[4 * KSTEPS]) {
        wait_full(V_FULL + s, (t / NS) & 1);
        await_turn();
        wgmma_fence_operand(o);
        wgmma_fence_operand(pv);
        wgmma_fence();
        issue_pv(o, lt_unused, pv, s);
        pass_turn(src == n_src - 1);
        wgmma_wait<0>();
        wgmma_fence_operand(o);
        wgmma_fence_operand(pv);
        release_v(s);
        CE_TICK(2)
        ++t;
      };
      int j = 1;
      for (; j + 1 < my_tiles; j += 2) {
        step(pa, pb, j);
        step(pb, pa, j + 1);
      }
      if (j < my_tiles) {
        step(pa, pb, j);
        drain(pb);
      } else {
        drain(pa);
      }
    } else {
      for (int j = 0; j < my_tiles; ++j, ++t) {
        const int s = t % NS;
        const uint32_t parity = (t / NS) & 1;
        const int valid = my_len - j * BKV;  // >= 1; >= 128 means no masking
        float sc[64];
        mbar_wait(&bars[K_FULL + s], parity);
        wgmma_fence();
        issue_s(sc, s);
        wgmma_wait<0>();
        if constexpr (FP8) {   // sc[4c + e + 2hh] is row r0 + 8hh, key 8c + 2quad + e: times the key's scale
          const float* kss = kscale + s * BKV;
#pragma unroll
          for (int c = 0; c < 16; ++c) {
            const float2 ks = *reinterpret_cast<const float2*>(kss + 8 * c + 2 * quad);
            sc[4 * c] *= ks.x;
            sc[4 * c + 2] *= ks.x;
            sc[4 * c + 1] *= ks.y;
            sc[4 * c + 3] *= ks.y;
          }
        }
        release_k(s);
        CE_TICK(0)
        uint32_t p[4 * KSTEPS];
        float alpha[2];
        softmax(sc, valid, m, l, p, alpha);
        if constexpr (!FP8) rescale(o, alpha);
        CE_TICK(1)
        float ot[64], lt[4];
        mbar_wait(&bars[V_FULL + s], parity);
        wgmma_fence();
        issue_pv(FP8 ? ot : o, lt, p, s);
        wgmma_wait<0>();
        release_v(s);
        if constexpr (FP8) {
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
        CE_TICK(2)
      }
    }

    // ---- normalise and store this source's result: bf16(o / l), FP8 bf16(o s_v / l)
    const float* vs = nullptr;   // FP8: s_v of channels 2quad + {0, 1} (+ 8c) of this head
    if constexpr (FP8) vs = a.v_scale + (size_t)b * a.H * HD + h * HD + 2 * quad;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float lr = l[hh];
      if constexpr (!FP8) {
        lr += __shfl_xor_sync(0xffffffffu, lr, 1);
        lr += __shfl_xor_sync(0xffffffffu, lr, 2);
      }
      const float inv = 1.0f / lr;
      const int row = q0 + r0 + 8 * hh;
      if (row >= Lq) continue;
      bf16* orow = a.out + ((size_t)b * Lq + row) * a.ldo + h * HD;
      if constexpr (!FP8) {
        if (a.peer_rows > 0)   // sequence parallel: the token's owner gets the row (peer store over NVLink)
          orow = a.out_peer[row / a.peer_rows] + ((size_t)b * a.peer_rows + row % a.peer_rows) * a.ldo + a.out_col0 + h * HD;
      }
#pragma unroll
      for (int c = 0; c < 16; ++c) {
        uint32_t* dst = reinterpret_cast<uint32_t*>(orow + 8 * c + 2 * quad);
        if constexpr (FP8) {
          const float2 sv = *reinterpret_cast<const float2*>(vs + 8 * c);
          *dst = pack_bf16x2(o[4 * c + 2 * hh] * sv.x * inv, o[4 * c + 2 * hh + 1] * sv.y * inv);
        } else {
          float y0 = o[4 * c + 2 * hh] * inv, y1 = o[4 * c + 2 * hh + 1] * inv;
          if (a.accumulate || src == 1) {   // each SDPA result is a bf16 tensor in the reference before the add
            const float2 prev = unpack_bf16x2(*dst);
            y0 = bf16_round(y0) + prev.x;
            y1 = bf16_round(y1) + prev.y;
          }
          *dst = pack_bf16x2(y0, y1);
        }
      }
    }
  }
  if (timed) {
    for (int i = 0; i < 3; ++i) timing[i] = tacc[i];
    timing[3] = T0 + T1;
  }
#undef CE_TICK
}

// PIPE: the pipelined schedule (the default); !PIPE: the serial one, kept as the reference the pipelined one is tested against
// (ce_debug_attention_kernel(1)).
template <bool PIPE>
__global__ void __launch_bounds__(ATTN_THREADS, 1)
attention_fwd_kernel(const __grid_constant__ CUtensorMap tma_q, const __grid_constant__ CUtensorMap tma_k,
                     const __grid_constant__ CUtensorMap tma_v, const __grid_constant__ CUtensorMap tma_k2,
                     const __grid_constant__ CUtensorMap tma_v2, AttnArgs a) {
  attention_tiles<bf16, PIPE>(&tma_q, &tma_k, &tma_v, &tma_k2, &tma_v2, a);
}

__global__ void __launch_bounds__(ATTN_THREADS, 1)
attention_fp8_kernel(const __grid_constant__ CUtensorMap tma_q, const __grid_constant__ CUtensorMap tma_k,
                     const __grid_constant__ CUtensorMap tma_vt, AttnFp8Args a) {
  attention_tiles<__nv_fp8_e4m3, false>(&tma_q, &tma_k, &tma_vt, &tma_k, &tma_vt, a);
}

// A token-major [B, L, H * 128] operand with row stride ld (elements), in 128-byte boxes of 128 rows (64 bf16 or 128 e4m3 wide).
template <class T>
int make_qkv_tmap(CUtensorMap* m, const T* base, int B, int L, int H, int ld) {
  const uint64_t dims[3] = {(uint64_t)H * HD, (uint64_t)L, (uint64_t)B};
  const uint64_t strides[2] = {(uint64_t)ld * sizeof(T), (uint64_t)L * ld * sizeof(T)};
  const uint32_t box[3] = {128 / sizeof(T), 128, 1};
  return sizeof(T) == 1 ? make_tmap_u8(m, base, 3, dims, strides, box) : make_tmap_bf16(m, base, 3, dims, strides, box);
}

// One CTA per (128-query tile, head, batch).
template <class T, class... Params>
int launch_tiles(void (*kernel)(Params...), int B, int H, int Lq, cudaStream_t stream, Params... params) {
  CE_ENSURE_SMEM(kernel, SmemLayout<T>::total);
  const dim3 grid((Lq + BQ - 1) / BQ, H, B);
  kernel<<<grid, ATTN_THREADS, SmemLayout<T>::total, stream>>>(params...);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

}  // namespace

int launch_attention(const AttnArgs& a, cudaStream_t stream, bool pipelined) {
  CE_REQUIRE(a.B > 0 && a.H > 0 && a.Lq > 0 && a.Lk > 0, "attention: empty problem");
  CE_REQUIRE(a.peer_rows == 0 || (a.Lk2 == 0 && !a.accumulate && (a.Lq + a.peer_rows - 1) / a.peer_rows <= 8),
             "attention: the sequence-parallel output scatter serves the self-attention, with at most 8 peers");
  CE_REQUIRE(a.head_dim == HD, "attention: only head_dim 128 is built");
  CE_REQUIRE(a.ldq % 8 == 0 && a.ldk % 8 == 0 && a.ldv % 8 == 0 && a.ldo % 8 == 0, "attention: leading dims % 8");
  CE_REQUIRE(a.q && a.k && a.v && a.out, "attention: null pointer");
  CUtensorMap tq, tk, tv, tk2, tv2;
  CE_TRY(make_qkv_tmap(&tq, a.q, a.B, a.Lq, a.H, a.ldq));
  CE_TRY(make_qkv_tmap(&tk, a.k, a.B, a.Lk, a.H, a.ldk));
  CE_TRY(make_qkv_tmap(&tv, a.v, a.B, a.Lk, a.H, a.ldv));
  if (a.Lk2 > 0) {
    CE_REQUIRE(a.k2 && a.v2 && a.ldk2 % 8 == 0 && a.ldv2 % 8 == 0, "attention: dual source needs k2 / v2");
    CE_TRY(make_qkv_tmap(&tk2, a.k2, a.B, a.Lk2, a.H, a.ldk2));
    CE_TRY(make_qkv_tmap(&tv2, a.v2, a.B, a.Lk2, a.H, a.ldv2));
  } else {
    tk2 = tk;
    tv2 = tv;
  }
  if (pipelined) return launch_tiles<bf16>(attention_fwd_kernel<true>, a.B, a.H, a.Lq, stream, tq, tk, tv, tk2, tv2, a);
  return launch_tiles<bf16>(attention_fwd_kernel<false>, a.B, a.H, a.Lq, stream, tq, tk, tv, tk2, tv2, a);
}

int launch_attention_fp8(const AttnFp8Args& a, cudaStream_t stream) {
  CE_REQUIRE(a.B > 0 && a.H > 0 && a.L > 0, "attention_fp8: empty problem");
  CE_REQUIRE(a.q && a.k && a.q_scale && a.k_scale && a.vt && a.v_scale && a.out, "attention_fp8: null pointer");
  CE_REQUIRE(a.ldqk % 16 == 0 && a.ldqk >= a.H * HD && a.lds >= a.H && a.ldo % 8 == 0 && a.ldo >= a.H * HD,
             "attention_fp8: ldqk % 16 and >= H * 128, lds >= H, ldo % 8 and >= H * 128");
  CE_REQUIRE(a.Lpad >= a.L && a.Lpad % 32 == 0, "attention_fp8: Lpad >= L, a multiple of 32");
  CUtensorMap tq, tk, tv;
  CE_TRY(make_qkv_tmap(&tq, a.q, a.B, a.L, a.H, a.ldqk));
  CE_TRY(make_qkv_tmap(&tk, a.k, a.B, a.L, a.H, a.ldqk));
  // V^T [B, H * 128, Lpad]: channel rows, keys contiguous
  const uint64_t dv[3] = {(uint64_t)a.Lpad, (uint64_t)a.H * HD, (uint64_t)a.B};
  const uint64_t sv[2] = {(uint64_t)a.Lpad, (uint64_t)a.H * HD * a.Lpad};
  const uint32_t box[3] = {128, 128, 1};
  CE_TRY(make_tmap_u8(&tv, a.vt, 3, dv, sv, box));
  return launch_tiles<__nv_fp8_e4m3>(attention_fp8_kernel, a.B, a.H, a.L, stream, tq, tk, tv, a);
}

}  // namespace ce
