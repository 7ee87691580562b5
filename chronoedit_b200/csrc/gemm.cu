// bf16 GEMM for sm_90a on the TMA -> shared-memory ring -> wgmma pipeline of ring_gemm.cuh, with a fused epilogue.
//
//   out[M,N] = epilogue( A[M,K] * W[N,K]^T )        A: activations (row-major), W: nn.Linear weight (row-major)
//
// Per k-block an A tile 128x64 and a W tile BNx64; the epilogue applies bias / activation / gate / residual / row statistics,
// split between the consumer warpgroups (up to the bf16 rounding) and warps 1-3 of the producer warpgroup (the rest, from a
// shared-memory staging tile), so that the tensor cores start the next tile while the last one is stored.
// The FP8 instantiation (gemm_fp8_kernel) reads e4m3 operands in k-blocks of 128 and multiplies the accumulator by a row scale
// and a column scale before the same epilogue: out[M,N] = epilogue( (Aq * Wq^T) * s_a[M] * s_w[N] ).
// Tile order is grouped along M so that concurrently resident tiles share W column panels through L2.
//
// Replaces the cuBLASLt calls behind every nn.Linear of the reference DiT block
// (chronoedit_diffusers/transformer_chronoedit.py:58-60, 84-87, 106, 292) plus the elementwise
// launches that follow them (:281, :286, :293).
#include "gemm.cuh"
#include "ring_gemm.cuh"

namespace ce {

namespace {

__device__ __forceinline__ void tile_coords(int t, int tiles_m, int tiles_n, int group_m, int& mb, int& nb) {
  const int per_group = group_m * tiles_n;
  const int g = t / per_group;
  const int first_m = g * group_m;
  const int gsize = min(tiles_m - first_m, group_m);
  const int r = t - g * per_group;
  mb = first_m + r % gsize;
  nb = r / gsize;
}

__device__ __forceinline__ float gelu_tanh_f(float x) {
  const float kBeta = 0.7978845608028654f;  // sqrt(2/pi)
  const float kKappa = 0.044715f;
  float inner = kBeta * (x + kKappa * x * x * x);
  return 0.5f * x * (1.0f + tanhf(inner));
}
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.7071067811865476f)); }

constexpr uint16_t NEG_ZERO = 0x8000u;          // bf16 -0.0

// Shared memory after the ring (Ring::tail()): the bf16 tile the consumers hand to the epilogue warps, then the tile's column
// and row operands (bias, bias_row and the FP8 scales, -0.0 / 0 outside [M, N)), which the epilogue warps load one tile ahead so
// that the consumers' part of the epilogue reads no global memory.  Two barriers order the hand-over:
//   staged   the consumers have written the tile (and are done with its operands): one arrive per consumer thread
//   drained  the epilogue warps have read the tile and loaded the next tile's operands: one arrive per epilogue thread
template <int BN>
struct Staging {
  static constexpr int CPR = BN / 8;   // 16-byte chunks (8 columns) per row; the swizzle below needs CPR >= 8
  static constexpr size_t BYTES = (size_t)BM * BN * 2 + BN * (2 + 4) + BM * (2 + 4);
  static constexpr int EPI_THREADS = 96, CONSUMER_THREADS = 256;
  uint8_t* tile;
  uint16_t* bias;   // [BN] bf16 bits
  float* s_w;       // [BN]
  uint16_t* bias_row;   // [BM] bf16 bits
  float* s_a;       // [BM]
  uint64_t *staged, *drained;

  template <int STAGES>
  __device__ __forceinline__ explicit Staging(const Ring<BN, STAGES>& ring) {
    tile = ring.tail();
    bias = reinterpret_cast<uint16_t*>(tile + BM * BN * 2);
    s_w = reinterpret_cast<float*>(bias + BN);
    bias_row = reinterpret_cast<uint16_t*>(s_w + BN);
    s_a = reinterpret_cast<float*>(bias_row + BM);
    staged = ring.empty + STAGES;
    drained = staged + 1;
  }
  // Byte offset of row r, chunk c.  Chunks are XOR-swizzled with r & 7 (rows are BN * 2 bytes, a multiple of 128), so both
  // access patterns are free of bank conflicts: the consumers' 4-byte writes (8 rows x 4 lanes per chunk, fragment order) and
  // the epilogue warps' 16-byte row-wise reads (8 consecutive chunks of one row per quarter warp).
  static __device__ __forceinline__ uint32_t off(int r, int c) { return r * (BN * 2) + ((c ^ (r & 7)) << 4); }
};

// Epilogue warps: the operands of tile t into shared memory.
template <int BN, bool FP8>
__device__ __forceinline__ void stage_operands(const Staging<BN>& st, const GemmArgs& g, const float* s_a, const float* s_w, int t,
                                               int tiles_m, int tiles_n) {
  int mb, nb;
  tile_coords(t, tiles_m, tiles_n, g.group_m, mb, nb);
  const int i = threadIdx.x - 32;
  for (int c = i; c < BN; c += Staging<BN>::EPI_THREADS) {
    const int n = nb * BN + c;
    st.bias[c] = g.bias && n < g.N ? __bfloat16_as_ushort(g.bias[n]) : NEG_ZERO;
    if (FP8) st.s_w[c] = n < g.N ? s_w[n] : 0.f;
  }
  for (int r = i; r < BM; r += Staging<BN>::EPI_THREADS) {
    const int m = mb * BM + r;
    st.bias_row[r] = g.bias_row && m < g.M ? __bfloat16_as_ushort(g.bias_row[m]) : NEG_ZERO;
    if (FP8) st.s_a[r] = m < g.M ? s_a[m] : 0.f;
  }
}

// Epilogue warps: GELU, residual / gate, stores and row statistics of one staged tile.  Warp w (1-3) takes the 8-row groups
// w - 1, w + 2, ...; per group, first the stores (each lane a 16-byte chunk, the residual loads of U chunks issued ahead of
// their stores, since out and resid may alias), the stored values written back to the staging tile, then the
// statistics with the consumers' lane layout (4 lanes per row, lane q summing columns 8j + 2q, 8j + 2q + 1 for ascending j, then
// the xor-1 and xor-2 shuffles), so they are the same bits as when the consumers computed them from their registers.
template <int BN>
__device__ __forceinline__ void drain_tile(const Staging<BN>& st, const GemmArgs& g, int mb, int nb) {
  constexpr int CPR = Staging<BN>::CPR;
  constexpr int ITERS = BN / 32;              // chunks per lane per group
  constexpr int U = ITERS < 4 ? ITERS : 4;    // residual loads in flight per lane (8 spill under the epilogue warps' 88 registers)
  const int lane = threadIdx.x & 31;
  const bool resid_epi = g.epi == EPI_BIAS_GATE_RESID || g.epi == EPI_BIAS_RESID;
  const bool gate_epi = g.epi == EPI_BIAS_GATE_RESID;
  const bool gelu = g.epi == EPI_BIAS_GELU_TANH || g.epi == EPI_BIAS_GELU_ERF;
  for (int grp = (threadIdx.x >> 5) - 1; grp < BM / 8; grp += 3) {
#pragma unroll 1
    for (int i0 = 0; i0 < ITERS; i0 += U) {
      uint4 rw[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int idx = lane + 32 * (i0 + u), m = mb * BM + grp * 8 + idx / CPR, n = nb * BN + (idx % CPR) * 8;
        rw[u] = resid_epi && m < g.M && n < g.N ? *reinterpret_cast<const uint4*>(g.resid + (size_t)m * g.ldr + n) : make_uint4(0, 0, 0, 0);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int idx = lane + 32 * (i0 + u), r = grp * 8 + idx / CPR, c = idx % CPR, m = mb * BM + r, n = nb * BN + c * 8;
        if (m >= g.M || n >= g.N) continue;
        uint4* sp = reinterpret_cast<uint4*>(st.tile + Staging<BN>::off(r, c));
        uint32_t v[4] = {sp->x, sp->y, sp->z, sp->w};
        const uint32_t x[4] = {rw[u].x, rw[u].y, rw[u].z, rw[u].w};
        float gv[8];   // the gate row of a batch is 1 KB per tile: after the first rows, L1 hits
        if (gate_epi) {
          const float4* gp = reinterpret_cast<const float4*>(g.gate + (size_t)(m / g.rows_per_batch) * g.gate_stride + n);
          const float4 g0 = gp[0], g1 = gp[1];
          gv[0] = g0.x; gv[1] = g0.y; gv[2] = g0.z; gv[3] = g0.w; gv[4] = g1.x; gv[5] = g1.y; gv[6] = g1.z; gv[7] = g1.w;
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 yv = unpack_bf16x2(v[e]);
          float y0 = yv.x, y1 = yv.y;
          if (gelu) {
            if (g.epi == EPI_BIAS_GELU_TANH) {
              y0 = bf16_round(gelu_tanh_f(y0));
              y1 = bf16_round(gelu_tanh_f(y1));
            } else {
              y0 = bf16_round(gelu_erf_f(y0));
              y1 = bf16_round(gelu_erf_f(y1));
            }
          }
          if (resid_epi) {
            const float2 xv = unpack_bf16x2(x[e]);
            if (gate_epi) {
              y0 = xv.x + y0 * gv[2 * e];
              y1 = xv.y + y1 * gv[2 * e + 1];
            } else {
              y0 = xv.x + y0;
              y1 = xv.y + y1;
            }
          }
          v[e] = pack_bf16x2(y0, y1);
        }
        *reinterpret_cast<uint4*>(g.out + (size_t)m * g.ldo + n) = make_uint4(v[0], v[1], v[2], v[3]);
        if (g.stats_mode) *sp = make_uint4(v[0], v[1], v[2], v[3]);
      }
    }
    if (!g.stats_mode) continue;
    __syncwarp();
    // row statistics of this tile (GemmArgs::stats_out): the four lanes that share a row keep partial sums about one pivot
    const int r = grp * 8 + (lane >> 2), q = lane & 3, m = mb * BM + r;
    const float st_pivot = g.stats_mode == 1 ? __uint_as_float((uint32_t)*reinterpret_cast<const uint16_t*>(st.tile + Staging<BN>::off(r, 0)) << 16)
                                             : 0.f;   // the row's first column
    float st_s = 0.f, st_ss = 0.f;
    int st_n = 0;
#pragma unroll 8
    for (int j = 0; j < CPR; ++j) {
      if (nb * BN + j * 8 < g.N) {
        const float2 z = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(st.tile + Staging<BN>::off(r, j) + 4 * q));
        const float d0 = z.x - st_pivot, d1 = z.y - st_pivot;
        st_s += d0 + d1;
        st_ss = fmaf(d0, d0, st_ss);
        st_ss = fmaf(d1, d1, st_ss);
        st_n += 8;
      }
    }
    st_s += __shfl_xor_sync(0xffffffffu, st_s, 1);   // the quad's partial sums are added in a fixed order
    st_ss += __shfl_xor_sync(0xffffffffu, st_ss, 1);
    st_s += __shfl_xor_sync(0xffffffffu, st_s, 2);
    st_ss += __shfl_xor_sync(0xffffffffu, st_ss, 2);
    if (m < g.M && st_n > 0 && q == 0) {
      float2 pr;
      if (g.stats_mode == 1) {   // (mean, M2) of this tile's st_n columns
        const float md = __fdividef(st_s, (float)st_n);
        pr = make_float2(st_pivot + md, fmaxf(st_ss - st_s * md, 0.f));
      } else {
        pr = make_float2(st_ss, 0.f);
      }
      g.stats_out[(size_t)m * g.stats_ld + nb] = pr;
    }
  }
}

// The kernel body for operands of type T (bf16, or e4m3 with the row scales s_a[M] and column scales s_w[N]).
// The epilogue is split where the value is bf16(acc [* s_a * s_w] + bias + bias_row), which everything after it reads:
//   consumers       after the main loop: the FP8 scales, the fp32 copy (out_f32), bias and bias_row, rounding to bf16, the
//                   rounded tile into the staging buffer; then straight into the next tile's main loop
//   epilogue warps  (warps 1-3 of warpgroup 0) GELU, residual / gate, the stores and the row statistics (drain_tile), while the
//                   consumers run the next tile
// The arithmetic and its rounding points are those of a single pass from the accumulators; the output is the same bits.
template <int BN, int STAGES, class T>
__device__ __forceinline__ void gemm_tiles(const CUtensorMap* tma_a, const CUtensorMap* tma_b, const GemmArgs& g, const float* s_a,
                                           const float* s_w) {
  constexpr int KB = BK_OF<T>;
  constexpr bool FP8 = sizeof(T) == 1;
  const int tiles_m = (g.M + BM - 1) / BM;
  const int tiles_n = (g.N + BN - 1) / BN;
  const int num_tiles = tiles_m * tiles_n;
  const int kblocks = (g.K + KB - 1) / KB;

  Ring<BN, STAGES> ring;
  const Staging<BN> st(ring);
  if (threadIdx.x == 0) {   // fenced and published by ring.start()
    mbar_init(st.staged, Staging<BN>::CONSUMER_THREADS);
    mbar_init(st.drained, Staging<BN>::EPI_THREADS);
  }
  if (!ring.start(
          tma_a, tma_b, num_tiles,
          [&](int t) {   // TMA producer
            int mb, nb;
            tile_coords(t, tiles_m, tiles_n, g.group_m, mb, nb);
            for (int kb = 0; kb < kblocks; ++kb) {
              const auto s = ring.acquire();
              tma_load_2d(s.a, tma_a, s.bar, kb * KB, mb * BM);
              tma_load_2d(s.b, tma_b, s.bar, kb * KB, nb * BN);
            }
          },
          [&] {   // epilogue warps; drained phase k: tile k - 1 drained and tile k's operands in shared memory
            stage_operands<BN, FP8>(st, g, s_a, s_w, blockIdx.x, tiles_m, tiles_n);
            mbar_arrive(st.drained);
            uint32_t phase = 0;
            for (int t : RingTiles{num_tiles}) {
              mbar_wait(st.staged, phase);
              phase ^= 1;
              if (t + (int)gridDim.x < num_tiles) stage_operands<BN, FP8>(st, g, s_a, s_w, t + gridDim.x, tiles_m, tiles_n);
              if (g.out) {
                int mb, nb;
                tile_coords(t, tiles_m, tiles_n, g.group_m, mb, nb);
                drain_tile<BN>(st, g, mb, nb);
              }
              mbar_arrive(st.drained);
            }
          }))
    return;
  // -------------------------------------------------------------------- consumers: main loop + their part of the epilogue
  const int r_in_tile = ring_row();   // rows r_in_tile and r_in_tile + 8 of the tile
  const int c_in_group = ring_col();
  float acc[BN / 2];
  uint32_t phase = 0;
  for (int t : RingTiles{num_tiles}) {
    int mb, nb;
    tile_coords(t, tiles_m, tiles_n, g.group_m, mb, nb);
    ring.template mma_tile<T>(acc, kblocks);
    mbar_wait(st.drained, phase);   // the previous tile is drained and this one's operands are in shared memory
    phase ^= 1;
    const int row0 = mb * BM + r_in_tile;
    float br[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) br[h] = __uint_as_float((uint32_t)st.bias_row[r_in_tile + 8 * h] << 16);
    if constexpr (FP8) {   // y = (acc * s_a[row]) * s_w[col], before everything else reads acc (out_f32 included)
      float sa[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) sa[h] = st.s_a[r_in_tile + 8 * h];
#pragma unroll
      for (int j0 = 0; j0 < BN / 8; j0 += 8) {
#pragma unroll
        for (int j = j0; j < j0 + 8 && j < BN / 8; ++j) {
          const float2 sw = *reinterpret_cast<const float2*>(st.s_w + j * 8 + c_in_group);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            acc[4 * j + 2 * h] = acc[4 * j + 2 * h] * sa[h] * sw.x;
            acc[4 * j + 2 * h + 1] = acc[4 * j + 2 * h + 1] * sa[h] * sw.y;
          }
        }
        asm volatile("" ::: "memory");   // at most 8 column scales in flight: all BN / 8 at once spill at BN = 256
      }
    }
    if (g.out_f32) {   // fp32 copy of acc + bias (validation path)
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int n = nb * BN + j * 8 + c_in_group;
        const float2 bv = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(st.bias + j * 8 + c_in_group));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = row0 + 8 * h;
          if (row < g.M && nb * BN + j * 8 < g.N)
            *reinterpret_cast<float2*>(g.out_f32 + (size_t)row * (g.ld_f32 ? g.ld_f32 : g.N) + n) =
                make_float2(acc[4 * j + 2 * h] + bv.x + br[h], acc[4 * j + 2 * h + 1] + bv.y + br[h]);
        }
      }
    }
    // bf16(acc + bias + bias_row) into the staging tile (-0.0 without a bias: x + -0.0 == x for every x, zeros included)
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const float2 bv = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(st.bias + j * 8 + c_in_group));
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float y0 = acc[4 * j + 2 * h] + bv.x, y1 = acc[4 * j + 2 * h + 1] + bv.y;
        y0 += br[h];
        y1 += br[h];
        *reinterpret_cast<uint32_t*>(st.tile + Staging<BN>::off(r_in_tile + 8 * h, j) + 2 * c_in_group) = pack_bf16x2(y0, y1);
      }
      if (j % 8 == 7) asm volatile("" ::: "memory");   // at most 8 bias words in flight (the FP8 kernel spills with all of them)
    }
    mbar_arrive(st.staged);
  }
}

template <int BN, int STAGES>
__global__ void __launch_bounds__(RING_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b, GemmArgs g) {
  gemm_tiles<BN, STAGES, bf16>(&tma_a, &tma_b, g, nullptr, nullptr);
}

template <int BN, int STAGES>
__global__ void __launch_bounds__(RING_THREADS, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b, GemmArgs g, const float* s_a,
                const float* s_w) {
  gemm_tiles<BN, STAGES, e4m3>(&tma_a, &tma_b, g, s_a, s_w);
}

template <class T>
int launch_gemm(const T* A, int lda, const float* s_a, const T* W, int ldw, const float* s_w, const GemmArgs& g, cudaStream_t stream) {
  constexpr bool fp8 = sizeof(T) == 1;
  CE_REQUIRE(g.M > 0 && g.N > 0 && g.K > 0, "gemm: empty problem");
  CE_REQUIRE(g.N % 8 == 0, "gemm: N must be a multiple of 8");
  if (fp8) CE_REQUIRE(lda % 16 == 0 && ldw % 16 == 0, "gemm: lda, ldw must be multiples of 16 (16-byte TMA strides)");
  else CE_REQUIRE(lda % 8 == 0 && ldw % 8 == 0, "gemm: lda, ldw must be multiples of 8 (16-byte TMA strides)");
  CE_REQUIRE((g.out != nullptr && g.ldo % 8 == 0) || (g.out == nullptr && g.out_f32 != nullptr), "gemm: out / ldo");
  CE_REQUIRE((reinterpret_cast<uintptr_t>(g.out) & 15) == 0, "gemm: out must be 16-byte aligned");
  CE_REQUIRE(g.out_f32 == nullptr || ((reinterpret_cast<uintptr_t>(g.out_f32) & 15) == 0 && g.ld_f32 % 4 == 0 && (g.ld_f32 == 0 || g.ld_f32 >= g.N)),
             "gemm: out_f32 must be 16-byte aligned with ld_f32 % 4 == 0, ld_f32 >= N");
  if (g.epi == EPI_BIAS_GATE_RESID || g.epi == EPI_BIAS_RESID)
    CE_REQUIRE(g.resid != nullptr && g.ldr % 8 == 0 && (reinterpret_cast<uintptr_t>(g.resid) & 15) == 0,
               "gemm: residual epilogue needs resid / ldr, resid 16-byte aligned");
  if (g.epi == EPI_BIAS_GATE_RESID)
    CE_REQUIRE(g.gate != nullptr && g.gate_stride % 4 == 0 && g.rows_per_batch > 0 && (reinterpret_cast<uintptr_t>(g.gate) & 15) == 0,
               "gemm: gate epilogue needs gate, 16-byte aligned");
  if (g.stats_mode) CE_REQUIRE(g.stats_out != nullptr && g.out != nullptr && g.stats_ld >= (g.N + gemm_tile_n(g.N) - 1) / gemm_tile_n(g.N) &&
                               (g.stats_mode == 1 || g.stats_mode == 2), "gemm: stats_out / stats_ld / stats_mode");
  GemmArgs a = g;
  // Tiles are rasterised in groups of group_m M-tiles x all N-tiles so that the A panel of a group stays in L2 while the W
  // panels stream past it (16 M-tiles x 128 rows x K = 5120 is 20 MB of A, inside the H100's 50 MB L2).
  if (a.group_m <= 0) a.group_m = 16;
  const int bn = gemm_tile_n(a.N);
  const auto tmap = fp8 ? make_tmap_2d_u8 : make_tmap_2d;
  CUtensorMap ta, tb;
  int rc = tmap(&ta, A, (uint64_t)a.M, (uint64_t)a.K, (uint64_t)lda, BM);
  if (rc) return rc;
  rc = tmap(&tb, W, (uint64_t)a.N, (uint64_t)a.K, (uint64_t)ldw, (uint32_t)bn);
  if (rc) return rc;
  const int tiles = ((a.M + BM - 1) / BM) * ((a.N + bn - 1) / bn);
  // Ring depth: what is left of the 227 KB beside the staging tile (64 KB at BN = 256, where one stage of 48 KB has to go).
  if constexpr (fp8) {
    if (bn == 256) return launch_ring_gemm<256, 3, Staging<256>::BYTES>(gemm_fp8_kernel<256, 3>, tiles, stream, ta, tb, a, s_a, s_w);
    if (bn == 128) return launch_ring_gemm<128, 6, Staging<128>::BYTES>(gemm_fp8_kernel<128, 6>, tiles, stream, ta, tb, a, s_a, s_w);
    return launch_ring_gemm<64, 8, Staging<64>::BYTES>(gemm_fp8_kernel<64, 8>, tiles, stream, ta, tb, a, s_a, s_w);
  } else {
    if (bn == 256) return launch_ring_gemm<256, 3, Staging<256>::BYTES>(gemm_bf16_kernel<256, 3>, tiles, stream, ta, tb, a);
    if (bn == 128) return launch_ring_gemm<128, 6, Staging<128>::BYTES>(gemm_bf16_kernel<128, 6>, tiles, stream, ta, tb, a);
    return launch_ring_gemm<64, 8, Staging<64>::BYTES>(gemm_bf16_kernel<64, 8>, tiles, stream, ta, tb, a);
  }
}

}  // namespace

int launch_gemm_bf16(const bf16* A, int lda, const bf16* W, int ldw, const GemmArgs& g, cudaStream_t stream) {
  return launch_gemm<bf16>(A, lda, nullptr, W, ldw, nullptr, g, stream);
}

int launch_gemm_fp8(const e4m3* Aq, int lda, const float* s_a, const e4m3* Wq, int ldw, const float* s_w, const GemmArgs& g,
                    cudaStream_t stream) {
  CE_REQUIRE(s_a != nullptr && s_w != nullptr && (reinterpret_cast<uintptr_t>(s_w) & 7) == 0,
             "gemm_fp8: a_scale and w_scale are required, w_scale 8-byte aligned");
  return launch_gemm<e4m3>(Aq, lda, s_a, Wq, ldw, s_w, g, stream);
}

int run_gemm(Launcher& run, const bf16* A, int lda, const bf16* W, int ldw, int M, int N, int K, bf16* out, int ldo, const bf16* bias, int epi,
             const bf16* resid, int ldr) {
  GemmArgs g;
  g.M = M; g.N = N; g.K = K; g.out = out; g.ldo = ldo; g.bias = bias;
  g.epi = epi; g.resid = resid; g.ldr = ldr;
  return run([&] { return launch_gemm_bf16(A, lda, W, ldw, g, run.s); });
}

int gemm_attention(Launcher& run, const GemmAttention& a) {
  const int I = a.H * a.dk, L8 = up8(a.L);
  CE_TRY(run_gemm(run, a.x, a.D, a.wqk, a.D, a.L, 2 * I, a.D, a.qk, 2 * I, a.bqk));
  GemmArgs g;
  g.M = I; g.N = L8; g.K = a.D; g.out = a.vT; g.ldo = L8; g.bias_row = a.bv;
  CE_TRY(run([&] { return launch_gemm_bf16(a.wv, a.D, a.x, a.D, g, run.s); }));
  CE_REQUIRE(a.q0 >= 0 && a.nq >= 1 && a.q0 + a.nq <= a.L, "gemm_attention: query rows outside [0, L)");
  CE_REQUIRE(a.nq == a.L || a.sc.rule == SOFTMAX_SCALED, "gemm_attention: a query range needs the scaled softmax (no position bias)");
  for (int h = 0; h < a.H; ++h) {
    g = GemmArgs();
    g.M = a.nq; g.N = L8; g.K = a.dk; g.out_f32 = a.S + (size_t)h * a.nq * L8; g.ld_f32 = L8;
    CE_TRY(run([&] { return launch_gemm_bf16(a.qk + (size_t)a.q0 * 2 * I + h * a.dk, 2 * I, a.qk + I + h * a.dk, 2 * I, g, run.s); }));
  }
  CE_TRY(run([&] { return launch_softmax_rows(a.S, L8, a.P, L8, a.H * a.nq, a.L, a.sc, run.s); }));
  for (int h = 0; h < a.H; ++h)
    CE_TRY(run_gemm(run, a.P + (size_t)h * a.nq * L8, L8, a.vT + (size_t)h * a.dk * L8, L8, a.nq, a.dk, a.kpv, a.out + h * a.dk, a.ldo));
  return CE_OK;
}

}  // namespace ce
