// bf16 GEMM for sm_90a on the TMA -> shared-memory ring -> wgmma pipeline of ring_gemm.cuh, with a fused epilogue.
//
//   out[M,N] = epilogue( A[M,K] * W[N,K]^T )        A: activations (row-major), W: nn.Linear weight (row-major)
//
// Per k-block an A tile 128x64 and a W tile BNx64; the epilogue applies bias / activation / gate / residual / row statistics.
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

constexpr uint32_t NEG_ZERO2 = 0x80008000u;   // two bf16 -0.0

// The kernel body for operands of type T (bf16, or e4m3 with the row scales s_a[M] and column scales s_w[N]).
template <int BN, int STAGES, class T>
__device__ __forceinline__ void gemm_tiles(const CUtensorMap* tma_a, const CUtensorMap* tma_b, const GemmArgs& g, const float* s_a,
                                           const float* s_w) {
  constexpr int KB = BK_OF<T>;
  const int lane = threadIdx.x & 31;
  const int tiles_m = (g.M + BM - 1) / BM;
  const int tiles_n = (g.N + BN - 1) / BN;
  const int num_tiles = tiles_m * tiles_n;
  const int kblocks = (g.K + KB - 1) / KB;

  Ring<BN, STAGES> ring;
  if (!ring.start(tma_a, tma_b, num_tiles, [&](int t) {   // TMA producer
        int mb, nb;
        tile_coords(t, tiles_m, tiles_n, g.group_m, mb, nb);
        for (int kb = 0; kb < kblocks; ++kb) {
          const auto s = ring.acquire();
          tma_load_2d(s.a, tma_a, s.bar, kb * KB, mb * BM);
          tma_load_2d(s.b, tma_b, s.bar, kb * KB, nb * BN);
        }
      }))
    return;
  // -------------------------------------------------------------------- consumers: main loop + epilogue
  // The epilogue works in passes so that its global loads are not serialised behind its stores.  out, resid and bias are all
  // bf16 pointers and do alias (out == resid in place in the DiT's residual GEMMs), so the compiler keeps every load behind every
  // earlier store: with one load and one store per column group, as before, a tile waited for 64 round trips to memory.
  //   pass 1  (no store) bias, rounding to bf16, GELU; packs the value as stored into one register per two columns, which frees
  //           half of the accumulator registers (the kernel has 168 per thread, 128 of them accumulators at BN = 256)
  //   pass 2  per row, chunks of CH column groups: the chunk's residual and gate loads, then its stores and row statistics
  // A thread reads each element before it writes it, so in-place stays correct.  Arithmetic, rounding points and the order of
  // the statistics sums are those of the single pass; the output is bit-identical.  CH = 16 spills at BN = 256.
  constexpr int CH = BN / 8 < 8 ? BN / 8 : 8;
  const int r_in_tile = ring_row();   // rows r_in_tile and r_in_tile + 8 of the tile
  const int c_in_group = ring_col();
  const bool resid_epi = g.epi == EPI_BIAS_GATE_RESID || g.epi == EPI_BIAS_RESID;
  float acc[BN / 2];
  for (int t : RingTiles{num_tiles}) {
    int mb, nb;
    tile_coords(t, tiles_m, tiles_n, g.group_m, mb, nb);
    ring.template mma_tile<T>(acc, kblocks);
    const int row0 = mb * BM + r_in_tile;
    if constexpr (sizeof(T) == 1) {   // y = (acc * s_a[row]) * s_w[col], before everything else reads acc (out_f32 included)
      float sa[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) sa[h] = row0 + 8 * h < g.M ? s_a[row0 + 8 * h] : 0.f;
#pragma unroll
      for (int j0 = 0; j0 < BN / 8; j0 += CH) {
#pragma unroll
        for (int j = j0; j < j0 + CH; ++j) {
          if (nb * BN + j * 8 < g.N) {
            const float2 sw = *reinterpret_cast<const float2*>(s_w + nb * BN + j * 8 + c_in_group);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              acc[4 * j + 2 * h] = acc[4 * j + 2 * h] * sa[h] * sw.x;
              acc[4 * j + 2 * h + 1] = acc[4 * j + 2 * h + 1] * sa[h] * sw.y;
            }
          }
        }
        asm volatile("" ::: "memory");   // at most CH column scales in flight: all BN / 8 at once spill at BN = 256
      }
    }
    if (g.out_f32) {   // fp32 copy of acc + bias (validation path), on its own so that pass 1 has no store
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int n = nb * BN + j * 8 + c_in_group;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = row0 + 8 * h;
          if (row < g.M && nb * BN + j * 8 < g.N) {
            const float2 bv = unpack_bf16x2(g.bias ? *reinterpret_cast<const uint32_t*>(g.bias + n) : NEG_ZERO2);
            const float br = g.bias_row ? __bfloat162float(g.bias_row[row]) : -0.f;
            *reinterpret_cast<float2*>(g.out_f32 + (size_t)row * (g.ld_f32 ? g.ld_f32 : g.N) + n) =
                make_float2(acc[4 * j + 2 * h] + bv.x + br, acc[4 * j + 2 * h + 1] + bv.y + br);
          }
        }
      }
    }
    uint32_t yp[BN / 8][2];   // [column group][row]: bf16(acc + bias), after GELU; raw acc where nothing is stored
    // ---- pass 1: bias (loaded once per chunk for both rows), rounding, activation
#pragma unroll
    for (int j0 = 0; j0 < BN / 8; j0 += CH) {
      uint32_t bias_w[CH];
#pragma unroll
      for (int jj = 0; jj < CH; ++jj) {
        const int n = nb * BN + (j0 + jj) * 8 + c_in_group;
        bias_w[jj] = g.bias && row0 < g.M && nb * BN + (j0 + jj) * 8 < g.N ? *reinterpret_cast<const uint32_t*>(g.bias + n) : NEG_ZERO2;
      }
#pragma unroll
      for (int jj = 0; jj < CH; ++jj) {
        const int j = j0 + jj;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = row0 + 8 * h;
          float y0 = acc[4 * j + 2 * h], y1 = acc[4 * j + 2 * h + 1];
          // The wgmma asm takes acc as "+f", so without this the values would stay live until the next tile's first wgmma
          // (which ignores them: scale_d = 0) and pass 2 could not have their registers.
          acc[4 * j + 2 * h] = acc[4 * j + 2 * h + 1] = 0.f;
          if (row < g.M && nb * BN + j * 8 < g.N) {
            const float2 bv = unpack_bf16x2(bias_w[jj]);   // -0.0 without a bias: x + -0.0 == x for every x, zeros included
            y0 += bv.x;
            y1 += bv.y;
            const float br = g.bias_row ? __bfloat162float(g.bias_row[row]) : -0.f;
            y0 += br;
            y1 += br;
            y0 = bf16_round(y0);  // nn.Linear returns bf16
            y1 = bf16_round(y1);
            if (g.epi == EPI_BIAS_GELU_TANH) {
              y0 = gelu_tanh_f(y0);
              y1 = gelu_tanh_f(y1);
            } else if (g.epi == EPI_BIAS_GELU_ERF) {
              y0 = gelu_erf_f(y0);
              y1 = gelu_erf_f(y1);
            }
          }
          yp[j][h] = pack_bf16x2(y0, y1);   // exact except after GELU, where it is the rounding of the store
        }
      }
    }
    if (!g.out) continue;
    // ---- pass 2: residual / gate, store, row statistics
#pragma unroll
    for (int h = 0; h < 2; ++h) {   // the thread's two rows
      const int row = row0 + 8 * h;
      const bool row_ok = row < g.M;
      const int batch = row_ok ? row / g.rows_per_batch : 0;
      // row statistics of this tile (GemmArgs::stats_out): the four lanes that share a row keep partial sums about one pivot
      float st_pivot = 0.f, st_s = 0.f, st_ss = 0.f;
      int st_n = 0;
#pragma unroll
      for (int j0 = 0; j0 < BN / 8; j0 += CH) {
        uint32_t resid_w[CH];
        float2 gate_v[CH];
#pragma unroll
        for (int jj = 0; jj < CH; ++jj) {   // the chunk's loads
          const int n = nb * BN + (j0 + jj) * 8 + c_in_group;
          const bool ld = resid_epi && row_ok && nb * BN + (j0 + jj) * 8 < g.N;
          resid_w[jj] = ld ? *reinterpret_cast<const uint32_t*>(g.resid + (size_t)row * g.ldr + n) : 0u;
          gate_v[jj] = ld && g.epi == EPI_BIAS_GATE_RESID ? *reinterpret_cast<const float2*>(g.gate + (size_t)batch * g.gate_stride + n)
                                                          : make_float2(0.f, 0.f);
        }
#pragma unroll
        for (int jj = 0; jj < CH; ++jj) {   // 8-column groups, two columns per lane
          const int j = j0 + jj;
          const int n = nb * BN + j * 8 + c_in_group;
          const bool ok = row_ok && nb * BN + j * 8 < g.N;
          const float2 yv = unpack_bf16x2(yp[j][h]);
          float y0 = yv.x, y1 = yv.y;
          if (ok) {
            if (resid_epi) {
              const float2 x = unpack_bf16x2(resid_w[jj]);
              if (g.epi == EPI_BIAS_GATE_RESID) {
                y0 = x.x + y0 * gate_v[jj].x;
                y1 = x.y + y1 * gate_v[jj].y;
              } else {
                y0 = x.x + y0;
                y1 = x.y + y1;
              }
            }
            *reinterpret_cast<uint32_t*>(g.out + (size_t)row * g.ldo + n) = pack_bf16x2(y0, y1);
          }
          if (g.stats_mode) {   // statistics of the values as stored (bf16), pivot-shifted inside the tile
            const float z0 = bf16_round(y0), z1 = bf16_round(y1);
            if (j == 0) st_pivot = g.stats_mode == 1 ? __shfl_sync(0xffffffffu, z0, lane & ~3) : 0.f;  // the row's first column
            if (ok) {
              const float d0 = z0 - st_pivot, d1 = z1 - st_pivot;
              st_s += d0 + d1;
              st_ss = fmaf(d0, d0, st_ss);
              st_ss = fmaf(d1, d1, st_ss);
              st_n += 8;
            }
          }
        }
      }
      if (g.stats_mode) {   // warp-uniform; the quad's partial sums are added in a fixed order
        st_s += __shfl_xor_sync(0xffffffffu, st_s, 1);
        st_ss += __shfl_xor_sync(0xffffffffu, st_ss, 1);
        st_s += __shfl_xor_sync(0xffffffffu, st_s, 2);
        st_ss += __shfl_xor_sync(0xffffffffu, st_ss, 2);
        if (row_ok && st_n > 0 && (lane & 3) == 0) {
          float2 pr;
          if (g.stats_mode == 1) {   // (mean, M2) of this tile's st_n columns
            const float md = __fdividef(st_s, (float)st_n);  // no call: a subroutine would serialise the wgmma pipeline
            pr = make_float2(st_pivot + md, fmaxf(st_ss - st_s * md, 0.f));
          } else {
            pr = make_float2(st_ss, 0.f);
          }
          g.stats_out[(size_t)row * g.stats_ld + nb] = pr;
        }
      }
    }
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
    CE_REQUIRE(g.resid != nullptr && g.ldr % 8 == 0, "gemm: residual epilogue needs resid / ldr");
  if (g.epi == EPI_BIAS_GATE_RESID)
    CE_REQUIRE(g.gate != nullptr && g.gate_stride % 4 == 0 && g.rows_per_batch > 0, "gemm: gate epilogue needs gate");
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
  if constexpr (fp8) {
    if (bn == 256) return launch_ring_gemm<256, 4>(gemm_fp8_kernel<256, 4>, tiles, stream, ta, tb, a, s_a, s_w);
    if (bn == 128) return launch_ring_gemm<128, 6>(gemm_fp8_kernel<128, 6>, tiles, stream, ta, tb, a, s_a, s_w);
    return launch_ring_gemm<64, 8>(gemm_fp8_kernel<64, 8>, tiles, stream, ta, tb, a, s_a, s_w);
  } else {
    if (bn == 256) return launch_ring_gemm<256, 4>(gemm_bf16_kernel<256, 4>, tiles, stream, ta, tb, a);
    if (bn == 128) return launch_ring_gemm<128, 6>(gemm_bf16_kernel<128, 6>, tiles, stream, ta, tb, a);
    return launch_ring_gemm<64, 8>(gemm_bf16_kernel<64, 8>, tiles, stream, ta, tb, a);
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
  for (int h = 0; h < a.H; ++h) {
    g = GemmArgs();
    g.M = a.L; g.N = L8; g.K = a.dk; g.out_f32 = a.S + (size_t)h * a.L * L8; g.ld_f32 = L8;
    CE_TRY(run([&] { return launch_gemm_bf16(a.qk + h * a.dk, 2 * I, a.qk + I + h * a.dk, 2 * I, g, run.s); }));
  }
  CE_TRY(run([&] { return launch_softmax_rows(a.S, L8, a.P, L8, a.H * a.L, a.L, a.sc, run.s); }));
  for (int h = 0; h < a.H; ++h)
    CE_TRY(run_gemm(run, a.P + (size_t)h * a.L * L8, L8, a.vT + (size_t)h * a.dk * L8, L8, a.L, a.dk, a.kpv, a.out + h * a.dk, a.ldo));
  return CE_OK;
}

}  // namespace ce
