// Interface of the wgmma GEMM used by the DiT path (gemm.cu).
#pragma once
#include "host_common.h"
#include <cuda_fp8.h>

#include "elementwise.cuh"
#include "ptx.cuh"

namespace ce {

typedef __nv_fp8_e4m3 e4m3;

// Fused epilogues.  "y" is the Linear output rounded to bf16 exactly as nn.Linear returns it in the
// reference's bf16 path; every variant keeps the reference's rounding points (SURVEY.md section 8a).
enum GemmEpilogue : int {
  EPI_BIAS = 0,             // out = bf16(acc + bias)
  EPI_BIAS_GELU_TANH = 1,   // out = bf16(gelu_tanh(float(bf16(acc + bias))))          ffn.net.0  (transformer_chronoedit.py:292)
  EPI_BIAS_GELU_ERF = 2,    // out = bf16(gelu_erf (float(bf16(acc + bias))))          image_embedder.ff.net.0 (:111-123)
  EPI_BIAS_GATE_RESID = 3,  // out = bf16(float(resid) + float(bf16(acc + bias)) * gate[batch, col])   (:281, :293)
  EPI_BIAS_RESID = 4,       // out = bf16(float(resid) + float(bf16(acc + bias)))                      (:286)
};

struct GemmArgs {
  int M = 0, N = 0, K = 0;
  bf16* out = nullptr;        // [M, ldo] bf16 (may be null when out_f32 is given)
  int ldo = 0;
  float* out_f32 = nullptr;   // optional [M, ld_f32] fp32 copy of (acc + bias) BEFORE any rounding (parity tests, fp32 validation mode)
  int ld_f32 = 0;             // leading dimension of out_f32 in elements (0 = N)
  const bf16* bias = nullptr; // [N] or null
  const bf16* bias_row = nullptr;  // [M] or null: added per output ROW (used for V^T = W_v x^T + b_v in the VAE attention)
  int epi = EPI_BIAS;
  const bf16* resid = nullptr;  // [M, ldr]
  int ldr = 0;
  const float* gate = nullptr;  // [batches, gate_stride] fp32, row -> batch = row / rows_per_batch
  int gate_stride = 0;
  int rows_per_batch = 1;
  // Row statistics of the STORED bf16 output, one float2 per (row, N tile) at stats_out[row * stats_ld + n_tile]:
  //   stats_mode 1: (mean, M2 = sum (y - mean)^2) of the tile's columns      -> FP32LayerNorm of the next operator
  //   stats_mode 2: (sum y^2, 0)                                             -> RMSNorm across heads
  // so that the row kernel that follows is a pure streaming pass (no reduction, no barrier); tiles are merged there in a fixed
  // order (deterministic).  N tile width = gemm_tile_n(N).
  float2* stats_out = nullptr;
  int stats_ld = 0;
  int stats_mode = 0;
  int group_m = 0;              // tile rasterisation: M-tiles per group (L2 reuse); 0 = chosen by launch_gemm_bf16
};

// N tile width launch_gemm_bf16 uses for a given N (the granularity of GemmArgs::stats_out)
inline int gemm_tile_n(int N) { return N >= 256 ? 256 : (N >= 128 ? 128 : 64); }

// out[M,N] = epilogue(A[M,K] (row-major, lda) x W[N,K]^T (row-major = nn.Linear weight, ldw)).
int launch_gemm_bf16(const bf16* A, int lda, const bf16* W, int ldw, const GemmArgs& g, cudaStream_t stream);

// The FP8 mode's GEMM: y[m,n] = (sum_k Aq[m,k] Wq[n,k] * s_a[m]) * s_w[n] with e4m3 operands (Aq row-major, lda; Wq row-major, ldw;
// lda, ldw multiples of 16) and fp32 scales s_a[M], s_w[N]; out[M,N] = epilogue(y) exactly as launch_gemm_bf16 applies it to acc.
int launch_gemm_fp8(const e4m3* Aq, int lda, const float* s_a, const e4m3* Wq, int ldw, const float* s_w, const GemmArgs& g,
                    cudaStream_t stream);

// One launch_gemm_bf16 through `run`, with only the epilogue fields bias / epi / resid.
int run_gemm(Launcher& run, const bf16* A, int lda, const bf16* W, int ldw, int M, int N, int K, bf16* out, int ldo, const bf16* bias = nullptr,
             int epi = EPI_BIAS, const bf16* resid = nullptr, int ldr = 0);

// Multi-head attention built from GEMMs over one sequence of L tokens, I = heads * dk, L8 = up8(L):
//   q|k = x [Wq;Wk]^T + bqk                -> qk [L, 2I]
//   V^T = Wv x^T + bv (per row)            -> vT [I, L8]   (x rows L..L8-1 are read: finite or not, they only reach columns
//                                                           of V^T that P.V does not sum over, or multiply zeros of P)
//   per head: S_h = q_h k_h^T (fp32)       -> S [H, L, L8]   (k rows L..L8-1 of qk are read but never written here: whatever
//                                                           they hold only reaches columns L..L8-1 of S, which the softmax
//                                                           does not read)
//   P = one row-softmax launch (rule sc)   -> P [H, L, L8]
//   per head: O_h = P_h[:, 0:kpv] V_h      -> out [L, I] (ld ldo)
// Only the query rows [q0, q0 + nq) are computed past q|k and V^T: S and P are [H, nq, L8] and out is [nq, I]; every row is the same
// sum over the same keys in the same order whatever range it is computed in (the VAE split over ranks computes its band of rows).
// x [L8, D] (ld D), Wqk [2I, D], Wv [I, D]; bqk / bv may be null.  Every launch goes through `run`.
struct GemmAttention {
  const bf16 *x, *wqk, *bqk, *wv, *bv;
  int L, D, H, dk;
  int kpv;   // keys P.V sums over: L, or L8 when P's padding columns are zero and V^T's are finite
  int q0, nq;   // query rows: [0, L) for the whole sequence
  SoftmaxScores sc;
  bf16 *qk, *vT, *P, *out;
  float* S;
  int ldo;
};
int gemm_attention(Launcher& run, const GemmAttention& a);

}  // namespace ce
