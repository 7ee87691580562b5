// The operators of the fp32 chains (dit_fp32.cu: the DiT's validation forward; encoders.cu: the fp32 CLIP vision encoder).
//
// Every matrix product runs on the wgmma GEMM of gemm.cu: an fp32 operand x is split into two bf16 terms hi = bf16(x),
// lo = bf16(x - hi) (|x - hi - lo| <= 2^-17 |x|), and A.W^T is evaluated as ONE bf16 GEMM over a K axis three times as long --
// A' = [A_hi | A_lo | A_hi], W' = [W_hi | W_hi | W_lo], i.e. A_hi.W_hi + A_lo.W_hi + A_hi.W_lo, fp32 accumulation in registers, fp32
// store (the dropped A_lo.W_lo term is 2^-18 relative).  Attention is S = Q.K^T (same split GEMM, fp32 S in HBM), an fp32 row
// softmax, and O = P.V with P and V^T split the same way.  Everything elementwise is a plain fp32 SIMT kernel.
//
// With terms = 6 every operand is split into three bf16 terms hi, mid, lo (|x - hi - mid - lo| <= 2^-25 |x|) and the six products
// down to 2^-16 are kept: hi.hi + hi.mid + mid.hi + mid.mid + hi.lo + lo.hi, about 2^-24 relative per product -- twice the MMA work of
// the 3-term split.  The wgmma accumulator then sets the error: it loses low bits at every k-step, relative to the sum so far, so
// one long accumulation drifts.  A 6-term product therefore runs the five small products as one GEMM (their own sum is 2^-8 of the
// result, and so are its losses), then hi.hi as one GEMM per K-chunk of kHiChunk, each added to the result with an fp32 add.  The
// 32-layer CLIP encoder needs this to stay within rtol 1e-3 / atol 1e-4 of transformers' fp32 run; the 3-term split does not.
#pragma once
#include "host_common.h"

namespace ce {

// One fp32 Linear: weight [N, K], bias [N] (or null).
struct Lin32 {
  const float *w = nullptr, *b = nullptr;
};

// bf16 elements of the split operand of `rows` rows of a K-long fp32 product (A' or W' above) in `terms` terms.
inline int64_t split_elems(int64_t rows, int K, int terms) { return rows * terms * up8(K); }
constexpr int kHiChunk = 256;   // K of one hi.hi GEMM of a 6-term product

struct Fp32Chain {
  Launcher run;
  bf16 *Ap, *Wp;   // split operands: A' and W' of the largest product
  float *S, *P;    // attention scores and probabilities of one head, [Lq, up8(Lk)]
  int terms = 3;   // bf16 products per fp32 product: 3 (hi / lo split) or 6 (hi / mid / lo split)
  float* part = nullptr;   // [M, N] fp32 of the largest product: one hi.hi chunk (terms = 6)

  // out[rows, terms * Kp] (bf16) = the split of x[rows, 0:K] (ldx) in the A (w_layout 0) or W (1) layout
  int split(const float* x, int ldx, int rows, int K, int Kp, bf16* out, int w_layout);
  // out[M, ldo] (fp32) = A'[M, terms * Kp] . W'[N, terms * Kp]^T of two splits
  int product(const bf16* A, const bf16* W, int M, int N, int Kp, float* out, int ldo);
  // out[M, ldo] (fp32) = act(A[M, K] (lda) . W[N, K]^T + bias);  act 0 none, 1 GELU(tanh), 2 GELU(erf), 3 SiLU
  int linear(const float* A, int lda, int M, int K, const Lin32& w, int N, float* out, int ldo, int act);
  // y[r, c] = act(y[r, c] + bias[c])   (bias may be null)
  int bias_act(float* y, int ldy, int rows, int N, const float* bias, int act);
  // x[r, c] += y[r, c] * (gate ? gate[(r / rows_per_batch) * gate_stride + c] : 1)
  int resid(float* x, const float* y, int rows, int D, const float* gate, int gate_stride, int rows_per_batch);
  // y = LN(x) * (1 + scale[b]) + shift[b]   or   LN(x) * w + b   (two-pass variance, fp32; b = row / rpb, rpb 0 = all rows)
  int layernorm(const float* x, float* y, int rows, int D, float eps, const float* scale, const float* shift, int mod_stride, int rpb,
                const float* w, const float* b);
  // out[b, i, h*hd:(h+1)*hd] = softmax(q k^T * scale) v   for every (b, h); q [B*Lq, D], k / v [B*Lk, D]
  int attention(const float* q, const float* k, const float* v, float* out, int B, int H, int Lq, int Lk, int D, int hd, float scale);
};

}  // namespace ce
