// The operators of the fp32 chains: see fp32_chain.cuh.
#include <math.h>

#include "elementwise.cuh"
#include "fp32_chain.cuh"
#include "gemm.cuh"

namespace ce {

namespace {

// out[r, :] (bf16, 3*Kp wide) from x[r, 0:K] fp32 (leading dim ldx); A layout [hi | lo | hi], W layout [hi | hi | lo]; columns
// K..Kp-1 of each third are zero
__global__ void split3_kernel(const float* __restrict__ x, int ldx, int rows, int K, int Kp, bf16* __restrict__ out, int w_layout) {
  const size_t total = (size_t)rows * Kp;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % Kp);
    const size_t r = i / Kp;
    float v = c < K ? x[r * ldx + c] : 0.f;
    const bf16 hi = __float2bfloat16_rn(v);
    const bf16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
    bf16* o = out + r * 3 * (size_t)Kp;
    o[c] = hi;
    o[Kp + c] = w_layout ? hi : lo;
    o[2 * Kp + c] = w_layout ? lo : hi;
  }
}
// W layout of the TRANSPOSE: out[n, :] over k from x[k, n]  (V^T for the P.V product); x [K, ldx], n < N
__global__ void split3_transposed_kernel(const float* __restrict__ x, int ldx, int K, int Kp, int N, bf16* __restrict__ out) {
  const size_t total = (size_t)N * Kp;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % Kp);
    const int n = (int)(i / Kp);
    float v = k < K ? x[(size_t)k * ldx + n] : 0.f;
    const bf16 hi = __float2bfloat16_rn(v);
    const bf16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
    bf16* o = out + (size_t)n * 3 * Kp;
    o[k] = hi;
    o[Kp + k] = hi;
    o[2 * Kp + k] = lo;
  }
}

// The 6-term split: hi = bf16(x), mid = bf16(x - hi), lo = bf16(x - hi - mid) (|x - hi - mid - lo| <= 2^-25 |x|); A layout
// [hi | hi | mid | mid | hi | lo], W layout [hi | mid | hi | mid | lo | hi], i.e. hi.hi + hi.mid + mid.hi + mid.mid + hi.lo + lo.hi (the
// dropped mid.lo, lo.mid and lo.lo terms are below 2^-24 relative).  Columns K..Kp-1 of each sixth are zero.
__device__ __forceinline__ void split6_store(float v, bf16* o, int Kp, int c, int w_layout) {
  const bf16 hi = __float2bfloat16_rn(v);
  const float r = v - __bfloat162float(hi);
  const bf16 mid = __float2bfloat16_rn(r);
  const bf16 lo = __float2bfloat16_rn(r - __bfloat162float(mid));
  o[c] = hi;
  o[Kp + c] = w_layout ? mid : hi;
  o[2 * Kp + c] = w_layout ? hi : mid;
  o[3 * Kp + c] = mid;
  o[4 * Kp + c] = w_layout ? lo : hi;
  o[5 * Kp + c] = w_layout ? hi : lo;
}
__global__ void split6_kernel(const float* __restrict__ x, int ldx, int rows, int K, int Kp, bf16* __restrict__ out, int w_layout) {
  const size_t total = (size_t)rows * Kp;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % Kp);
    const size_t r = i / Kp;
    split6_store(c < K ? x[r * ldx + c] : 0.f, out + r * 6 * (size_t)Kp, Kp, c, w_layout);
  }
}
__global__ void split6_transposed_kernel(const float* __restrict__ x, int ldx, int K, int Kp, int N, bf16* __restrict__ out) {
  const size_t total = (size_t)N * Kp;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % Kp);
    const int n = (int)(i / Kp);
    split6_store(k < K ? x[(size_t)k * ldx + n] : 0.f, out + (size_t)n * 6 * Kp, Kp, k, 1);
  }
}

__device__ __forceinline__ float act_f(float y, int act) {
  if (act == 1) return 0.5f * y * (1.0f + tanhf(0.7978845608028654f * (y + 0.044715f * y * y * y)));  // GELU(tanh)
  if (act == 2) return 0.5f * y * (1.0f + erff(y * 0.7071067811865476f));                              // GELU(erf)
  if (act == 3) return y / (1.0f + expf(-y));                                                          // SiLU
  return y;
}
// y[r, c] = act(y[r, c] + bias[c])
__global__ void bias_act_kernel(float* __restrict__ y, int ldy, int rows, int N, const float* __restrict__ bias, int act) {
  const size_t total = (size_t)rows * N;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % N);
    const size_t r = i / N;
    float v = y[r * ldy + c] + (bias ? bias[c] : 0.f);
    y[r * ldy + c] = act_f(v, act);
  }
}
// out[r, c] += part[r, c]   (out with leading dim ldo, part [rows, N])
__global__ void add_rows_kernel(float* __restrict__ out, int ldo, const float* __restrict__ part, int rows, int N) {
  const size_t total = (size_t)rows * N;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
    out[(i / N) * ldo + i % N] += part[i];
}
// x[r, c] += y[r, c] * (gate ? gate[b(r), c] : 1)
__global__ void resid_kernel(float* __restrict__ x, const float* __restrict__ y, int rows, int D, const float* __restrict__ gate,
                             int gate_stride, int rows_per_batch) {
  const size_t total = (size_t)rows * D;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % D);
    const size_t r = i / D;
    const float g = gate ? gate[(r / rows_per_batch) * gate_stride + c] : 1.0f;
    x[i] = x[i] + y[i] * g;
  }
}
// one warp per row: y = LN(x) * (1 + scale) + shift   or   LN(x) * w + b   (two-pass variance, fp32)
__global__ void layernorm_f32_kernel(const float* __restrict__ x, float* __restrict__ y, int rows, int D, float eps,
                                     const float* __restrict__ scale, const float* __restrict__ shift, int mod_stride, int rows_per_batch,
                                     const float* __restrict__ w, const float* __restrict__ b) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* xr = x + (size_t)row * D;
  float s = 0.f;
  for (int i = lane; i < D; i += 32) s += xr[i];
  const float mean = warp_sum(s) / D;
  float ss = 0.f;
  for (int i = lane; i < D; i += 32) {
    const float d = xr[i] - mean;
    ss += d * d;
  }
  const float rstd = rsqrtf(warp_sum(ss) / D + eps);
  const int bi = row / rows_per_batch;
  for (int i = lane; i < D; i += 32) {
    float v = (xr[i] - mean) * rstd;
    if (scale) v = v * (1.0f + scale[(size_t)bi * mod_stride + i]) + shift[(size_t)bi * mod_stride + i];
    else if (w) v = v * w[i] + b[i];
    y[(size_t)row * D + i] = v;
  }
}

}  // namespace

int Fp32Chain::split(const float* x, int ldx, int rows, int K, int Kp, bf16* out, int w_layout) {
  return run.kernel(terms == 6 ? split6_kernel : split3_kernel, grid_for((size_t)rows * Kp), TPB, x, ldx, rows, K, Kp, out, w_layout);
}

int Fp32Chain::product(const bf16* A, const bf16* W, int M, int N, int Kp, float* out, int ldo) {
  const int ld = terms * Kp;
  GemmArgs g;
  g.M = M; g.N = N; g.out_f32 = out; g.ld_f32 = ldo;
  if (terms == 3) {
    g.K = 3 * Kp;
    return run([&] { return launch_gemm_bf16(A, ld, W, ld, g, run.s); });
  }
  CE_REQUIRE(part != nullptr, "fp32 chain: a 6-term product needs the partial buffer");
  g.K = 5 * Kp;   // the five small products first, then hi.hi chunk by chunk
  CE_TRY(run([&] { return launch_gemm_bf16(A + Kp, ld, W + Kp, ld, g, run.s); }));
  g.out_f32 = part; g.ld_f32 = N;
  for (int k0 = 0; k0 < Kp; k0 += kHiChunk) {
    g.K = Kp - k0 < kHiChunk ? Kp - k0 : kHiChunk;
    CE_TRY(run([&] { return launch_gemm_bf16(A + k0, ld, W + k0, ld, g, run.s); }));
    CE_TRY(run.kernel(add_rows_kernel, grid_for((size_t)M * N), TPB, out, ldo, (const float*)part, M, N));
  }
  return CE_OK;
}

int Fp32Chain::linear(const float* A, int lda, int M, int K, const Lin32& w, int N, float* out, int ldo, int act) {
  const int Kp = up8(K);
  CE_TRY(split(A, lda, M, K, Kp, Ap, 0));
  CE_TRY(split(w.w, K, N, K, Kp, Wp, 1));
  CE_TRY(product(Ap, Wp, M, N, Kp, out, ldo));
  if (w.b || act) CE_TRY(bias_act(out, ldo, M, N, w.b, act));
  return CE_OK;
}

int Fp32Chain::bias_act(float* y, int ldy, int rows, int N, const float* bias, int act) {
  return run.kernel(bias_act_kernel, grid_for((size_t)rows * N), TPB, y, ldy, rows, N, bias, act);
}

int Fp32Chain::resid(float* x, const float* y, int rows, int D, const float* gate, int gate_stride, int rows_per_batch) {
  return run.kernel(resid_kernel, grid_for((size_t)rows * D), TPB, x, y, rows, D, gate, gate_stride, rows_per_batch);
}

int Fp32Chain::layernorm(const float* x, float* y, int rows, int D, float eps, const float* scale, const float* shift, int mod_stride, int rpb,
                         const float* w, const float* b) {
  return run.kernel(layernorm_f32_kernel, (rows + 7) / 8, 256, x, y, rows, D, eps, scale, shift, mod_stride, rpb > 0 ? rpb : rows, w, b);
}

int Fp32Chain::attention(const float* q, const float* k, const float* v, float* out, int B, int H, int Lq, int Lk, int D, int hd, float scale) {
  const int Lk8 = up8(Lk), T = terms;
  for (int b = 0; b < B; ++b)
    for (int hh = 0; hh < H; ++hh) {
      const float* qh = q + (size_t)b * Lq * D + hh * hd;
      const float* kh = k + (size_t)b * Lk * D + hh * hd;
      const float* vh = v + (size_t)b * Lk * D + hh * hd;
      // S[Lq, Lk8]: rows Lk..Lk8-1 of the "weight" operand are zero-padded by splitting Lk rows over a zeroed tail
      CE_CHECK_CUDA(cudaMemsetAsync(Wp, 0, (size_t)Lk8 * T * up8(hd) * sizeof(bf16), run.s));
      {
        const int Kp = up8(hd);
        CE_TRY(split(qh, D, Lq, hd, Kp, Ap, 0));
        CE_TRY(split(kh, D, Lk, hd, Kp, Wp, 1));
        CE_TRY(product(Ap, Wp, Lq, Lk8, Kp, S, Lk8));
      }
      CE_TRY(run([&] { return launch_softmax_rows_f32(S, Lk8, P, Lk8, Lq, Lk, scale, run.s); }));
      {  // O = P . V : P [Lq, Lk8] (padded columns are 0), V^T as the "weight" operand [hd, Lk8] (keys >= Lk zero-filled)
        CE_TRY(split(P, Lk8, Lq, Lk8, Lk8, Ap, 0));
        CE_TRY(run.kernel(terms == 6 ? split6_transposed_kernel : split3_transposed_kernel, grid_for((size_t)hd * Lk8), TPB, vh, D, Lk, Lk8, hd, Wp));
        CE_TRY(product(Ap, Wp, Lq, hd, Lk8, out + (size_t)b * Lq * D + hh * hd, D));
      }
    }
  return CE_OK;
}

}  // namespace ce
