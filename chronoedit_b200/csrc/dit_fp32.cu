// ce_dit_forward_fp32: VALIDATION mode of the DiT forward -- fp32 inputs, fp32 weights, fp32 residual stream and fp32
// stores everywhere, so that the north_star tolerance (rtol 1e-3 / atol 1e-4) can be asserted END TO END against the
// reference's fp32 run (the bf16 path cannot meet it: the reference does not meet it against itself across precisions,
// SURVEY.md section 7 hard part 3).  Same operator order as ChronoEditTransformer3DModel.forward
// (/root/reference/chronoedit_diffusers/transformer_chronoedit.py:397-476) evaluated in fp32 like the reference's own fp32 run.
//
// Every matrix product still runs on the wgmma GEMM of gemm.cu: an fp32 operand x is split into two bf16 terms
// hi = bf16(x), lo = bf16(x - hi) (|x - hi - lo| <= 2^-17 |x|), and A.W^T is evaluated as ONE bf16 GEMM over a K axis three times
// as long -- A' = [A_hi | A_lo | A_hi], W' = [W_hi | W_hi | W_lo], i.e. A_hi.W_hi + A_lo.W_hi + A_hi.W_lo, fp32 accumulation in
// registers, fp32 store (the dropped A_lo.W_lo term is 2^-18 relative).  Attention is S = Q.K^T (same split GEMM, fp32 S in HBM),
// an fp32 row softmax, and O = P.V with P and V^T split the same way.  Everything elementwise is a plain fp32 SIMT kernel.
// This path trades speed for precision (3x the MMA work, S materialised) and exists for parity checks only.
#include <math.h>

#include <string>

#include "../../include/chronoedit_b200.h"
#include "elementwise.cuh"
#include "gemm.cuh"

using namespace ce;

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
// in place, one warp per row: x = x * rsqrt(mean(x^2) + eps) * w, then optional interleaved RoPE (cos/sin [L, hd/2])
__global__ void rmsnorm_rope_f32_kernel(float* __restrict__ x, int ldx, int rows, int D, float eps, const float* __restrict__ w,
                                        const float* __restrict__ rc, const float* __restrict__ rs, int L, int hd) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float* xr = x + (size_t)row * ldx;
  float ss = 0.f;
  for (int i = lane; i < D; i += 32) ss += xr[i] * xr[i];
  const float rstd = rsqrtf(warp_sum(ss) / D + eps);
  const int tok = rc ? row % L : 0, half = hd >> 1;
  for (int p = lane; p < D / 2; p += 32) {
    float re = xr[2 * p] * rstd * w[2 * p], im = xr[2 * p + 1] * rstd * w[2 * p + 1];
    if (rc) {
      const int pi = p % half;
      const float c = rc[(size_t)tok * half + pi], sn = rs[(size_t)tok * half + pi];
      const float a = re * c - im * sn, bb = re * sn + im * c;
      re = a;
      im = bb;
    }
    xr[2 * p] = re;
    xr[2 * p + 1] = im;
  }
}
// P[r, c] = softmax_c(S[r, c] * scale) over c < cols, 0 for cols <= c < ldp   (one block per row, fp32)
__global__ void softmax_rows_f32_kernel(const float* __restrict__ S, int lds, float* __restrict__ P, int ldp, int cols, float scale) {
  __shared__ float red[32];
  const float* s = S + (size_t)blockIdx.x * lds;
  float* p = P + (size_t)blockIdx.x * ldp;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < cols; i += blockDim.x) mx = fmaxf(mx, s[i]);
  mx = warp_max(mx);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = warp_max((threadIdx.x & 31) < (blockDim.x >> 5) ? red[threadIdx.x & 31] : -INFINITY);
  __syncthreads();
  float sum = 0.f;
  for (int i = threadIdx.x; i < cols; i += blockDim.x) sum += expf((s[i] - mx) * scale);
  sum = warp_sum(sum);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = warp_sum((threadIdx.x & 31) < (blockDim.x >> 5) ? red[threadIdx.x & 31] : 0.f);
  const float inv = 1.0f / sum;
  for (int i = threadIdx.x; i < ldp; i += blockDim.x) p[i] = i < cols ? expf((s[i] - mx) * scale) * inv : 0.f;
}
__global__ void patchify_f32_kernel(const float* __restrict__ x, float* __restrict__ patches, int B, int C, int T, int H, int W) {
  const int hp = H >> 1, wp = W >> 1, K = C * 4;
  const size_t total = (size_t)B * T * hp * wp * K;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % K);
    size_t r = i / K;
    const int j = (int)(r % wp); r /= wp;
    const int ii = (int)(r % hp); r /= hp;
    const int f = (int)(r % T);
    const int b = (int)(r / T);
    const int c = k >> 2, dh = (k >> 1) & 1, dw = k & 1;
    patches[i] = x[((((size_t)b * C + c) * T + f) * H + (2 * ii + dh)) * W + (2 * j + dw)];
  }
}
__global__ void unpatchify_f32_kernel(const float* __restrict__ y, int ldy, float* __restrict__ out, int B, int C, int T, int H, int W) {
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
// dst[b, c, d] = table[c, d] + src[b, (per_chunk ? c*n : 0) + d]
__global__ void add_table_f32_kernel(const float* __restrict__ table, const float* __restrict__ src, int src_ld, int per_chunk,
                                     float* __restrict__ dst, int B, int n, int chunks) {
  const size_t total = (size_t)B * chunks * n;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int d = (int)(i % n);
    size_t r = i / n;
    const int c = (int)(r % chunks);
    const int b = (int)(r / chunks);
    dst[i] = table[(size_t)c * n + d] + src[(size_t)b * src_ld + (per_chunk ? c * n : 0) + d];
  }
}
__global__ void add_inplace_kernel(float* __restrict__ a, const float* __restrict__ b, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) a[i] += b[i];
}

struct Ws32 {
  float *x, *xn, *q, *k, *v, *attn, *attn2, *h, *patches, *yout, *text1, *ctx_text, *img0, *img1, *img2, *ctx_img, *kt, *vt, *ki, *vi;
  float *sin_emb, *h1, *temb, *tproj, *mod, *modf, *S, *P;
  bf16 *Ap, *Wp;
  int64_t bytes;
};

Ws32 carve32(const ce_dit_config& c, void* base, int B, int L, int Lt, int Li) {
  const int64_t D = (int64_t)c.num_attention_heads * c.attention_head_dim, F = c.ffn_dim, M = (int64_t)B * L;
  const int64_t Kp = (int64_t)c.in_channels * 4, No = (int64_t)c.out_channels * 4, I = c.image_dim > 0 ? c.image_dim : 8;
  Bump b(base);
  Ws32 w;
  w.x = b.take<float>(M * D); w.xn = b.take<float>(M * D); w.q = b.take<float>(M * D); w.k = b.take<float>(M * D); w.v = b.take<float>(M * D);
  w.attn = b.take<float>(M * D); w.attn2 = b.take<float>(M * D); w.h = b.take<float>(M * F);
  w.patches = b.take<float>(M * Kp); w.yout = b.take<float>(M * No);
  w.text1 = b.take<float>((int64_t)B * Lt * D); w.ctx_text = b.take<float>((int64_t)B * Lt * D);
  w.img0 = b.take<float>((int64_t)B * Li * I); w.img1 = b.take<float>((int64_t)B * Li * I);
  w.img2 = b.take<float>((int64_t)B * Li * D); w.ctx_img = b.take<float>((int64_t)B * Li * D);
  w.kt = b.take<float>((int64_t)B * Lt * D); w.vt = b.take<float>((int64_t)B * Lt * D);
  w.ki = b.take<float>((int64_t)B * Li * D); w.vi = b.take<float>((int64_t)B * Li * D);
  w.sin_emb = b.take<float>((int64_t)B * c.freq_dim); w.h1 = b.take<float>((int64_t)B * D); w.temb = b.take<float>((int64_t)B * D);
  w.tproj = b.take<float>((int64_t)B * 6 * D); w.mod = b.take<float>((int64_t)B * 6 * D); w.modf = b.take<float>((int64_t)B * 2 * D);
  const int64_t Lmax = up8((int)std::max<int64_t>(L, std::max(Lt, Li)));
  w.S = b.take<float>((int64_t)L * Lmax); w.P = b.take<float>((int64_t)L * Lmax);
  // split operands: the largest A' is max(M*3F, L*3*Lmax), the largest W' max over weights / V^T
  const int64_t kmax = std::max<int64_t>(std::max<int64_t>(F, D), std::max<int64_t>(c.text_dim, Lmax));
  const int64_t a_elems = std::max<int64_t>(M, (int64_t)B * std::max(Lt, Li)) * 3 * up8((int)kmax);
  const int64_t w_elems = std::max<int64_t>(std::max<int64_t>(F, 6 * D), Lmax) * 3 * up8((int)kmax);
  w.Ap = b.take<bf16>(a_elems); w.Wp = b.take<bf16>(w_elems);
  w.bytes = b.bytes();
  return w;
}

}  // namespace

// handle internals (dit.cu)
const float* ce_dit_internal_weight_f32(const ce_dit* h, const std::string& name, int64_t expect_numel);
int ce_dit_internal_rope(ce_dit* h, int frames, int hp, int wp, cudaStream_t s, const float** cos_out, const float** sin_out);
const ce_dit_config* ce_dit_internal_config(const ce_dit* h);

#define RUN32(call)      \
  do {                   \
    int _rc = (call);    \
    if (_rc) return _rc; \
  } while (0)
#define KCHECK() CE_CHECK_CUDA(cudaGetLastError())

namespace {

struct Ctx32 {
  ce_dit* h;
  Ws32 ws;
  cudaStream_t s;
  int rc = 0;
  const float* W(const std::string& n, int64_t numel) {
    const float* p = ce_dit_internal_weight_f32(h, n, numel);
    if (!p && !rc) rc = fail(CE_ERR_MISSING_WEIGHT, "fp32 validation mode: missing fp32 weight " + n);
    return p;
  }
  // out[M, ldo] (fp32) = act(A[M, K] (lda) . W[N, K]^T + bias)
  int linear(const float* A, int lda, int M, int K, const std::string& wname, int N, float* out, int ldo, int act) {
    const float* Wt = W(wname + ".weight", (int64_t)N * K);
    const float* bias = W(wname + ".bias", N);
    if (rc) return rc;
    return matmul(A, lda, M, K, Wt, K, N, out, ldo, bias, act);
  }
  int matmul(const float* A, int lda, int M, int K, const float* Wt, int ldw, int N, float* out, int ldo, const float* bias, int act) {
    const int Kp = up8(K);
    split3_kernel<<<grid_for((size_t)M * Kp), TPB, 0, s>>>(A, lda, M, K, Kp, ws.Ap, 0);
    split3_kernel<<<grid_for((size_t)N * Kp), TPB, 0, s>>>(Wt, ldw, N, K, Kp, ws.Wp, 1);
    KCHECK();
    GemmArgs g;
    g.M = M; g.N = N; g.K = 3 * Kp;
    g.out = nullptr; g.ldo = 0; g.out_f32 = out; g.ld_f32 = ldo;
    g.bias = nullptr; g.epi = EPI_BIAS;
    RUN32(launch_gemm_bf16(ws.Ap, 3 * Kp, ws.Wp, 3 * Kp, g, s));
    if (bias || act) {
      bias_act_kernel<<<grid_for((size_t)M * N), TPB, 0, s>>>(out, ldo, M, N, bias, act);
      KCHECK();
    }
    return CE_OK;
  }
  int layernorm(const float* x, float* y, int rows, int D, float eps, const float* scale, const float* shift, int mod_stride, int rpb,
                const float* w, const float* b) {
    layernorm_f32_kernel<<<(rows + 7) / 8, 256, 0, s>>>(x, y, rows, D, eps, scale, shift, mod_stride, rpb > 0 ? rpb : rows, w, b);
    KCHECK();
    return CE_OK;
  }
  int rms(float* x, int ldx, int rows, int D, float eps, const float* w, const float* rc_, const float* rs_, int L, int hd) {
    rmsnorm_rope_f32_kernel<<<(rows + 7) / 8, 256, 0, s>>>(x, ldx, rows, D, eps, w, rc_, rs_, L, hd);
    KCHECK();
    return CE_OK;
  }
  // out[b, i, h*hd:(h+1)*hd] = softmax(q k^T * scale) v   for every (b, h); q [B*Lq, D], k / v [B*Lk, D]
  int attention(const float* q, const float* k, const float* v, float* out, int B, int H, int Lq, int Lk, int D, int hd, float scale) {
    const int Lk8 = up8(Lk);
    for (int b = 0; b < B; ++b)
      for (int hh = 0; hh < H; ++hh) {
        const float* qh = q + (size_t)b * Lq * D + hh * hd;
        const float* kh = k + (size_t)b * Lk * D + hh * hd;
        const float* vh = v + (size_t)b * Lk * D + hh * hd;
        // S[Lq, Lk8]: rows Lk..Lk8-1 of the "weight" operand are zero-padded by giving split3 rows = Lk8 over a zeroed tail
        CE_CHECK_CUDA(cudaMemsetAsync(ws.Wp, 0, (size_t)Lk8 * 3 * up8(hd) * sizeof(bf16), s));
        {
          const int Kp = up8(hd);
          split3_kernel<<<grid_for((size_t)Lq * Kp), TPB, 0, s>>>(qh, D, Lq, hd, Kp, ws.Ap, 0);
          split3_kernel<<<grid_for((size_t)Lk * Kp), TPB, 0, s>>>(kh, D, Lk, hd, Kp, ws.Wp, 1);
          KCHECK();
          GemmArgs g;
          g.M = Lq; g.N = Lk8; g.K = 3 * Kp; g.out_f32 = ws.S; g.ld_f32 = Lk8;
          RUN32(launch_gemm_bf16(ws.Ap, 3 * Kp, ws.Wp, 3 * Kp, g, s));
        }
        softmax_rows_f32_kernel<<<Lq, 256, 0, s>>>(ws.S, Lk8, ws.P, Lk8, Lk, scale);
        KCHECK();
        {  // O = P . V : P [Lq, Lk8] (padded columns are 0), V^T as the "weight" operand [hd, Lk8] (keys >= Lk zero-filled)
          split3_kernel<<<grid_for((size_t)Lq * Lk8), TPB, 0, s>>>(ws.P, Lk8, Lq, Lk8, Lk8, ws.Ap, 0);
          split3_transposed_kernel<<<grid_for((size_t)hd * Lk8), TPB, 0, s>>>(vh, D, Lk, Lk8, hd, ws.Wp);
          KCHECK();
          GemmArgs g;
          g.M = Lq; g.N = hd; g.K = 3 * Lk8; g.out_f32 = out + (size_t)b * Lq * D + hh * hd; g.ld_f32 = D;
          RUN32(launch_gemm_bf16(ws.Ap, 3 * Lk8, ws.Wp, 3 * Lk8, g, s));
        }
      }
    return CE_OK;
  }
};

}  // namespace

extern "C" {

int64_t ce_dit_fp32_workspace_bytes(const ce_dit* h, int batch, int frames, int height, int width, int text_len) {
  if (!h || batch < 1 || frames < 1 || height < 2 || width < 2 || text_len < 1) return -1;
  const ce_dit_config& c = *ce_dit_internal_config(h);
  const int L = frames * (height / c.patch_h) * (width / c.patch_w);
  return carve32(c, nullptr, batch, L, text_len, 257).bytes;
}

int ce_dit_forward_fp32(ce_dit* h, const float* hidden_states, const float* timestep, const float* encoder_hidden_states,
                        const float* encoder_hidden_states_image, float* sample, int batch, int frames, int height, int width, int text_len,
                        void* workspace, int64_t workspace_bytes, float* block_out, void* stream_v) {
  CE_REQUIRE(h && hidden_states && timestep && encoder_hidden_states && sample && workspace, "ce_dit_forward_fp32: null argument");
  int rc = check_device();
  if (rc) return rc;
  const ce_dit_config& c = *ce_dit_internal_config(h);
  CE_REQUIRE(batch >= 1 && batch <= 8 && (frames == 2 || frames == c.rope_temporal_skip_len) && height % c.patch_h == 0 && width % c.patch_w == 0,
             "ce_dit_forward_fp32: geometry (same rules as ce_dit_forward)");
  CE_REQUIRE((c.image_dim > 0) == (encoder_hidden_states_image != nullptr), "ce_dit_forward_fp32: image states iff image_dim");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_v);
  const int B = batch, hp = height / c.patch_h, wp = width / c.patch_w, L = frames * hp * wp, M = B * L;
  const int H = c.num_attention_heads, hd = c.attention_head_dim, D = H * hd, F = c.ffn_dim, Lt = text_len, Li = 257;
  const int Kp = c.in_channels * 4, No = c.out_channels * 4;
  Ctx32 X{h, carve32(c, workspace, B, L, Lt, Li), s};
  Ws32& ws = X.ws;
  if (ws.bytes > workspace_bytes) return fail(CE_ERR_WORKSPACE, "fp32 validation workspace too small: need " + std::to_string(ws.bytes));
  CE_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "workspace must be 256-byte aligned");
  const float *rope_c, *rope_s;
  RUN32(ce_dit_internal_rope(h, frames, hp, wp, s, &rope_c, &rope_s));
  const float scale = 1.0f / sqrtf((float)hd);
  const std::string ce_ = "condition_embedder.";

  // patch embedding (:429-430)
  patchify_f32_kernel<<<grid_for((size_t)M * Kp), TPB, 0, s>>>(hidden_states, ws.patches, B, c.in_channels, frames, height, width);
  KCHECK();
  RUN32(X.linear(ws.patches, Kp, M, Kp, "patch_embedding", D, ws.x, D, 0));
  // condition embedder (:147-165): everything fp32, no bf16 rounding anywhere
  RUN32(launch_timestep_sinusoid(timestep, ws.sin_emb, B, c.freq_dim, s));
  RUN32(X.linear(ws.sin_emb, c.freq_dim, B, c.freq_dim, ce_ + "time_embedder.linear_1", D, ws.h1, D, 3));
  RUN32(X.linear(ws.h1, D, B, D, ce_ + "time_embedder.linear_2", D, ws.temb, D, 0));
  CE_CHECK_CUDA(cudaMemcpyAsync(ws.h1, ws.temb, (size_t)B * D * 4, cudaMemcpyDeviceToDevice, s));
  bias_act_kernel<<<grid_for((size_t)B * D), TPB, 0, s>>>(ws.h1, D, B, D, nullptr, 3);   // act_fn(temb)
  KCHECK();
  RUN32(X.linear(ws.h1, D, B, D, ce_ + "time_proj", 6 * D, ws.tproj, 6 * D, 0));
  RUN32(X.linear(encoder_hidden_states, c.text_dim, B * Lt, c.text_dim, ce_ + "text_embedder.linear_1", D, ws.text1, D, 1));
  RUN32(X.linear(ws.text1, D, B * Lt, D, ce_ + "text_embedder.linear_2", D, ws.ctx_text, D, 0));
  if (c.image_dim > 0) {
    const int I = c.image_dim;
    RUN32(X.layernorm(encoder_hidden_states_image, ws.img0, B * Li, I, 1e-5f, nullptr, nullptr, 0, 0, X.W(ce_ + "image_embedder.norm1.weight", I),
                      X.W(ce_ + "image_embedder.norm1.bias", I)));
    RUN32(X.linear(ws.img0, I, B * Li, I, ce_ + "image_embedder.ff.net.0.proj", I, ws.img1, I, 2));
    RUN32(X.linear(ws.img1, I, B * Li, I, ce_ + "image_embedder.ff.net.2", D, ws.img2, D, 0));
    RUN32(X.layernorm(ws.img2, ws.ctx_img, B * Li, D, 1e-5f, nullptr, nullptr, 0, 0, X.W(ce_ + "image_embedder.norm2.weight", D),
                      X.W(ce_ + "image_embedder.norm2.bias", D)));
  }
  if (X.rc) return X.rc;

  for (int i = 0; i < c.num_layers; ++i) {
    const std::string p = "blocks." + std::to_string(i) + ".";
    const float* table = X.W(p + "scale_shift_table", 6 * (int64_t)D);
    if (X.rc) return X.rc;
    add_table_f32_kernel<<<grid_for((size_t)B * 6 * D), TPB, 0, s>>>(table, ws.tproj, 6 * D, 1, ws.mod, B, D, 6);   // [B, 6, D]
    KCHECK();
    const float* mod = ws.mod;
    // 1. self-attention (:279-281)
    RUN32(X.layernorm(ws.x, ws.xn, M, D, c.eps, mod + 1 * D, mod + 0 * D, 6 * D, L, nullptr, nullptr));
    RUN32(X.linear(ws.xn, D, M, D, p + "attn1.to_q", D, ws.q, D, 0));
    RUN32(X.linear(ws.xn, D, M, D, p + "attn1.to_k", D, ws.k, D, 0));
    RUN32(X.linear(ws.xn, D, M, D, p + "attn1.to_v", D, ws.v, D, 0));
    RUN32(X.rms(ws.q, D, M, D, c.eps, X.W(p + "attn1.norm_q.weight", D), rope_c, rope_s, L, hd));
    RUN32(X.rms(ws.k, D, M, D, c.eps, X.W(p + "attn1.norm_k.weight", D), rope_c, rope_s, L, hd));
    RUN32(X.attention(ws.q, ws.k, ws.v, ws.attn, B, H, L, L, D, hd, scale));
    RUN32(X.linear(ws.attn, D, M, D, p + "attn1.to_out.0", D, ws.xn, D, 0));
    resid_kernel<<<grid_for((size_t)M * D), TPB, 0, s>>>(ws.x, ws.xn, M, D, mod + 2 * D, 6 * D, L);
    KCHECK();
    // 2. cross-attention (:284-286)
    RUN32(X.layernorm(ws.x, ws.xn, M, D, c.eps, nullptr, nullptr, 0, 0, X.W(p + "norm2.weight", D), X.W(p + "norm2.bias", D)));
    RUN32(X.linear(ws.xn, D, M, D, p + "attn2.to_q", D, ws.q, D, 0));
    RUN32(X.rms(ws.q, D, M, D, c.eps, X.W(p + "attn2.norm_q.weight", D), nullptr, nullptr, 0, hd));
    RUN32(X.linear(ws.ctx_text, D, B * Lt, D, p + "attn2.to_k", D, ws.kt, D, 0));
    RUN32(X.linear(ws.ctx_text, D, B * Lt, D, p + "attn2.to_v", D, ws.vt, D, 0));
    RUN32(X.rms(ws.kt, D, B * Lt, D, c.eps, X.W(p + "attn2.norm_k.weight", D), nullptr, nullptr, 0, hd));
    RUN32(X.attention(ws.q, ws.kt, ws.vt, ws.attn, B, H, L, Lt, D, hd, scale));
    if (c.image_dim > 0) {
      RUN32(X.linear(ws.ctx_img, D, B * Li, D, p + "attn2.add_k_proj", D, ws.ki, D, 0));
      RUN32(X.linear(ws.ctx_img, D, B * Li, D, p + "attn2.add_v_proj", D, ws.vi, D, 0));
      RUN32(X.rms(ws.ki, D, B * Li, D, c.eps, X.W(p + "attn2.norm_added_k.weight", D), nullptr, nullptr, 0, hd));
      RUN32(X.attention(ws.q, ws.ki, ws.vi, ws.attn2, B, H, L, Li, D, hd, scale));
      add_inplace_kernel<<<grid_for((size_t)M * D), TPB, 0, s>>>(ws.attn, ws.attn2, (size_t)M * D);
      KCHECK();
    }
    RUN32(X.linear(ws.attn, D, M, D, p + "attn2.to_out.0", D, ws.xn, D, 0));
    resid_kernel<<<grid_for((size_t)M * D), TPB, 0, s>>>(ws.x, ws.xn, M, D, nullptr, 0, 1);
    KCHECK();
    // 3. feed-forward (:289-293)
    RUN32(X.layernorm(ws.x, ws.xn, M, D, c.eps, mod + 4 * D, mod + 3 * D, 6 * D, L, nullptr, nullptr));
    RUN32(X.linear(ws.xn, D, M, D, p + "ffn.net.0.proj", F, ws.h, F, 1));
    RUN32(X.linear(ws.h, F, M, F, p + "ffn.net.2", D, ws.xn, D, 0));
    resid_kernel<<<grid_for((size_t)M * D), TPB, 0, s>>>(ws.x, ws.xn, M, D, mod + 5 * D, 6 * D, L);
    KCHECK();
    if (X.rc) return X.rc;
    if (i == 0 && block_out) CE_CHECK_CUDA(cudaMemcpyAsync(block_out, ws.x, (size_t)M * D * 4, cudaMemcpyDeviceToDevice, s));
  }
  // head (:451-467)
  add_table_f32_kernel<<<grid_for((size_t)B * 2 * D), TPB, 0, s>>>(X.W("scale_shift_table", 2 * (int64_t)D), ws.temb, D, 0, ws.modf, B, D, 2);
  KCHECK();
  if (X.rc) return X.rc;
  RUN32(X.layernorm(ws.x, ws.xn, M, D, c.eps, ws.modf + D, ws.modf, 2 * D, L, nullptr, nullptr));
  RUN32(X.linear(ws.xn, D, M, D, "proj_out", No, ws.yout, No, 0));
  unpatchify_f32_kernel<<<grid_for((size_t)B * c.out_channels * frames * height * width), TPB, 0, s>>>(ws.yout, No, sample, B, c.out_channels, frames,
                                                                                                       height, width);
  KCHECK();
  return X.rc;
}

}  // extern "C"
