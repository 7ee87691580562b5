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
#include <vector>

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

// One Linear of the fp32 model: weight [N, K], bias [N].
struct Lin32 {
  const float *w = nullptr, *b = nullptr;
};
struct Layer32 {
  const float* table;   // scale_shift_table [6, D]
  Lin32 q, k, v, out1, q2, k2, v2, add_k, add_v, out2, ffn1, ffn2;
  const float *norm_q, *norm_k, *norm2_w, *norm2_b, *norm_q2, *norm_k2, *norm_added_k;
};
// Every fp32 parameter ce_dit_forward_fp32 reads, under its reference name.
struct Weights32 {
  Lin32 patch, time1, time2, time_proj, text1, text2, img_ff0, img_ff2, proj_out;
  const float *img_norm1_w{}, *img_norm1_b{}, *img_norm2_w{}, *img_norm2_b{}, *head_table{};
  std::vector<Layer32> layers;
};

int resolve_weights32(const WeightMap& map, const ce_dit_config& c, Weights32& w) {
  const int64_t D = (int64_t)c.num_attention_heads * c.attention_head_dim, F = c.ffn_dim, I = c.image_dim;
  WeightLookup r{map};
  auto lin = [&](const std::string& m, int64_t N, int64_t K) { return Lin32{r.f32(m + ".weight", N * K), r.f32(m + ".bias", N)}; };
  const std::string ce_ = "condition_embedder.";
  w.patch = lin("patch_embedding", D, (int64_t)c.in_channels * 4);
  w.time1 = lin(ce_ + "time_embedder.linear_1", D, c.freq_dim);
  w.time2 = lin(ce_ + "time_embedder.linear_2", D, D);
  w.time_proj = lin(ce_ + "time_proj", 6 * D, D);
  w.text1 = lin(ce_ + "text_embedder.linear_1", D, c.text_dim);
  w.text2 = lin(ce_ + "text_embedder.linear_2", D, D);
  if (I > 0) {
    w.img_norm1_w = r.f32(ce_ + "image_embedder.norm1.weight", I);
    w.img_norm1_b = r.f32(ce_ + "image_embedder.norm1.bias", I);
    w.img_ff0 = lin(ce_ + "image_embedder.ff.net.0.proj", I, I);
    w.img_ff2 = lin(ce_ + "image_embedder.ff.net.2", D, I);
    w.img_norm2_w = r.f32(ce_ + "image_embedder.norm2.weight", D);
    w.img_norm2_b = r.f32(ce_ + "image_embedder.norm2.bias", D);
  }
  for (int i = 0; i < c.num_layers; ++i) {
    const std::string p = "blocks." + std::to_string(i) + ".";
    Layer32 l{};
    l.table = r.f32(p + "scale_shift_table", 6 * D);
    l.q = lin(p + "attn1.to_q", D, D);
    l.k = lin(p + "attn1.to_k", D, D);
    l.v = lin(p + "attn1.to_v", D, D);
    l.norm_q = r.f32(p + "attn1.norm_q.weight", D);
    l.norm_k = r.f32(p + "attn1.norm_k.weight", D);
    l.out1 = lin(p + "attn1.to_out.0", D, D);
    l.norm2_w = r.f32(p + "norm2.weight", D);
    l.norm2_b = r.f32(p + "norm2.bias", D);
    l.q2 = lin(p + "attn2.to_q", D, D);
    l.norm_q2 = r.f32(p + "attn2.norm_q.weight", D);
    l.k2 = lin(p + "attn2.to_k", D, D);
    l.v2 = lin(p + "attn2.to_v", D, D);
    l.norm_k2 = r.f32(p + "attn2.norm_k.weight", D);
    if (I > 0) {
      l.add_k = lin(p + "attn2.add_k_proj", D, D);
      l.add_v = lin(p + "attn2.add_v_proj", D, D);
      l.norm_added_k = r.f32(p + "attn2.norm_added_k.weight", D);
    }
    l.out2 = lin(p + "attn2.to_out.0", D, D);
    l.ffn1 = lin(p + "ffn.net.0.proj", F, D);
    l.ffn2 = lin(p + "ffn.net.2", D, F);
    w.layers.push_back(l);
  }
  w.head_table = r.f32("scale_shift_table", 2 * D);
  w.proj_out = lin("proj_out", (int64_t)c.out_channels * 4, D);
  return r.rc;
}

// The launches of the fp32 forward.  They are not counted: ce_dit_last_launch_count reports the last bf16 forward.
struct Ctx32 {
  Ws32 ws;
  Launcher run;
  // out[M, ldo] (fp32) = act(A[M, K] (lda) . W[N, K]^T + bias)
  int linear(const float* A, int lda, int M, int K, const Lin32& w, int N, float* out, int ldo, int act) {
    const int Kp = up8(K);
    CE_TRY(run.kernel(split3_kernel, grid_for((size_t)M * Kp), TPB, A, lda, M, K, Kp, ws.Ap, 0));
    CE_TRY(run.kernel(split3_kernel, grid_for((size_t)N * Kp), TPB, w.w, K, N, K, Kp, ws.Wp, 1));
    GemmArgs g;
    g.M = M; g.N = N; g.K = 3 * Kp;
    g.out = nullptr; g.ldo = 0; g.out_f32 = out; g.ld_f32 = ldo;
    g.bias = nullptr; g.epi = EPI_BIAS;
    CE_TRY(run([&] { return launch_gemm_bf16(ws.Ap, 3 * Kp, ws.Wp, 3 * Kp, g, run.s); }));
    if (w.b || act) CE_TRY(run.kernel(bias_act_kernel, grid_for((size_t)M * N), TPB, out, ldo, M, N, w.b, act));
    return CE_OK;
  }
  int layernorm(const float* x, float* y, int rows, int D, float eps, const float* scale, const float* shift, int mod_stride, int rpb,
                const float* w, const float* b) {
    return run.kernel(layernorm_f32_kernel, (rows + 7) / 8, 256, x, y, rows, D, eps, scale, shift, mod_stride, rpb > 0 ? rpb : rows, w, b);
  }
  int rms(float* x, int ldx, int rows, int D, float eps, const float* w, const float* rc_, const float* rs_, int L, int hd) {
    return run.kernel(rmsnorm_rope_f32_kernel, (rows + 7) / 8, 256, x, ldx, rows, D, eps, w, rc_, rs_, L, hd);
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
        CE_CHECK_CUDA(cudaMemsetAsync(ws.Wp, 0, (size_t)Lk8 * 3 * up8(hd) * sizeof(bf16), run.s));
        {
          const int Kp = up8(hd);
          CE_TRY(run.kernel(split3_kernel, grid_for((size_t)Lq * Kp), TPB, qh, D, Lq, hd, Kp, ws.Ap, 0));
          CE_TRY(run.kernel(split3_kernel, grid_for((size_t)Lk * Kp), TPB, kh, D, Lk, hd, Kp, ws.Wp, 1));
          GemmArgs g;
          g.M = Lq; g.N = Lk8; g.K = 3 * Kp; g.out_f32 = ws.S; g.ld_f32 = Lk8;
          CE_TRY(run([&] { return launch_gemm_bf16(ws.Ap, 3 * Kp, ws.Wp, 3 * Kp, g, run.s); }));
        }
        CE_TRY(run([&] { return launch_softmax_rows_f32(ws.S, Lk8, ws.P, Lk8, Lq, Lk, scale, run.s); }));
        {  // O = P . V : P [Lq, Lk8] (padded columns are 0), V^T as the "weight" operand [hd, Lk8] (keys >= Lk zero-filled)
          CE_TRY(run.kernel(split3_kernel, grid_for((size_t)Lq * Lk8), TPB, ws.P, Lk8, Lq, Lk8, Lk8, ws.Ap, 0));
          CE_TRY(run.kernel(split3_transposed_kernel, grid_for((size_t)hd * Lk8), TPB, vh, D, Lk, Lk8, hd, ws.Wp));
          GemmArgs g;
          g.M = Lq; g.N = hd; g.K = 3 * Lk8; g.out_f32 = out + (size_t)b * Lq * D + hh * hd; g.ld_f32 = D;
          CE_TRY(run([&] { return launch_gemm_bf16(ws.Ap, 3 * Lk8, ws.Wp, 3 * Lk8, g, run.s); }));
        }
      }
    return CE_OK;
  }
};

}  // namespace

// handle internals (dit.cu)
const WeightMap& ce_dit_internal_weights_f32(const ce_dit* h);
int ce_dit_internal_rope(ce_dit* h, int frames, int hp, int wp, cudaStream_t s, const float** cos_out, const float** sin_out);
const ce_dit_config* ce_dit_internal_config(const ce_dit* h);
int ce_dit_internal_bp_world(const ce_dit* h);
bool ce_dit_internal_lora_set(const ce_dit* h);

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
  CE_REQUIRE(ce_dit_internal_bp_world(h) <= 1,
             "ce_dit_forward_fp32: the validation forward is not built for the batch split: switch it off (ce_dit_bp_configure with world 1)");
  CE_REQUIRE(!ce_dit_internal_lora_set(h),
             "ce_dit_forward_fp32: the validation forward is not built for run-time LoRA: clear it first (ce_dit_set_lora with n = 0)");
  const ce_dit_config& c = *ce_dit_internal_config(h);
  CE_REQUIRE(batch >= 1 && batch <= 8 && (frames == 2 || frames == c.rope_temporal_skip_len) && height % c.patch_h == 0 && width % c.patch_w == 0,
             "ce_dit_forward_fp32: geometry (same rules as ce_dit_forward)");
  CE_REQUIRE((c.image_dim > 0) == (encoder_hidden_states_image != nullptr), "ce_dit_forward_fp32: image states iff image_dim");
  Weights32 W;
  CE_TRY(resolve_weights32(ce_dit_internal_weights_f32(h), c, W));
  CE_TRY(check_device());
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_v);
  const int B = batch, hp = height / c.patch_h, wp = width / c.patch_w, L = frames * hp * wp, M = B * L;
  const int H = c.num_attention_heads, hd = c.attention_head_dim, D = H * hd, F = c.ffn_dim, Lt = text_len, Li = 257;
  const int Kp = c.in_channels * 4, No = c.out_channels * 4;
  Ctx32 X{carve32(c, workspace, B, L, Lt, Li), Launcher{s, nullptr}};
  Ws32& ws = X.ws;
  if (ws.bytes > workspace_bytes) return fail(CE_ERR_WORKSPACE, "fp32 validation workspace too small: need " + std::to_string(ws.bytes));
  CE_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "workspace must be 256-byte aligned");
  const float *rope_c, *rope_s;
  CE_TRY(ce_dit_internal_rope(h, frames, hp, wp, s, &rope_c, &rope_s));
  const float scale = 1.0f / sqrtf((float)hd);

  // patch embedding (:429-430)
  CE_TRY(X.run.kernel(patchify_f32_kernel, grid_for((size_t)M * Kp), TPB, hidden_states, ws.patches, B, c.in_channels, frames, height, width));
  CE_TRY(X.linear(ws.patches, Kp, M, Kp, W.patch, D, ws.x, D, 0));
  // condition embedder (:147-165): everything fp32, no bf16 rounding anywhere
  CE_TRY(X.run([&] { return launch_timestep_sinusoid(timestep, ws.sin_emb, B, c.freq_dim, s); }));
  CE_TRY(X.linear(ws.sin_emb, c.freq_dim, B, c.freq_dim, W.time1, D, ws.h1, D, 3));
  CE_TRY(X.linear(ws.h1, D, B, D, W.time2, D, ws.temb, D, 0));
  CE_CHECK_CUDA(cudaMemcpyAsync(ws.h1, ws.temb, (size_t)B * D * 4, cudaMemcpyDeviceToDevice, s));
  CE_TRY(X.run.kernel(bias_act_kernel, grid_for((size_t)B * D), TPB, ws.h1, D, B, D, nullptr, 3));   // act_fn(temb)
  CE_TRY(X.linear(ws.h1, D, B, D, W.time_proj, 6 * D, ws.tproj, 6 * D, 0));
  CE_TRY(X.linear(encoder_hidden_states, c.text_dim, B * Lt, c.text_dim, W.text1, D, ws.text1, D, 1));
  CE_TRY(X.linear(ws.text1, D, B * Lt, D, W.text2, D, ws.ctx_text, D, 0));
  if (c.image_dim > 0) {
    const int I = c.image_dim;
    CE_TRY(X.layernorm(encoder_hidden_states_image, ws.img0, B * Li, I, 1e-5f, nullptr, nullptr, 0, 0, W.img_norm1_w, W.img_norm1_b));
    CE_TRY(X.linear(ws.img0, I, B * Li, I, W.img_ff0, I, ws.img1, I, 2));
    CE_TRY(X.linear(ws.img1, I, B * Li, I, W.img_ff2, D, ws.img2, D, 0));
    CE_TRY(X.layernorm(ws.img2, ws.ctx_img, B * Li, D, 1e-5f, nullptr, nullptr, 0, 0, W.img_norm2_w, W.img_norm2_b));
  }

  for (int i = 0; i < c.num_layers; ++i) {
    const Layer32& l = W.layers[i];
    CE_TRY(X.run.kernel(add_table_f32_kernel, grid_for((size_t)B * 6 * D), TPB, l.table, ws.tproj, 6 * D, 1, ws.mod, B, D, 6));   // [B, 6, D]
    const float* mod = ws.mod;
    // 1. self-attention (:279-281)
    CE_TRY(X.layernorm(ws.x, ws.xn, M, D, c.eps, mod + 1 * D, mod + 0 * D, 6 * D, L, nullptr, nullptr));
    CE_TRY(X.linear(ws.xn, D, M, D, l.q, D, ws.q, D, 0));
    CE_TRY(X.linear(ws.xn, D, M, D, l.k, D, ws.k, D, 0));
    CE_TRY(X.linear(ws.xn, D, M, D, l.v, D, ws.v, D, 0));
    CE_TRY(X.rms(ws.q, D, M, D, c.eps, l.norm_q, rope_c, rope_s, L, hd));
    CE_TRY(X.rms(ws.k, D, M, D, c.eps, l.norm_k, rope_c, rope_s, L, hd));
    CE_TRY(X.attention(ws.q, ws.k, ws.v, ws.attn, B, H, L, L, D, hd, scale));
    CE_TRY(X.linear(ws.attn, D, M, D, l.out1, D, ws.xn, D, 0));
    CE_TRY(X.run.kernel(resid_kernel, grid_for((size_t)M * D), TPB, ws.x, ws.xn, M, D, mod + 2 * D, 6 * D, L));
    // 2. cross-attention (:284-286)
    CE_TRY(X.layernorm(ws.x, ws.xn, M, D, c.eps, nullptr, nullptr, 0, 0, l.norm2_w, l.norm2_b));
    CE_TRY(X.linear(ws.xn, D, M, D, l.q2, D, ws.q, D, 0));
    CE_TRY(X.rms(ws.q, D, M, D, c.eps, l.norm_q2, nullptr, nullptr, 0, hd));
    CE_TRY(X.linear(ws.ctx_text, D, B * Lt, D, l.k2, D, ws.kt, D, 0));
    CE_TRY(X.linear(ws.ctx_text, D, B * Lt, D, l.v2, D, ws.vt, D, 0));
    CE_TRY(X.rms(ws.kt, D, B * Lt, D, c.eps, l.norm_k2, nullptr, nullptr, 0, hd));
    CE_TRY(X.attention(ws.q, ws.kt, ws.vt, ws.attn, B, H, L, Lt, D, hd, scale));
    if (c.image_dim > 0) {
      CE_TRY(X.linear(ws.ctx_img, D, B * Li, D, l.add_k, D, ws.ki, D, 0));
      CE_TRY(X.linear(ws.ctx_img, D, B * Li, D, l.add_v, D, ws.vi, D, 0));
      CE_TRY(X.rms(ws.ki, D, B * Li, D, c.eps, l.norm_added_k, nullptr, nullptr, 0, hd));
      CE_TRY(X.attention(ws.q, ws.ki, ws.vi, ws.attn2, B, H, L, Li, D, hd, scale));
      CE_TRY(X.run.kernel(add_inplace_kernel, grid_for((size_t)M * D), TPB, ws.attn, ws.attn2, (size_t)M * D));
    }
    CE_TRY(X.linear(ws.attn, D, M, D, l.out2, D, ws.xn, D, 0));
    CE_TRY(X.run.kernel(resid_kernel, grid_for((size_t)M * D), TPB, ws.x, ws.xn, M, D, nullptr, 0, 1));
    // 3. feed-forward (:289-293)
    CE_TRY(X.layernorm(ws.x, ws.xn, M, D, c.eps, mod + 4 * D, mod + 3 * D, 6 * D, L, nullptr, nullptr));
    CE_TRY(X.linear(ws.xn, D, M, D, l.ffn1, F, ws.h, F, 1));
    CE_TRY(X.linear(ws.h, F, M, F, l.ffn2, D, ws.xn, D, 0));
    CE_TRY(X.run.kernel(resid_kernel, grid_for((size_t)M * D), TPB, ws.x, ws.xn, M, D, mod + 5 * D, 6 * D, L));
    if (i == 0 && block_out) CE_CHECK_CUDA(cudaMemcpyAsync(block_out, ws.x, (size_t)M * D * 4, cudaMemcpyDeviceToDevice, s));
  }
  // head (:451-467)
  CE_TRY(X.run.kernel(add_table_f32_kernel, grid_for((size_t)B * 2 * D), TPB, W.head_table, ws.temb, D, 0, ws.modf, B, D, 2));
  CE_TRY(X.layernorm(ws.x, ws.xn, M, D, c.eps, ws.modf + D, ws.modf, 2 * D, L, nullptr, nullptr));
  CE_TRY(X.linear(ws.xn, D, M, D, W.proj_out, No, ws.yout, No, 0));
  return X.run.kernel(unpatchify_f32_kernel, grid_for((size_t)B * c.out_channels * frames * height * width), TPB, ws.yout, No, sample, B,
                      c.out_channels, frames, height, width);
}

}  // extern "C"
