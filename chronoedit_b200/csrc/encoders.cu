// ce_encoder: the two once-per-edit encoders in front of the sampling loop (SURVEY.md section 8(f) row 3), on the same wgmma
// GEMM as the DiT:
//   UMT5 text encoder   -- `self.text_encoder(input_ids, mask).last_hidden_state`  (chronoedit_diffusers/pipeline_chronoedit.py:205-244;
//                          transformers UMT5EncoderModel: T5LayerNorm, per-layer relative-position bias, un-scaled QK^T, gated GELU)
//   CLIP vision encoder -- `self.image_encoder(**image, output_hidden_states=True).hidden_states[-2]`  (:246-254; transformers
//                          CLIPVisionModel: patch conv + class token + position embedding, pre-LN blocks, penultimate hidden state)
// Every Linear is one launch of the wgmma GEMM (fused bias / GELU / residual epilogues); LayerNorm / T5 RMSNorm are the row
// kernels of elementwise.cu.  Head dims are 64 (UMT5) and 80 (CLIP ViT-H), sequence lengths 512 and 257: attention is S = Q K^T
// per head (fp32 accumulator out of the GEMM), one row-softmax launch per layer over ALL heads (which applies the reference's
// bf16 rounding of the scores, the T5 position bias / key mask or the CLIP scale), and O = P V per head with V^T produced for all
// heads by one GEMM (V^T = W_v x^T).  All rounding points of the reference's bf16 eager path are kept.
#include <math.h>

#include <map>
#include <string>
#include <vector>

#include "../../include/chronoedit_b200.h"
#include "elementwise.cuh"
#include "gemm.cuh"

using namespace ce;

struct ce_encoder {
  ce_encoder_config cfg;
  std::map<std::string, const void*> w;
  std::map<std::string, int64_t> wn;
  int64_t launches = 0;
};

namespace {

__global__ void embedding_kernel(const int64_t* __restrict__ ids, const bf16* __restrict__ table, bf16* __restrict__ out, int n, int D, int64_t vocab) {
  const size_t total = (size_t)n * (D / 8);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % (D / 8));
    const size_t r = i / (D / 8);
    int64_t id = ids[r];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    reinterpret_cast<uint4*>(out + r * D)[c] = reinterpret_cast<const uint4*>(table + id * D)[c];
  }
}
// a[i] = bf16(float(a[i]) * float(b[i]))      (gated GELU: hidden_gelu * hidden_linear)
__global__ void mul_kernel(bf16* __restrict__ a, const bf16* __restrict__ b, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    a[i] = __float2bfloat16_rn(__bfloat162float(a[i]) * __bfloat162float(b[i]));
}
// x = bf16(x * sigmoid(1.702 x))     (CLIP "quick_gelu")
__global__ void quick_gelu_kernel(bf16* __restrict__ x, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float v = __bfloat162float(x[i]);
    x[i] = __float2bfloat16_rn(v / (1.0f + __expf(-1.702f * v)));
  }
}
// Row softmax over all heads of one sample.  S fp32 [H, Lq, lds] (GEMM accumulators), P bf16 [H, Lq, ldp].
//   mode 0 (T5):   s = bf16(bf16(acc) + bias[h, (j - i) + Lq - 1]), keys j >= valid are masked out (their probability is 0, as
//                  adding finfo(bf16).min does in the reference)
//   mode 1 (CLIP): s = bf16(bf16(acc) * scale)
// p = bf16(softmax_fp32(s)); columns cols..ldp-1 are written as 0.
__global__ void __launch_bounds__(256)
attn_softmax_kernel(const float* __restrict__ S, int lds, bf16* __restrict__ P, int ldp, int Lq, int cols, int mode, float scale,
                    const bf16* __restrict__ bias, int bias_ld, int valid) {
  __shared__ float red[32];
  const int row = blockIdx.x;   // h * Lq + i
  const int h = row / Lq, i = row % Lq;
  const float* s = S + (size_t)row * lds;
  bf16* p = P + (size_t)row * ldp;
  const bf16* bh = bias ? bias + (size_t)h * bias_ld + (Lq - 1 - i) : nullptr;
  const int nk = mode == 0 ? (valid < cols ? valid : cols) : cols;
  auto score = [&](int j) {
    float v = bf16_round(s[j]);
    if (mode == 0) v = bf16_round(v + __bfloat162float(bh[j]));
    else v = bf16_round(v * scale);
    return v;
  };
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < nk; j += blockDim.x) mx = fmaxf(mx, score(j));
  mx = warp_max(mx);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = warp_max((threadIdx.x & 31) < (blockDim.x >> 5) ? red[threadIdx.x & 31] : -INFINITY);
  __syncthreads();
  float sum = 0.f;
  for (int j = threadIdx.x; j < nk; j += blockDim.x) sum += expf(score(j) - mx);
  sum = warp_sum(sum);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = warp_sum((threadIdx.x & 31) < (blockDim.x >> 5) ? red[threadIdx.x & 31] : 0.f);
  const float inv = 1.0f / sum;
  for (int j = threadIdx.x; j < ldp; j += blockDim.x) p[j] = __float2bfloat16_rn(j < nk ? expf(score(j) - mx) * inv : 0.f);
}
// CLIP embeddings: x[b, 0, :] = cls + pos[0];  x[b, 1 + p, :] = bf16(patch[b, p, :] + pos[1 + p])   (bf16 adds)
__global__ void clip_embed_kernel(const bf16* __restrict__ patch, const bf16* __restrict__ cls, const bf16* __restrict__ pos, bf16* __restrict__ x,
                                  int B, int L, int D) {
  const size_t total = (size_t)B * L * D;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int d = (int)(i % D);
    size_t r = i / D;
    const int t = (int)(r % L);
    const int b = (int)(r / L);
    const float e = t == 0 ? __bfloat162float(cls[d]) : __bfloat162float(patch[((size_t)b * (L - 1) + (t - 1)) * D + d]);
    x[i] = __float2bfloat16_rn(e + __bfloat162float(pos[(size_t)t * D + d]));
  }
}
// im2row for the patch convolution: rows = patches, K = 3 * ps * ps (c, dy, dx), pixel_values [B, 3, S, S] bf16
__global__ void clip_patchify_kernel(const bf16* __restrict__ px, bf16* __restrict__ A, int B, int S, int ps, int Kp) {
  const int g = S / ps, K = 3 * ps * ps;
  const size_t total = (size_t)B * g * g * Kp;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % Kp);
    size_t r = i / Kp;
    const int gx = (int)(r % g); r /= g;
    const int gy = (int)(r % g);
    const int b = (int)(r / g);
    bf16 v = __float2bfloat16_rn(0.f);
    if (k < K) {
      const int c = k / (ps * ps), dy = (k / ps) % ps, dx = k % ps;
      v = px[(((size_t)b * 3 + c) * S + gy * ps + dy) * S + gx * ps + dx];
    }
    A[i] = v;
  }
}

struct EncWs {
  bf16 *x, *xn, *qk, *vT, *attn, *h0, *h1, *P, *patches, *pe;
  float* S;
  int64_t bytes;
};
EncWs carve(const ce_encoder_config& c, void* base, int B, int L) {
  const int64_t D = c.d_model, I = (int64_t)c.num_heads * c.d_kv, F = c.d_ff, L8 = up8(L), M = (int64_t)B * L8;
  Bump b(base);
  EncWs w;
  w.x = b.take<bf16>(M * D);
  w.xn = b.take<bf16>(M * D);
  w.qk = b.take<bf16>(M * 2 * I);
  w.vT = b.take<bf16>(I * L8);
  w.attn = b.take<bf16>(M * I);
  w.h0 = b.take<bf16>(M * F);
  w.h1 = b.take<bf16>(M * F);
  w.S = b.take<float>((int64_t)c.num_heads * L * L8);
  w.P = b.take<bf16>((int64_t)c.num_heads * L * L8);
  const int64_t Kp = up8(3 * c.patch_size * c.patch_size);
  w.patches = b.take<bf16>(c.kind == 1 ? (int64_t)B * (L - 1) * Kp : 8);
  w.pe = b.take<bf16>(c.kind == 1 ? (int64_t)B * (L - 1) * D : 8);
  w.bytes = b.bytes();
  return w;
}

struct Enc {
  ce_encoder* h;
  cudaStream_t s;
  int rc = 0;
  const bf16* W(const std::string& n, int64_t numel) {
    auto it = h->w.find(n);
    if (it == h->w.end() || h->wn[n] != numel) {
      if (!rc) rc = fail(CE_ERR_MISSING_WEIGHT, "encoder: missing or mis-sized weight " + n + " (expected " + std::to_string(numel) + " elements)");
      return nullptr;
    }
    return reinterpret_cast<const bf16*>(it->second);
  }
  int gemm(const bf16* A, int lda, const bf16* Wt, int ldw, int M, int N, int K, bf16* out, int ldo, const bf16* bias, int epi, const bf16* resid,
           int ldr, float* out_f32 = nullptr, int ld_f32 = 0, const bf16* bias_row = nullptr) {
    if (rc) return rc;
    GemmArgs g;
    g.M = M; g.N = N; g.K = K; g.out = out; g.ldo = ldo; g.out_f32 = out_f32; g.ld_f32 = ld_f32; g.bias = bias; g.bias_row = bias_row;
    g.epi = epi; g.resid = resid; g.ldr = ldr;
    int r = launch_gemm_bf16(A, lda, Wt, ldw, g, s);
    if (r && !rc) rc = r;
    if (!r) ++h->launches;
    return r;
  }
  void count() { ++h->launches; }
};

// One attention sub-layer on xn [L8 rows per sample]: q|k = xn [Wq;Wk]^T (+bias), V^T = Wv xn^T (+bias per row), per head S, softmax, P V.
// wqk [2I, D], wv [I, D]; result in ws.attn [L8, I] for sample b.
int attention_sublayer(Enc& E, const EncWs& ws, const ce_encoder_config& c, int b, int L, const bf16* wqk, const bf16* bqk, const bf16* wv,
                       const bf16* bv, int mode, float scale, const bf16* bias, int valid) {
  const int D = c.d_model, H = c.num_heads, dk = c.d_kv, I = H * dk, L8 = up8(L);
  const bf16* xn = ws.xn + (size_t)b * L8 * D;
  bf16* qk = ws.qk + (size_t)b * L8 * 2 * I;
  E.gemm(xn, D, wqk, D, L8, 2 * I, D, qk, 2 * I, bqk, EPI_BIAS, nullptr, 0);
  E.gemm(wv, D, xn, D, I, L8, D, ws.vT, L8, nullptr, EPI_BIAS, nullptr, 0, nullptr, 0, bv);   // V^T [I, L8] (+ b_v per row)
  for (int hh = 0; hh < H && !E.rc; ++hh)
    E.gemm(qk + hh * dk, 2 * I, qk + I + hh * dk, 2 * I, L, L8, dk, nullptr, 0, nullptr, EPI_BIAS, nullptr, 0, ws.S + (size_t)hh * L * L8, L8);
  if (E.rc) return E.rc;
  attn_softmax_kernel<<<H * L, 256, 0, E.s>>>(ws.S, L8, ws.P, L8, L, L, mode, scale, bias, 2 * L - 1, valid);
  CE_CHECK_CUDA(cudaGetLastError());
  E.count();
  bf16* attn = ws.attn + (size_t)b * L8 * I;
  for (int hh = 0; hh < H && !E.rc; ++hh)
    E.gemm(ws.P + (size_t)hh * L * L8, L8, ws.vT + (size_t)hh * dk * L8, L8, L, dk, L8, attn + hh * dk, I, nullptr, EPI_BIAS, nullptr, 0);
  return E.rc;
}

}  // namespace

extern "C" {

int ce_encoder_create(const ce_encoder_config* cfg, ce_encoder** out) {
  CE_REQUIRE(cfg && out, "ce_encoder_create: null argument");
  CE_REQUIRE(cfg->kind == 0 || cfg->kind == 1, "ce_encoder_create: kind 0 (UMT5 text) or 1 (CLIP vision)");
  CE_REQUIRE(cfg->d_model % 8 == 0 && cfg->d_kv % 8 == 0 && cfg->d_ff % 8 == 0 && cfg->num_heads > 0 && cfg->num_layers > 0, "ce_encoder_create: dims % 8");
  if (cfg->kind == 1) CE_REQUIRE(cfg->image_size % cfg->patch_size == 0 && cfg->patch_size > 0, "ce_encoder_create: image / patch size");
  ce_encoder* h = new ce_encoder();
  h->cfg = *cfg;
  *out = h;
  return CE_OK;
}
void ce_encoder_destroy(ce_encoder* h) { delete h; }

int ce_encoder_set_weight(ce_encoder* h, const char* name, const void* ptr, int64_t numel) {
  CE_REQUIRE(h && name && ptr, "ce_encoder_set_weight: null argument");
  CE_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "ce_encoder_set_weight: pointer must be 16-byte aligned");
  h->w[name] = ptr;
  h->wn[name] = numel;
  return CE_OK;
}

int64_t ce_encoder_workspace_bytes(const ce_encoder* h, int batch, int seq_len) {
  if (!h || batch < 1 || seq_len < 1) return -1;
  return carve(h->cfg, nullptr, batch, seq_len).bytes;
}
int64_t ce_encoder_last_launch_count(const ce_encoder* h) { return h ? h->launches : 0; }

// UMT5EncoderModel.forward(input_ids [B, L] int64, attention_mask -> valid_len[b] leading valid tokens) -> last_hidden_state [B, L, D]
int ce_umt5_encode(ce_encoder* h, const int64_t* input_ids, const int32_t* valid_len_host, void* last_hidden_state, int batch, int seq_len,
                   const void* bias_tables, void* workspace, int64_t workspace_bytes, void* stream_v) {
  CE_REQUIRE(h && input_ids && valid_len_host && last_hidden_state && workspace && bias_tables, "ce_umt5_encode: null argument");
  int rc = check_device();
  if (rc) return rc;
  const ce_encoder_config& c = h->cfg;
  CE_REQUIRE(c.kind == 0, "ce_umt5_encode: handle is not a UMT5 encoder");
  CE_REQUIRE(seq_len % 8 == 0, "ce_umt5_encode: seq_len must be a multiple of 8 (the pipeline pads to 512)");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_v);
  const int B = batch, L = seq_len, D = c.d_model, H = c.num_heads, I = H * c.d_kv, F = c.d_ff;
  EncWs ws = carve(c, workspace, B, L);
  if (ws.bytes > workspace_bytes) return fail(CE_ERR_WORKSPACE, "ce_umt5_encode: workspace too small, need " + std::to_string(ws.bytes));
  Enc E{h, s};
  h->launches = 0;
  embedding_kernel<<<grid_for((size_t)B * L * D / 8), TPB, 0, s>>>(input_ids, E.W("shared.weight", (int64_t)c.vocab_size * D), ws.x, B * L, D, c.vocab_size);
  if (E.rc) return E.rc;
  CE_CHECK_CUDA(cudaGetLastError());
  E.count();
  const bf16* bias_all = reinterpret_cast<const bf16*>(bias_tables);   // [layers, H, 2L-1] bf16: relative_attention_bias[bucket(j - i)] per layer
  for (int l = 0; l < c.num_layers && !E.rc; ++l) {
    const std::string p = "encoder.block." + std::to_string(l) + ".layer.";
    // self-attention sub-layer: x = x + o(attn(T5LayerNorm(x)))
    CE_CHECK_CUDA(cudaMemcpyAsync(ws.xn, ws.x, (size_t)B * L * D * 2, cudaMemcpyDeviceToDevice, s));
    int r = launch_rmsnorm_rope(ws.xn, D, B * L, D, c.eps, E.W(p + "0.layer_norm.weight", D), nullptr, nullptr, 0, 128, s);
    if (r) return r;
    E.count();
    const bf16* wqk = E.W(p + "0.SelfAttention.qk.weight", 2 * (int64_t)I * D);
    const bf16* wv = E.W(p + "0.SelfAttention.v.weight", (int64_t)I * D);
    const bf16* wo = E.W(p + "0.SelfAttention.o.weight", (int64_t)D * I);
    if (E.rc) return E.rc;
    for (int b = 0; b < B && !E.rc; ++b)
      attention_sublayer(E, ws, c, b, L, wqk, nullptr, wv, nullptr, 0, 1.0f, bias_all + (size_t)l * H * (2 * L - 1), valid_len_host[b]);
    E.gemm(ws.attn, I, wo, I, B * L, D, I, ws.x, D, nullptr, EPI_BIAS_RESID, ws.x, D);
    // feed-forward sub-layer: x = x + wo(gelu_new(wi_0(n)) * wi_1(n))
    CE_CHECK_CUDA(cudaMemcpyAsync(ws.xn, ws.x, (size_t)B * L * D * 2, cudaMemcpyDeviceToDevice, s));
    r = launch_rmsnorm_rope(ws.xn, D, B * L, D, c.eps, E.W(p + "1.layer_norm.weight", D), nullptr, nullptr, 0, 128, s);
    if (r) return r;
    E.count();
    E.gemm(ws.xn, D, E.W(p + "1.DenseReluDense.wi_0.weight", (int64_t)F * D), D, B * L, F, D, ws.h0, F, nullptr, EPI_BIAS_GELU_TANH, nullptr, 0);
    E.gemm(ws.xn, D, E.W(p + "1.DenseReluDense.wi_1.weight", (int64_t)F * D), D, B * L, F, D, ws.h1, F, nullptr, EPI_BIAS, nullptr, 0);
    if (E.rc) return E.rc;
    mul_kernel<<<grid_for((size_t)B * L * F), TPB, 0, s>>>(ws.h0, ws.h1, (size_t)B * L * F);
    CE_CHECK_CUDA(cudaGetLastError());
    E.count();
    E.gemm(ws.h0, F, E.W(p + "1.DenseReluDense.wo.weight", (int64_t)D * F), F, B * L, D, F, ws.x, D, nullptr, EPI_BIAS_RESID, ws.x, D);
  }
  if (E.rc) return E.rc;
  CE_CHECK_CUDA(cudaMemcpyAsync(last_hidden_state, ws.x, (size_t)B * L * D * 2, cudaMemcpyDeviceToDevice, s));
  rc = launch_rmsnorm_rope(reinterpret_cast<bf16*>(last_hidden_state), D, B * L, D, c.eps, E.W("encoder.final_layer_norm.weight", D), nullptr, nullptr, 0,
                           128, s);
  if (rc) return rc;
  E.count();
  return E.rc;
}

// CLIPVisionModel(pixel_values [B, 3, S, S], output_hidden_states=True).hidden_states[hidden_index]   (hidden_index = -2 in the pipeline:
// the output of encoder layer num_layers-1; index 0 = the embeddings after pre_layrnorm) -> out [B, 1 + (S/ps)^2, D]
int ce_clip_vision_encode(ce_encoder* h, const void* pixel_values, void* out, int batch, int layers_to_run, void* workspace,
                          int64_t workspace_bytes, void* stream_v) {
  CE_REQUIRE(h && pixel_values && out && workspace, "ce_clip_vision_encode: null argument");
  int rc = check_device();
  if (rc) return rc;
  const ce_encoder_config& c = h->cfg;
  CE_REQUIRE(c.kind == 1, "ce_clip_vision_encode: handle is not a CLIP vision encoder");
  CE_REQUIRE(layers_to_run >= 0 && layers_to_run <= c.num_layers, "ce_clip_vision_encode: layers_to_run");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_v);
  const int B = batch, g = c.image_size / c.patch_size, L = 1 + g * g, L8 = up8(L), D = c.d_model, H = c.num_heads, I = H * c.d_kv, F = c.d_ff;
  const int K = 3 * c.patch_size * c.patch_size, Kp = up8(K);
  EncWs ws = carve(c, workspace, B, L);
  if (ws.bytes > workspace_bytes) return fail(CE_ERR_WORKSPACE, "ce_clip_vision_encode: workspace too small, need " + std::to_string(ws.bytes));
  Enc E{h, s};
  h->launches = 0;
  const std::string vm = "vision_model.";
  // embeddings: patch conv as im2row + GEMM (no bias), class token, position embedding, pre_layrnorm.  Rows are laid out with L8 per
  // sample so that per-sample tensors can be handed to the GEMM with their padding rows in place (zeroed once).
  CE_CHECK_CUDA(cudaMemsetAsync(ws.x, 0, (size_t)B * L8 * D * 2, s));
  CE_CHECK_CUDA(cudaMemsetAsync(ws.xn, 0, (size_t)B * L8 * D * 2, s));
  CE_CHECK_CUDA(cudaMemsetAsync(ws.attn, 0, (size_t)B * L8 * I * 2, s));   // padding rows of every per-sample tensor stay finite
  clip_patchify_kernel<<<grid_for((size_t)B * g * g * Kp), TPB, 0, s>>>(reinterpret_cast<const bf16*>(pixel_values), ws.patches, B, c.image_size, c.patch_size, Kp);
  CE_CHECK_CUDA(cudaGetLastError());
  E.count();
  E.gemm(ws.patches, Kp, E.W(vm + "embeddings.patch_embedding.weight", (int64_t)D * Kp), Kp, B * g * g, D, Kp, ws.pe, D, nullptr, EPI_BIAS, nullptr, 0);
  if (E.rc) return E.rc;
  for (int b = 0; b < B; ++b) {
    clip_embed_kernel<<<grid_for((size_t)L * D), TPB, 0, s>>>(ws.pe + (size_t)b * (L - 1) * D, E.W(vm + "embeddings.class_embedding", D),
                                                              E.W(vm + "embeddings.position_embedding.weight", (int64_t)L * D), ws.xn + (size_t)b * L8 * D, 1, L, D);
    if (E.rc) return E.rc;
    CE_CHECK_CUDA(cudaGetLastError());
    E.count();
  }
  auto ln = [&](const bf16* src, bf16* dst, const std::string& name) -> int {   // LayerNorm(eps) with fp32 affine copies registered by the host
    const float* w = reinterpret_cast<const float*>(E.W(name + ".weight_f32", D));   // fp32 copies [D] (torch's LayerNorm computes in fp32)
    const float* bb = reinterpret_cast<const float*>(E.W(name + ".bias_f32", D));
    if (E.rc) return E.rc;
    for (int b = 0; b < B; ++b) {
      int r = launch_layernorm(src + (size_t)b * L8 * D, D, dst + (size_t)b * L8 * D, D, L, D, c.eps, nullptr, nullptr, 0, 0, w, bb, s);
      if (r) return r;
      E.count();
    }
    return CE_OK;
  };
  if ((rc = ln(ws.xn, ws.x, vm + "pre_layrnorm"))) return rc;
  const float scale = 1.0f / sqrtf((float)c.d_kv);
  for (int l = 0; l < layers_to_run && !E.rc; ++l) {
    const std::string p = vm + "encoder.layers." + std::to_string(l) + ".";
    if ((rc = ln(ws.x, ws.xn, p + "layer_norm1"))) return rc;
    const bf16* wqk = E.W(p + "self_attn.qk_proj.weight", 2 * (int64_t)I * D);
    const bf16* bqk = E.W(p + "self_attn.qk_proj.bias", 2 * (int64_t)I);
    const bf16* wv = E.W(p + "self_attn.v_proj.weight", (int64_t)I * D);
    const bf16* bv = E.W(p + "self_attn.v_proj.bias", I);
    if (E.rc) return E.rc;
    for (int b = 0; b < B && !E.rc; ++b) attention_sublayer(E, ws, c, b, L, wqk, bqk, wv, bv, 1, scale, nullptr, L);
    E.gemm(ws.attn, I, E.W(p + "self_attn.out_proj.weight", (int64_t)D * I), I, B * L8, D, I, ws.x, D, E.W(p + "self_attn.out_proj.bias", D),
           EPI_BIAS_RESID, ws.x, D);
    if ((rc = ln(ws.x, ws.xn, p + "layer_norm2"))) return rc;
    const int act_epi = c.hidden_act == 1 ? EPI_BIAS_GELU_ERF : EPI_BIAS;   // 0 quick_gelu (separate pass), 1 gelu (erf)
    E.gemm(ws.xn, D, E.W(p + "mlp.fc1.weight", (int64_t)F * D), D, B * L8, F, D, ws.h0, F, E.W(p + "mlp.fc1.bias", F), act_epi, nullptr, 0);
    if (E.rc) return E.rc;
    if (c.hidden_act == 0) {
      quick_gelu_kernel<<<grid_for((size_t)B * L8 * F), TPB, 0, s>>>(ws.h0, (size_t)B * L8 * F);
      CE_CHECK_CUDA(cudaGetLastError());
      E.count();
    }
    E.gemm(ws.h0, F, E.W(p + "mlp.fc2.weight", (int64_t)D * F), F, B * L8, D, F, ws.x, D, E.W(p + "mlp.fc2.bias", D), EPI_BIAS_RESID, ws.x, D);
  }
  if (E.rc) return E.rc;
  for (int b = 0; b < B; ++b)
    CE_CHECK_CUDA(cudaMemcpyAsync(reinterpret_cast<bf16*>(out) + (size_t)b * L * D, ws.x + (size_t)b * L8 * D, (size_t)L * D * 2, cudaMemcpyDeviceToDevice, s));
  return E.rc;
}

}  // extern "C"
