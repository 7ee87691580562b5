// ce_encoder: the two once-per-edit encoders in front of the sampling loop (SURVEY.md section 8(f) row 3), on the same wgmma
// GEMM as the DiT:
//   UMT5 text encoder   -- `self.text_encoder(input_ids, mask).last_hidden_state`  (chronoedit_diffusers/pipeline_chronoedit.py:205-244;
//                          transformers UMT5EncoderModel: T5LayerNorm, per-layer relative-position bias, un-scaled QK^T, gated GELU)
//   CLIP vision encoder -- `self.image_encoder(**image, output_hidden_states=True).hidden_states[-2]`  (:246-254; transformers
//                          CLIPVisionModel: patch conv + class token + position embedding, pre-LN blocks, penultimate hidden state)
// Every Linear is one launch of the wgmma GEMM (fused bias / GELU / residual epilogues); LayerNorm / T5 RMSNorm are the row
// kernels of elementwise.cu.  Head dims are 64 (UMT5) and 80 (CLIP ViT-H), sequence lengths 512 and 257: attention is
// gemm_attention (gemm.cu) per sample, whose one row-softmax launch over all heads applies the reference's bf16 rounding of the
// scores and the T5 position bias / key mask or the CLIP scale.  All rounding points of the reference's bf16 eager path are kept.
//
// ce_clip_vision_encode_fp32 is the same CLIP chain in fp32 -- fp32 pixels, weights, residual stream and output -- as the
// reference CLI loads the image encoder (scripts/run_inference_diffusers.py:333-337, torch_dtype=torch.float32).  Its products,
// attention and LayerNorms are the fp32 chain of fp32_chain.cuh (split-bf16 GEMMs, fp32 softmax), shared with the DiT's fp32 mode.
#include <math.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/chronoedit_b200.h"
#include "elementwise.cuh"
#include "fp32_chain.cuh"
#include "gemm.cuh"

using namespace ce;

struct ce_encoder {
  ce_encoder_config cfg;
  WeightMap w;
  WeightMap w32;   // fp32 CLIP parameters (ce_encoder_set_weight_fp32), under their transformers names
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

// Every weight a forward reads, resolved from the names registered with ce_encoder_set_weight.
struct Umt5Layer {
  const bf16 *ln0, *qk, *v, *o, *ln1, *wi0, *wi1, *wo;
};
struct ClipLayer {
  const float *ln1_w, *ln1_b, *ln2_w, *ln2_b;   // fp32 copies registered by the host (torch's LayerNorm computes in fp32)
  const bf16 *qk_w, *qk_b, *v_w, *v_b, *out_w, *out_b, *fc1_w, *fc1_b, *fc2_w, *fc2_b;
};
struct EncWeights {
  const bf16* embed = nullptr;          // UMT5 shared.weight [vocab, D]; CLIP patch_embedding.weight [D, Kp]
  const bf16* final_ln = nullptr;       // UMT5
  const bf16 *cls = nullptr, *pos = nullptr;
  const float *pre_ln_w = nullptr, *pre_ln_b = nullptr;   // CLIP
  std::vector<Umt5Layer> umt5;
  std::vector<ClipLayer> clip;
};

int resolve_weights(const ce_encoder* h, EncWeights& w) {
  const ce_encoder_config& c = h->cfg;
  const int64_t D = c.d_model, I = (int64_t)c.num_heads * c.d_kv, F = c.d_ff;
  WeightLookup r{h->w};
  auto b16 = [&](const std::string& n, int64_t numel) { return r.any<bf16>(n, numel); };
  auto f32 = [&](const std::string& n, int64_t numel) { return r.any<float>(n, numel); };
  if (c.kind == 0) {
    w.embed = b16("shared.weight", (int64_t)c.vocab_size * D);
    for (int l = 0; l < c.num_layers; ++l) {
      const std::string p = "encoder.block." + std::to_string(l) + ".layer.";
      w.umt5.push_back({b16(p + "0.layer_norm.weight", D), b16(p + "0.SelfAttention.qk.weight", 2 * I * D),
                        b16(p + "0.SelfAttention.v.weight", I * D), b16(p + "0.SelfAttention.o.weight", D * I),
                        b16(p + "1.layer_norm.weight", D), b16(p + "1.DenseReluDense.wi_0.weight", F * D),
                        b16(p + "1.DenseReluDense.wi_1.weight", F * D), b16(p + "1.DenseReluDense.wo.weight", D * F)});
    }
    w.final_ln = b16("encoder.final_layer_norm.weight", D);
    return r.rc;
  }
  const std::string vm = "vision_model.";
  const int64_t g = c.image_size / c.patch_size, Kp = up8(3 * c.patch_size * c.patch_size);
  w.embed = b16(vm + "embeddings.patch_embedding.weight", D * Kp);
  w.cls = b16(vm + "embeddings.class_embedding", D);
  w.pos = b16(vm + "embeddings.position_embedding.weight", (1 + g * g) * D);
  w.pre_ln_w = f32(vm + "pre_layrnorm.weight_f32", D);
  w.pre_ln_b = f32(vm + "pre_layrnorm.bias_f32", D);
  for (int l = 0; l < c.num_layers; ++l) {
    const std::string p = vm + "encoder.layers." + std::to_string(l) + ".";
    ClipLayer L;
    L.ln1_w = f32(p + "layer_norm1.weight_f32", D);
    L.ln1_b = f32(p + "layer_norm1.bias_f32", D);
    L.qk_w = b16(p + "self_attn.qk_proj.weight", 2 * I * D);
    L.qk_b = b16(p + "self_attn.qk_proj.bias", 2 * I);
    L.v_w = b16(p + "self_attn.v_proj.weight", I * D);
    L.v_b = b16(p + "self_attn.v_proj.bias", I);
    L.out_w = b16(p + "self_attn.out_proj.weight", D * I);
    L.out_b = b16(p + "self_attn.out_proj.bias", D);
    L.ln2_w = f32(p + "layer_norm2.weight_f32", D);
    L.ln2_b = f32(p + "layer_norm2.bias_f32", D);
    L.fc1_w = b16(p + "mlp.fc1.weight", F * D);
    L.fc1_b = b16(p + "mlp.fc1.bias", F);
    L.fc2_w = b16(p + "mlp.fc2.weight", D * F);
    L.fc2_b = b16(p + "mlp.fc2.bias", D);
    w.clip.push_back(L);
  }
  return r.rc;
}

// The self-attention of sample b on ws.xn [L8 rows per sample] into ws.attn [L8, I]; wqk [2I, D], wv [I, D].
GemmAttention attention_of(const EncWs& ws, const ce_encoder_config& c, int b, int L, const bf16* wqk, const bf16* bqk, const bf16* wv,
                           const bf16* bv) {
  const int D = c.d_model, I = c.num_heads * c.d_kv, L8 = up8(L);
  GemmAttention a;
  a.x = ws.xn + (size_t)b * L8 * D;
  a.wqk = wqk; a.bqk = bqk; a.wv = wv; a.bv = bv;
  a.L = L; a.D = D; a.H = c.num_heads; a.dk = c.d_kv; a.kpv = L8; a.q0 = 0; a.nq = L;
  a.qk = ws.qk + (size_t)b * L8 * 2 * I; a.vT = ws.vT; a.S = ws.S; a.P = ws.P;
  a.out = ws.attn + (size_t)b * L8 * I; a.ldo = I;
  return a;
}

// ---- fp32 CLIP ----------------------------------------------------------------------------------------------------------------
// im2row for the patch convolution in fp32: patches[(b, gy, gx), (c, dy, dx)] = px[b, c, gy*ps + dy, gx*ps + dx], K = 3 * ps * ps
__global__ void clip_patchify_f32_kernel(const float* __restrict__ px, float* __restrict__ A, int B, int S, int ps) {
  const int g = S / ps, K = 3 * ps * ps;
  const size_t total = (size_t)B * g * g * K;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % K);
    size_t r = i / K;
    const int gx = (int)(r % g); r /= g;
    const int gy = (int)(r % g);
    const int b = (int)(r / g);
    const int c = k / (ps * ps), dy = (k / ps) % ps, dx = k % ps;
    A[i] = px[(((size_t)b * 3 + c) * S + gy * ps + dy) * S + gx * ps + dx];
  }
}
// x[b, 0, :] = cls + pos[0];  x[b, 1 + p, :] = patch[b, p, :] + pos[1 + p]   (fp32; x is [B, L, D], patch [B, L-1, D])
__global__ void clip_embed_f32_kernel(const float* __restrict__ patch, const float* __restrict__ cls, const float* __restrict__ pos,
                                      float* __restrict__ x, int B, int L, int D) {
  const size_t total = (size_t)B * L * D;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int d = (int)(i % D);
    const size_t r = i / D;
    const int t = (int)(r % L);
    const int b = (int)(r / L);
    const float e = t == 0 ? cls[d] : patch[((size_t)b * (L - 1) + (t - 1)) * D + d];
    x[i] = e + pos[(size_t)t * D + d];
  }
}
// x = x * sigmoid(1.702 x)   (CLIP "quick_gelu", fp32 as torch evaluates it)
__global__ void quick_gelu_f32_kernel(float* __restrict__ x, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float v = x[i];
    x[i] = v * (1.0f / (1.0f + expf(-1.702f * v)));
  }
}

// Rows are B * L, packed (the fp32 GEMM stores any row count, so no per-sample padding).
struct ClipWs32 {
  float *x, *xn, *q, *k, *v, *attn, *y, *h, *part, *patches, *S, *P;
  bf16 *Ap, *Wp;
  int64_t bytes;
};
ClipWs32 carve_clip32(const ce_encoder_config& c, void* base, int B) {
  const int g = c.image_size / c.patch_size, L = 1 + g * g, L8 = up8(L), D = c.d_model, F = c.d_ff, hd = c.d_kv;
  const int K = 3 * c.patch_size * c.patch_size;
  const int64_t M = (int64_t)B * L, P = (int64_t)B * g * g;
  Bump b(base);
  ClipWs32 w;
  w.x = b.take<float>(M * D); w.xn = b.take<float>(M * D);
  w.q = b.take<float>(M * D); w.k = b.take<float>(M * D); w.v = b.take<float>(M * D);
  w.attn = b.take<float>(M * D); w.y = b.take<float>(M * D); w.h = b.take<float>(M * F); w.part = b.take<float>(std::max((int64_t)L * L8, M * std::max(D, F)));
  w.patches = b.take<float>(P * K);
  w.S = b.take<float>((int64_t)L * L8); w.P = b.take<float>((int64_t)L * L8);
  // the split operands of the largest product on each side: the Linears (patch, q / k / v / out, fc1, fc2), S and P.V
  const int64_t a_elems = std::max({split_elems(P, K, 6), split_elems(M, D, 6), split_elems(M, F, 6), split_elems(L, hd, 6), split_elems(L, L8, 6)});
  const int64_t w_elems = std::max({split_elems(D, K, 6), split_elems(D, D, 6), split_elems(F, D, 6), split_elems(D, F, 6), split_elems(L8, hd, 6),
                                    split_elems(hd, L8, 6)});
  w.Ap = b.take<bf16>(a_elems); w.Wp = b.take<bf16>(w_elems);
  w.bytes = b.bytes();
  return w;
}

struct ClipLayer32 {
  const float *ln1_w, *ln1_b, *ln2_w, *ln2_b;
  Lin32 q, k, v, out, fc1, fc2;
};
// Every fp32 parameter ce_clip_vision_encode_fp32 reads, under its transformers name, unfused.
struct ClipWeights32 {
  Lin32 patch;   // patch_embedding.weight [D, 3, ps, ps] read as [D, 3 * ps * ps]; no bias
  const float *cls = nullptr, *pos = nullptr, *pre_ln_w = nullptr, *pre_ln_b = nullptr;
  std::vector<ClipLayer32> layers;
};
int resolve_clip32(const ce_encoder* h, ClipWeights32& w) {
  const ce_encoder_config& c = h->cfg;
  const int64_t D = c.d_model, F = c.d_ff, g = c.image_size / c.patch_size;
  WeightLookup r{h->w32};
  auto lin = [&](const std::string& m, int64_t N, int64_t K) { return Lin32{r.f32(m + ".weight", N * K), r.f32(m + ".bias", N)}; };
  const std::string vm = "vision_model.";
  w.patch.w = r.f32(vm + "embeddings.patch_embedding.weight", D * 3 * c.patch_size * c.patch_size);
  w.cls = r.f32(vm + "embeddings.class_embedding", D);
  w.pos = r.f32(vm + "embeddings.position_embedding.weight", (1 + g * g) * D);
  w.pre_ln_w = r.f32(vm + "pre_layrnorm.weight", D);
  w.pre_ln_b = r.f32(vm + "pre_layrnorm.bias", D);
  for (int l = 0; l < c.num_layers; ++l) {
    const std::string p = vm + "encoder.layers." + std::to_string(l) + ".";
    ClipLayer32 L;
    L.ln1_w = r.f32(p + "layer_norm1.weight", D);
    L.ln1_b = r.f32(p + "layer_norm1.bias", D);
    L.q = lin(p + "self_attn.q_proj", D, D);
    L.k = lin(p + "self_attn.k_proj", D, D);
    L.v = lin(p + "self_attn.v_proj", D, D);
    L.out = lin(p + "self_attn.out_proj", D, D);
    L.ln2_w = r.f32(p + "layer_norm2.weight", D);
    L.ln2_b = r.f32(p + "layer_norm2.bias", D);
    L.fc1 = lin(p + "mlp.fc1", F, D);
    L.fc2 = lin(p + "mlp.fc2", D, F);
    w.layers.push_back(L);
  }
  return r.rc;
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
  CE_REQUIRE(h, "ce_encoder_set_weight: null handle");
  return register_weight(h->w, "ce_encoder_set_weight", name, ptr, -1, numel);
}

int64_t ce_encoder_workspace_bytes(const ce_encoder* h, int batch, int seq_len) {
  if (!h || batch < 1 || seq_len < 1) return -1;
  return carve(h->cfg, nullptr, batch, seq_len).bytes;
}
int64_t ce_encoder_last_launch_count(const ce_encoder* h) { return h ? h->launches : 0; }

int ce_encoder_set_weight_fp32(ce_encoder* h, const char* name, const float* ptr, int64_t numel) {
  CE_REQUIRE(h, "ce_encoder_set_weight_fp32: null handle");
  return register_weight(h->w32, "ce_encoder_set_weight_fp32", name, ptr, 1, numel);
}

int64_t ce_clip_vision_fp32_workspace_bytes(const ce_encoder* h, int batch) {
  if (!h || h->cfg.kind != 1 || batch < 1) return -1;
  return carve_clip32(h->cfg, nullptr, batch).bytes;
}

// UMT5EncoderModel.forward(input_ids [B, L] int64, attention_mask -> valid_len[b] leading valid tokens) -> last_hidden_state [B, L, D]
int ce_umt5_encode(ce_encoder* h, const int64_t* input_ids, const int32_t* valid_len_host, void* last_hidden_state, int batch, int seq_len,
                   const void* bias_tables, void* workspace, int64_t workspace_bytes, void* stream_v) {
  CE_REQUIRE(h && input_ids && valid_len_host && last_hidden_state && workspace && bias_tables, "ce_umt5_encode: null argument");
  const ce_encoder_config& c = h->cfg;
  CE_REQUIRE(c.kind == 0, "ce_umt5_encode: handle is not a UMT5 encoder");
  CE_REQUIRE(seq_len % 8 == 0, "ce_umt5_encode: seq_len must be a multiple of 8 (the pipeline pads to 512)");
  EncWeights W;
  CE_TRY(resolve_weights(h, W));
  CE_TRY(check_device());
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_v);
  const int B = batch, L = seq_len, D = c.d_model, H = c.num_heads, I = H * c.d_kv, F = c.d_ff;
  EncWs ws = carve(c, workspace, B, L);
  if (ws.bytes > workspace_bytes) return fail(CE_ERR_WORKSPACE, "ce_umt5_encode: workspace too small, need " + std::to_string(ws.bytes));
  Launcher run{s, &h->launches};
  h->launches = 0;
  CE_TRY(run.kernel(embedding_kernel, grid_for((size_t)B * L * D / 8), TPB, input_ids, W.embed, ws.x, B * L, D, (int64_t)c.vocab_size));
  const bf16* bias_all = reinterpret_cast<const bf16*>(bias_tables);   // [layers, H, 2L-1] bf16: relative_attention_bias[bucket(j - i)] per layer
  for (int l = 0; l < c.num_layers; ++l) {
    const Umt5Layer& lw = W.umt5[l];
    // self-attention sub-layer: x = x + o(attn(T5LayerNorm(x)))
    CE_CHECK_CUDA(cudaMemcpyAsync(ws.xn, ws.x, (size_t)B * L * D * 2, cudaMemcpyDeviceToDevice, s));
    CE_TRY(run([&] { return launch_rmsnorm_rope(ws.xn, D, B * L, D, c.eps, lw.ln0, nullptr, 1, nullptr, nullptr, 0, 128, RowPartials{}, s); }));
    for (int b = 0; b < B; ++b) {
      GemmAttention a = attention_of(ws, c, b, L, lw.qk, nullptr, lw.v, nullptr);
      a.sc.rule = SOFTMAX_T5;
      a.sc.bias = bias_all + (size_t)l * H * (2 * L - 1);
      a.sc.bias_ld = 2 * L - 1;
      a.sc.Lq = L;
      a.sc.valid = valid_len_host[b];
      CE_TRY(gemm_attention(run, a));
    }
    CE_TRY(run_gemm(run, ws.attn, I, lw.o, I, B * L, D, I, ws.x, D, nullptr, EPI_BIAS_RESID, ws.x, D));
    // feed-forward sub-layer: x = x + wo(gelu_new(wi_0(n)) * wi_1(n))
    CE_CHECK_CUDA(cudaMemcpyAsync(ws.xn, ws.x, (size_t)B * L * D * 2, cudaMemcpyDeviceToDevice, s));
    CE_TRY(run([&] { return launch_rmsnorm_rope(ws.xn, D, B * L, D, c.eps, lw.ln1, nullptr, 1, nullptr, nullptr, 0, 128, RowPartials{}, s); }));
    CE_TRY(run_gemm(run, ws.xn, D, lw.wi0, D, B * L, F, D, ws.h0, F, nullptr, EPI_BIAS_GELU_TANH));
    CE_TRY(run_gemm(run, ws.xn, D, lw.wi1, D, B * L, F, D, ws.h1, F, nullptr, EPI_BIAS));
    CE_TRY(run.kernel(mul_kernel, grid_for((size_t)B * L * F), TPB, ws.h0, ws.h1, (size_t)B * L * F));
    CE_TRY(run_gemm(run, ws.h0, F, lw.wo, F, B * L, D, F, ws.x, D, nullptr, EPI_BIAS_RESID, ws.x, D));
  }
  CE_CHECK_CUDA(cudaMemcpyAsync(last_hidden_state, ws.x, (size_t)B * L * D * 2, cudaMemcpyDeviceToDevice, s));
  return run([&] {
    return launch_rmsnorm_rope(reinterpret_cast<bf16*>(last_hidden_state), D, B * L, D, c.eps, W.final_ln, nullptr, 1, nullptr, nullptr, 0, 128, RowPartials{}, s);
  });
}

// CLIPVisionModel(pixel_values [B, 3, S, S], output_hidden_states=True).hidden_states[hidden_index]   (hidden_index = -2 in the pipeline:
// the output of encoder layer num_layers-1; index 0 = the embeddings after pre_layrnorm) -> out [B, 1 + (S/ps)^2, D]
int ce_clip_vision_encode(ce_encoder* h, const void* pixel_values, void* out, int batch, int layers_to_run, void* workspace,
                          int64_t workspace_bytes, void* stream_v) {
  CE_REQUIRE(h && pixel_values && out && workspace, "ce_clip_vision_encode: null argument");
  const ce_encoder_config& c = h->cfg;
  CE_REQUIRE(c.kind == 1, "ce_clip_vision_encode: handle is not a CLIP vision encoder");
  CE_REQUIRE(layers_to_run >= 0 && layers_to_run <= c.num_layers, "ce_clip_vision_encode: layers_to_run");
  EncWeights W;
  CE_TRY(resolve_weights(h, W));
  CE_TRY(check_device());
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_v);
  const int B = batch, g = c.image_size / c.patch_size, L = 1 + g * g, L8 = up8(L), D = c.d_model, H = c.num_heads, I = H * c.d_kv, F = c.d_ff;
  const int K = 3 * c.patch_size * c.patch_size, Kp = up8(K);
  EncWs ws = carve(c, workspace, B, L);
  if (ws.bytes > workspace_bytes) return fail(CE_ERR_WORKSPACE, "ce_clip_vision_encode: workspace too small, need " + std::to_string(ws.bytes));
  Launcher run{s, &h->launches};
  h->launches = 0;
  // embeddings: patch conv as im2row + GEMM (no bias), class token, position embedding, pre_layrnorm.  Rows are laid out with L8 per
  // sample so that per-sample tensors can be handed to the GEMM with their padding rows in place (zeroed once).
  CE_CHECK_CUDA(cudaMemsetAsync(ws.x, 0, (size_t)B * L8 * D * 2, s));
  CE_CHECK_CUDA(cudaMemsetAsync(ws.xn, 0, (size_t)B * L8 * D * 2, s));
  CE_CHECK_CUDA(cudaMemsetAsync(ws.attn, 0, (size_t)B * L8 * I * 2, s));   // padding rows of every per-sample tensor stay finite
  CE_TRY(run.kernel(clip_patchify_kernel, grid_for((size_t)B * g * g * Kp), TPB, reinterpret_cast<const bf16*>(pixel_values), ws.patches, B,
                    c.image_size, c.patch_size, Kp));
  CE_TRY(run_gemm(run, ws.patches, Kp, W.embed, Kp, B * g * g, D, Kp, ws.pe, D, nullptr, EPI_BIAS));
  for (int b = 0; b < B; ++b)
    CE_TRY(run.kernel(clip_embed_kernel, grid_for((size_t)L * D), TPB, ws.pe + (size_t)b * (L - 1) * D, W.cls, W.pos, ws.xn + (size_t)b * L8 * D, 1, L,
                      D));
  auto ln = [&](const bf16* src, bf16* dst, const float* w, const float* bb) -> int {   // LayerNorm(eps) per sample
    for (int b = 0; b < B; ++b)
      CE_TRY(run([&] { return launch_layernorm(src + (size_t)b * L8 * D, D, dst + (size_t)b * L8 * D, D, L, D, c.eps, nullptr, nullptr, 0, 0, w, bb, 0, RowPartials{}, s); }));
    return CE_OK;
  };
  CE_TRY(ln(ws.xn, ws.x, W.pre_ln_w, W.pre_ln_b));
  const float scale = 1.0f / sqrtf((float)c.d_kv);
  for (int l = 0; l < layers_to_run; ++l) {
    const ClipLayer& lw = W.clip[l];
    CE_TRY(ln(ws.x, ws.xn, lw.ln1_w, lw.ln1_b));
    for (int b = 0; b < B; ++b) {
      GemmAttention a = attention_of(ws, c, b, L, lw.qk_w, lw.qk_b, lw.v_w, lw.v_b);
      a.sc.rule = SOFTMAX_CLIP;
      a.sc.scale = scale;
      CE_TRY(gemm_attention(run, a));
    }
    CE_TRY(run_gemm(run, ws.attn, I, lw.out_w, I, B * L8, D, I, ws.x, D, lw.out_b, EPI_BIAS_RESID, ws.x, D));
    CE_TRY(ln(ws.x, ws.xn, lw.ln2_w, lw.ln2_b));
    const int act_epi = c.hidden_act == 1 ? EPI_BIAS_GELU_ERF : EPI_BIAS;   // 0 quick_gelu (separate pass), 1 gelu (erf)
    CE_TRY(run_gemm(run, ws.xn, D, lw.fc1_w, D, B * L8, F, D, ws.h0, F, lw.fc1_b, act_epi));
    if (c.hidden_act == 0) CE_TRY(run.kernel(quick_gelu_kernel, grid_for((size_t)B * L8 * F), TPB, ws.h0, (size_t)B * L8 * F));
    CE_TRY(run_gemm(run, ws.h0, F, lw.fc2_w, F, B * L8, D, F, ws.x, D, lw.fc2_b, EPI_BIAS_RESID, ws.x, D));
  }
  for (int b = 0; b < B; ++b)
    CE_CHECK_CUDA(cudaMemcpyAsync(reinterpret_cast<bf16*>(out) + (size_t)b * L * D, ws.x + (size_t)b * L8 * D, (size_t)L * D * 2, cudaMemcpyDeviceToDevice, s));
  return CE_OK;
}

// The same call in fp32, on the parameters registered with ce_encoder_set_weight_fp32: transformers' CLIPVisionModel loaded in fp32.
int ce_clip_vision_encode_fp32(ce_encoder* h, const float* pixel_values, float* out, int batch, int layers_to_run, void* workspace,
                               int64_t workspace_bytes, void* stream_v) {
  CE_REQUIRE(h && pixel_values && out && workspace, "ce_clip_vision_encode_fp32: null argument");
  const ce_encoder_config& c = h->cfg;
  CE_REQUIRE(c.kind == 1, "ce_clip_vision_encode_fp32: handle is not a CLIP vision encoder");
  CE_REQUIRE(batch >= 1, "ce_clip_vision_encode_fp32: batch >= 1");
  CE_REQUIRE(layers_to_run >= 0 && layers_to_run <= c.num_layers, "ce_clip_vision_encode_fp32: layers_to_run");
  CE_REQUIRE(!h->w32.empty(), "ce_clip_vision_encode_fp32: the handle has no fp32 weights (register them with ce_encoder_set_weight_fp32)");
  ClipWeights32 W;
  CE_TRY(resolve_clip32(h, W));
  const ClipWs32 ws = carve_clip32(c, workspace, batch);
  if (ws.bytes > workspace_bytes)
    return fail(CE_ERR_WORKSPACE, "ce_clip_vision_encode_fp32: workspace too small, need " + std::to_string(ws.bytes));
  CE_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "ce_clip_vision_encode_fp32: workspace must be 256-byte aligned");
  CE_TRY(check_device());
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_v);
  const int B = batch, g = c.image_size / c.patch_size, L = 1 + g * g, M = B * L, D = c.d_model, H = c.num_heads, hd = c.d_kv, F = c.d_ff;
  const int K = 3 * c.patch_size * c.patch_size;
  Fp32Chain X{Launcher{s, &h->launches}, ws.Ap, ws.Wp, ws.S, ws.P, 6, ws.part};
  h->launches = 0;
  // embeddings: patch conv as im2row + GEMM (no bias), class token, position embedding, pre_layrnorm
  CE_TRY(X.run.kernel(clip_patchify_f32_kernel, grid_for((size_t)B * g * g * K), TPB, pixel_values, ws.patches, B, c.image_size, c.patch_size));
  CE_TRY(X.linear(ws.patches, K, B * g * g, K, W.patch, D, ws.y, D, 0));
  CE_TRY(X.run.kernel(clip_embed_f32_kernel, grid_for((size_t)M * D), TPB, ws.y, W.cls, W.pos, ws.xn, B, L, D));
  CE_TRY(X.layernorm(ws.xn, ws.x, M, D, c.eps, nullptr, nullptr, 0, 0, W.pre_ln_w, W.pre_ln_b));
  const float scale = 1.0f / sqrtf((float)hd);
  for (int l = 0; l < layers_to_run; ++l) {
    const ClipLayer32& lw = W.layers[l];
    // x = x + out_proj(attn(LayerNorm1(x)))
    CE_TRY(X.layernorm(ws.x, ws.xn, M, D, c.eps, nullptr, nullptr, 0, 0, lw.ln1_w, lw.ln1_b));
    CE_TRY(X.linear(ws.xn, D, M, D, lw.q, D, ws.q, D, 0));
    CE_TRY(X.linear(ws.xn, D, M, D, lw.k, D, ws.k, D, 0));
    CE_TRY(X.linear(ws.xn, D, M, D, lw.v, D, ws.v, D, 0));
    CE_TRY(X.attention(ws.q, ws.k, ws.v, ws.attn, B, H, L, L, D, hd, scale));
    CE_TRY(X.linear(ws.attn, D, M, D, lw.out, D, ws.y, D, 0));
    CE_TRY(X.resid(ws.x, ws.y, M, D, nullptr, 0, 1));
    // x = x + fc2(act(fc1(LayerNorm2(x))))
    CE_TRY(X.layernorm(ws.x, ws.xn, M, D, c.eps, nullptr, nullptr, 0, 0, lw.ln2_w, lw.ln2_b));
    CE_TRY(X.linear(ws.xn, D, M, D, lw.fc1, F, ws.h, F, c.hidden_act == 1 ? 2 : 0));   // 1 gelu (erf); 0 quick_gelu, a pass of its own
    if (c.hidden_act == 0) CE_TRY(X.run.kernel(quick_gelu_f32_kernel, grid_for((size_t)M * F), TPB, ws.h, (size_t)M * F));
    CE_TRY(X.linear(ws.h, F, M, F, lw.fc2, D, ws.y, D, 0));
    CE_TRY(X.resid(ws.x, ws.y, M, D, nullptr, 0, 1));
  }
  CE_CHECK_CUDA(cudaMemcpyAsync(out, ws.x, (size_t)M * D * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return CE_OK;
}

// Test aid: one gemm_attention as the VAE mid-block, UMT5 or CLIP runs it, on caller-owned buffers.
int ce_gemm_attention_bf16(const ce_gemm_attention_args* args, void* stream) {
  CE_TRY(check_device());
  CE_REQUIRE(args != nullptr, "ce_gemm_attention_bf16: null args");
  const ce_gemm_attention_args& g = *args;
  CE_REQUIRE(g.x && g.wqk && g.wv && g.qk && g.vT && g.S && g.P && g.out, "ce_gemm_attention_bf16: null buffer");
  CE_REQUIRE(g.L > 0 && g.H > 0 && g.D > 0 && g.dk > 0 && g.D % 8 == 0 && g.dk % 8 == 0, "ce_gemm_attention_bf16: L, H > 0; D, dk % 8");
  CE_REQUIRE(g.kpv >= g.L && g.kpv <= up8(g.L) && g.ldo >= g.H * g.dk, "ce_gemm_attention_bf16: kpv in [L, up8(L)], ldo >= H * dk");
  CE_REQUIRE(g.rule >= SOFTMAX_SCALED && g.rule <= SOFTMAX_CLIP, "ce_gemm_attention_bf16: rule 0, 1 or 2");
  if (g.rule == SOFTMAX_T5)
    CE_REQUIRE(g.bias && g.bias_ld >= 2 * g.L - 1 && g.valid >= 1, "ce_gemm_attention_bf16: T5 needs bias, bias_ld >= 2L - 1, valid >= 1");
  GemmAttention a;
  a.x = reinterpret_cast<const bf16*>(g.x);
  a.wqk = reinterpret_cast<const bf16*>(g.wqk); a.bqk = reinterpret_cast<const bf16*>(g.bqk);
  a.wv = reinterpret_cast<const bf16*>(g.wv); a.bv = reinterpret_cast<const bf16*>(g.bv);
  a.L = g.L; a.D = g.D; a.H = g.H; a.dk = g.dk; a.kpv = g.kpv; a.q0 = 0; a.nq = g.L;
  a.sc.rule = static_cast<SoftmaxRule>(g.rule);
  a.sc.scale = g.scale;
  a.sc.bias = reinterpret_cast<const bf16*>(g.bias); a.sc.bias_ld = g.bias_ld; a.sc.Lq = g.L; a.sc.valid = g.valid;
  a.qk = reinterpret_cast<bf16*>(g.qk); a.vT = reinterpret_cast<bf16*>(g.vT); a.S = g.S; a.P = reinterpret_cast<bf16*>(g.P);
  a.out = reinterpret_cast<bf16*>(g.out); a.ldo = g.ldo;
  Launcher run{reinterpret_cast<cudaStream_t>(stream), nullptr};
  return gemm_attention(run, a);
}

}  // extern "C"
