// ce_dit: the ChronoEdit DiT per-step forward as a chain of hand-written sm_90a kernels behind the C ABI.
//
// Mirrors ChronoEditTransformer3DModel.forward (/root/reference/chronoedit_diffusers/transformer_chronoedit.py:397-476)
// with every rounding point of the reference's bf16 path kept (SURVEY.md section 8a).  Per block
// (ChronoEditTransformerBlock.forward, :267-295) the launches are:
//   LN+modulate -> QKV GEMM (one launch, N=3D) -> RMSNorm+RoPE(q|k) -> attention -> out-proj GEMM with gate*y+x epilogue
//   -> LN(affine) -> q GEMM -> RMSNorm(q) -> [text k|v GEMM, RMSNorm(k)] [image k|v GEMM, RMSNorm(k)] -> attention(text +
//   image, one launch) -> out-proj GEMM with y+x epilogue -> LN+modulate -> FFN-1 GEMM with bias+GELU epilogue -> FFN-2 GEMM
//   with gate*y+x epilogue.
// When D % 256 == 0 the GEMM before each LN / RMSNorm also writes that norm's row statistics; other widths take row kernels
// that reduce over the row themselves.  RMSNorm+RoPE(q|k) is one launch either way.
// With FP8 attention on (ce_dit_set_attention_fp8) the self-attention becomes quantize(q|k) -> quantize(v) -> attention_fp8.
#include <math.h>

#include <algorithm>
#include <atomic>
#include <map>
#include <string>
#include <vector>

#include "../../include/chronoedit_b200.h"
#include "attention.cuh"
#include "elementwise.cuh"
#include "gemm.cuh"
#include "seqpar.cuh"

namespace ce {
const std::string& last_error();
// One block GEMM's run-time LoRA entry (ce_dit_set_lora): a_cat [rank, K] and the pre-scaled b_cat [N, rank], bf16 device memory
struct LoraGemm {
  const void* a_cat = nullptr;
  const void* b_cat = nullptr;
  int rank = 0;
};
}

using namespace ce;

struct ce_dit {
  ce_dit_config cfg;
  WeightMap w;     // dtype 2 (e4m3) for FP8 mode's block weights
  WeightMap w32;   // fp32 validation mode: every parameter in fp32 under its reference name
  // RoPE tables, cached per latent geometry
  int rope_f = 0, rope_h = 0, rope_w = 0, rope_dev = -1;
  float* rope_cos = nullptr;
  float* rope_sin = nullptr;
  int64_t launches = 0;
  // parity aid: output of selected blocks copied out (ce_dit_set_capture)
  std::vector<std::pair<int, void*>> capture;
  // sequence parallelism (ce_dit_sp_configure): world == 1 means off
  ce::SeqPar sp;
  // batch split (ce_dit_bp_configure): rank r computes samples [r B / world, (r + 1) B / world) of each call; world == 1 means off
  ce::SeqPar bp;
  // call-pair group (ce_dit_cp_configure): rank 0 computes the prompt call of a CFG pair, rank 1 the negative-prompt call, and
  // ce_dit_cp_exchange swaps the two samples; world == 1 means off.  Exclusive with `bp`.
  ce::SeqPar cp;
  // optional per-category device timing (CUDA events on the launch stream around every kernel)
  bool profiling = false;
  std::vector<cudaEvent_t> ev;       // pairs (begin, end)
  std::vector<int> ev_cat;
  std::vector<double> ev_work;       // algorithmic flops (cat 0,1) or bytes (cat 2) of the launch
  size_t ev_used = 0;
  // FP8 mode: the current forward's workspace slices for a GEMM's quantized A operand and its row scales
  uint8_t* fp8_q = nullptr;
  float* fp8_scale = nullptr;
  // FP8 self-attention (ce_dit_set_attention_fp8): independent of the weights' dtype
  bool attn_fp8 = false;
  // TeaCache record mode (ce_dit_set_residual_record): every forward leaves x_after_blocks - x_before_blocks here
  void* resid_rec = nullptr;
  int64_t resid_rec_bytes = 0;
  // run-time LoRA (ce_dit_set_lora): [num_layers * CE_LORA_TARGETS] entries, empty when off; lora_rmax = their largest rank
  std::vector<ce::LoraGemm> lora;
  int lora_rmax = 0;
  // the current forward's workspace slices for one GEMM's down-projection [Mx, lora_rmax] and low-rank term [Mx, max(3D, F)]
  bf16* lora_mid = nullptr;
  bf16* lora_term = nullptr;
};

enum { CAT_GEMM = 0, CAT_ATTN = 1, CAT_ROWS = 2, CAT_OTHER = 3, NUM_CATS = 4 };
// ce_dit_set_lora's targets (include/chronoedit_b200.h): the GEMMs of LayerWeights in its order
enum { LORA_QKV = 0, LORA_OUT1, LORA_Q2, LORA_KV, LORA_ADD_KV, LORA_OUT2, LORA_FFN1, LORA_FFN2 };
static_assert(LORA_FFN2 + 1 == CE_LORA_TARGETS, "one LoRA target per block GEMM");

namespace {

int D_of(const ce_dit_config& c) { return c.num_attention_heads * c.attention_head_dim; }

struct Workspace {
  bf16 *x, *xn, *qkv, *attn, *hbuf, *patches, *yout;
  bf16 *text1, *ctx_text, *img0, *img1, *img2, *ctx_img, *kv_text, *kv_img;
  bf16 *temb_bf16, *tproj;
  float *sin_emb, *h1, *temb_f32, *mod, *modf;
  float2 *stats_x, *stats_qkv, *stats_q2;   // epilogue row statistics (GemmArgs::stats_out): [M, D/256], [M, 3D/256], [M, D/256]
  uint8_t* fp8_q;     // FP8 mode only: [M, max(D, F)] e4m3, the A operand of one block GEMM at a time
  float* fp8_scale;   //                [M] its row scales
  uint8_t* qk8;       // FP8 attention only: [M, 2D] e4m3 q | k of the self-attention
  float* qk_scale;    //                     [M, 2H] their (token, head) scales
  uint8_t* vt8;       //                     [B, H, 128, Lpad] e4m3 V^T
  float* v_scale;     //                     [B, D] its (sample, channel) scales
  bf16* lora_mid;     // run-time LoRA only: [Mx, R_max] x A_cat^T of one GEMM (Mx = max(M, B Lt, B Li))
  bf16* lora_term;    //                     [Mx, max(3D, F)] its low-rank term
  int64_t bytes;
};

// Sequence parallelism (ce_dit_sp_configure): the tokens of one edit are split over the ranks, and the only exchange is around the
// self-attention (heads <-> tokens, "Ulysses" layout, reference: chronoedit_diffsynth/wan_video_new_chronoedit.py:330-355,
// 1448-1498).  The RMSNorm+RoPE kernel scatters q | k by head, a copy scatters v, the attention epilogue scatters the output rows back
// to the ranks that own the tokens, and a copy all-gathers the head output.  Byte offsets inside a rank's peer region:
struct SpLayout {
  int64_t q, k, v;      // gathered q / k / v of the heads this rank owns: [B, L, D / world] bf16 each
  int64_t attn;         // attention output of the tokens this rank owns: [B * L / world, D] bf16
  int64_t yout;         // full head output [B * L, out_channels * 4] bf16 (every rank gets all of it)
  int64_t flags;        // uint32 [8 * 32]
  int64_t bytes;
};

SpLayout sp_layout(int64_t B, int64_t L, int64_t D, int64_t No, int world) {
  auto al = [](int64_t v) { return (v + 1023) & ~int64_t(1023); };
  SpLayout l;
  const int64_t g = al(B * L * (D / world) * 2);
  l.q = 0;
  l.k = g;
  l.v = 2 * g;
  l.attn = 3 * g;
  l.yout = l.attn + al(B * (L / world) * D * 2);
  l.flags = l.yout + al(B * L * No * 2);
  l.bytes = l.flags + 1024;
  return l;
}

// Batch split (ce_dit_bp_configure) and call pair (ce_dit_cp_configure): a rank's peer region is the flags block (uint32 [8 * 32],
// first), then two sample slots, each [batch, out_channels, frames, height, width] bf16 rounded up to 1024 bytes (the full batch of a
// split call, or one whole call of a pair).  The slot size follows from the region size, so a region sized for one geometry serves
// every call whose full sample fits.
constexpr int64_t kSlotFlagsBytes = 1024;
int64_t slot_bytes(int64_t region_bytes) { return std::max<int64_t>(0, (region_bytes - kSlotFlagsBytes) / 2) & ~int64_t(1023); }

// Keys of the FP8 attention's V^T rows: L rounded up to the 32-key groups of its layout.
int vt_keys(int L) { return (L + 31) / 32 * 32; }

Workspace carve(const ce_dit_config& c, void* base, int B, int L, int Lt, int Li, bool fp8, bool attn_fp8, int lora_rmax = 0) {
  const int64_t D = D_of(c), F = c.ffn_dim, M = (int64_t)B * L;
  const int64_t Kp = (int64_t)c.in_channels * c.patch_t * c.patch_h * c.patch_w;
  const int64_t No = (int64_t)c.out_channels * c.patch_t * c.patch_h * c.patch_w;
  Bump b(base);
  Workspace w;
  w.x = b.take<bf16>(M * D);
  w.xn = b.take<bf16>(M * D);
  w.qkv = b.take<bf16>(M * 3 * D);
  w.attn = b.take<bf16>(M * D);
  w.hbuf = b.take<bf16>(M * F);
  w.patches = b.take<bf16>(M * Kp);
  w.yout = b.take<bf16>(M * No);
  w.text1 = b.take<bf16>((int64_t)B * Lt * D);
  w.ctx_text = b.take<bf16>((int64_t)B * Lt * D);
  const int64_t I = c.image_dim > 0 ? c.image_dim : 8;
  w.img0 = b.take<bf16>((int64_t)B * Li * I);
  w.img1 = b.take<bf16>((int64_t)B * Li * I);
  w.img2 = b.take<bf16>((int64_t)B * Li * D);
  w.ctx_img = b.take<bf16>((int64_t)B * Li * D);
  w.kv_text = b.take<bf16>((int64_t)B * Lt * 2 * D);
  w.kv_img = b.take<bf16>((int64_t)B * Li * 2 * D);
  w.temb_bf16 = b.take<bf16>((int64_t)B * D);
  w.tproj = b.take<bf16>((int64_t)B * 6 * D);
  w.sin_emb = b.take<float>((int64_t)B * c.freq_dim);
  w.h1 = b.take<float>((int64_t)B * D);
  w.temb_f32 = b.take<float>((int64_t)B * D);
  w.mod = b.take<float>((int64_t)c.num_layers * B * 6 * D);
  w.modf = b.take<float>((int64_t)B * 2 * D);
  const int64_t td = (D + 255) / 256;
  w.stats_x = b.take<float2>(M * td);
  w.stats_qkv = b.take<float2>(M * 3 * td);
  w.stats_q2 = b.take<float2>(M * td);
  w.fp8_q = fp8 ? b.take<uint8_t>(M * (D > F ? D : F)) : nullptr;
  w.fp8_scale = fp8 ? b.take<float>(M) : nullptr;
  const int64_t H = c.num_attention_heads;
  w.qk8 = attn_fp8 ? b.take<uint8_t>(M * 2 * D) : nullptr;
  w.qk_scale = attn_fp8 ? b.take<float>(M * 2 * H) : nullptr;
  w.vt8 = attn_fp8 ? b.take<uint8_t>((int64_t)B * D * vt_keys(L)) : nullptr;
  w.v_scale = attn_fp8 ? b.take<float>((int64_t)B * D) : nullptr;
  const int64_t Mx = std::max<int64_t>(M, (int64_t)B * std::max(Lt, Li));
  w.lora_mid = lora_rmax ? b.take<bf16>(Mx * lora_rmax) : nullptr;
  w.lora_term = lora_rmax ? b.take<bf16>(Mx * std::max<int64_t>(3 * D, F)) : nullptr;
  w.bytes = b.bytes();
  return w;
}

// The device staging buffer of ce_dit_forward_host_ex: the inputs, then the sample (left there for the caller at sample_offset).
struct Staging {
  int64_t n_x, n_t, n_i, n_o;   // elements of hidden_states, encoder_hidden_states, encoder_hidden_states_image, sample
  bf16 *x, *text, *image, *sample;
  float* timestep;
  int64_t sample_offset, bytes;
};

Staging carve_staging(const ce_dit_config& c, void* base, int batch, int frames, int height, int width, int text_len) {
  Staging st;
  st.n_x = (int64_t)batch * c.in_channels * frames * height * width;
  st.n_t = (int64_t)batch * text_len * c.text_dim;
  st.n_i = (int64_t)batch * 257 * c.image_dim;
  st.n_o = (int64_t)batch * c.out_channels * frames * height * width;
  Bump b(base);
  st.x = b.take<bf16>(st.n_x);
  st.timestep = b.take<float>(batch);
  st.text = b.take<bf16>(st.n_t);
  st.image = b.take<bf16>(st.n_i > 0 ? st.n_i : 8);
  st.sample_offset = b.bytes();
  st.sample = b.take<bf16>(st.n_o);
  st.bytes = b.bytes();
  return st;
}

// One GEMM weight [N, K] of the forward with its bias [N]: bf16, or e4m3 with fp32 per-output-channel scales [N] (FP8 mode).
struct Linear {
  const void* weight = nullptr;
  int dtype = 0;   // 0 bf16, 2 e4m3
  const bf16* bias = nullptr;
  const float* weight_scale = nullptr;
};

struct LayerWeights {
  Linear qkv, out1, q2, kv, add_kv, out2, ffn1, ffn2;   // attn1.to_qkv, attn1.to_out.0, attn2.to_q, attn2.to_kv, attn2.add_kv_proj,
                                                        // attn2.to_out.0, ffn.net.0.proj, ffn.net.2
  const bf16 *norm_q1{}, *norm_k1{}, *norm_q2{}, *norm_k2{}, *norm_added_k{};
  const float *norm2_w{}, *norm2_b{};
};

// Every parameter the forward reads, resolved from the names registered with ce_dit_set_weight.
struct Weights {
  bool fp8 = false;   // the six block GEMM weights of every layer are e4m3: chosen by layer 0's attn1.to_qkv.weight
  Linear patch, text1, text2, img_ff0, img_ff2, proj_out;
  const float *time1_w{}, *time1_b{}, *time2_w{}, *time2_b{};
  const bf16 *time_proj_w{}, *time_proj_b{};
  const float *img_norm1_w{}, *img_norm1_b{}, *img_norm2_w{}, *img_norm2_b{};
  const float *block_table{}, *head_table{};   // blocks.scale_shift_table [layers, 6, D], scale_shift_table [2, D]
  std::vector<LayerWeights> layers;
};

// module `m` of shape [N, K]: "<m>.weight", for e4m3 "<m>.weight_scale", then "<m>.bias"
Linear lookup_linear(WeightLookup& r, const std::string& m, int64_t N, int64_t K, bool e4m3 = false) {
  Linear l;
  l.dtype = e4m3 ? 2 : 0;
  l.weight = r.get(m + ".weight", l.dtype, N * K);
  if (e4m3) l.weight_scale = r.f32(m + ".weight_scale", N);
  l.bias = r.b16(m + ".bias", N);
  return l;
}

int resolve_weights(const ce_dit* h, Weights& w) {
  const ce_dit_config& c = h->cfg;
  const int64_t D = D_of(c), F = c.ffn_dim;
  const int64_t Kp = (int64_t)c.in_channels * c.patch_t * c.patch_h * c.patch_w;
  const int64_t No = (int64_t)c.out_channels * c.patch_t * c.patch_h * c.patch_w;
  auto qkv0 = h->w.find("blocks.0.attn1.to_qkv.weight");
  w.fp8 = qkv0 != h->w.end() && qkv0->second.dtype == 2;
  WeightLookup r{h->w};
  w.patch = lookup_linear(r, "patch_embedding", D, Kp);
  const std::string ce_ = "condition_embedder.";
  w.time1_w = r.f32(ce_ + "time_embedder.linear_1.weight", D * c.freq_dim);
  w.time1_b = r.f32(ce_ + "time_embedder.linear_1.bias", D);
  w.time2_w = r.f32(ce_ + "time_embedder.linear_2.weight", D * D);
  w.time2_b = r.f32(ce_ + "time_embedder.linear_2.bias", D);
  w.time_proj_w = r.b16(ce_ + "time_proj.weight", 6 * D * D);
  w.time_proj_b = r.b16(ce_ + "time_proj.bias", 6 * D);
  w.text1 = lookup_linear(r, ce_ + "text_embedder.linear_1", D, c.text_dim);
  w.text2 = lookup_linear(r, ce_ + "text_embedder.linear_2", D, D);
  if (c.image_dim > 0) {
    const int64_t I = c.image_dim;
    w.img_norm1_w = r.f32(ce_ + "image_embedder.norm1.weight", I);
    w.img_norm1_b = r.f32(ce_ + "image_embedder.norm1.bias", I);
    w.img_ff0 = lookup_linear(r, ce_ + "image_embedder.ff.net.0.proj", I, I);
    w.img_ff2 = lookup_linear(r, ce_ + "image_embedder.ff.net.2", D, I);
    w.img_norm2_w = r.f32(ce_ + "image_embedder.norm2.weight", D);
    w.img_norm2_b = r.f32(ce_ + "image_embedder.norm2.bias", D);
  }
  w.block_table = r.f32("blocks.scale_shift_table", (int64_t)c.num_layers * 6 * D);
  w.layers.resize(c.num_layers);
  for (int i = 0; i < c.num_layers; ++i) {
    const std::string p = "blocks." + std::to_string(i) + ".";
    LayerWeights& l = w.layers[i];
    l.qkv = lookup_linear(r, p + "attn1.to_qkv", 3 * D, D, w.fp8);
    l.norm_q1 = r.b16(p + "attn1.norm_q.weight", D);
    l.norm_k1 = r.b16(p + "attn1.norm_k.weight", D);
    l.out1 = lookup_linear(r, p + "attn1.to_out.0", D, D, w.fp8);
    l.norm2_w = r.f32(p + "norm2.weight", D);
    l.norm2_b = r.f32(p + "norm2.bias", D);
    l.q2 = lookup_linear(r, p + "attn2.to_q", D, D, w.fp8);
    l.norm_q2 = r.b16(p + "attn2.norm_q.weight", D);
    l.norm_k2 = r.b16(p + "attn2.norm_k.weight", D);
    l.kv = lookup_linear(r, p + "attn2.to_kv", 2 * D, D);
    if (c.image_dim > 0) {
      l.add_kv = lookup_linear(r, p + "attn2.add_kv_proj", 2 * D, c.added_kv_proj_dim);
      l.norm_added_k = r.b16(p + "attn2.norm_added_k.weight", D);
    }
    l.out2 = lookup_linear(r, p + "attn2.to_out.0", D, D, w.fp8);
    l.ffn1 = lookup_linear(r, p + "ffn.net.0.proj", F, D, w.fp8);
    l.ffn2 = lookup_linear(r, p + "ffn.net.2", D, F, w.fp8);
  }
  w.head_table = r.f32("scale_shift_table", 2 * D);
  w.proj_out = lookup_linear(r, "proj_out", No, D);
  return r.rc;
}

int validate_geometry(const ce_dit* h, int batch, int frames, int height, int width, int text_len) {
  const ce_dit_config& c = h->cfg;
  CE_REQUIRE(batch >= 1 && batch <= 8, "dit: batch must be 1..8");
  CE_REQUIRE(frames == 2 || frames == c.rope_temporal_skip_len,
             "dit: num_frames must be 2 or rope_temporal_skip_len (transformer_chronoedit.py:205)");
  CE_REQUIRE(height > 0 && width > 0 && height % c.patch_h == 0 && width % c.patch_w == 0, "dit: latent H/W vs patch size");
  CE_REQUIRE(text_len > 0, "dit: text_len");
  CE_REQUIRE(height / c.patch_h <= c.rope_max_seq_len && width / c.patch_w <= c.rope_max_seq_len, "dit: rope_max_seq_len");
  return CE_OK;
}

// ChronoEditRotaryPosEmbed (transformer_chronoedit.py:168-213): fp64 angles -> fp32 cos/sin [L, hd/2].
int rope_table_host(int hd, int frames, int hp, int wp, int max_seq_len, int skip_len, double theta, std::vector<float>& cs,
                    std::vector<float>& sn) {
  CE_REQUIRE(frames == 2 || frames == skip_len, "rope: num_frames must be 2 or temporal_skip_len");
  CE_REQUIRE(hp <= max_seq_len && wp <= max_seq_len && skip_len <= max_seq_len, "rope: positions exceed max_seq_len");
  const int h_dim = 2 * (hd / 6), w_dim = h_dim, t_dim = hd - h_dim - w_dim;
  const int nt = t_dim / 2, nh = h_dim / 2, nw = w_dim / 2, half = hd / 2;
  const int64_t L = (int64_t)frames * hp * wp;
  cs.resize(L * half);
  sn.resize(L * half);
  auto inv_freq = [&](int i, int dim) { return 1.0 / pow(theta, (double)(2 * i) / (double)dim); };
  for (int f = 0; f < frames; ++f) {
    const int tpos = (frames == 2) ? (f == 0 ? 0 : skip_len - 1) : f;
    for (int y = 0; y < hp; ++y)
      for (int x = 0; x < wp; ++x) {
        const int64_t tok = ((int64_t)f * hp + y) * wp + x;
        float* c = &cs[tok * half];
        float* s = &sn[tok * half];
        for (int i = 0; i < nt; ++i) {
          const double a = tpos * inv_freq(i, t_dim);
          c[i] = (float)cos(a);
          s[i] = (float)sin(a);
        }
        for (int i = 0; i < nh; ++i) {
          const double a = y * inv_freq(i, h_dim);
          c[nt + i] = (float)cos(a);
          s[nt + i] = (float)sin(a);
        }
        for (int i = 0; i < nw; ++i) {
          const double a = x * inv_freq(i, w_dim);
          c[nt + nh + i] = (float)cos(a);
          s[nt + nh + i] = (float)sin(a);
        }
      }
  }
  return CE_OK;
}

int ensure_rope(ce_dit* h, int frames, int hp, int wp, cudaStream_t stream) {
  int dev = 0;
  CE_CHECK_CUDA(cudaGetDevice(&dev));
  if (h->rope_cos && h->rope_dev == dev && h->rope_f == frames && h->rope_h == hp && h->rope_w == wp) return CE_OK;
  std::vector<float> cs, sn;
  int rc = rope_table_host(h->cfg.attention_head_dim, frames, hp, wp, h->cfg.rope_max_seq_len, h->cfg.rope_temporal_skip_len,
                           10000.0, cs, sn);
  if (rc) return rc;
  if (h->rope_cos) {  // other geometry, or the handle moved to another device (model.to(...)): rebuild there
    CE_CHECK_CUDA(cudaStreamSynchronize(stream));
    cudaFree(h->rope_cos);  // cudaFree accepts pointers of any device
    cudaFree(h->rope_sin);
    h->rope_cos = h->rope_sin = nullptr;
  }
  CE_CHECK_CUDA(cudaMalloc(&h->rope_cos, cs.size() * sizeof(float)));
  CE_CHECK_CUDA(cudaMalloc(&h->rope_sin, sn.size() * sizeof(float)));
  CE_CHECK_CUDA(cudaMemcpyAsync(h->rope_cos, cs.data(), cs.size() * sizeof(float), cudaMemcpyHostToDevice, stream));
  CE_CHECK_CUDA(cudaMemcpyAsync(h->rope_sin, sn.data(), sn.size() * sizeof(float), cudaMemcpyHostToDevice, stream));
  CE_CHECK_CUDA(cudaStreamSynchronize(stream));  // host vectors go out of scope
  h->rope_dev = dev;
  h->rope_f = frames;
  h->rope_h = hp;
  h->rope_w = wp;
  return CE_OK;
}

}  // namespace

// Every launch of the forward goes through run(): under ce_dit_profile_begin it records a (begin, end) event pair around the
// launch with its category and work (algorithmic flops for GEMM and attention, bytes for the row kernels), and it counts the
// launch once it is enqueued.
template <class Launch>
static int run(ce_dit* h, cudaStream_t s, int cat, double work, Launch&& launch) {
  const bool prof = h->profiling && h->ev_used + 2 <= h->ev.size();
  if (prof) {
    cudaEventRecord(h->ev[h->ev_used], s);
    h->ev_cat[h->ev_used / 2] = cat;
    h->ev_work[h->ev_used / 2] = work;
  }
  const int rc = launch();
  if (rc) return rc;
  if (prof) {
    cudaEventRecord(h->ev[h->ev_used + 1], s);
    h->ev_used += 2;
  }
  ++h->launches;
  return CE_OK;
}
#define LAUNCH(cat, work, call)                                              \
  do {                                                                       \
    const int _rc = run(h, s, (cat), (work), [&] { return (call); });       \
    if (_rc) return _rc;                                                     \
  } while (0)

static double attention_flops(const AttnArgs& a) { return 4.0 * a.B * a.H * (double)a.Lq * (a.Lk + a.Lk2) * a.head_dim; }

// out[M, N] = epilogue(A[M, K] x W^T + bias) with A and out dense.  `e` brings the epilogue fields (epi, resid, gate,
// stats_out / stats_mode); the statistics come one per N tile of gemm_tile_n(N).  An e4m3 weight takes two launches: the
// per-row quantization of A into the workspace, then the FP8 GEMM.
// With a LoRA entry `lo` of rank R > 0 (ce_dit_set_lora), two bf16 GEMMs come first: mid = bf16(A a_cat^T) [M, R], from the bf16 A
// (before any quantization), and term = bf16(mid b_cat^T) [M, N]; the main GEMM's epilogue adds the term (LoraAddend).
static int linear(ce_dit* h, cudaStream_t s, const Linear& w, const bf16* A, int M, int N, int K, bf16* out, GemmArgs e,
                  const LoraGemm* lo = nullptr) {
  GemmArgs g = e;
  g.M = M; g.N = N; g.K = K;
  g.out = out; g.ldo = N;
  g.bias = w.bias;
  if (g.stats_out) g.stats_ld = (N + gemm_tile_n(N) - 1) / gemm_tile_n(N);
  LoraAddend la;
  const LoraAddend* lp = nullptr;
  if (lo && lo->rank > 0) {
    const int R = lo->rank;
    GemmArgs d;
    d.M = M; d.N = R; d.K = K; d.out = h->lora_mid; d.ldo = R;
    LAUNCH(CAT_GEMM, 2.0 * M * (double)R * K, launch_gemm_bf16(A, K, static_cast<const bf16*>(lo->a_cat), K, d, s));
    GemmArgs u;
    u.M = M; u.N = N; u.K = R; u.out = h->lora_term; u.ldo = N;
    LAUNCH(CAT_GEMM, 2.0 * M * (double)N * R, launch_gemm_bf16(h->lora_mid, R, static_cast<const bf16*>(lo->b_cat), R, u, s));
    la.t = h->lora_term;
    la.ld = N;
    lp = &la;
  }
  if (w.dtype == 2) {
    LAUNCH(CAT_ROWS, 3.0 * M * (double)K + 4.0 * M, launch_quantize_rows_fp8(A, K, M, K, h->fp8_q, K, h->fp8_scale, s));
    LAUNCH(CAT_GEMM, 2.0 * M * (double)N * K,
           launch_gemm_fp8(reinterpret_cast<const e4m3*>(h->fp8_q), K, h->fp8_scale, static_cast<const e4m3*>(w.weight), K,
                           w.weight_scale, g, s, lp));
  } else {
    LAUNCH(CAT_GEMM, 2.0 * M * (double)N * K, launch_gemm_bf16(A, K, static_cast<const bf16*>(w.weight), K, g, s, lp));
  }
  return CE_OK;
}

// The time path of the condition embedder (:147-159): sinusoid, time embedder (fp32, temb rounded to bf16) and, when `tproj` is
// given, time_proj into tproj [B, 6D] bf16 (the reference's timestep_proj).
static int time_path(ce_dit* h, cudaStream_t s, const Weights& W, const float* timestep, int B, float* sin_emb, float* h1,
                     float* temb_f32, bf16* temb_bf16, bf16* tproj) {
  const ce_dit_config& c = h->cfg;
  const int D = D_of(c);
  LAUNCH(CAT_OTHER, 0.0, launch_timestep_sinusoid(timestep, sin_emb, B, c.freq_dim, s));
  LAUNCH(CAT_OTHER, 0.0, launch_small_linear(sin_emb, c.freq_dim, W.time1_w, W.time1_b, 0, D, B, /*act=*/1, 0, h1, nullptr, s));
  LAUNCH(CAT_OTHER, 0.0, launch_small_linear(h1, D, W.time2_w, W.time2_b, 0, D, B, 0, 0, temb_f32, temb_bf16, s));  // temb = (...).type_as(bf16)
  if (tproj)
    LAUNCH(CAT_OTHER, 0.0, launch_small_linear(temb_f32, D, W.time_proj_w, W.time_proj_b, 1, 6 * D, B, 0, /*in_silu_bf16=*/1, nullptr, tproj, s));
  return CE_OK;
}

// Batch split: the refusals of a split call, all before its first launch.  `sample_elems`: elements of one output sample.
static int bp_check(const ce_dit* h, const char* who, int batch, int64_t sample_elems, bool block_capture, cudaStream_t s) {
  const SeqPar& bp = h->bp;
  if (batch % bp.world != 0)
    return fail(CE_ERR_INVALID, std::string(who) + ": batch split: a batch of " + std::to_string(batch) + " does not divide over " +
                                    std::to_string(bp.world) + " ranks.  Only a call that carries the whole CFG pair is split: the unchanged "
                                    "diffusers pipeline's batch-1 calls are not split (it calls with the prompt and the negative prompt "
                                    "one at a time).  Run the pair as one batch-2 call, or switch the split off (ce_dit_bp_configure with "
                                    "world 1)");
  const int64_t need = (int64_t)batch * sample_elems * (int64_t)sizeof(bf16), slot = slot_bytes(bp.region_bytes);
  if (need > slot)
    return fail(CE_ERR_WORKSPACE, std::string(who) + ": batch split: the call's sample needs a slot of " + std::to_string(need) +
                                      " bytes, the peer region holds slots of " + std::to_string(slot) + " (ce_dit_bp_region_bytes)");
  CE_REQUIRE(!block_capture, std::string(who) + ": batch split: no block capture / block0_out (each rank runs only its own samples)");
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  CE_CHECK_CUDA(cudaStreamIsCapturing(s, &cs));
  CE_REQUIRE(cs == cudaStreamCaptureStatusNone,
             std::string(who) + ": batch split: the stream is capturing (the exchange's barrier epoch advances every call, so it cannot be "
                                "replayed from a graph)");
  return CE_OK;
}

// The exchange of a slot group (the batch split's `bp`, the call pair's `cp`).  `part` bytes at `own` go to offset rank * stride of
// every peer's slot of the current set; one barrier; then for every peer w the `part` bytes at offset w * stride of the own slot go to
// dst + w * stride.  The batch split passes its samples' place in the caller's buffer (stride = part); the call pair passes the two
// samples of the pair (stride 0: a slot holds the one sample of the other call).
// The set alternates with the barrier epoch's parity, so one barrier per exchange suffices: a rank reads set p of exchange n before it
// reaches the barrier of exchange n + 1, and no peer writes set p again before it has passed that barrier.
static int slot_exchange(ce_dit* h, SeqPar& g, const void* own, void* dst, int64_t part, int64_t stride, cudaStream_t s) {
  const int64_t set = kSlotFlagsBytes + (int64_t)(g.epoch & 1) * slot_bytes(g.region_bytes);
  SpCopy put[8], get[8];
  int n = 0;
  for (int w = 0; w < g.world; ++w) {
    if (w == g.rank) continue;
    put[n].src = own;
    put[n].dst = g.region[w] + set + g.rank * stride;
    put[n].bytes = part;
    get[n].src = g.region[g.rank] + set + w * stride;
    get[n].dst = reinterpret_cast<uint8_t*>(dst) + w * stride;
    get[n].bytes = part;
    ++n;
  }
  LAUNCH(CAT_OTHER, 0.0, launch_sp_copy(put, n, s));
  LAUNCH(CAT_OTHER, 0.0, launch_sp_barrier(g, 0, s));
  LAUNCH(CAT_OTHER, 0.0, launch_sp_copy(get, n, s));
  return CE_OK;
}

// Batch split: the exchange that ends every split call.  This rank's samples, already at their offset in the caller's buffer, go into
// every peer's slot; the other ranks' samples come from the own slot into the caller's buffer.
static int bp_exchange(ce_dit* h, void* sample, int batch, int64_t sample_elems, cudaStream_t s) {
  SeqPar& bp = h->bp;
  const int64_t part = (int64_t)(batch / bp.world) * sample_elems * (int64_t)sizeof(bf16);
  return slot_exchange(h, bp, reinterpret_cast<uint8_t*>(sample) + bp.rank * part, sample, part, part, s);
}

// ---- internals shared with dit_fp32.cu
const WeightMap& ce_dit_internal_weights_f32(const ce_dit* h) { return h->w32; }
int ce_dit_internal_rope(ce_dit* h, int frames, int hp, int wp, cudaStream_t s, const float** cos_out, const float** sin_out) {
  int rc = ensure_rope(h, frames, hp, wp, s);
  if (rc) return rc;
  *cos_out = h->rope_cos;
  *sin_out = h->rope_sin;
  return CE_OK;
}
const ce_dit_config* ce_dit_internal_config(const ce_dit* h) { return &h->cfg; }
int ce_dit_internal_bp_world(const ce_dit* h) { return h->bp.world; }
bool ce_dit_internal_lora_set(const ce_dit* h) { return !h->lora.empty(); }

extern "C" {

int ce_abi_version(void) { return CE_ABI_VERSION; }

int ce_dit_set_weight_fp32(ce_dit* h, const char* name, const float* ptr, int64_t numel) {
  CE_REQUIRE(h, "ce_dit_set_weight_fp32: null handle");
  return register_weight(h->w32, "ce_dit_set_weight_fp32", name, ptr, 1, numel);
}
const char* ce_last_error(void) { return ce::last_error().c_str(); }
int ce_device_check(void) { return check_device(); }

int ce_dit_create(const ce_dit_config* cfg, ce_dit** out) {
  CE_REQUIRE(cfg && out, "ce_dit_create: null argument");
  CE_REQUIRE(cfg->attention_head_dim == 128, "ce_dit_create: only attention_head_dim 128 is built");
  CE_REQUIRE(cfg->patch_t == 1 && cfg->patch_h == 2 && cfg->patch_w == 2, "ce_dit_create: only patch_size (1,2,2) is built");
  CE_REQUIRE(cfg->num_attention_heads > 0 && cfg->num_layers > 0 && cfg->ffn_dim % 8 == 0 && cfg->text_dim % 8 == 0, "ce_dit_create: dims");
  CE_REQUIRE(cfg->image_dim == 0 || (cfg->image_dim % 8 == 0 && cfg->added_kv_proj_dim == D_of(*cfg)),
             "ce_dit_create: image_dim % 8 and added_kv_proj_dim == inner dim (the image embedder projects to inner dim)");
  CE_REQUIRE((cfg->in_channels * 4) % 8 == 0 && (cfg->out_channels * 4) % 8 == 0, "ce_dit_create: channel counts");
  CE_REQUIRE(cfg->freq_dim % 4 == 0, "ce_dit_create: freq_dim % 4");
  ce_dit* h = new ce_dit();
  h->cfg = *cfg;
  *out = h;
  return CE_OK;
}

void ce_dit_destroy(ce_dit* h) {
  if (!h) return;
  if (h->rope_cos) cudaFree(h->rope_cos);
  if (h->rope_sin) cudaFree(h->rope_sin);
  for (cudaEvent_t e : h->ev) cudaEventDestroy(e);
  delete h;
}

int ce_dit_set_weight(ce_dit* h, const char* name, const void* ptr, int dtype, int64_t numel) {
  CE_REQUIRE(h, "ce_dit_set_weight: null handle");
  return register_weight(h->w, "ce_dit_set_weight", name, ptr, dtype, numel);
}

int ce_dit_weights_complete(const ce_dit* h) {
  CE_REQUIRE(h, "null handle");
  Weights w;
  return resolve_weights(h, w);
}

int64_t ce_dit_workspace_bytes(const ce_dit* h, int batch, int frames, int height, int width, int text_len) {
  if (!h || validate_geometry(h, batch, frames, height, width, text_len)) return -1;
  Weights w;
  resolve_weights(h, w);   // only w.fp8 is read here, and it is set even before every weight has been registered
  const int L = frames * (height / h->cfg.patch_h) * (width / h->cfg.patch_w);
  return carve(h->cfg, nullptr, batch, L, text_len, 257, w.fp8, h->attn_fp8, h->lora_rmax).bytes;
}

int64_t ce_dit_last_launch_count(const ce_dit* h) { return h ? h->launches : 0; }

int64_t ce_dit_context_cache_bytes(const ce_dit* h, int batch, int text_len) {
  if (!h || batch < 1 || text_len < 1) return -1;
  const int64_t D = D_of(h->cfg);
  const int64_t per_layer = (int64_t)batch * (text_len + (h->cfg.image_dim > 0 ? 257 : 0)) * 2 * D * (int64_t)sizeof(bf16);
  return ((per_layer + 255) & ~int64_t(255)) * h->cfg.num_layers;
}

int64_t ce_dit_sp_region_bytes(const ce_dit* h, int batch, int frames, int height, int width, int world) {
  if (!h || world < 2 || world > 8 || batch < 1) return -1;
  const ce_dit_config& c = h->cfg;
  const int64_t L = (int64_t)frames * (height / c.patch_h) * (width / c.patch_w);
  if (L % world != 0 || c.num_attention_heads % world != 0) return -1;
  return sp_layout(batch, L, D_of(c), (int64_t)c.out_channels * 4, world).bytes;
}

int ce_dit_sp_configure(ce_dit* h, int rank, int world, void* const* region_ptrs, int64_t region_bytes) {
  CE_REQUIRE(h, "ce_dit_sp_configure: null handle");
  SeqPar sp = h->sp;
  CE_TRY(sp_configure(sp, "ce_dit_sp_configure", rank, world, region_ptrs, region_bytes));
  CE_REQUIRE(h->cfg.num_attention_heads % sp.world == 0, "ce_dit_sp_configure: the head count must be divisible by the number of ranks");
  h->sp = sp;
  return CE_OK;
}

int ce_dit_sp_host_barrier(ce_dit* h, int timeout_ms) { return sp_set_host_barrier(h ? &h->sp : nullptr, "ce_dit_sp_host_barrier", timeout_ms); }

int64_t ce_dit_bp_region_bytes(const ce_dit* h, int batch, int frames, int height, int width, int world) {
  if (!h || world < 2 || world > 8 || batch < 1 || batch > 8 || batch % world != 0 || frames < 1 || height < 1 || width < 1) return -1;
  const int64_t sample = (int64_t)batch * h->cfg.out_channels * frames * height * width * (int64_t)sizeof(bf16);
  return kSlotFlagsBytes + 2 * ((sample + 1023) & ~int64_t(1023));
}

int ce_dit_bp_configure(ce_dit* h, int rank, int world, void* const* region_ptrs, int64_t region_bytes) {
  CE_REQUIRE(h, "ce_dit_bp_configure: null handle");
  CE_REQUIRE(world == 1 || h->cp.world <= 1,
             "ce_dit_bp_configure: the call-pair split is configured (ce_dit_cp_configure): the two CFG splits are exclusive, switch it off first");
  return sp_configure(h->bp, "ce_dit_bp_configure", rank, world, region_ptrs, region_bytes);
}

int ce_dit_bp_host_barrier(ce_dit* h, int timeout_ms) { return sp_set_host_barrier(h ? &h->bp : nullptr, "ce_dit_bp_host_barrier", timeout_ms); }

int64_t ce_dit_cp_region_bytes(const ce_dit* h, int batch, int frames, int height, int width) {
  if (!h || batch < 1 || batch > 8 || frames < 1 || height < 1 || width < 1) return -1;
  const int64_t sample = (int64_t)batch * h->cfg.out_channels * frames * height * width * (int64_t)sizeof(bf16);
  return kSlotFlagsBytes + 2 * ((sample + 1023) & ~int64_t(1023));
}

int ce_dit_cp_configure(ce_dit* h, int rank, int world, void* const* region_ptrs, int64_t region_bytes) {
  CE_REQUIRE(h, "ce_dit_cp_configure: null handle");
  CE_REQUIRE(world == 1 || h->bp.world <= 1,
             "ce_dit_cp_configure: the batch split is configured (ce_dit_bp_configure): the two CFG splits are exclusive, switch it off first");
  SeqPar cp = h->cp;
  CE_TRY(sp_configure(cp, "ce_dit_cp_configure", rank, world, region_ptrs, region_bytes));
  CE_REQUIRE(cp.world <= 2, "ce_dit_cp_configure: a CFG pair has two calls: world must be 1 (off) or 2");
  h->cp = cp;
  return CE_OK;
}

int ce_dit_cp_exchange(ce_dit* h, const void* own_sample, void* other_sample, int batch, int frames, int height, int width, void* stream_v) {
  CE_REQUIRE(h && own_sample && other_sample, "ce_dit_cp_exchange: null argument");
  CE_REQUIRE(h->cp.world == 2, "ce_dit_cp_exchange: the call-pair split is not configured (ce_dit_cp_configure with world 2)");
  CE_REQUIRE(batch >= 1 && batch <= 8 && frames >= 1 && height >= 1 && width >= 1, "ce_dit_cp_exchange: geometry");
  CE_REQUIRE(((reinterpret_cast<uintptr_t>(own_sample) | reinterpret_cast<uintptr_t>(other_sample)) & 1) == 0,
             "ce_dit_cp_exchange: the samples must be bf16-aligned");
  const int64_t need = (int64_t)batch * h->cfg.out_channels * frames * height * width * (int64_t)sizeof(bf16);
  const int64_t slot = slot_bytes(h->cp.region_bytes);
  if (need > slot)
    return fail(CE_ERR_WORKSPACE, "ce_dit_cp_exchange: the call's sample needs a slot of " + std::to_string(need) +
                                      " bytes, the peer region holds slots of " + std::to_string(slot) + " (ce_dit_cp_region_bytes)");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_v);
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  CE_CHECK_CUDA(cudaStreamIsCapturing(s, &cs));
  CE_REQUIRE(cs == cudaStreamCaptureStatusNone,
             "ce_dit_cp_exchange: the stream is capturing (the exchange's barrier epoch advances every pair, so it cannot be replayed from "
             "a graph)");
  return slot_exchange(h, h->cp, own_sample, other_sample, need, 0, s);
}

int ce_dit_cp_host_barrier(ce_dit* h, int timeout_ms) { return sp_set_host_barrier(h ? &h->cp : nullptr, "ce_dit_cp_host_barrier", timeout_ms); }

int ce_dit_set_capture(ce_dit* h, const int32_t* layers, void* const* dst, int n) {
  CE_REQUIRE(h && n >= 0 && (n == 0 || (layers && dst)), "ce_dit_set_capture: arguments");
  h->capture.clear();
  for (int i = 0; i < n; ++i) {
    CE_REQUIRE(layers[i] >= 0 && layers[i] < h->cfg.num_layers && dst[i], "ce_dit_set_capture: layer index / null destination");
    h->capture.push_back({layers[i], dst[i]});
  }
  return CE_OK;
}

int ce_dit_profile_begin(ce_dit* h, int max_launches) {
  CE_REQUIRE(h && max_launches > 0, "ce_dit_profile_begin: arguments");
  while ((int)h->ev.size() < 2 * max_launches) {
    cudaEvent_t e;
    CE_CHECK_CUDA(cudaEventCreate(&e));
    h->ev.push_back(e);
  }
  h->ev_cat.assign(h->ev.size() / 2, 0);
  h->ev_work.assign(h->ev.size() / 2, 0.0);
  h->ev_used = 0;
  h->profiling = true;
  return CE_OK;
}

int ce_dit_profile_end(ce_dit* h, double* ms_out, double* work_out, int64_t* count_out) {
  CE_REQUIRE(h && ms_out && work_out && count_out, "ce_dit_profile_end: arguments");
  h->profiling = false;
  for (int c = 0; c < NUM_CATS; ++c) {
    ms_out[c] = 0.0;
    work_out[c] = 0.0;
    count_out[c] = 0;
  }
  if (h->ev_used == 0) return CE_OK;
  CE_CHECK_CUDA(cudaEventSynchronize(h->ev[h->ev_used - 1]));
  for (size_t i = 0; i + 1 < h->ev_used + 1 && i < h->ev_used; i += 2) {
    float ms = 0.f;
    CE_CHECK_CUDA(cudaEventElapsedTime(&ms, h->ev[i], h->ev[i + 1]));
    const int c = h->ev_cat[i / 2];
    ms_out[c] += ms;
    work_out[c] += h->ev_work[i / 2];
    count_out[c] += 1;
  }
  h->ev_used = 0;
  return CE_OK;
}

int ce_dit_forward(ce_dit* h, const void* hidden_states, const float* timestep, const void* encoder_hidden_states,
                   const void* encoder_hidden_states_image, void* sample, int batch, int frames, int height, int width,
                   int text_len, void* workspace, int64_t workspace_bytes, void* block0_out, void* stream_v) {
  return ce_dit_forward_ex(h, hidden_states, timestep, encoder_hidden_states, encoder_hidden_states_image, sample, batch, frames, height,
                           width, text_len, workspace, workspace_bytes, block0_out, nullptr, 0, 0, stream_v);
}

// The forward of the samples this rank computes (all of them without the batch split).
static int forward_samples(ce_dit* h, const void* hidden_states, const float* timestep, const void* encoder_hidden_states,
                           const void* encoder_hidden_states_image, void* sample, int batch, int frames, int height, int width,
                           int text_len, void* workspace, int64_t workspace_bytes, void* block0_out, void* ctx_cache,
                           int64_t ctx_cache_bytes, int ctx_reuse, void* stream_v) {
  CE_REQUIRE(h && hidden_states && timestep && encoder_hidden_states && sample && workspace, "ce_dit_forward: null argument");
  CE_REQUIRE(ctx_reuse == 0 || ctx_cache != nullptr, "ce_dit_forward_ex: ctx_reuse needs a context cache");
  int rc = check_device();
  if (rc) return rc;
  if ((rc = validate_geometry(h, batch, frames, height, width, text_len))) return rc;
  Weights W;
  if ((rc = resolve_weights(h, W))) return rc;
  const ce_dit_config& c = h->cfg;
  CE_REQUIRE((c.image_dim > 0) == (encoder_hidden_states_image != nullptr),
             "ce_dit_forward: encoder_hidden_states_image must be given iff the model has an image embedder");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_v);
  const int B = batch, hp = height / c.patch_h, wp = width / c.patch_w;
  const int Lfull = frames * hp * wp, D = D_of(c), F = c.ffn_dim, H = c.num_attention_heads, Lt = text_len, Li = 257;
  const int Kp = c.in_channels * 4, No = c.out_channels * 4;
  // sequence parallel: this rank owns tokens [tok0, tok0 + L) of every sample; everything below is written for "L local tokens"
  SeqPar& sp = h->sp;
  const bool spx = sp.world > 1;
  if (spx) {
    CE_REQUIRE(!h->attn_fp8, "sequence parallelism is not built for FP8 attention: run it on one GPU or switch it off (ce_dit_set_attention_fp8)");
    CE_REQUIRE(Lfull % sp.world == 0, "sequence parallel: the tokens must divide by the rank count");
    CE_REQUIRE(D % 256 == 0, "sequence parallel: the width must be a multiple of 256 (the q | k scatter needs the GEMM's row statistics)");
    CE_REQUIRE(Lfull >= 256, "sequence parallel: at least 256 tokens (the self-attention kernel with the output scatter)");
    CE_REQUIRE(!h->profiling && h->capture.empty() && block0_out == nullptr, "sequence parallel: no per-launch profiling / block capture");
  }
  const int L = spx ? Lfull / sp.world : Lfull, tok0 = spx ? sp.rank * L : 0, M = B * L;
  const SpLayout lay = spx ? sp_layout(B, Lfull, D, No, sp.world) : SpLayout();
  if (spx && lay.bytes > sp.region_bytes) return fail(CE_ERR_WORKSPACE, "sequence parallel: peer region too small (ce_dit_sp_region_bytes)");
  CE_REQUIRE(!(spx && W.fp8), "sequence parallelism is not built for FP8 weights: run the FP8 mode on one GPU");
  CE_REQUIRE(!(spx && !h->lora.empty()), "sequence parallelism is not built for run-time LoRA: clear it first (ce_dit_set_lora with n = 0)");
  Workspace ws = carve(c, workspace, B, L, Lt, Li, W.fp8, h->attn_fp8, h->lora_rmax);
  if (ws.bytes > workspace_bytes)
    return fail(CE_ERR_WORKSPACE, "workspace too small: need " + std::to_string(ws.bytes) + " bytes, got " + std::to_string(workspace_bytes));
  CE_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "workspace must be 256-byte aligned");
  bf16* const rec = reinterpret_cast<bf16*>(h->resid_rec);
  if (rec) {
    CE_REQUIRE(!spx, "TeaCache residual record: sequence parallelism is not built for it");
    CE_REQUIRE(h->resid_rec_bytes >= (int64_t)M * D * (int64_t)sizeof(bf16),
               "TeaCache residual record: buffer too small for this forward (needs batch * tokens * inner dim bf16)");
  }
  if ((rc = ensure_rope(h, frames, hp, wp, s))) return rc;   // always the full table [Lfull, 64]
  h->fp8_q = ws.fp8_q;
  h->fp8_scale = ws.fp8_scale;
  h->lora_mid = ws.lora_mid;
  h->lora_term = ws.lora_term;
  // run-time LoRA entry of layer i's GEMM `target`, or null
  auto lora_of = [&](int i, int target) { return h->lora.empty() ? nullptr : &h->lora[(size_t)i * CE_LORA_TARGETS + target]; };
  // step-invariant context (text / image embedders and every block's cross-attention K/V, :52-60, :147-165): kept in the
  // caller's cache across the steps of one edit when one is given; recomputed into the workspace otherwise
  const int64_t kv_t_elems = (int64_t)B * Lt * 2 * D, kv_i_elems = c.image_dim > 0 ? (int64_t)B * Li * 2 * D : 0;
  const int64_t ctx_layer_bytes = ((kv_t_elems + kv_i_elems) * (int64_t)sizeof(bf16) + 255) & ~int64_t(255);
  if (ctx_cache) {
    CE_REQUIRE((reinterpret_cast<uintptr_t>(ctx_cache) & 255) == 0, "ce_dit_forward_ex: context cache must be 256-byte aligned");
    CE_REQUIRE(ctx_cache_bytes >= ctx_layer_bytes * c.num_layers, "ce_dit_forward_ex: context cache too small (ce_dit_context_cache_bytes)");
  }
  auto kv_text_of = [&](int layer) { return ctx_cache ? reinterpret_cast<bf16*>(reinterpret_cast<uint8_t*>(ctx_cache) + layer * ctx_layer_bytes) : ws.kv_text; };
  auto kv_img_of = [&](int layer) { return ctx_cache ? kv_text_of(layer) + kv_t_elems : ws.kv_img; };
  const bool ctx_compute = !(ctx_cache && ctx_reuse);
  // Row statistics for the LayerNorms / RMSNorms inside the blocks come from the epilogue of the GEMM that wrote the row whenever
  // the N tiles (256 wide) line up with the q | k | v boundaries; the row kernels are then streaming passes (elementwise.cuh).
  // Other widths get no partials, and the row kernels reduce over the row themselves.  The row kernels take D <= 8192.
  const bool st = D % 256 == 0;
  const int tD = D / 256;
  auto partials = [&](const float2* stats, int ld) { return st ? RowPartials{stats, ld, tD, 256} : RowPartials{}; };
  auto ln = [&](const bf16* x, bf16* y, const float* scale, const float* shift, int mod_stride, int rpb, const float* w, const float* b, int is1p) {
    return launch_layernorm(x, D, y, D, M, D, c.eps, scale, shift, mod_stride, rpb, w, b, is1p, partials(ws.stats_x, tD), s);
  };
  // linear() epilogues: `stats` receives the output's row statistics (mode 1 for a LayerNorm, 2 for an RMSNorm) on the
  // statistics path; the residual ones update the residual stream ws.x in place, gated by a modulation chunk [B, 6D] or not
  auto epi = [&](int e, float2* stats = nullptr, int mode = 0) {
    GemmArgs g;
    g.epi = e;
    if (st && stats) {
      g.stats_out = stats;
      g.stats_mode = mode;
    }
    return g;
  };
  auto resid_epi = [&](const float* gate) {
    GemmArgs g = epi(gate ? EPI_BIAS_GATE_RESID : EPI_BIAS_RESID, ws.stats_x, 1);
    g.resid = ws.x; g.ldr = D;
    if (gate) {
      g.gate = gate; g.gate_stride = 6 * D; g.rows_per_batch = L;
    }
    return g;
  };
  h->launches = 0;
  const float attn_scale = 1.0f / sqrtf((float)c.attention_head_dim);

  // ---- patch embedding (Conv3d k=s=(1,2,2) as im2row + GEMM, :429-430)
  LAUNCH(CAT_OTHER, 0.0, launch_patchify(reinterpret_cast<const bf16*>(hidden_states), ws.patches, B, c.in_channels, frames, height, width, tok0, L, s));
  if ((rc = linear(h, s, W.patch, ws.patches, M, D, Kp, ws.x, epi(EPI_BIAS, ws.stats_x, 1)))) return rc;
  if (rec) CE_CHECK_CUDA(cudaMemcpyAsync(rec, ws.x, (size_t)M * D * sizeof(bf16), cudaMemcpyDeviceToDevice, s));   // x_before_blocks

  // ---- condition embedder (:147-165)
  if ((rc = time_path(h, s, W, timestep, B, ws.sin_emb, ws.h1, ws.temb_f32, ws.temb_bf16, ws.tproj))) return rc;
  LAUNCH(CAT_OTHER, 0.0, launch_add_table(W.block_table, c.num_layers, ws.tproj, 6 * D, ws.mod, B, D, 6, s, /*scale chunks 1,4 -> 1+scale*/ 0x12u));
  LAUNCH(CAT_OTHER, 0.0, launch_add_table(W.head_table, 1, ws.temb_bf16, D, ws.modf, B, D, 2, s, /*chunk 1 = scale*/ 0x2u));
  // text: Linear -> GELU(tanh) -> Linear
  if (ctx_compute) {
    const bf16* text = reinterpret_cast<const bf16*>(encoder_hidden_states);
    if ((rc = linear(h, s, W.text1, text, B * Lt, D, c.text_dim, ws.text1, epi(EPI_BIAS_GELU_TANH)))) return rc;
    if ((rc = linear(h, s, W.text2, ws.text1, B * Lt, D, D, ws.ctx_text, epi(EPI_BIAS)))) return rc;
  }
  if (ctx_compute && c.image_dim > 0) {  // image: FP32LayerNorm -> Linear -> GELU(erf) -> Linear -> FP32LayerNorm (:111-123)
    const int I = c.image_dim;
    LAUNCH(CAT_OTHER, 0.0, launch_layernorm(reinterpret_cast<const bf16*>(encoder_hidden_states_image), I, ws.img0, I, B * Li, I, 1e-5f, nullptr, nullptr, 0, 0,
                                            W.img_norm1_w, W.img_norm1_b, 0, RowPartials{}, s));
    if ((rc = linear(h, s, W.img_ff0, ws.img0, B * Li, I, I, ws.img1, epi(EPI_BIAS_GELU_ERF)))) return rc;
    if ((rc = linear(h, s, W.img_ff2, ws.img1, B * Li, D, I, ws.img2, epi(EPI_BIAS)))) return rc;
    LAUNCH(CAT_OTHER, 0.0, launch_layernorm(ws.img2, D, ws.ctx_img, D, B * Li, D, 1e-5f, nullptr, nullptr, 0, 0, W.img_norm2_w, W.img_norm2_b, 0,
                                            RowPartials{}, s));
  }

  // ---- transformer blocks (:447-448)
  for (int i = 0; i < c.num_layers; ++i) {
    const LayerWeights& lw = W.layers[i];
    const float* mod = ws.mod + (size_t)i * B * 6 * D;  // [B, 6, D]: shift, scale, gate, c_shift, c_scale, c_gate
    // 1. self-attention
    LAUNCH(CAT_ROWS, 4.0 * M * D, ln(ws.x, ws.xn, mod + 1 * D, mod + 0 * D, 6 * D, L, nullptr, nullptr, 1));
    if ((rc = linear(h, s, lw.qkv, ws.xn, M, 3 * D, D, ws.qkv, epi(EPI_BIAS, ws.stats_qkv, 2), lora_of(i, LORA_QKV)))) return rc;
    const bf16* attn_in = ws.attn;
    if (spx) {
      // heads <-> tokens exchange by peer stores: q | k normalised + rotated and scattered by head, v scattered by head, barrier,
      // attention over ALL tokens for this rank's heads with the output rows scattered back to the ranks that own the tokens, barrier
      const int Hl = H / sp.world, Dl = D / sp.world;
      SpScatter sc;
      sc.world = sp.world; sc.heads_per_rank = Hl; sc.L_total = Lfull; sc.rows_per_batch = L; sc.tok0 = tok0;
      SpCopy vj[8];   // v columns of rank w's heads into rows [tok0, tok0 + L) of every sample of its v buffer
      for (int w = 0; w < sp.world; ++w) {
        sc.dst[0][w] = reinterpret_cast<bf16*>(sp.region[w] + lay.q);
        sc.dst[1][w] = reinterpret_cast<bf16*>(sp.region[w] + lay.k);
        vj[w].src = ws.qkv + 2 * D + w * Dl;
        vj[w].dst = sp.region[w] + lay.v + (int64_t)tok0 * Dl * 2;
        vj[w].bytes = Dl * 2;
        vj[w].n0 = L; vj[w].sp0 = 3 * D * 2; vj[w].dp0 = Dl * 2;
        vj[w].n1 = B; vj[w].sp1 = (int64_t)L * 3 * D * 2; vj[w].dp1 = (int64_t)Lfull * Dl * 2;
      }
      LAUNCH(CAT_OTHER, 0.0, launch_rmsnorm_rope(ws.qkv, 3 * D, M, D, c.eps, lw.norm_q1, lw.norm_k1, 2, h->rope_cos, h->rope_sin, Lfull,
                                                 c.attention_head_dim, partials(ws.stats_qkv, 3 * tD), s, &sc));
      LAUNCH(CAT_OTHER, 0.0, launch_sp_copy(vj, sp.world, s));
      LAUNCH(CAT_OTHER, 0.0, launch_sp_barrier(sp, lay.flags, s));
      AttnArgs a;
      a.B = B; a.H = Hl; a.Lq = Lfull; a.Lk = Lfull;
      a.q = reinterpret_cast<const bf16*>(sp.region[sp.rank] + lay.q); a.ldq = Dl;
      a.k = reinterpret_cast<const bf16*>(sp.region[sp.rank] + lay.k); a.ldk = Dl;
      a.v = reinterpret_cast<const bf16*>(sp.region[sp.rank] + lay.v); a.ldv = Dl;
      a.out = reinterpret_cast<bf16*>(sp.region[sp.rank] + lay.attn); a.ldo = D;
      for (int w = 0; w < sp.world; ++w) a.out_peer[w] = reinterpret_cast<bf16*>(sp.region[w] + lay.attn);
      a.peer_rows = L;
      a.out_col0 = sp.rank * Dl;
      a.scale = attn_scale;
      LAUNCH(CAT_ATTN, attention_flops(a), launch_attention(a, s));
      LAUNCH(CAT_OTHER, 0.0, launch_sp_barrier(sp, lay.flags, s));
      attn_in = reinterpret_cast<const bf16*>(sp.region[sp.rank] + lay.attn);
    } else {
      LAUNCH(CAT_ROWS, 8.0 * M * D, launch_rmsnorm_rope(ws.qkv, 3 * D, M, D, c.eps, lw.norm_q1, lw.norm_k1, 2, h->rope_cos, h->rope_sin, L,
                                                        c.attention_head_dim, partials(ws.stats_qkv, 3 * tD), s));
      if (h->attn_fp8) {   // quantize q | k per (token, head) and v per (sample, channel), then the e4m3 attention
        const int Lpad = vt_keys(L);
        LAUNCH(CAT_ROWS, 6.0 * M * D + 8.0 * M * H, launch_quantize_heads_fp8(ws.qkv, 3 * D, M, 2 * H, ws.qk8, 2 * D, ws.qk_scale, s));
        LAUNCH(CAT_ROWS, 4.0 * M * D + 1.0 * B * Lpad * D + 4.0 * B * D,
               launch_quantize_v_fp8(ws.qkv + 2 * D, 3 * D, B, L, H, ws.vt8, Lpad, ws.v_scale, s));
        AttnFp8Args a;
        a.B = B; a.H = H; a.L = L;
        a.q = ws.qk8; a.k = ws.qk8 + D; a.ldqk = 2 * D;
        a.q_scale = ws.qk_scale; a.k_scale = ws.qk_scale + H; a.lds = 2 * H;
        a.vt = ws.vt8; a.Lpad = Lpad; a.v_scale = ws.v_scale;
        a.out = ws.attn; a.ldo = D;
        a.scale = attn_scale;
        LAUNCH(CAT_ATTN, 4.0 * B * H * (double)L * L * c.attention_head_dim, launch_attention_fp8(a, s));
      } else {
        AttnArgs a;
        a.B = B; a.H = H; a.Lq = L; a.Lk = L;
        a.q = ws.qkv; a.ldq = 3 * D;
        a.k = ws.qkv + D; a.ldk = 3 * D;
        a.v = ws.qkv + 2 * D; a.ldv = 3 * D;
        a.out = ws.attn; a.ldo = D;
        a.scale = attn_scale;
        LAUNCH(CAT_ATTN, attention_flops(a), launch_attention(a, s));
      }
    }
    if ((rc = linear(h, s, lw.out1, attn_in, M, D, D, ws.x, resid_epi(mod + 2 * D), lora_of(i, LORA_OUT1)))) return rc;
    // 2. cross-attention
    LAUNCH(CAT_ROWS, 4.0 * M * D, ln(ws.x, ws.xn, nullptr, nullptr, 0, 0, lw.norm2_w, lw.norm2_b, 0));
    bf16* q2 = ws.qkv;  // [M, D]
    if ((rc = linear(h, s, lw.q2, ws.xn, M, D, D, q2, epi(EPI_BIAS, ws.stats_q2, 2), lora_of(i, LORA_Q2)))) return rc;
    LAUNCH(CAT_ROWS, 4.0 * M * D, launch_rmsnorm_rope(q2, D, M, D, c.eps, lw.norm_q2, nullptr, 1, nullptr, nullptr, 0, c.attention_head_dim,
                                                      partials(ws.stats_q2, tD), s));
    bf16* kv_text = kv_text_of(i);
    bf16* kv_img = kv_img_of(i);
    if (ctx_compute) {
      if ((rc = linear(h, s, lw.kv, ws.ctx_text, B * Lt, 2 * D, D, kv_text, epi(EPI_BIAS), lora_of(i, LORA_KV)))) return rc;
      LAUNCH(CAT_OTHER, 0.0, launch_rmsnorm_rope(kv_text, 2 * D, B * Lt, D, c.eps, lw.norm_k2, nullptr, 1, nullptr, nullptr, 0, c.attention_head_dim,
                                                     RowPartials{}, s));
      if (c.image_dim > 0) {
        if ((rc = linear(h, s, lw.add_kv, ws.ctx_img, B * Li, 2 * D, D, kv_img, epi(EPI_BIAS), lora_of(i, LORA_ADD_KV)))) return rc;
        LAUNCH(CAT_OTHER, 0.0, launch_rmsnorm_rope(kv_img, 2 * D, B * Li, D, c.eps, lw.norm_added_k, nullptr, 1, nullptr, nullptr, 0, c.attention_head_dim,
                                                       RowPartials{}, s));
      }
    }
    {  // text and image cross-attention in ONE launch: two key/value sources, two softmaxes, results added (:84-104)
      AttnArgs a;
      a.B = B; a.H = H; a.Lq = L; a.Lk = Lt;
      a.q = q2; a.ldq = D;
      a.k = kv_text; a.ldk = 2 * D;
      a.v = kv_text + D; a.ldv = 2 * D;
      if (c.image_dim > 0) {
        a.k2 = kv_img; a.ldk2 = 2 * D;
        a.v2 = kv_img + D; a.ldv2 = 2 * D;
        a.Lk2 = Li;
      }
      a.out = ws.attn; a.ldo = D;
      a.scale = attn_scale;
      LAUNCH(CAT_ATTN, attention_flops(a), launch_attention(a, s));
    }
    if ((rc = linear(h, s, lw.out2, ws.attn, M, D, D, ws.x, resid_epi(nullptr), lora_of(i, LORA_OUT2)))) return rc;
    // 3. feed-forward
    LAUNCH(CAT_ROWS, 4.0 * M * D, ln(ws.x, ws.xn, mod + 4 * D, mod + 3 * D, 6 * D, L, nullptr, nullptr, 1));
    if ((rc = linear(h, s, lw.ffn1, ws.xn, M, F, D, ws.hbuf, epi(EPI_BIAS_GELU_TANH), lora_of(i, LORA_FFN1)))) return rc;
    if ((rc = linear(h, s, lw.ffn2, ws.hbuf, M, D, F, ws.x, resid_epi(mod + 5 * D), lora_of(i, LORA_FFN2)))) return rc;
    if (i == 0 && block0_out)
      CE_CHECK_CUDA(cudaMemcpyAsync(block0_out, ws.x, (size_t)M * D * sizeof(bf16), cudaMemcpyDeviceToDevice, s));
    for (const auto& cap : h->capture)
      if (cap.first == i) CE_CHECK_CUDA(cudaMemcpyAsync(cap.second, ws.x, (size_t)M * D * sizeof(bf16), cudaMemcpyDeviceToDevice, s));
  }
  if (rec) LAUNCH(CAT_ROWS, 6.0 * M * D, launch_sub_from(ws.x, rec, (int64_t)M * D, s));   // residual = bf16(x_after - x_before)

  // ---- output head (:451-467): modf = [B, 2, D] with shift = chunk 0, scale = chunk 1
  LAUNCH(CAT_ROWS, 4.0 * M * D, ln(ws.x, ws.xn, ws.modf + D, ws.modf, 2 * D, L, nullptr, nullptr, 1));
  if ((rc = linear(h, s, W.proj_out, ws.xn, M, No, D, ws.yout, epi(EPI_BIAS)))) return rc;
  if (spx) {   // every rank gets the whole head output (rows all-gathered by peer stores), then un-patchifies the full sample
    SpCopy yj[8];   // this rank's rows into rows [tok0, tok0 + L) of every sample of every rank's yout
    for (int w = 0; w < sp.world; ++w) {
      yj[w].src = ws.yout;
      yj[w].dst = sp.region[w] + lay.yout + (int64_t)tok0 * No * 2;
      yj[w].bytes = (int64_t)L * No * 2;
      yj[w].n0 = B; yj[w].sp0 = (int64_t)L * No * 2; yj[w].dp0 = (int64_t)Lfull * No * 2;
    }
    LAUNCH(CAT_OTHER, 0.0, launch_sp_copy(yj, sp.world, s));
    LAUNCH(CAT_OTHER, 0.0, launch_sp_barrier(sp, lay.flags, s));
    LAUNCH(CAT_OTHER, 0.0, launch_unpatchify(reinterpret_cast<const bf16*>(sp.region[sp.rank] + lay.yout), No, reinterpret_cast<bf16*>(sample), B,
                                             c.out_channels, frames, height, width, s));
    LAUNCH(CAT_OTHER, 0.0, launch_sp_barrier(sp, lay.flags, s));   // nobody overwrites a peer's yout (next forward) before it has been read
    return CE_OK;
  }
  LAUNCH(CAT_OTHER, 0.0, launch_unpatchify(ws.yout, No, reinterpret_cast<bf16*>(sample), B, c.out_channels, frames, height, width, s));
  return CE_OK;
}

// Byte address of sample `first` of a [batch, ...] tensor with `per_sample` bytes per sample (NULL stays NULL).
static const void* sample_at(const void* p, int first, int64_t per_sample) {
  return p ? static_cast<const uint8_t*>(p) + first * per_sample : nullptr;
}

int ce_dit_forward_ex(ce_dit* h, const void* hidden_states, const float* timestep, const void* encoder_hidden_states,
                      const void* encoder_hidden_states_image, void* sample, int batch, int frames, int height, int width,
                      int text_len, void* workspace, int64_t workspace_bytes, void* block0_out, void* ctx_cache,
                      int64_t ctx_cache_bytes, int ctx_reuse, void* stream_v) {
  if (!h || h->bp.world <= 1)
    return forward_samples(h, hidden_states, timestep, encoder_hidden_states, encoder_hidden_states_image, sample, batch, frames, height,
                           width, text_len, workspace, workspace_bytes, block0_out, ctx_cache, ctx_cache_bytes, ctx_reuse, stream_v);
  // batch split: this rank's samples through the forward above (the token split, when configured too, runs on them unchanged), then
  // the exchange
  CE_REQUIRE(hidden_states && timestep && encoder_hidden_states && sample && workspace, "ce_dit_forward: null argument");
  CE_TRY(validate_geometry(h, batch, frames, height, width, text_len));
  const ce_dit_config& c = h->cfg;
  const int64_t pixels = (int64_t)frames * height * width, out_elems = c.out_channels * pixels;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_v);
  CE_TRY(bp_check(h, "ce_dit_forward_ex", batch, out_elems, block0_out != nullptr || !h->capture.empty(), s));
  const int Bl = batch / h->bp.world, s0 = h->bp.rank * Bl;
  CE_TRY(forward_samples(h, sample_at(hidden_states, s0, c.in_channels * pixels * 2), timestep + s0,
                         sample_at(encoder_hidden_states, s0, (int64_t)text_len * c.text_dim * 2),
                         sample_at(encoder_hidden_states_image, s0, (int64_t)257 * c.image_dim * 2),
                         const_cast<void*>(sample_at(sample, s0, out_elems * 2)), Bl, frames, height, width, text_len, workspace,
                         workspace_bytes, nullptr, ctx_cache, ctx_cache_bytes, ctx_reuse, stream_v));
  return bp_exchange(h, sample, batch, out_elems, s);
}

// ---------------------------------------------------------------------------------------------- TeaCache
static bool aligned256(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 255) == 0; }

// The probe's scratch: sinusoid [B, freq_dim] f32, h1 and temb [B, D] f32, temb [B, D] bf16.
static int64_t probe_bytes(const ce_dit_config& c, int B, float** sin_emb, float** h1, float** temb_f32, bf16** temb_bf16, void* base) {
  Bump b(base);
  float* p0 = b.take<float>((int64_t)B * c.freq_dim);
  float* p1 = b.take<float>((int64_t)B * D_of(c));
  float* p2 = b.take<float>((int64_t)B * D_of(c));
  bf16* p3 = b.take<bf16>((int64_t)B * D_of(c));
  if (sin_emb) { *sin_emb = p0; *h1 = p1; *temb_f32 = p2; *temb_bf16 = p3; }
  return b.bytes();
}

int64_t ce_dit_teacache_probe_bytes(const ce_dit* h, int batch) {
  if (!h || batch < 1 || batch > 8) return -1;
  return probe_bytes(h->cfg, batch, nullptr, nullptr, nullptr, nullptr, nullptr);
}

int ce_dit_teacache_probe(ce_dit* h, const float* timestep, int batch, const void* prev_tproj, void* tproj_out, float* sums_out,
                          void* workspace, int64_t workspace_bytes, void* stream_v) {
  CE_REQUIRE(h && timestep && tproj_out && workspace, "ce_dit_teacache_probe: null argument");
  CE_REQUIRE(h->sp.world <= 1, "ce_dit_teacache_probe: TeaCache is not built for sequence parallelism");
  CE_REQUIRE(batch >= 1 && batch <= 8, "ce_dit_teacache_probe: batch must be 1..8");
  CE_REQUIRE(prev_tproj == nullptr || sums_out != nullptr, "ce_dit_teacache_probe: prev_tproj needs sums_out");
  CE_REQUIRE(aligned256(tproj_out) && aligned256(workspace) && aligned256(prev_tproj) && aligned256(sums_out),
             "ce_dit_teacache_probe: tproj_out, prev_tproj, sums_out and workspace must be 256-byte aligned");
  const int64_t need = probe_bytes(h->cfg, batch, nullptr, nullptr, nullptr, nullptr, nullptr);
  if (workspace_bytes < need)
    return fail(CE_ERR_WORKSPACE, "ce_dit_teacache_probe: workspace too small: need " + std::to_string(need) + " bytes, got " +
                                      std::to_string(workspace_bytes));
  int rc = check_device();
  if (rc) return rc;
  Weights W;
  if ((rc = resolve_weights(h, W))) return rc;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_v);
  float *sin_emb, *h1, *temb_f32;
  bf16* temb_bf16;
  probe_bytes(h->cfg, batch, &sin_emb, &h1, &temb_f32, &temb_bf16, workspace);
  bf16* tproj = reinterpret_cast<bf16*>(tproj_out);
  if ((rc = time_path(h, s, W, timestep, batch, sin_emb, h1, temb_f32, temb_bf16, tproj))) return rc;
  if (prev_tproj)
    LAUNCH(CAT_OTHER, 0.0, launch_l1_pair_sums(tproj, reinterpret_cast<const bf16*>(prev_tproj), (int64_t)batch * 6 * D_of(h->cfg), sums_out, s));
  return CE_OK;
}

int ce_dit_set_residual_record(ce_dit* h, void* buf, int64_t bytes) {
  CE_REQUIRE(h, "ce_dit_set_residual_record: null handle");
  CE_REQUIRE(buf == nullptr || (aligned256(buf) && bytes > 0), "ce_dit_set_residual_record: the buffer must be 256-byte aligned and non-empty");
  CE_REQUIRE(buf == nullptr || h->sp.world <= 1, "ce_dit_set_residual_record: TeaCache is not built for sequence parallelism");
  h->resid_rec = buf;
  h->resid_rec_bytes = buf ? bytes : 0;
  return CE_OK;
}

static int forward_cached_samples(ce_dit* h, const void* hidden_states, const float* timestep, const void* residual,
                                  int64_t residual_bytes, void* sample, int batch, int frames, int height, int width, int text_len,
                                  void* workspace, int64_t workspace_bytes, void* stream_v) {
  CE_REQUIRE(h && hidden_states && timestep && residual && sample && workspace, "ce_dit_forward_cached: null argument");
  CE_REQUIRE(h->sp.world <= 1, "ce_dit_forward_cached: TeaCache is not built for sequence parallelism");
  CE_REQUIRE(aligned256(residual) && aligned256(workspace), "ce_dit_forward_cached: residual and workspace must be 256-byte aligned");
  int rc = validate_geometry(h, batch, frames, height, width, text_len);
  if (rc) return rc;
  const ce_dit_config& c = h->cfg;
  const int B = batch, hp = height / c.patch_h, wp = width / c.patch_w;
  const int L = frames * hp * wp, M = B * L, D = D_of(c), Kp = c.in_channels * 4, No = c.out_channels * 4;
  CE_REQUIRE(residual_bytes >= (int64_t)M * D * (int64_t)sizeof(bf16),
             "ce_dit_forward_cached: residual too small for this geometry (batch * tokens * inner dim bf16)");
  Weights W;
  if ((rc = resolve_weights(h, W))) return rc;
  Workspace ws = carve(c, workspace, B, L, text_len, 257, W.fp8, h->attn_fp8);
  if (ws.bytes > workspace_bytes)
    return fail(CE_ERR_WORKSPACE, "ce_dit_forward_cached: workspace too small: need " + std::to_string(ws.bytes) + " bytes, got " +
                                      std::to_string(workspace_bytes));
  if ((rc = check_device())) return rc;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_v);
  h->fp8_q = ws.fp8_q;
  h->fp8_scale = ws.fp8_scale;
  const bool st = D % 256 == 0;
  const RowPartials px = st ? RowPartials{ws.stats_x, D / 256, D / 256, 256} : RowPartials{};
  h->launches = 0;
  // x = bf16(x0 + residual): the patch-embedding GEMM's residual epilogue, which also leaves the head LayerNorm's row statistics
  LAUNCH(CAT_OTHER, 0.0, launch_patchify(reinterpret_cast<const bf16*>(hidden_states), ws.patches, B, c.in_channels, frames, height, width, 0, L, s));
  GemmArgs g;
  g.epi = EPI_BIAS_RESID;
  g.resid = reinterpret_cast<const bf16*>(residual);
  g.ldr = D;
  if (st) {
    g.stats_out = ws.stats_x;
    g.stats_mode = 1;
  }
  if ((rc = linear(h, s, W.patch, ws.patches, M, D, Kp, ws.x, g))) return rc;
  if ((rc = time_path(h, s, W, timestep, B, ws.sin_emb, ws.h1, ws.temb_f32, ws.temb_bf16, nullptr))) return rc;
  LAUNCH(CAT_OTHER, 0.0, launch_add_table(W.head_table, 1, ws.temb_bf16, D, ws.modf, B, D, 2, s, /*chunk 1 = scale*/ 0x2u));
  LAUNCH(CAT_ROWS, 4.0 * M * D, launch_layernorm(ws.x, D, ws.xn, D, M, D, c.eps, ws.modf + D, ws.modf, 2 * D, L, nullptr, nullptr, 1, px, s));
  GemmArgs gh;
  gh.epi = EPI_BIAS;
  if ((rc = linear(h, s, W.proj_out, ws.xn, M, No, D, ws.yout, gh))) return rc;
  LAUNCH(CAT_OTHER, 0.0, launch_unpatchify(ws.yout, No, reinterpret_cast<bf16*>(sample), B, c.out_channels, frames, height, width, s));
  return CE_OK;
}

int ce_dit_forward_cached(ce_dit* h, const void* hidden_states, const float* timestep, const void* residual, int64_t residual_bytes,
                          void* sample, int batch, int frames, int height, int width, int text_len, void* workspace,
                          int64_t workspace_bytes, void* stream_v) {
  if (!h || h->bp.world <= 1)
    return forward_cached_samples(h, hidden_states, timestep, residual, residual_bytes, sample, batch, frames, height, width, text_len,
                                  workspace, workspace_bytes, stream_v);
  // batch split: the residual is this rank's, [batch / world * tokens, D]; a skipped call ends in the same exchange as a computed one
  CE_REQUIRE(hidden_states && timestep && residual && sample && workspace, "ce_dit_forward_cached: null argument");
  CE_TRY(validate_geometry(h, batch, frames, height, width, text_len));
  const ce_dit_config& c = h->cfg;
  const int64_t pixels = (int64_t)frames * height * width, out_elems = c.out_channels * pixels;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_v);
  CE_TRY(bp_check(h, "ce_dit_forward_cached", batch, out_elems, false, s));
  const int Bl = batch / h->bp.world, s0 = h->bp.rank * Bl;
  CE_TRY(forward_cached_samples(h, sample_at(hidden_states, s0, c.in_channels * pixels * 2), timestep + s0, residual, residual_bytes,
                                const_cast<void*>(sample_at(sample, s0, out_elems * 2)), Bl, frames, height, width, text_len, workspace,
                                workspace_bytes, stream_v));
  return bp_exchange(h, sample, batch, out_elems, s);
}

int64_t ce_dit_host_staging_bytes(const ce_dit* h, int batch, int frames, int height, int width, int text_len) {
  if (!h) return -1;
  return carve_staging(h->cfg, nullptr, batch, frames, height, width, text_len).bytes;
}

int64_t ce_dit_host_staging_sample_offset(const ce_dit* h, int batch, int frames, int height, int width, int text_len) {
  if (!h) return -1;
  return carve_staging(h->cfg, nullptr, batch, frames, height, width, text_len).sample_offset;
}

int ce_dit_forward_host(ce_dit* h, const void* hidden_states_host, const float* timestep_host, const void* encoder_hidden_states_host,
                        const void* encoder_hidden_states_image_host, void* sample_host, int batch, int frames, int height, int width,
                        int text_len, void* staging, int64_t staging_bytes, void* workspace, int64_t workspace_bytes, void* stream_v) {
  return ce_dit_forward_host_ex(h, hidden_states_host, timestep_host, encoder_hidden_states_host, encoder_hidden_states_image_host, sample_host,
                                batch, frames, height, width, text_len, staging, staging_bytes, workspace, workspace_bytes, nullptr, 0, 0, stream_v);
}

int ce_dit_forward_host_ex(ce_dit* h, const void* hidden_states_host, const float* timestep_host, const void* encoder_hidden_states_host,
                           const void* encoder_hidden_states_image_host, void* sample_host, int batch, int frames, int height, int width,
                           int text_len, void* staging, int64_t staging_bytes, void* workspace, int64_t workspace_bytes, void* ctx_cache,
                           int64_t ctx_cache_bytes, int ctx_reuse, void* stream_v) {
  CE_REQUIRE(h && hidden_states_host && timestep_host && encoder_hidden_states_host && sample_host && staging, "ce_dit_forward_host: null argument");
  const Staging st = carve_staging(h->cfg, staging, batch, frames, height, width, text_len);
  CE_REQUIRE(staging_bytes >= st.bytes, "ce_dit_forward_host: staging too small");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_v);
  CE_CHECK_CUDA(cudaMemcpyAsync(st.x, hidden_states_host, st.n_x * 2, cudaMemcpyHostToDevice, s));
  CE_CHECK_CUDA(cudaMemcpyAsync(st.timestep, timestep_host, batch * 4, cudaMemcpyHostToDevice, s));
  // the encoder states are copied every call (they are part of the call's inputs); with ctx_reuse the kernels do not read them
  CE_CHECK_CUDA(cudaMemcpyAsync(st.text, encoder_hidden_states_host, st.n_t * 2, cudaMemcpyHostToDevice, s));
  const bool image = encoder_hidden_states_image_host && st.n_i > 0;
  if (image) CE_CHECK_CUDA(cudaMemcpyAsync(st.image, encoder_hidden_states_image_host, st.n_i * 2, cudaMemcpyHostToDevice, s));
  int rc = ce_dit_forward_ex(h, st.x, st.timestep, st.text, image ? st.image : nullptr, st.sample, batch, frames, height, width,
                             text_len, workspace, workspace_bytes, nullptr, ctx_cache, ctx_cache_bytes, ctx_reuse, stream_v);
  if (rc) return rc;
  CE_CHECK_CUDA(cudaMemcpyAsync(sample_host, st.sample, st.n_o * 2, cudaMemcpyDeviceToHost, s));
  CE_CHECK_CUDA(cudaStreamSynchronize(s));
  return CE_OK;
}

// ---------------------------------------------------------------------------------------------- operator exports
int ce_linear_bf16(const void* A, int lda, const void* W, int ldw, const void* bias, void* out, int ldo, float* out_f32, int M, int N,
                   int K, int epilogue, const void* resid, int ldr, const float* gate, int gate_stride, int rows_per_batch, void* stream) {
  ce_linear_args a = {};
  a.A = A; a.lda = lda;
  a.W = W; a.ldw = ldw;
  a.M = M; a.N = N; a.K = K;
  a.out = out; a.ldo = ldo;
  a.out_f32 = out_f32;
  a.bias = bias;
  a.epilogue = epilogue;
  a.resid = resid; a.ldr = ldr;
  a.gate = gate; a.gate_stride = gate_stride; a.rows_per_batch = rows_per_batch;
  return ce_linear_ex_bf16(&a, stream);
}

static GemmArgs gemm_args_of(const ce_linear_args* a) {
  GemmArgs g;
  g.M = a->M; g.N = a->N; g.K = a->K;
  g.out = reinterpret_cast<bf16*>(a->out); g.ldo = a->ldo;
  g.out_f32 = a->out_f32; g.ld_f32 = a->ld_f32;
  g.bias = reinterpret_cast<const bf16*>(a->bias);
  g.bias_row = reinterpret_cast<const bf16*>(a->bias_row);
  g.epi = a->epilogue;
  g.resid = reinterpret_cast<const bf16*>(a->resid); g.ldr = a->ldr;
  g.gate = a->gate; g.gate_stride = a->gate_stride; g.rows_per_batch = a->rows_per_batch > 0 ? a->rows_per_batch : 1;
  g.stats_out = reinterpret_cast<float2*>(a->stats_out); g.stats_ld = a->stats_ld; g.stats_mode = a->stats_mode;
  g.group_m = a->group_m;
  return g;
}

// Test aid: one GEMM with every GemmArgs field, including the epilogue row statistics and the tile rasterisation.
int ce_linear_ex_bf16(const ce_linear_args* a, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  CE_REQUIRE(a != nullptr, "ce_linear_ex_bf16: null args");
  return launch_gemm_bf16(reinterpret_cast<const bf16*>(a->A), a->lda, reinterpret_cast<const bf16*>(a->W), a->ldw, gemm_args_of(a),
                          reinterpret_cast<cudaStream_t>(stream));
}

// Test aids of the FP8 mode: its GEMM with every epilogue option, and its row quantization.
int ce_linear_fp8_ex(const ce_linear_fp8_args* a, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  CE_REQUIRE(a != nullptr, "ce_linear_fp8_ex: null args");
  return launch_gemm_fp8(reinterpret_cast<const e4m3*>(a->base.A), a->base.lda, a->a_scale, reinterpret_cast<const e4m3*>(a->base.W),
                         a->base.ldw, a->w_scale, gemm_args_of(&a->base), reinterpret_cast<cudaStream_t>(stream));
}

int ce_linear_lora_bf16(const ce_linear_args* a, const void* term, int ldt, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  CE_REQUIRE(a != nullptr, "ce_linear_lora_bf16: null args");
  LoraAddend lo;
  lo.t = reinterpret_cast<const bf16*>(term);
  lo.ld = ldt;
  return launch_gemm_bf16(reinterpret_cast<const bf16*>(a->A), a->lda, reinterpret_cast<const bf16*>(a->W), a->ldw, gemm_args_of(a),
                          reinterpret_cast<cudaStream_t>(stream), &lo);
}

int ce_linear_lora_fp8(const ce_linear_fp8_args* a, const void* term, int ldt, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  CE_REQUIRE(a != nullptr, "ce_linear_lora_fp8: null args");
  LoraAddend lo;
  lo.t = reinterpret_cast<const bf16*>(term);
  lo.ld = ldt;
  return launch_gemm_fp8(reinterpret_cast<const e4m3*>(a->base.A), a->base.lda, a->a_scale, reinterpret_cast<const e4m3*>(a->base.W),
                         a->base.ldw, a->w_scale, gemm_args_of(&a->base), reinterpret_cast<cudaStream_t>(stream), &lo);
}

int ce_dit_set_lora(ce_dit* h, const void* const* a_cat, const void* const* b_cat, const int32_t* rank, int n) {
  CE_REQUIRE(h, "ce_dit_set_lora: null handle");
  const ce_dit_config& c = h->cfg;
  if (n == 0) {
    h->lora.clear();
    h->lora_rmax = 0;
    return CE_OK;
  }
  CE_REQUIRE(n == c.num_layers * CE_LORA_TARGETS && a_cat && b_cat && rank,
             "ce_dit_set_lora: the tables need num_layers * CE_LORA_TARGETS entries (or n = 0 to clear)");
  auto aligned16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  std::vector<LoraGemm> t(n);
  int rmax = 0;
  for (int i = 0; i < n; ++i) {
    const int target = i % CE_LORA_TARGETS;
    const std::string at = "ce_dit_set_lora: entry " + std::to_string(i) + " (layer " + std::to_string(i / CE_LORA_TARGETS) +
                           ", target " + std::to_string(target) + "): ";
    if (rank[i] < 0 || rank[i] % 8 != 0) return fail(CE_ERR_INVALID, at + "rank must be a multiple of 8 (zero-padded), 0 for none");
    if (rank[i] == 0) continue;
    if (!a_cat[i] || !b_cat[i] || !aligned16(a_cat[i]) || !aligned16(b_cat[i]))
      return fail(CE_ERR_INVALID, at + "a_cat / b_cat must be non-null, 16-byte aligned device pointers");
    if (target == LORA_ADD_KV && c.image_dim <= 0) return fail(CE_ERR_INVALID, at + "the model has no image projection (add_kv_proj)");
    t[i].a_cat = a_cat[i];
    t[i].b_cat = b_cat[i];
    t[i].rank = rank[i];
    rmax = std::max(rmax, (int)rank[i]);
  }
  if (rmax == 0) t.clear();
  h->lora = std::move(t);
  h->lora_rmax = rmax;
  return CE_OK;
}

int ce_dit_set_attention_fp8(ce_dit* h, int enabled) {
  CE_REQUIRE(h, "ce_dit_set_attention_fp8: null handle");
  h->attn_fp8 = enabled != 0;
  return CE_OK;
}

// Test aids of the FP8 self-attention: its two quantizers and the attention on their outputs.
int ce_quantize_heads_fp8(const void* x, int ldx, int rows, int heads, void* q, int ldq, float* scale, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  return launch_quantize_heads_fp8(reinterpret_cast<const bf16*>(x), ldx, rows, heads, reinterpret_cast<uint8_t*>(q), ldq, scale,
                                   reinterpret_cast<cudaStream_t>(stream));
}

int ce_quantize_v_fp8(const void* v, int ldv, int B, int L, int H, void* vt, int Lpad, float* scale, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  return launch_quantize_v_fp8(reinterpret_cast<const bf16*>(v), ldv, B, L, H, reinterpret_cast<uint8_t*>(vt), Lpad, scale,
                               reinterpret_cast<cudaStream_t>(stream));
}

int ce_attention_fp8(const void* q, const void* k, int ldqk, const float* q_scale, const float* k_scale, int lds, const void* vt, int Lpad,
                     const float* v_scale, void* out, int ldo, int B, int H, int L, float scale, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  AttnFp8Args a;
  a.B = B; a.H = H; a.L = L;
  a.q = reinterpret_cast<const uint8_t*>(q); a.k = reinterpret_cast<const uint8_t*>(k); a.ldqk = ldqk;
  a.q_scale = q_scale; a.k_scale = k_scale; a.lds = lds;
  a.vt = reinterpret_cast<const uint8_t*>(vt); a.Lpad = Lpad; a.v_scale = v_scale;
  a.out = reinterpret_cast<bf16*>(out); a.ldo = ldo;
  a.scale = scale;
  return launch_attention_fp8(a, reinterpret_cast<cudaStream_t>(stream));
}

int ce_quantize_rows_fp8(const void* x, int ldx, int rows, int K, void* q, int ldq, float* scale, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  return launch_quantize_rows_fp8(reinterpret_cast<const bf16*>(x), ldx, rows, K, reinterpret_cast<uint8_t*>(q), ldq, scale,
                                  reinterpret_cast<cudaStream_t>(stream));
}

static std::atomic<long long*> g_attn_timing{nullptr};   // process-wide; read by calls from any host thread
// Profiling aid: subsequent ce_attention_bf16 calls record the phase cycles of the first consumer thread of block 0 into `buf`
// ([16] int64 on the device); pass NULL to stop.
int ce_debug_attention_timing(long long* buf) {
  g_attn_timing.store(buf);
  return CE_OK;
}

// Test and measurement aid: the schedule of the bf16 attention kernel for later ce_attention_bf16 / ce_attention_dual_bf16 calls
// (process-wide, like the timing hook).  The DiT forward does not read it: it always runs the pipelined schedule.
static std::atomic<bool> g_attn_serial{false};
int ce_debug_attention_kernel(int version) {
  if (version != -1 && version != 0 && version != 1)
    return ce::fail(ce::CE_ERR_INVALID, "attention kernel version must be -1, 0 (pipelined) or 1 (serial)");
  g_attn_serial.store(version == 1);
  return CE_OK;
}

int ce_attention_bf16(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, void* out, int ldo, int B, int H, int Lq,
                      int Lk, float scale, int accumulate, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  AttnArgs a;
  a.B = B; a.H = H; a.Lq = Lq; a.Lk = Lk;
  a.q = reinterpret_cast<const bf16*>(q); a.ldq = ldq;
  a.k = reinterpret_cast<const bf16*>(k); a.ldk = ldk;
  a.v = reinterpret_cast<const bf16*>(v); a.ldv = ldv;
  a.out = reinterpret_cast<bf16*>(out); a.ldo = ldo;
  a.scale = scale;
  a.accumulate = accumulate;
  a.timing = g_attn_timing.load();
  return launch_attention(a, reinterpret_cast<cudaStream_t>(stream), !g_attn_serial.load());
}

int ce_attention_dual_bf16(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, const void* k2, int ldk2, const void* v2,
                           int ldv2, void* out, int ldo, int B, int H, int Lq, int Lk, int Lk2, float scale, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  AttnArgs a;
  a.B = B; a.H = H; a.Lq = Lq; a.Lk = Lk; a.Lk2 = Lk2;
  a.q = reinterpret_cast<const bf16*>(q); a.ldq = ldq;
  a.k = reinterpret_cast<const bf16*>(k); a.ldk = ldk;
  a.v = reinterpret_cast<const bf16*>(v); a.ldv = ldv;
  a.k2 = reinterpret_cast<const bf16*>(k2); a.ldk2 = ldk2;
  a.v2 = reinterpret_cast<const bf16*>(v2); a.ldv2 = ldv2;
  a.out = reinterpret_cast<bf16*>(out); a.ldo = ldo;
  a.scale = scale;
  return launch_attention(a, reinterpret_cast<cudaStream_t>(stream), !g_attn_serial.load());
}

int ce_layernorm_bf16(const void* x, int ldx, void* y, int ldy, int rows, int D, float eps, const float* scale, const float* shift,
                      int mod_stride, int rows_per_batch, const float* weight, const float* bias, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  return launch_layernorm(reinterpret_cast<const bf16*>(x), ldx, reinterpret_cast<bf16*>(y), ldy, rows, D, eps, scale, shift, mod_stride,
                          rows_per_batch, weight, bias, 0, RowPartials{}, reinterpret_cast<cudaStream_t>(stream));
}

int ce_rmsnorm_rope_bf16(void* x, int ldx, int rows, int D, float eps, const void* weight, const float* rope_cos, const float* rope_sin,
                         int L, int head_dim, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  return launch_rmsnorm_rope(reinterpret_cast<bf16*>(x), ldx, rows, D, eps, reinterpret_cast<const bf16*>(weight), nullptr, 1, rope_cos,
                             rope_sin, L, head_dim, RowPartials{}, reinterpret_cast<cudaStream_t>(stream));
}

// Test aids: the two row kernels with their statistics from GEMM epilogue partials (GemmArgs::stats_out), or reduced in the kernel
// when stats is null.
int ce_layernorm_stats_bf16(const void* x, int ldx, void* y, int ldy, int rows, int D, float eps, const float* scale, const float* shift,
                            int mod_stride, int rows_per_batch, const float* weight, const float* bias, int scale_is_1p, const float* stats,
                            int stats_ld, int tiles, int tile_n, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  return launch_layernorm(reinterpret_cast<const bf16*>(x), ldx, reinterpret_cast<bf16*>(y), ldy, rows, D, eps, scale, shift, mod_stride,
                          rows_per_batch, weight, bias, scale_is_1p, RowPartials{reinterpret_cast<const float2*>(stats), stats_ld, tiles, tile_n},
                          reinterpret_cast<cudaStream_t>(stream));
}

int ce_rmsnorm_rope_stats_bf16(void* x, int ldx, int rows, int D, float eps, const void* weight0, const void* weight1, int nmat,
                               const float* rope_cos, const float* rope_sin, int L, int head_dim, const float* stats, int stats_ld, int tiles,
                               void* stream) {
  int rc = check_device();
  if (rc) return rc;
  return launch_rmsnorm_rope(reinterpret_cast<bf16*>(x), ldx, rows, D, eps, reinterpret_cast<const bf16*>(weight0),
                             reinterpret_cast<const bf16*>(weight1), nmat, rope_cos, rope_sin, L, head_dim,
                             RowPartials{reinterpret_cast<const float2*>(stats), stats_ld, tiles, 0}, reinterpret_cast<cudaStream_t>(stream));
}

int ce_rope_table_host(int head_dim, int frames, int height_patches, int width_patches, int max_seq_len, int temporal_skip_len, float theta,
                       float* cos_out_host, float* sin_out_host) {
  CE_REQUIRE(cos_out_host && sin_out_host, "ce_rope_table_host: null output");
  std::vector<float> cs, sn;
  int rc = rope_table_host(head_dim, frames, height_patches, width_patches, max_seq_len, temporal_skip_len, (double)theta, cs, sn);
  if (rc) return rc;
  for (size_t i = 0; i < cs.size(); ++i) {
    cos_out_host[i] = cs[i];
    sin_out_host[i] = sn[i];
  }
  return CE_OK;
}

}  // extern "C"
