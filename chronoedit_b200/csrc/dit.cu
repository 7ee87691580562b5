// ce_dit: the ChronoEdit DiT per-step forward as a chain of hand-written sm_90a kernels behind the C ABI.
//
// Mirrors ChronoEditTransformer3DModel.forward (/root/reference/chronoedit_diffusers/transformer_chronoedit.py:397-476)
// with every rounding point of the reference's bf16 path kept (SURVEY.md section 8a).  Per block
// (ChronoEditTransformerBlock.forward, :267-295) the launches are:
//   LN+modulate -> QKV GEMM (one launch, N=3D) -> RMSNorm+RoPE(q), RMSNorm+RoPE(k) -> attention -> out-proj GEMM with
//   gate*y+x epilogue -> LN(affine) -> q GEMM -> RMSNorm(q) -> [text k|v GEMM, RMSNorm(k)] [image k|v GEMM, RMSNorm(k)]
//   -> attention(text) -> attention(image, += ) -> out-proj GEMM with y+x epilogue -> LN+modulate -> FFN-1 GEMM with
//   bias+GELU epilogue -> FFN-2 GEMM with gate*y+x epilogue.
#include <math.h>
#include <stdlib.h>

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
}

using namespace ce;

struct WeightRef {
  const void* ptr = nullptr;
  int dtype = 0;  // 0 bf16, 1 fp32, 2 e4m3 (FP8 mode's block weights)
  int64_t numel = 0;
};

struct ce_dit {
  ce_dit_config cfg;
  std::map<std::string, WeightRef> w;
  std::map<std::string, WeightRef> w32;   // fp32 validation mode: every parameter in fp32 under its reference name
  // RoPE tables, cached per latent geometry
  int rope_f = 0, rope_h = 0, rope_w = 0, rope_dev = -1;
  float* rope_cos = nullptr;
  float* rope_sin = nullptr;
  int64_t launches = 0;
  // parity aid: output of selected blocks copied out (ce_dit_set_capture)
  std::vector<std::pair<int, void*>> capture;
  // sequence parallelism (ce_dit_sp_configure): world == 1 means off
  ce::SeqPar sp;
  // optional per-category device timing (CUDA events on the launch stream around every kernel)
  bool profiling = false;
  std::vector<cudaEvent_t> ev;       // pairs (begin, end)
  std::vector<int> ev_cat;
  std::vector<double> ev_work;       // algorithmic flops (cat 0,1) or bytes (cat 2) of the launch
  size_t ev_used = 0;
  // FP8 mode: the current forward's workspace slices for a GEMM's quantized A operand and its row scales
  uint8_t* fp8_q = nullptr;
  float* fp8_scale = nullptr;
};

enum { CAT_GEMM = 0, CAT_ATTN = 1, CAT_ROWS = 2, CAT_OTHER = 3, NUM_CATS = 4 };

namespace {

int D_of(const ce_dit_config& c) { return c.num_attention_heads * c.attention_head_dim; }

struct Bump {
  uint8_t* base;
  int64_t off = 0;
  explicit Bump(void* b) : base(reinterpret_cast<uint8_t*>(b)) {}
  template <typename T>
  T* take(int64_t n) {
    off = (off + 255) & ~int64_t(255);
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += n * (int64_t)sizeof(T);
    return p;
  }
};

struct Workspace {
  bf16 *x, *xn, *qkv, *attn, *hbuf, *patches, *yout;
  bf16 *text1, *ctx_text, *img0, *img1, *img2, *ctx_img, *kv_text, *kv_img;
  bf16 *temb_bf16, *tproj;
  float *sin_emb, *h1, *temb_f32, *mod, *modf;
  float2 *stats_x, *stats_qkv, *stats_q2;   // epilogue row statistics (GemmArgs::stats_out): [M, D/256], [M, 3D/256], [M, D/256]
  uint8_t* fp8_q;     // FP8 mode only: [M, max(D, F)] e4m3, the A operand of one block GEMM at a time
  float* fp8_scale;   //                [M] its row scales
  int64_t bytes;
};

Workspace carve(const ce_dit_config& c, void* base, int B, int L, int Lt, int Li, bool fp8) {
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
  w.bytes = (b.off + 255) & ~int64_t(255);
  return w;
}

struct WeightSpec {
  std::string name;
  int dtype;
  int64_t numel;
};

// The handle holds FP8 weights when layer 0's QKV weight was registered as e4m3; ce_dit_weights_complete checks the rest.
bool holds_fp8(const ce_dit* h) {
  auto it = h->w.find("blocks.0.attn1.to_qkv.weight");
  return it != h->w.end() && it->second.dtype == 2;
}

std::vector<WeightSpec> required_weights(const ce_dit_config& c, bool fp8) {
  const int64_t D = D_of(c), F = c.ffn_dim;
  const int64_t Kp = (int64_t)c.in_channels * c.patch_t * c.patch_h * c.patch_w;
  const int64_t No = (int64_t)c.out_channels * c.patch_t * c.patch_h * c.patch_w;
  std::vector<WeightSpec> v;
  auto add = [&](const std::string& n, int dt, int64_t ne) { v.push_back({n, dt, ne}); };
  auto add_block_linear = [&](const std::string& m, int64_t N, int64_t K) {   // one of the six FP8-mode GEMMs: [N, K]
    if (fp8) {
      add(m + ".weight", 2, N * K);
      add(m + ".weight_scale", 1, N);
    } else {
      add(m + ".weight", 0, N * K);
    }
  };
  add("patch_embedding.weight", 0, D * Kp);
  add("patch_embedding.bias", 0, D);
  const std::string ce_ = "condition_embedder.";
  add(ce_ + "time_embedder.linear_1.weight", 1, D * c.freq_dim);
  add(ce_ + "time_embedder.linear_1.bias", 1, D);
  add(ce_ + "time_embedder.linear_2.weight", 1, D * D);
  add(ce_ + "time_embedder.linear_2.bias", 1, D);
  add(ce_ + "time_proj.weight", 0, 6 * D * D);
  add(ce_ + "time_proj.bias", 0, 6 * D);
  add(ce_ + "text_embedder.linear_1.weight", 0, D * c.text_dim);
  add(ce_ + "text_embedder.linear_1.bias", 0, D);
  add(ce_ + "text_embedder.linear_2.weight", 0, D * D);
  add(ce_ + "text_embedder.linear_2.bias", 0, D);
  if (c.image_dim > 0) {
    const int64_t I = c.image_dim;
    add(ce_ + "image_embedder.norm1.weight", 1, I);
    add(ce_ + "image_embedder.norm1.bias", 1, I);
    add(ce_ + "image_embedder.ff.net.0.proj.weight", 0, I * I);
    add(ce_ + "image_embedder.ff.net.0.proj.bias", 0, I);
    add(ce_ + "image_embedder.ff.net.2.weight", 0, D * I);
    add(ce_ + "image_embedder.ff.net.2.bias", 0, D);
    add(ce_ + "image_embedder.norm2.weight", 1, D);
    add(ce_ + "image_embedder.norm2.bias", 1, D);
  }
  add("blocks.scale_shift_table", 1, (int64_t)c.num_layers * 6 * D);
  for (int i = 0; i < c.num_layers; ++i) {
    const std::string p = "blocks." + std::to_string(i) + ".";
    add_block_linear(p + "attn1.to_qkv", 3 * D, D);
    add(p + "attn1.to_qkv.bias", 0, 3 * D);
    add(p + "attn1.norm_q.weight", 0, D);
    add(p + "attn1.norm_k.weight", 0, D);
    add_block_linear(p + "attn1.to_out.0", D, D);
    add(p + "attn1.to_out.0.bias", 0, D);
    add(p + "norm2.weight", 1, D);
    add(p + "norm2.bias", 1, D);
    add_block_linear(p + "attn2.to_q", D, D);
    add(p + "attn2.to_q.bias", 0, D);
    add(p + "attn2.norm_q.weight", 0, D);
    add(p + "attn2.norm_k.weight", 0, D);
    add(p + "attn2.to_kv.weight", 0, 2 * D * D);
    add(p + "attn2.to_kv.bias", 0, 2 * D);
    if (c.image_dim > 0) {
      add(p + "attn2.add_kv_proj.weight", 0, 2 * D * (int64_t)c.added_kv_proj_dim);
      add(p + "attn2.add_kv_proj.bias", 0, 2 * D);
      add(p + "attn2.norm_added_k.weight", 0, D);
    }
    add_block_linear(p + "attn2.to_out.0", D, D);
    add(p + "attn2.to_out.0.bias", 0, D);
    add_block_linear(p + "ffn.net.0.proj", F, D);
    add(p + "ffn.net.0.proj.bias", 0, F);
    add_block_linear(p + "ffn.net.2", D, F);
    add(p + "ffn.net.2.bias", 0, D);
  }
  add("scale_shift_table", 1, 2 * D);
  add("proj_out.weight", 0, No * D);
  add("proj_out.bias", 0, No);
  return v;
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

#define W_BF16(name) reinterpret_cast<const bf16*>(h->w.at(name).ptr)
#define W_F32(name) reinterpret_cast<const float*>(h->w.at(name).ptr)
static inline void prof_begin(ce_dit* h, int cat, double work, cudaStream_t s) {
  if (!h->profiling || h->ev_used + 2 > h->ev.size()) return;
  cudaEventRecord(h->ev[h->ev_used], s);
  h->ev_cat[h->ev_used / 2] = cat;
  h->ev_work[h->ev_used / 2] = work;
}
static inline void prof_end(ce_dit* h, cudaStream_t s) {
  if (!h->profiling || h->ev_used + 2 > h->ev.size()) return;
  cudaEventRecord(h->ev[h->ev_used + 1], s);
  h->ev_used += 2;
}
#define RUNC(cat, work, call)          \
  do {                                 \
    prof_begin(h, (cat), (work), s);   \
    int _rc = (call);                  \
    if (_rc) return _rc;               \
    prof_end(h, s);                    \
    ++h->launches;                     \
  } while (0)
#define RUN(call) RUNC(CAT_OTHER, 0.0, call)
#define RUN2(call)           \
  do {                       \
    int _rc = (call);        \
    if (_rc) return _rc;     \
    ++h->launches;           \
  } while (0)

static int linear(ce_dit* h, const bf16* A, int lda, const std::string& wname, int M, int N, int K, bf16* out, int ldo, int epi,
                  const bf16* resid, int ldr, const float* gate, int gate_stride, int rows_per_batch, cudaStream_t s,
                  float2* stats_out = nullptr, int stats_mode = 0) {
  GemmArgs g;
  if (stats_out) {
    g.stats_out = stats_out;
    g.stats_mode = stats_mode;
    g.stats_ld = (N + gemm_tile_n(N) - 1) / gemm_tile_n(N);
  }
  g.M = M; g.N = N; g.K = K;
  g.out = out; g.ldo = ldo;
  g.bias = W_BF16(wname + ".bias");
  g.epi = epi;
  g.resid = resid; g.ldr = ldr;
  g.gate = gate; g.gate_stride = gate_stride; g.rows_per_batch = rows_per_batch;
  const WeightRef& w = h->w.at(wname + ".weight");
  if (w.dtype == 2) {   // FP8 mode: quantize A per row into the workspace, then the e4m3 GEMM (one launch more than bf16)
    prof_begin(h, CAT_ROWS, 3.0 * M * (double)K + 4.0 * M, s);
    int rc = launch_quantize_rows_fp8(A, lda, M, K, h->fp8_q, K, h->fp8_scale, s);
    if (rc) return rc;
    prof_end(h, s);
    ++h->launches;
    prof_begin(h, CAT_GEMM, 2.0 * M * (double)N * K, s);
    rc = launch_gemm_fp8(reinterpret_cast<const e4m3*>(h->fp8_q), K, h->fp8_scale, reinterpret_cast<const e4m3*>(w.ptr), K,
                         W_F32(wname + ".weight_scale"), g, s);
    if (rc == 0) prof_end(h, s);
    return rc;
  }
  prof_begin(h, CAT_GEMM, 2.0 * M * (double)N * K, s);
  int rc = launch_gemm_bf16(A, lda, reinterpret_cast<const bf16*>(w.ptr), K, g, s);
  if (rc == 0) prof_end(h, s);
  return rc;
}
static int attention(ce_dit* h, const AttnArgs& a, cudaStream_t s) {
  prof_begin(h, CAT_ATTN, 4.0 * a.B * a.H * (double)a.Lq * (a.Lk + a.Lk2) * a.head_dim, s);
  int rc = launch_attention(a, s);
  if (rc == 0) prof_end(h, s);
  return rc;
}

// ---- internals shared with dit_fp32.cu
const float* ce_dit_internal_weight_f32(const ce_dit* h, const std::string& name, int64_t expect_numel) {
  auto it = h->w32.find(name);
  if (it == h->w32.end() || it->second.numel != expect_numel) return nullptr;
  return reinterpret_cast<const float*>(it->second.ptr);
}
int ce_dit_internal_rope(ce_dit* h, int frames, int hp, int wp, cudaStream_t s, const float** cos_out, const float** sin_out) {
  int rc = ensure_rope(h, frames, hp, wp, s);
  if (rc) return rc;
  *cos_out = h->rope_cos;
  *sin_out = h->rope_sin;
  return CE_OK;
}
const ce_dit_config* ce_dit_internal_config(const ce_dit* h) { return &h->cfg; }

extern "C" {

int ce_abi_version(void) { return CE_ABI_VERSION; }

int ce_dit_set_weight_fp32(ce_dit* h, const char* name, const float* ptr, int64_t numel) {
  CE_REQUIRE(h && name && ptr, "ce_dit_set_weight_fp32: null argument");
  CE_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "ce_dit_set_weight_fp32: pointer must be 16-byte aligned");
  WeightRef r;
  r.ptr = ptr;
  r.dtype = 1;
  r.numel = numel;
  h->w32[name] = r;
  return CE_OK;
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
  CE_REQUIRE(h && name && ptr, "ce_dit_set_weight: null argument");
  CE_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "ce_dit_set_weight: pointer must be 16-byte aligned");
  WeightRef r;
  r.ptr = ptr;
  r.dtype = dtype;
  r.numel = numel;
  h->w[name] = r;
  return CE_OK;
}

int ce_dit_weights_complete(const ce_dit* h) {
  CE_REQUIRE(h, "null handle");
  const bool fp8 = holds_fp8(h);
  for (const WeightSpec& s : required_weights(h->cfg, fp8)) {
    auto it = h->w.find(s.name);
    if (it == h->w.end()) return fail(CE_ERR_MISSING_WEIGHT, "missing weight: " + s.name);
    if (it->second.dtype != s.dtype)
      return fail(CE_ERR_MISSING_WEIGHT, "weight " + s.name + " has dtype " + std::to_string(it->second.dtype) + ", expected " +
                                             std::to_string(s.dtype) + " (0 bf16, 1 fp32, 2 e4m3" +
                                             (s.dtype == 2 || it->second.dtype == 2
                                                  ? "; the six block GEMM weights of every layer are either all bf16 or all e4m3)"
                                                  : ")"));
    if (it->second.numel != s.numel)
      return fail(CE_ERR_MISSING_WEIGHT, "weight " + s.name + " has " + std::to_string(it->second.numel) + " elements, expected " +
                                             std::to_string(s.numel));
  }
  return CE_OK;
}

int64_t ce_dit_workspace_bytes(const ce_dit* h, int batch, int frames, int height, int width, int text_len) {
  if (!h || validate_geometry(h, batch, frames, height, width, text_len)) return -1;
  const int L = frames * (height / h->cfg.patch_h) * (width / h->cfg.patch_w);
  return carve(h->cfg, nullptr, batch, L, text_len, 257, holds_fp8(h)).bytes;
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
  if (world <= 1) {
    h->sp = SeqPar();
    return CE_OK;
  }
  CE_REQUIRE(world <= 8 && rank >= 0 && rank < world && region_ptrs && region_bytes > 0, "ce_dit_sp_configure: arguments");
  CE_REQUIRE(h->cfg.num_attention_heads % world == 0, "ce_dit_sp_configure: the head count must be divisible by the number of ranks");
  h->sp = SeqPar();
  h->sp.rank = rank;
  h->sp.world = world;
  h->sp.region_bytes = region_bytes;
  for (int w = 0; w < world; ++w) {
    CE_REQUIRE(region_ptrs[w] != nullptr, "ce_dit_sp_configure: null region pointer");
    h->sp.region[w] = reinterpret_cast<uint8_t*>(region_ptrs[w]);
  }
  return CE_OK;
}

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

int ce_dit_forward_ex(ce_dit* h, const void* hidden_states, const float* timestep, const void* encoder_hidden_states,
                      const void* encoder_hidden_states_image, void* sample, int batch, int frames, int height, int width,
                      int text_len, void* workspace, int64_t workspace_bytes, void* block0_out, void* ctx_cache,
                      int64_t ctx_cache_bytes, int ctx_reuse, void* stream_v) {
  CE_REQUIRE(h && hidden_states && timestep && encoder_hidden_states && sample && workspace, "ce_dit_forward: null argument");
  CE_REQUIRE(ctx_reuse == 0 || ctx_cache != nullptr, "ce_dit_forward_ex: ctx_reuse needs a context cache");
  int rc = check_device();
  if (rc) return rc;
  if ((rc = validate_geometry(h, batch, frames, height, width, text_len))) return rc;
  if ((rc = ce_dit_weights_complete(h))) return rc;
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
    CE_REQUIRE(Lfull % sp.world == 0 && D % 256 == 0, "sequence parallel: tokens must divide by the rank count and the width by 256");
    CE_REQUIRE(Lfull >= 256, "sequence parallel: at least 256 tokens (the self-attention kernel with the output scatter)");
    CE_REQUIRE(!h->profiling && h->capture.empty() && block0_out == nullptr, "sequence parallel: no per-launch profiling / block capture");
  }
  const int L = spx ? Lfull / sp.world : Lfull, tok0 = spx ? sp.rank * L : 0, M = B * L;
  const SpLayout lay = spx ? sp_layout(B, Lfull, D, No, sp.world) : SpLayout();
  if (spx && lay.bytes > sp.region_bytes) return fail(CE_ERR_WORKSPACE, "sequence parallel: peer region too small (ce_dit_sp_region_bytes)");
  const bool fp8 = holds_fp8(h);
  CE_REQUIRE(!(spx && fp8), "sequence parallelism is not built for FP8 weights: run the FP8 mode on one GPU");
  Workspace ws = carve(c, workspace, B, L, Lt, Li, fp8);
  if (ws.bytes > workspace_bytes)
    return fail(CE_ERR_WORKSPACE, "workspace too small: need " + std::to_string(ws.bytes) + " bytes, got " + std::to_string(workspace_bytes));
  CE_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "workspace must be 256-byte aligned");
  if ((rc = ensure_rope(h, frames, hp, wp, s))) return rc;   // always the full table [Lfull, 64]
  h->fp8_q = ws.fp8_q;
  h->fp8_scale = ws.fp8_scale;
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
  // Row statistics for the LayerNorms / RMSNorms come from the epilogue of the GEMM that wrote the row whenever the N tiles (256 wide)
  // line up with the q | k | v boundaries; the row kernels are then streaming passes (elementwise.cuh).  CE_DIT_STATS=0: the
  // round-1 kernels that reduce over the row themselves (A/B, and the path for widths that are not a multiple of 256).
  static const bool stats_env = [] {
    const char* e = getenv("CE_DIT_STATS");
    return !(e && e[0] == '0');
  }();
  const bool st = stats_env && D % 256 == 0 && D / 256 <= 32;
  const int tD = D / 256;
  auto ln = [&](const bf16* x, bf16* y, const float* scale, const float* shift, int mod_stride, int rpb, const float* w, const float* b, int is1p) {
    return st ? launch_layernorm_stats(x, D, y, D, M, D, c.eps, scale, shift, mod_stride, rpb, w, b, is1p, ws.stats_x, tD, tD, 256, s)
              : launch_layernorm(x, D, y, D, M, D, c.eps, scale, shift, mod_stride, rpb, w, b, s, is1p);
  };
  h->launches = 0;
  const float attn_scale = 1.0f / sqrtf((float)c.attention_head_dim);
  const std::string ce_ = "condition_embedder.";

  // ---- patch embedding (Conv3d k=s=(1,2,2) as im2row + GEMM, :429-430)
  if (spx) RUN(launch_patchify_range(reinterpret_cast<const bf16*>(hidden_states), ws.patches, B, c.in_channels, frames, height, width, tok0, L, s));
  else RUN(launch_patchify(reinterpret_cast<const bf16*>(hidden_states), ws.patches, B, c.in_channels, frames, height, width, s));
  RUN2(linear(h, ws.patches, Kp, "patch_embedding", M, D, Kp, ws.x, D, EPI_BIAS, nullptr, 0, nullptr, 0, 1, s, st ? ws.stats_x : nullptr, 1));

  // ---- condition embedder (:147-165)
  RUN(launch_timestep_sinusoid(timestep, ws.sin_emb, B, c.freq_dim, s));
  RUN(launch_small_linear(ws.sin_emb, c.freq_dim, W_F32(ce_ + "time_embedder.linear_1.weight"), W_F32(ce_ + "time_embedder.linear_1.bias"),
                          0, D, B, /*act=*/1, 0, ws.h1, nullptr, s));
  RUN(launch_small_linear(ws.h1, D, W_F32(ce_ + "time_embedder.linear_2.weight"), W_F32(ce_ + "time_embedder.linear_2.bias"), 0, D, B, 0, 0,
                          ws.temb_f32, ws.temb_bf16, s));  // temb = (...).type_as(bf16)
  RUN(launch_small_linear(ws.temb_f32, D, W_BF16(ce_ + "time_proj.weight"), W_BF16(ce_ + "time_proj.bias"), 1, 6 * D, B, 0, /*in_silu_bf16=*/1,
                          nullptr, ws.tproj, s));
  RUN(launch_add_table(W_F32("blocks.scale_shift_table"), c.num_layers, ws.tproj, 6 * D, ws.mod, B, D, 6, s, /*scale chunks 1,4 -> 1+scale*/ 0x12u));
  RUN(launch_add_table(W_F32("scale_shift_table"), 1, ws.temb_bf16, D, ws.modf, B, D, 2, s, /*chunk 1 = scale*/ 0x2u));
  // text: Linear -> GELU(tanh) -> Linear
  if (ctx_compute) {
  RUN2(linear(h, reinterpret_cast<const bf16*>(encoder_hidden_states), c.text_dim, ce_ + "text_embedder.linear_1", B * Lt, D, c.text_dim,
             ws.text1, D, EPI_BIAS_GELU_TANH, nullptr, 0, nullptr, 0, 1, s));
  RUN2(linear(h, ws.text1, D, ce_ + "text_embedder.linear_2", B * Lt, D, D, ws.ctx_text, D, EPI_BIAS, nullptr, 0, nullptr, 0, 1, s));
  }
  if (ctx_compute && c.image_dim > 0) {  // image: FP32LayerNorm -> Linear -> GELU(erf) -> Linear -> FP32LayerNorm (:111-123)
    const int I = c.image_dim;
    RUN(launch_layernorm(reinterpret_cast<const bf16*>(encoder_hidden_states_image), I, ws.img0, I, B * Li, I, 1e-5f, nullptr, nullptr, 0, 0,
                         W_F32(ce_ + "image_embedder.norm1.weight"), W_F32(ce_ + "image_embedder.norm1.bias"), s));
    RUN2(linear(h, ws.img0, I, ce_ + "image_embedder.ff.net.0.proj", B * Li, I, I, ws.img1, I, EPI_BIAS_GELU_ERF, nullptr, 0, nullptr, 0, 1, s));
    RUN2(linear(h, ws.img1, I, ce_ + "image_embedder.ff.net.2", B * Li, D, I, ws.img2, D, EPI_BIAS, nullptr, 0, nullptr, 0, 1, s));
    RUN(launch_layernorm(ws.img2, D, ws.ctx_img, D, B * Li, D, 1e-5f, nullptr, nullptr, 0, 0, W_F32(ce_ + "image_embedder.norm2.weight"),
                         W_F32(ce_ + "image_embedder.norm2.bias"), s));
  }

  // ---- transformer blocks (:447-448)
  for (int i = 0; i < c.num_layers; ++i) {
    const std::string p = "blocks." + std::to_string(i) + ".";
    const float* mod = ws.mod + (size_t)i * B * 6 * D;  // [B, 6, D]: shift, scale, gate, c_shift, c_scale, c_gate
    // 1. self-attention
    RUNC(CAT_ROWS, 4.0 * M * D, ln(ws.x, ws.xn, mod + 1 * D, mod + 0 * D, 6 * D, L, nullptr, nullptr, 1));
    RUN2(linear(h, ws.xn, D, p + "attn1.to_qkv", M, 3 * D, D, ws.qkv, 3 * D, EPI_BIAS, nullptr, 0, nullptr, 0, 1, s, st ? ws.stats_qkv : nullptr, 2));
    const bf16* attn_in = ws.attn;
    if (spx) {
      // heads <-> tokens exchange by peer stores: q | k normalised + rotated and scattered by head, v scattered by head, barrier,
      // attention over ALL tokens for this rank's heads with the output rows scattered back to the ranks that own the tokens, barrier
      const int Hl = H / sp.world, Dl = D / sp.world;
      SpScatter sc;
      sc.world = sp.world; sc.heads_per_rank = Hl; sc.L_total = Lfull; sc.rows_per_batch = L; sc.tok0 = tok0;
      bf16* vdst[8];
      for (int w = 0; w < sp.world; ++w) {
        sc.dst[0][w] = reinterpret_cast<bf16*>(sp.region[w] + lay.q);
        sc.dst[1][w] = reinterpret_cast<bf16*>(sp.region[w] + lay.k);
        vdst[w] = reinterpret_cast<bf16*>(sp.region[w] + lay.v);
      }
      RUN(launch_rmsnorm_rope_stats(ws.qkv, 3 * D, M, D, c.eps, W_BF16(p + "attn1.norm_q.weight"), W_BF16(p + "attn1.norm_k.weight"), 2, h->rope_cos,
                                    h->rope_sin, Lfull, c.attention_head_dim, ws.stats_qkv, 3 * tD, tD, s, &sc));
      RUN(launch_sp_scatter_cols(ws.qkv + 2 * D, 3 * D, B, L, D, vdst, sp.world, Dl, Lfull, tok0, s));
      RUN(launch_sp_barrier(sp, lay, s));
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
      RUN2(attention(h, a, s));
      RUN(launch_sp_barrier(sp, lay, s));
      attn_in = reinterpret_cast<const bf16*>(sp.region[sp.rank] + lay.attn);
    } else {
    if (st) {
      RUNC(CAT_ROWS, 8.0 * M * D, launch_rmsnorm_rope_stats(ws.qkv, 3 * D, M, D, c.eps, W_BF16(p + "attn1.norm_q.weight"), W_BF16(p + "attn1.norm_k.weight"), 2,
                                                             h->rope_cos, h->rope_sin, L, c.attention_head_dim, ws.stats_qkv, 3 * tD, tD, s));
    } else {
      RUNC(CAT_ROWS, 4.0 * M * D, launch_rmsnorm_rope(ws.qkv, 3 * D, M, D, c.eps, W_BF16(p + "attn1.norm_q.weight"), h->rope_cos, h->rope_sin, L, c.attention_head_dim, s));
      RUNC(CAT_ROWS, 4.0 * M * D, launch_rmsnorm_rope(ws.qkv + D, 3 * D, M, D, c.eps, W_BF16(p + "attn1.norm_k.weight"), h->rope_cos, h->rope_sin, L, c.attention_head_dim, s));
    }
    {
      AttnArgs a;
      a.B = B; a.H = H; a.Lq = L; a.Lk = L;
      a.q = ws.qkv; a.ldq = 3 * D;
      a.k = ws.qkv + D; a.ldk = 3 * D;
      a.v = ws.qkv + 2 * D; a.ldv = 3 * D;
      a.out = ws.attn; a.ldo = D;
      a.scale = attn_scale;
      RUN2(attention(h, a, s));
    }
    }
    RUN2(linear(h, attn_in, D, p + "attn1.to_out.0", M, D, D, ws.x, D, EPI_BIAS_GATE_RESID, ws.x, D, mod + 2 * D, 6 * D, L, s, st ? ws.stats_x : nullptr, 1));
    // 2. cross-attention
    RUNC(CAT_ROWS, 4.0 * M * D, ln(ws.x, ws.xn, nullptr, nullptr, 0, 0, W_F32(p + "norm2.weight"), W_F32(p + "norm2.bias"), 0));
    bf16* q2 = ws.qkv;  // [M, D]
    RUN2(linear(h, ws.xn, D, p + "attn2.to_q", M, D, D, q2, D, EPI_BIAS, nullptr, 0, nullptr, 0, 1, s, st ? ws.stats_q2 : nullptr, 2));
    if (st) {
      RUNC(CAT_ROWS, 4.0 * M * D, launch_rmsnorm_rope_stats(q2, D, M, D, c.eps, W_BF16(p + "attn2.norm_q.weight"), nullptr, 1, nullptr, nullptr, 0,
                                                             c.attention_head_dim, ws.stats_q2, tD, tD, s));
    } else {
      RUNC(CAT_ROWS, 4.0 * M * D, launch_rmsnorm_rope(q2, D, M, D, c.eps, W_BF16(p + "attn2.norm_q.weight"), nullptr, nullptr, 0, c.attention_head_dim, s));
    }
    bf16* kv_text = kv_text_of(i);
    bf16* kv_img = kv_img_of(i);
    if (ctx_compute) {
      RUN2(linear(h, ws.ctx_text, D, p + "attn2.to_kv", B * Lt, 2 * D, D, kv_text, 2 * D, EPI_BIAS, nullptr, 0, nullptr, 0, 1, s));
      RUN(launch_rmsnorm_rope(kv_text, 2 * D, B * Lt, D, c.eps, W_BF16(p + "attn2.norm_k.weight"), nullptr, nullptr, 0, c.attention_head_dim, s));
      if (c.image_dim > 0) {
        RUN2(linear(h, ws.ctx_img, D, p + "attn2.add_kv_proj", B * Li, 2 * D, D, kv_img, 2 * D, EPI_BIAS, nullptr, 0, nullptr, 0, 1, s));
        RUN(launch_rmsnorm_rope(kv_img, 2 * D, B * Li, D, c.eps, W_BF16(p + "attn2.norm_added_k.weight"), nullptr, nullptr, 0, c.attention_head_dim, s));
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
      RUN2(attention(h, a, s));
    }
    RUN2(linear(h, ws.attn, D, p + "attn2.to_out.0", M, D, D, ws.x, D, EPI_BIAS_RESID, ws.x, D, nullptr, 0, 1, s, st ? ws.stats_x : nullptr, 1));
    // 3. feed-forward
    RUNC(CAT_ROWS, 4.0 * M * D, ln(ws.x, ws.xn, mod + 4 * D, mod + 3 * D, 6 * D, L, nullptr, nullptr, 1));
    RUN2(linear(h, ws.xn, D, p + "ffn.net.0.proj", M, F, D, ws.hbuf, F, EPI_BIAS_GELU_TANH, nullptr, 0, nullptr, 0, 1, s));
    RUN2(linear(h, ws.hbuf, F, p + "ffn.net.2", M, D, F, ws.x, D, EPI_BIAS_GATE_RESID, ws.x, D, mod + 5 * D, 6 * D, L, s, st ? ws.stats_x : nullptr, 1));
    if (i == 0 && block0_out)
      CE_CHECK_CUDA(cudaMemcpyAsync(block0_out, ws.x, (size_t)M * D * sizeof(bf16), cudaMemcpyDeviceToDevice, s));
    for (const auto& cap : h->capture)
      if (cap.first == i) CE_CHECK_CUDA(cudaMemcpyAsync(cap.second, ws.x, (size_t)M * D * sizeof(bf16), cudaMemcpyDeviceToDevice, s));
  }

  // ---- output head (:451-467): modf = [B, 2, D] with shift = chunk 0, scale = chunk 1
  RUNC(CAT_ROWS, 4.0 * M * D, ln(ws.x, ws.xn, ws.modf + D, ws.modf, 2 * D, L, nullptr, nullptr, 1));
  RUN2(linear(h, ws.xn, D, "proj_out", M, No, D, ws.yout, No, EPI_BIAS, nullptr, 0, nullptr, 0, 1, s));
  if (spx) {   // every rank gets the whole head output (rows all-gathered by peer stores), then un-patchifies the full sample
    bf16* ydst[8];
    for (int w = 0; w < sp.world; ++w) ydst[w] = reinterpret_cast<bf16*>(sp.region[w] + lay.yout);
    RUN(launch_sp_broadcast_rows(ws.yout, B, L, No, ydst, sp.world, Lfull, tok0, s));
    RUN(launch_sp_barrier(sp, lay, s));
    RUN(launch_unpatchify(reinterpret_cast<const bf16*>(sp.region[sp.rank] + lay.yout), No, reinterpret_cast<bf16*>(sample), B, c.out_channels, frames,
                          height, width, s));
    RUN(launch_sp_barrier(sp, lay, s));   // nobody overwrites a peer's yout (next forward) before it has been read
    return CE_OK;
  }
  RUN(launch_unpatchify(ws.yout, No, reinterpret_cast<bf16*>(sample), B, c.out_channels, frames, height, width, s));
  return CE_OK;
}

int64_t ce_dit_host_staging_bytes(const ce_dit* h, int batch, int frames, int height, int width, int text_len) {
  if (!h) return -1;
  const ce_dit_config& c = h->cfg;
  int64_t b = 0;
  auto al = [](int64_t v) { return (v + 255) & ~int64_t(255); };
  b += al((int64_t)batch * c.in_channels * frames * height * width * 2);
  b += al((int64_t)batch * 4);
  b += al((int64_t)batch * text_len * c.text_dim * 2);
  b += al((int64_t)batch * 257 * (c.image_dim > 0 ? c.image_dim : 8) * 2);
  b += al((int64_t)batch * c.out_channels * frames * height * width * 2);
  return b;
}

int64_t ce_dit_host_staging_sample_offset(const ce_dit* h, int batch, int frames, int height, int width, int text_len) {
  if (!h) return -1;
  const ce_dit_config& c = h->cfg;
  Bump b(nullptr);
  b.take<bf16>((int64_t)batch * c.in_channels * frames * height * width);
  b.take<float>(batch);
  b.take<bf16>((int64_t)batch * text_len * c.text_dim);
  const int64_t n_i = (int64_t)batch * 257 * c.image_dim;
  b.take<bf16>(n_i > 0 ? n_i : 8);
  b.off = (b.off + 255) & ~int64_t(255);
  return b.off;
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
  const ce_dit_config& c = h->cfg;
  CE_REQUIRE(staging_bytes >= ce_dit_host_staging_bytes(h, batch, frames, height, width, text_len), "ce_dit_forward_host: staging too small");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_v);
  Bump b(staging);
  const int64_t n_x = (int64_t)batch * c.in_channels * frames * height * width;
  const int64_t n_t = (int64_t)batch * text_len * c.text_dim;
  const int64_t n_i = (int64_t)batch * 257 * c.image_dim;
  const int64_t n_o = (int64_t)batch * c.out_channels * frames * height * width;
  bf16* d_x = b.take<bf16>(n_x);
  float* d_ts = b.take<float>(batch);
  bf16* d_t = b.take<bf16>(n_t);
  bf16* d_i = b.take<bf16>(n_i > 0 ? n_i : 8);
  bf16* d_o = b.take<bf16>(n_o);
  CE_CHECK_CUDA(cudaMemcpyAsync(d_x, hidden_states_host, n_x * 2, cudaMemcpyHostToDevice, s));
  CE_CHECK_CUDA(cudaMemcpyAsync(d_ts, timestep_host, batch * 4, cudaMemcpyHostToDevice, s));
  // the encoder states are copied every call (they are part of the call's inputs); with ctx_reuse the kernels do not read them
  CE_CHECK_CUDA(cudaMemcpyAsync(d_t, encoder_hidden_states_host, n_t * 2, cudaMemcpyHostToDevice, s));
  if (encoder_hidden_states_image_host && n_i > 0)
    CE_CHECK_CUDA(cudaMemcpyAsync(d_i, encoder_hidden_states_image_host, n_i * 2, cudaMemcpyHostToDevice, s));
  int rc = ce_dit_forward_ex(h, d_x, d_ts, d_t, (encoder_hidden_states_image_host && n_i > 0) ? d_i : nullptr, d_o, batch, frames, height, width,
                             text_len, workspace, workspace_bytes, nullptr, ctx_cache, ctx_cache_bytes, ctx_reuse, stream_v);
  if (rc) return rc;
  CE_CHECK_CUDA(cudaMemcpyAsync(sample_host, d_o, n_o * 2, cudaMemcpyDeviceToHost, s));
  CE_CHECK_CUDA(cudaStreamSynchronize(s));
  return CE_OK;
}

// ---------------------------------------------------------------------------------------------- operator exports
int ce_linear_bf16(const void* A, int lda, const void* W, int ldw, const void* bias, void* out, int ldo, float* out_f32, int M, int N,
                   int K, int epilogue, const void* resid, int ldr, const float* gate, int gate_stride, int rows_per_batch, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  GemmArgs g;
  g.M = M; g.N = N; g.K = K;
  g.out = reinterpret_cast<bf16*>(out); g.ldo = ldo;
  g.out_f32 = out_f32;
  g.bias = reinterpret_cast<const bf16*>(bias);
  g.epi = epilogue;
  g.resid = reinterpret_cast<const bf16*>(resid); g.ldr = ldr;
  g.gate = gate; g.gate_stride = gate_stride; g.rows_per_batch = rows_per_batch > 0 ? rows_per_batch : 1;
  return launch_gemm_bf16(reinterpret_cast<const bf16*>(A), lda, reinterpret_cast<const bf16*>(W), ldw, g, reinterpret_cast<cudaStream_t>(stream));
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

int ce_quantize_rows_fp8(const void* x, int ldx, int rows, int K, void* q, int ldq, float* scale, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  return launch_quantize_rows_fp8(reinterpret_cast<const bf16*>(x), ldx, rows, K, reinterpret_cast<uint8_t*>(q), ldq, scale,
                                  reinterpret_cast<cudaStream_t>(stream));
}

static long long* g_attn_timing = nullptr;
// Profiling aid: subsequent ce_attention_bf16 calls record the phase cycles of the first consumer thread of block 0 into `buf`
// ([16] int64 on the device); pass NULL to stop.
int ce_debug_attention_timing(long long* buf) {
  g_attn_timing = buf;
  return CE_OK;
}

// Test aid: attention.cu is the only attention kernel of the sm_90a build (version 0, also the default -1).
int ce_debug_attention_kernel(int version) {
  if (version != -1 && version != 0) return ce::fail(ce::CE_ERR_INVALID, "attention kernel version must be -1 or 0");
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
  a.timing = g_attn_timing;
  return launch_attention(a, reinterpret_cast<cudaStream_t>(stream));
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
  return launch_attention(a, reinterpret_cast<cudaStream_t>(stream));
}

int ce_layernorm_bf16(const void* x, int ldx, void* y, int ldy, int rows, int D, float eps, const float* scale, const float* shift,
                      int mod_stride, int rows_per_batch, const float* weight, const float* bias, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  return launch_layernorm(reinterpret_cast<const bf16*>(x), ldx, reinterpret_cast<bf16*>(y), ldy, rows, D, eps, scale, shift, mod_stride,
                          rows_per_batch, weight, bias, reinterpret_cast<cudaStream_t>(stream));
}

int ce_rmsnorm_rope_bf16(void* x, int ldx, int rows, int D, float eps, const void* weight, const float* rope_cos, const float* rope_sin,
                         int L, int head_dim, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  return launch_rmsnorm_rope(reinterpret_cast<bf16*>(x), ldx, rows, D, eps, reinterpret_cast<const bf16*>(weight), rope_cos, rope_sin, L,
                             head_dim, reinterpret_cast<cudaStream_t>(stream));
}

// Test aids: the two row kernels that take their statistics from GEMM epilogue partials (GemmArgs::stats_out).
int ce_layernorm_stats_bf16(const void* x, int ldx, void* y, int ldy, int rows, int D, float eps, const float* scale, const float* shift,
                            int mod_stride, int rows_per_batch, const float* weight, const float* bias, int scale_is_1p, const float* stats,
                            int stats_ld, int tiles, int tile_n, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  return launch_layernorm_stats(reinterpret_cast<const bf16*>(x), ldx, reinterpret_cast<bf16*>(y), ldy, rows, D, eps, scale, shift, mod_stride,
                                rows_per_batch, weight, bias, scale_is_1p, reinterpret_cast<const float2*>(stats), stats_ld, tiles, tile_n,
                                reinterpret_cast<cudaStream_t>(stream));
}

int ce_rmsnorm_rope_stats_bf16(void* x, int ldx, int rows, int D, float eps, const void* weight0, const void* weight1, int nmat,
                               const float* rope_cos, const float* rope_sin, int L, int head_dim, const float* stats, int stats_ld, int tiles,
                               void* stream) {
  int rc = check_device();
  if (rc) return rc;
  return launch_rmsnorm_rope_stats(reinterpret_cast<bf16*>(x), ldx, rows, D, eps, reinterpret_cast<const bf16*>(weight0),
                                   reinterpret_cast<const bf16*>(weight1), nmat, rope_cos, rope_sin, L, head_dim,
                                   reinterpret_cast<const float2*>(stats), stats_ld, tiles, reinterpret_cast<cudaStream_t>(stream));
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
