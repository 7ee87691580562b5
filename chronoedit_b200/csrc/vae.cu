// ce_vae: Wan2.1 3D causal VAE encode / decode as a chain of sm_90a kernels behind the C ABI.
//
// Follows WanVAE_.encode / .decode of /root/reference/chronoedit/_src/tokenizers/wan2pt1.py:502-560 (the arithmetic twin
// of diffusers AutoencoderKLWan, which the pipeline calls at pipeline_chronoedit.py:436-443, 776-781): chunked causal
// streaming (frame 0 alone, then 4-frame chunks when encoding; one latent frame per iteration when decoding) with a
// 2-frame history per causal convolution.  Activations are channels-last bf16; every convolution with Cin >= 64 is the
// wgmma implicit GEMM of conv.cu reading its input (history frames + chunk) in place; the three small-Cin convolutions
// (3->dim, z->top, 2z->2z) go through im2row + the wgmma GEMM; RMS_norm+SiLU / upsample are the row kernels of
// vae_kernels.cu; the single-head mid attention is gemm_attention (gemm.cu) with H = 1.
#include <math.h>

#include <map>
#include <string>
#include <vector>

#include "../../include/chronoedit_b200.h"
#include "conv.cuh"
#include "gemm.cuh"
#include "vae_kernels.cuh"

using namespace ce;

struct ce_vae {
  ce_vae_config cfg;
  WeightMap w;
  int64_t launches = 0;
};

namespace {

struct Act {
  bf16* p = nullptr;
  int T = 0, H = 0, W = 0, C = 0;
  size_t frame() const { return (size_t)H * W * C; }
  size_t numel() const { return (size_t)T * frame(); }
  size_t pixels() const { return (size_t)T * H * W; }
};

struct StreamBuf {  // input buffer of one streaming (causal) convolution: `hist` history frames, then the chunk
  bf16* p = nullptr;
  int hist = 0, tcap = 0, H = 0, W = 0, C = 0;
  bool primed = false;  // false until the first chunk went through (used for the "Rep" / pass-through first chunks)
};

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

// One encode or decode call.  `dry` = planning pass: the same walk without launches, in which the two bump allocators measure the
// workspace and every weight is looked up with its packed element count before anything is launched.
struct Run {
  ce_vae* h;
  cudaStream_t s;
  bool dry;
  Bump persist;   // from the front of the workspace: stream buffers, collected outputs
  Bump scratch;   // after the persistent region; reset per chunk
  int64_t scratch_max = 0;
  std::map<std::string, StreamBuf> streams;
  WeightLookup weights{h->w};
  Launcher run{s, &h->launches};
  int rc = 0;

  Run(ce_vae* h_, cudaStream_t s_, uint8_t* persist_base, uint8_t* scratch_base)
      : h(h_), s(s_), dry(persist_base == nullptr), persist(persist_base), scratch(scratch_base) {}

  void* take_scratch_bytes(size_t bytes) {
    void* p = scratch.take<uint8_t>((int64_t)bytes);
    if (scratch.off > scratch_max) scratch_max = scratch.off;
    return p;
  }
  Act scratch_act(int T, int H, int W, int C) {
    Act a;
    a.T = T; a.H = H; a.W = W; a.C = C;
    a.p = reinterpret_cast<bf16*>(take_scratch_bytes(a.numel() * 2));
    return a;
  }
  void reset_scratch() { scratch.off = 0; }
  int64_t workspace_bytes() const { return persist.bytes() + ((scratch_max + 255) & ~int64_t(255)) + 256; }

  template <class Launch>
  void launch(Launch&& l) {
    if (!dry && !rc) rc = run(l);
  }

  // ---- streaming conv input buffers
  StreamBuf& stream(const std::string& name, int hist, int tcap, int H, int W_, int C) {
    auto it = streams.find(name);
    if (it != streams.end()) return it->second;
    StreamBuf b;
    b.hist = hist; b.tcap = tcap; b.H = H; b.W = W_; b.C = C;
    const size_t elems = (size_t)(hist + tcap) * H * W_ * C;
    b.p = persist.take<bf16>((int64_t)elems);
    if (!dry && hist > 0) {
      cudaError_t e = cudaMemsetAsync(b.p, 0, (size_t)hist * H * W_ * C * 2, s);  // zero history = causal zero padding
      if (e != cudaSuccess && !rc) rc = fail(CE_ERR_CUDA, cudaGetErrorString(e));
    }
    return streams.emplace(name, b).first->second;
  }
  Act chunk_of(StreamBuf& b, int T) {
    Act a;
    a.T = T; a.H = b.H; a.W = b.W; a.C = b.C;
    a.p = b.p ? b.p + (size_t)b.hist * a.frame() : nullptr;
    if (T > b.tcap && !rc) rc = fail(CE_ERR_INVALID, "vae: chunk larger than the planned stream buffer");
    return a;
  }
  // history <- last `hist` frames of [history ; chunk of T frames]
  void push_history(StreamBuf& b, int T) {
    if (dry || b.hist == 0) return;
    const size_t fb = (size_t)b.H * b.W * b.C * 2;
    for (int i = 0; i < b.hist; ++i) {  // ascending order: sources are always at or after the destination
      const int src = T + i;            // frame index inside [hist ; chunk]
      cudaError_t e = cudaMemcpyAsync(reinterpret_cast<uint8_t*>(b.p) + (size_t)i * fb, reinterpret_cast<uint8_t*>(b.p) + (size_t)src * fb, fb,
                                      cudaMemcpyDeviceToDevice, s);
      if (e != cudaSuccess && !rc) rc = fail(CE_ERR_CUDA, cudaGetErrorString(e));
    }
  }
  void copy(const Act& src, bf16* dst) {
    if (dry) return;
    cudaError_t e = cudaMemcpyAsync(dst, src.p, src.numel() * 2, cudaMemcpyDeviceToDevice, s);
    if (e != cudaSuccess && !rc) rc = fail(CE_ERR_CUDA, cudaGetErrorString(e));
  }

  // ---- primitive ops
  void rms(const Act& x, const std::string& gamma_name, bf16* y, bool silu) {
    const bf16* g = weights.any<bf16>(gamma_name, x.C);
    launch([&] { return launch_rms_silu_cl(x.p, g, y, x.pixels(), x.C, silu ? 1 : 0, s); });
  }
  // implicit-GEMM conv reading `in` = [Tin frames] (history included) -> out
  void conv(const std::string& name, const bf16* in, int Tin, int Hin, int Win, int Cin, Act& out, int kt, int kh, int kw, int st, int sh,
            int sw, int ph, int pw, const bf16* resid = nullptr, int split_time = 0) {
    ConvArgs a;
    a.Cout = split_time ? out.C * 2 : out.C; a.Cin_pad = round_up(Cin, 64);
    a.w = weights.any<bf16>(name + ".weight", (int64_t)a.Cout * kt * kh * kw * a.Cin_pad);
    a.bias = weights.any<bf16>(name + ".bias", a.Cout);
    a.x = in; a.Tin = Tin; a.Hin = Hin; a.Win = Win; a.Cin = Cin;
    a.kt = kt; a.kh = kh; a.kw = kw; a.st = st; a.sh = sh; a.sw = sw; a.ph = ph; a.pw = pw;
    a.t_base = 0;
    a.y = out.p; a.Tout = split_time ? out.T / 2 : out.T; a.Hout = out.H; a.Wout = out.W;
    a.resid = resid; a.split_time = split_time;
    launch([&] { return launch_conv3d_cl(a, s); });
  }
  // streaming causal conv (kt = 3): x is already in the stream buffer's chunk region
  void causal_conv(const std::string& name, StreamBuf& b, int T, Act& out, int kh, const bf16* resid = nullptr, int split_time = 0) {
    conv(name, b.p, b.hist + T, b.H, b.W, b.C, out, 3, kh, kh, 1, 1, 1, kh / 2, kh / 2, resid, split_time);
    push_history(b, T);
    b.primed = true;
  }
  void gemm(const bf16* A, int lda, const bf16* Wt, int ldw, int M, int N, int K, bf16* out, int ldo, const bf16* bias, int epi = EPI_BIAS,
            const bf16* resid = nullptr, int ldr = 0) {
    if (!dry && !rc) rc = run_gemm(run, A, lda, Wt, ldw, M, N, K, out, ldo, bias, epi, resid, ldr);
  }

  // ---- blocks
  // ResidualBlock.forward (wan2pt1.py:201-220)
  Act res_block(const std::string& n, const Act& x, int Cout, int tcap) {
    StreamBuf& sa = stream(n + ".residual.2", 2, tcap, x.H, x.W, x.C);
    Act a_in = chunk_of(sa, x.T);
    rms(x, n + ".residual.0.gamma", a_in.p, true);
    Act t1 = scratch_act(x.T, x.H, x.W, Cout);
    causal_conv(n + ".residual.2", sa, x.T, t1, 3);
    StreamBuf& sb = stream(n + ".residual.6", 2, tcap, x.H, x.W, Cout);
    Act b_in = chunk_of(sb, x.T);
    rms(t1, n + ".residual.3.gamma", b_in.p, true);
    const bf16* hres = x.p;
    if (x.C != Cout) {
      Act sc = scratch_act(x.T, x.H, x.W, Cout);
      conv(n + ".shortcut", x.p, x.T, x.H, x.W, x.C, sc, 1, 1, 1, 1, 1, 1, 0, 0);
      hres = sc.p;
    }
    Act out = scratch_act(x.T, x.H, x.W, Cout);
    causal_conv(n + ".residual.6", sb, x.T, out, 3, hres);
    return out;
  }

  // AttentionBlock.forward (wan2pt1.py:240-259): per frame, single head of width C over H*W tokens
  Act attn_block(const std::string& n, const Act& x) {
    const int C = x.C, P = x.H * x.W, Ppad = round_up(P, 8);
    Act xn = scratch_act(x.T, x.H, x.W, C);
    rms(x, n + ".norm.gamma", xn.p, false);
    Act out = scratch_act(x.T, x.H, x.W, C);
    GemmAttention a;
    a.wqk = weights.any<bf16>(n + ".to_qkv.weight", (int64_t)3 * C * C);
    a.bqk = weights.any<bf16>(n + ".to_qkv.bias", 3 * C);
    a.wv = a.wqk ? a.wqk + (size_t)2 * C * C : nullptr;
    a.bv = a.bqk ? a.bqk + 2 * C : nullptr;
    const bf16* wproj = weights.any<bf16>(n + ".proj.weight", (int64_t)C * C);
    const bf16* bproj = weights.any<bf16>(n + ".proj.bias", C);
    a.L = P; a.D = C; a.H = 1; a.dk = C; a.kpv = P;
    a.sc.rule = SOFTMAX_SCALED;
    a.sc.scale = 1.0f / sqrtf((float)C);
    a.qk = reinterpret_cast<bf16*>(take_scratch_bytes((size_t)P * 2 * C * 2));
    a.vT = reinterpret_cast<bf16*>(take_scratch_bytes((size_t)C * Ppad * 2));
    a.S = reinterpret_cast<float*>(take_scratch_bytes((size_t)P * Ppad * 4));
    a.P = reinterpret_cast<bf16*>(take_scratch_bytes((size_t)P * Ppad * 2));
    a.out = reinterpret_cast<bf16*>(take_scratch_bytes((size_t)P * C * 2));
    a.ldo = C;
    for (int f = 0; f < x.T && !dry && !rc; ++f) {
      a.x = xn.p + (size_t)f * P * C;
      rc = gemm_attention(run, a);
      gemm(a.out, C, wproj, C, P, C, C, out.p + (size_t)f * P * C, C, bproj, EPI_BIAS_RESID, x.p + (size_t)f * P * C, C);   // proj + identity
    }
    return out;
  }

  // Resample upsample2d / upsample3d (wan2pt1.py:112-143)
  Act upsample(const std::string& n, Act x, bool temporal, int tcap_in) {
    const int C = x.C;
    if (temporal) {
      StreamBuf& st = stream(n + ".time_conv", 2, tcap_in, x.H, x.W, C);
      if (!st.primed) {
        st.primed = true;  // first chunk: "Rep" -- no temporal doubling, history stays zero (:116-120, 128-129)
      } else {
        Act in = chunk_of(st, x.T);
        copy(x, in.p);
        Act y = scratch_act(2 * x.T, x.H, x.W, C);
        causal_conv(n + ".time_conv", st, x.T, y, 1, nullptr, /*split_time=*/1);
        x = y;
      }
    }
    Act up = scratch_act(x.T, 2 * x.H, 2 * x.W, C);
    launch([&] { return launch_upsample2x_cl(x.p, up.p, x.T, x.H, x.W, C, s); });
    Act out = scratch_act(x.T, 2 * x.H, 2 * x.W, C / 2);
    conv(n + ".resample.1", up.p, up.T, up.H, up.W, C, out, 1, 3, 3, 1, 1, 1, 1, 1);
    return out;
  }

  // Resample downsample2d / downsample3d (wan2pt1.py:145-159)
  Act downsample(const std::string& n, const Act& x, bool temporal, int tcap_out_spatial) {
    const int C = x.C;
    const int Ho = (x.H + 1 - 3) / 2 + 1, Wo = (x.W + 1 - 3) / 2 + 1;
    if (!temporal) {
      Act out = scratch_act(x.T, Ho, Wo, C);
      conv(n + ".resample.1", x.p, x.T, x.H, x.W, C, out, 1, 3, 3, 1, 2, 2, 0, 0);  // ZeroPad2d(0,1,0,1) = OOB zero fill
      return out;
    }
    StreamBuf& st = stream(n + ".time_conv", 1, tcap_out_spatial, Ho, Wo, C);
    Act sp = chunk_of(st, x.T);
    conv(n + ".resample.1", x.p, x.T, x.H, x.W, C, sp, 1, 3, 3, 1, 2, 2, 0, 0);
    if (!st.primed) {  // first chunk passes through and becomes the history (:147-150)
      st.primed = true;
      Act out = scratch_act(x.T, Ho, Wo, C);
      copy(sp, out.p);
      push_history(st, x.T);
      return out;
    }
    const int To = (1 + x.T - 3) / 2 + 1;
    Act out = scratch_act(To, Ho, Wo, C);
    conv(n + ".time_conv", st.p, 1 + x.T, Ho, Wo, C, out, 3, 1, 1, 2, 1, 1, 0, 0);
    push_history(st, x.T);
    return out;
  }

  // small-Cin conv: im2row + GEMM.  x addressed by strides (planar or channels-last)
  void small_conv(const std::string& name, const bf16* x, size_t sc, size_t st_, size_t sh, size_t sw, int Tin, int Hin, int Win, int Cin,
                  int t_base, int kt, int kh, bf16* out, int ldo, int Tout, int Cout) {
    const int K = kt * kh * kh * Cin, Kpad = round_up(K, 8);
    bf16* A = reinterpret_cast<bf16*>(take_scratch_bytes((size_t)Tout * Hin * Win * Kpad * 2));
    const bf16* w = weights.any<bf16>(name + ".weight", (int64_t)Cout * Kpad);
    const bf16* b = weights.any<bf16>(name + ".bias", Cout);
    launch([&] { return launch_im2row(x, sc, st_, sh, sw, Tin, Hin, Win, Cin, A, Kpad, Tout, Hin, Win, kt, kh, kh, kh / 2, kh / 2, t_base, s); });
    gemm(A, Kpad, w, Kpad, Tout * Hin * Win, Cout, Kpad, out, ldo, b);
  }
};

int top_dim(const ce_vae_config& c) { return c.dim * c.dim_mult[3]; }

struct LayerSpec {
  bool res;
  int cin, cout;      // res
  int mode;           // resample: 0 = 2d, 1 = 3d
};

// Encoder3d.__init__ (wan2pt1.py:281-303)
std::vector<LayerSpec> encoder_layers(const ce_vae_config& c) {
  std::vector<LayerSpec> v;
  int dims[5] = {c.dim, c.dim * c.dim_mult[0], c.dim * c.dim_mult[1], c.dim * c.dim_mult[2], c.dim * c.dim_mult[3]};
  for (int i = 0; i < 4; ++i) {
    int cin = dims[i];
    for (int r = 0; r < c.num_res_blocks; ++r) {
      v.push_back({true, cin, dims[i + 1], 0});
      cin = dims[i + 1];
    }
    if (i != 3) v.push_back({false, dims[i + 1], dims[i + 1], c.temporal_downsample[i] ? 1 : 0});
  }
  return v;
}
// Decoder3d.__init__ (wan2pt1.py:379-408)
std::vector<LayerSpec> decoder_layers(const ce_vae_config& c) {
  std::vector<LayerSpec> v;
  int dims[5] = {c.dim * c.dim_mult[3], c.dim * c.dim_mult[3], c.dim * c.dim_mult[2], c.dim * c.dim_mult[1], c.dim * c.dim_mult[0]};
  for (int i = 0; i < 4; ++i) {
    int cin = dims[i];
    if (i >= 1) cin /= 2;
    for (int r = 0; r < c.num_res_blocks + 1; ++r) {
      v.push_back({true, cin, dims[i + 1], 0});
      cin = dims[i + 1];
    }
    if (i != 3) v.push_back({false, dims[i + 1], dims[i + 1], c.temporal_downsample[2 - i] ? 1 : 0});
  }
  return v;
}

// ---------------------------------------------------------------------------------------------- decode
// WanVAE_.decode (wan2pt1.py:543-560) + Decoder3d.forward (:412-456); z planar [zc, Tl, h, w] -> video planar [3, 1+4(Tl-1), 8h, 8w]
int run_decode(Run& R, const bf16* z, bf16* video, int Tl, int h, int w, int clamp) {
  const ce_vae_config& c = R.h->cfg;
  const int top = top_dim(c), zc = c.z_dim;
  const int T_px = 1 + 4 * (Tl - 1);
  const size_t zplane = (size_t)Tl * h * w;
  std::vector<LayerSpec> layers = decoder_layers(c);
  int t_out = 0;
  for (int i = 0; i < Tl && !R.rc; ++i) {
    R.reset_scratch();
    int cap = 1;  // frames a non-first chunk carries at the current depth (x2 after every upsample3d): stream capacity
    // conv2 (1x1x1 on the planar z) -> straight into the stream buffer of decoder.conv1
    StreamBuf& s1 = R.stream("decoder.conv1", 2, 1, h, w, zc);
    Act x0 = R.chunk_of(s1, 1);
    R.small_conv("conv2", z, zplane, (size_t)h * w, (size_t)w, 1, Tl, h, w, zc, /*t_base=*/i, 1, 1, x0.p, zc, 1, zc);
    // decoder.conv1: 3x3x3 causal with Cin = z_dim: im2row over [history ; chunk] (channels-last) + GEMM
    Act x = R.scratch_act(1, h, w, top);
    R.small_conv("decoder.conv1", s1.p, 1, (size_t)h * w * zc, (size_t)w * zc, (size_t)zc, s1.hist + 1, h, w, zc, 0, 3, 3, x.p, top, 1, top);
    R.push_history(s1, 1);
    x = R.res_block("decoder.middle.0", x, top, cap);
    x = R.attn_block("decoder.middle.1", x);
    x = R.res_block("decoder.middle.2", x, top, cap);
    int idx = 0;
    for (const LayerSpec& l : layers) {
      const std::string n = "decoder.upsamples." + std::to_string(idx++);
      if (l.res) {
        x = R.res_block(n, x, l.cout, cap);
      } else {
        x = R.upsample(n, x, l.mode == 1, cap);
        if (l.mode == 1) cap *= 2;
      }
    }
    // head: RMS + SiLU + conv dim->3, planar clamped store straight into the output video
    StreamBuf& sh = R.stream("decoder.head.2", 2, cap, x.H, x.W, x.C);
    Act hin = R.chunk_of(sh, x.T);
    R.rms(x, "decoder.head.0.gamma", hin.p, true);
    {
      ConvArgs a;
      a.x = sh.p; a.Tin = sh.hist + x.T; a.Hin = x.H; a.Win = x.W; a.Cin = x.C;
      a.Cout = 3; a.Cin_pad = round_up(x.C, 64);
      a.w = R.weights.any<bf16>("decoder.head.2.weight", (int64_t)3 * 27 * a.Cin_pad);
      a.bias = R.weights.any<bf16>("decoder.head.2.bias", 3);
      a.kt = 3; a.kh = 3; a.kw = 3; a.ph = 1; a.pw = 1;
      a.y = video; a.Tout = x.T; a.Hout = x.H; a.Wout = x.W;
      a.planar_out = 1; a.clamp = clamp; a.planar_T = T_px; a.planar_t0 = t_out;
      R.launch([&] { return launch_conv3d_cl(a, R.s); });
      R.push_history(sh, x.T);
    }
    t_out += x.T;
  }
  if (!R.rc && t_out != T_px) return fail(CE_ERR_INVALID, "vae decode: produced frame count mismatch");
  return R.rc;
}

// ---------------------------------------------------------------------------------------------- encode
// WanVAE_.encode (wan2pt1.py:502-533) + Encoder3d.forward (:315-357); video planar [3, T, H, W] -> mean planar [zc, Tl, H/8, W/8]
int run_encode(Run& R, const bf16* video, bf16* mu, int T, int H, int Wd) {
  const ce_vae_config& c = R.h->cfg;
  const int top = top_dim(c), zc = c.z_dim;
  const int Tl = 1 + (T - 1) / 4, h = H / 8, w = Wd / 8;
  std::vector<LayerSpec> layers = encoder_layers(c);
  bf16* enc_out = R.persist.take<bf16>((int64_t)Tl * h * w * 2 * zc);  // head outputs of every chunk, channels-last
  int t_lat = 0;
  for (int f0 = 0; f0 < T && !R.rc;) {
    const int Tc = f0 == 0 ? 1 : 4;
    R.reset_scratch();
    int cap = 4;
    Act x = R.scratch_act(Tc, H, Wd, c.dim);
    // encoder.conv1: 3x3x3 causal with Cin = 3 straight from the planar video (its own past frames are the history)
    R.small_conv("encoder.conv1", video, (size_t)T * H * Wd, (size_t)H * Wd, (size_t)Wd, 1, T, H, Wd, 3, /*t_base=*/f0 - 2, 3, 3, x.p, c.dim, Tc,
                 c.dim);
    int idx = 0;
    for (const LayerSpec& l : layers) {
      const std::string n = "encoder.downsamples." + std::to_string(idx++);
      if (l.res) {
        x = R.res_block(n, x, l.cout, cap);
      } else {
        x = R.downsample(n, x, l.mode == 1, cap);
        if (l.mode == 1) cap = cap > 1 ? cap / 2 : 1;
      }
    }
    x = R.res_block("encoder.middle.0", x, top, cap);
    x = R.attn_block("encoder.middle.1", x);
    x = R.res_block("encoder.middle.2", x, top, cap);
    StreamBuf& sh = R.stream("encoder.head.2", 2, cap, x.H, x.W, x.C);
    Act hin = R.chunk_of(sh, x.T);
    R.rms(x, "encoder.head.0.gamma", hin.p, true);
    Act o;
    o.T = x.T; o.H = x.H; o.W = x.W; o.C = 2 * zc;
    o.p = R.dry ? nullptr : enc_out + (size_t)t_lat * h * w * 2 * zc;
    if (x.H != h || x.W != w) return fail(CE_ERR_INVALID, "vae encode: spatial size mismatch (H, W must be multiples of 8)");
    R.causal_conv("encoder.head.2", sh, x.T, o, 3);
    t_lat += x.T;
    f0 += Tc;
  }
  if (!R.rc && t_lat != Tl) return fail(CE_ERR_INVALID, "vae encode: produced frame count mismatch");
  // conv1 (1x1x1, 2z -> 2z) then keep the first z channels (posterior mean)
  R.reset_scratch();
  const size_t P = (size_t)Tl * h * w;
  bf16* q = reinterpret_cast<bf16*>(R.take_scratch_bytes(P * 2 * zc * 2));
  const bf16* w1 = R.weights.any<bf16>("conv1.weight", (int64_t)4 * zc * zc);
  R.gemm(enc_out, 2 * zc, w1, 2 * zc, (int)P, 2 * zc, 2 * zc, q, 2 * zc, R.weights.any<bf16>("conv1.bias", 2 * zc));
  R.launch([&] { return launch_cl_to_planar(q, 2 * zc, mu, P, 2 * zc, R.s); });  // moments = mean | logvar
  return R.rc;
}

int check_geometry(const ce_vae* h, int T, int H, int W, bool decode) {
  CE_REQUIRE(h != nullptr, "vae: null handle");
  if (decode) {
    CE_REQUIRE(T >= 1 && H >= 1 && W >= 1, "vae decode: empty latent");
  } else {
    CE_REQUIRE(T >= 1 && (T - 1) % 4 == 0, "vae encode: frame count must be 1 + 4k (the reference fails otherwise)");
    CE_REQUIRE(H % 8 == 0 && W % 8 == 0 && H >= 8 && W >= 8, "vae encode: H, W must be multiples of 8");
  }
  return CE_OK;
}

}  // namespace

extern "C" {

int ce_vae_create(const ce_vae_config* cfg, ce_vae** out) {
  CE_REQUIRE(cfg && out, "ce_vae_create: null argument");
  CE_REQUIRE(cfg->dim % 8 == 0 && cfg->dim >= 16, "ce_vae_create: dim must be a multiple of 8 (16-byte channel vectors)");
  CE_REQUIRE(cfg->z_dim % 8 == 0 && cfg->z_dim <= 32, "ce_vae_create: z_dim % 8, <= 32");
  CE_REQUIRE(cfg->num_res_blocks >= 1, "ce_vae_create: num_res_blocks");
  ce_vae* h = new ce_vae();
  h->cfg = *cfg;
  *out = h;
  return CE_OK;
}

void ce_vae_destroy(ce_vae* h) { delete h; }

int ce_vae_set_weight(ce_vae* h, const char* name, const void* ptr, int64_t numel) {
  CE_REQUIRE(h, "ce_vae_set_weight: null handle");
  return register_weight(h->w, "ce_vae_set_weight", name, ptr, -1, numel);
}

int64_t ce_vae_workspace_bytes(ce_vae* h, int decode, int frames, int height, int width) {
  if (check_geometry(h, frames, height, width, decode != 0)) return -1;
  Run plan(h, nullptr, nullptr, nullptr);
  int rc = decode ? run_decode(plan, nullptr, nullptr, frames, height, width, 0) : run_encode(plan, nullptr, nullptr, frames, height, width);
  return rc || plan.weights.rc ? -1 : plan.workspace_bytes();
}

static int run(ce_vae* h, bool decode, const void* in, void* out, int frames, int height, int width, int clamp, void* workspace,
               int64_t workspace_bytes, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  if ((rc = check_geometry(h, frames, height, width, decode))) return rc;
  CE_REQUIRE(in && out && workspace, "vae: null argument");
  CE_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "vae: workspace must be 256-byte aligned");
  // plan first: sizes of the persistent region (stream buffers) and of the per-chunk scratch
  Run plan(h, nullptr, nullptr, nullptr);
  rc = decode ? run_decode(plan, nullptr, nullptr, frames, height, width, 0) : run_encode(plan, nullptr, nullptr, frames, height, width);
  if (rc || (rc = plan.weights.rc)) return rc;
  const int64_t need = plan.workspace_bytes();
  if (need > workspace_bytes)
    return fail(CE_ERR_WORKSPACE, "vae: workspace too small: need " + std::to_string(need) + " bytes, got " + std::to_string(workspace_bytes));
  uint8_t* base = reinterpret_cast<uint8_t*>(workspace);
  Run R(h, reinterpret_cast<cudaStream_t>(stream), base, base + plan.persist.bytes());
  h->launches = 0;
  return decode ? run_decode(R, reinterpret_cast<const bf16*>(in), reinterpret_cast<bf16*>(out), frames, height, width, clamp)
                : run_encode(R, reinterpret_cast<const bf16*>(in), reinterpret_cast<bf16*>(out), frames, height, width);
}

int ce_vae_encode(ce_vae* h, const void* video, void* mean, int frames, int height, int width, void* workspace, int64_t workspace_bytes,
                  void* stream) {
  return run(h, false, video, mean, frames, height, width, 0, workspace, workspace_bytes, stream);
}

int ce_vae_decode(ce_vae* h, const void* z, void* video, int latent_frames, int latent_height, int latent_width, int clamp, void* workspace,
                  int64_t workspace_bytes, void* stream) {
  return run(h, true, z, video, latent_frames, latent_height, latent_width, clamp, workspace, workspace_bytes, stream);
}

int64_t ce_vae_last_launch_count(const ce_vae* h) { return h ? h->launches : 0; }

// One implicit-GEMM convolution (parity tests / profiling).  Layouts as in conv.cuh.
int ce_conv3d_cl_bf16(const void* x, int Tin, int Hin, int Win, int Cin, const void* w, const void* bias, int Cout, int kt, int kh, int kw, int st,
                      int sh, int sw, int ph, int pw, int t_base, void* y, int Tout, int Hout, int Wout, const void* resid, int split_time,
                      void* stream) {
  ce_conv3d_args a = {};
  a.x = x; a.Tin = Tin; a.Hin = Hin; a.Win = Win; a.Cin = Cin;
  a.w = w; a.bias = bias; a.Cout = Cout; a.Cin_pad = round_up(Cin, 64);
  a.kt = kt; a.kh = kh; a.kw = kw; a.st = st; a.sh = sh; a.sw = sw; a.ph = ph; a.pw = pw; a.t_base = t_base;
  a.y = y; a.Tout = Tout; a.Hout = Hout; a.Wout = Wout;
  a.resid = resid; a.split_time = split_time;
  return ce_conv3d_cl_ex_bf16(&a, stream);
}

// Test aids: the VAE's operators one at a time, through the launchers the handle uses (and their argument checks).
int ce_conv3d_cl_ex_bf16(const ce_conv3d_args* args, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  CE_REQUIRE(args != nullptr, "ce_conv3d_cl_ex_bf16: null args");
  ConvArgs a;
  a.x = reinterpret_cast<const bf16*>(args->x); a.Tin = args->Tin; a.Hin = args->Hin; a.Win = args->Win; a.Cin = args->Cin;
  a.w = reinterpret_cast<const bf16*>(args->w); a.bias = reinterpret_cast<const bf16*>(args->bias);
  a.Cout = args->Cout; a.Cin_pad = args->Cin_pad;
  a.kt = args->kt; a.kh = args->kh; a.kw = args->kw; a.st = args->st; a.sh = args->sh; a.sw = args->sw; a.ph = args->ph; a.pw = args->pw;
  a.t_base = args->t_base;
  a.y = reinterpret_cast<bf16*>(args->y); a.Tout = args->Tout; a.Hout = args->Hout; a.Wout = args->Wout;
  a.resid = reinterpret_cast<const bf16*>(args->resid); a.split_time = args->split_time;
  a.planar_out = args->planar_out; a.clamp = args->clamp; a.planar_T = args->planar_T; a.planar_t0 = args->planar_t0;
  return launch_conv3d_cl(a, reinterpret_cast<cudaStream_t>(stream));
}

int ce_rms_silu_cl_bf16(const void* x, const void* gamma, void* y, int64_t pixels, int C, int apply_silu, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  CE_REQUIRE(x && gamma && y && pixels >= 0, "ce_rms_silu_cl_bf16: null pointer / negative pixel count");
  return launch_rms_silu_cl(reinterpret_cast<const bf16*>(x), reinterpret_cast<const bf16*>(gamma), reinterpret_cast<bf16*>(y), (size_t)pixels,
                            C, apply_silu, reinterpret_cast<cudaStream_t>(stream));
}

int ce_upsample2x_cl_bf16(const void* x, void* y, int T, int H, int W, int C, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  CE_REQUIRE(x && y && T >= 0 && H >= 0 && W >= 0, "ce_upsample2x_cl_bf16: null pointer / negative size");
  return launch_upsample2x_cl(reinterpret_cast<const bf16*>(x), reinterpret_cast<bf16*>(y), T, H, W, C, reinterpret_cast<cudaStream_t>(stream));
}

int ce_im2row_bf16(const void* x, int64_t sc, int64_t st, int64_t sh, int64_t sw, int Tin, int Hin, int Win, int Cin, void* A, int Kpad, int Tout,
                   int Hout, int Wout, int kt, int kh, int kw, int ph, int pw, int t_base, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  CE_REQUIRE(x && A && sc >= 0 && st >= 0 && sh >= 0 && sw >= 0 && Tout >= 0 && Hout >= 0 && Wout >= 0,
             "ce_im2row_bf16: null pointer / negative stride or size");
  return launch_im2row(reinterpret_cast<const bf16*>(x), (size_t)sc, (size_t)st, (size_t)sh, (size_t)sw, Tin, Hin, Win, Cin,
                       reinterpret_cast<bf16*>(A), Kpad, Tout, Hout, Wout, kt, kh, kw, ph, pw, t_base, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
