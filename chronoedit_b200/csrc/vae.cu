// ce_vae: Wan2.1 3D causal VAE encode / decode as a chain of sm_90a kernels behind the C ABI.
//
// Follows WanVAE_.encode / .decode of /root/reference/chronoedit/_src/tokenizers/wan2pt1.py:502-560 (the arithmetic twin
// of diffusers AutoencoderKLWan, which the pipeline calls at pipeline_chronoedit.py:436-443, 776-781): chunked causal
// streaming (frame 0 alone, then 4-frame chunks when encoding; one latent frame per iteration when decoding) with a
// 2-frame history per causal convolution.  Activations are channels-last bf16; every convolution with Cin >= 64 is the
// wgmma implicit GEMM of conv.cu reading its input (history frames + chunk) in place; the three small-Cin convolutions
// (3->dim, z->top, 2z->2z) go through im2row + the wgmma GEMM; RMS_norm+SiLU / upsample are the row kernels of
// vae_kernels.cu; the single-head mid attention is gemm_attention (gemm.cu) with H = 1.
//
// fp32 (ce_vae_*_fp32, AutoencoderKLWan loaded in fp32) runs the same walk: only Run's primitives know the precision (see Run).
// Every entry point plans and runs through vae_call, which refuses in one order for all of them.
//
// Split over the ranks of a node (ce_vae_sp_configure): rank r owns latent rows [r h / W, (r + 1) h / W) and the matching rows at
// every resolution of the encoder and decoder.  Every buffer that feeds a convolution with three kernel rows holds the band plus one
// halo row above and below; the neighbours store their edge rows into this rank's peer region, a barrier orders it, and a local copy
// moves them into the halo rows (zero past the global top and bottom: the convolution's own zero padding).  The mid attention
// gathers its normalised frame into every rank's region and computes the rank's query rows only; the outputs are gathered the same
// way.  Every output element sums the same terms in the same order as on one GPU, so each rank returns the single-GPU bits.
//
// Tiled (ce_vae_encode_tiled / ce_vae_decode_tiled, diffusers' enable_tiling): run_tiled walks a grid of overlapping tiles, runs the
// untiled chain on each and blends it with its neighbours (tile_blend_kernel, vae_kernels.cu); see the section above run_tiled.
#include <math.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "../../include/chronoedit_b200.h"
#include "conv.cuh"
#include "fp32_chain.cuh"
#include "gemm.cuh"
#include "seqpar.cuh"
#include "vae_kernels.cuh"

using namespace ce;

struct ce_vae {
  ce_vae_config cfg;
  WeightMap w;
  WeightMap w32;   // the fp32 VAE's (ce_vae_set_weight_fp32)
  int64_t launches = 0;
  SeqPar sp;   // the split over ranks (ce_vae_sp_configure): world == 1 means off
};

namespace {

// An activation [T, H, W, C]: p is what a convolution reads (bf16, or the fp32 activation's split pair [T, H, W, 2, C]), f the fp32
// values where they exist.
struct Act {
  bf16* p = nullptr;
  float* f = nullptr;
  int T = 0, H = 0, W = 0, C = 0;
  size_t frame() const { return (size_t)H * W * C; }
  size_t pixels() const { return (size_t)T * H * W; }
};

struct StreamBuf {  // input buffer of one streaming (causal) convolution: `hist` history frames, then the chunk
  bf16* p = nullptr;
  int hist = 0, tcap = 0, H = 0, W = 0, C = 0;
  int pair = 1;         // 2 in fp32: the frames hold the split pair [H, W, 2, C]
  bool halo = false;    // split: every frame is a band with one halo row above and below (H counts them)
  bool primed = false;  // false until the first chunk went through (used for the "Rep" / pass-through first chunks)
  size_t frame() const { return (size_t)H * W * pair * C; }
};

// Byte offsets inside a rank's peer region for one pixel geometry H x W, the same for every frame count.
struct VaeSpLayout {
  int64_t flags = 0;        // uint32 [8 * 32] barrier flags; first, so that every geometry finds them in the same place
  int64_t halo = 0;         // [2 sets][from above, from below][halo_slot]: the neighbours' edge rows of one chunk
  int64_t halo_slot = 0;
  int64_t frame = 0;        // [2 sets][frame_bytes]: the mid attention's normalised frame [up8(h w), top] bf16
  int64_t frame_bytes = 0;
  int64_t video = 0;        // [3, video_frames, H, W] bf16: the pixels of one decode chunk
  int video_frames = 0;
  int64_t moments = 0;      // [2 sets][moments_bytes]: one latent frame of encode moments [2 z_dim, h, w] bf16
  int64_t moments_bytes = 0;
  int64_t bytes = 0;
};

struct Planar {   // a convolution's planar [C, T, H, W] store: output frame t goes to frame t0 + t of T
  int T, t0, clamp;
};

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }
template <class T>
T* at(T* p, size_t off) {   // planning passes carry null pointers
  return p ? p + off : nullptr;
}

// One encode or decode call in bf16 or fp32.  A planning pass (dry) is the same walk without launches, in which the bump allocators
// measure the workspace and every weight is looked up with its packed element count before anything is launched.  Only the primitives
// below (rms, conv, the upsample, the mid attention, the stems and the encode's tail) know the precision: bf16 activations, or fp32
// activations whose convolutions read their split pair (launch_conv3d_cl_f32, conv.cuh), with the causal history kept as the pair and
// the mid attention Fp32Chain's (6-term split products, fp32 row softmax).
struct Run {
  ce_vae* h;
  bool fp32;
  cudaStream_t s;
  bool dry = true;
  Bump persist{nullptr};   // from the front of the workspace: stream buffers, converted inputs, collected outputs
  // Scratch after the persistent region, reset per chunk.  fp32 uses two arenas in turn, one per block: a block's temporaries and
  // output go into the arena its input is not in, which it resets first (what that arena held was the input of the block before,
  // consumed by now); a whole chunk's fp32 activations at 720p would not fit beside the fp32 stream buffers.  bf16 uses one.
  Bump arena[2] = {Bump(nullptr), Bump(nullptr)};
  int cur = 0;
  int64_t arena_max[2] = {0, 0};
  std::map<std::string, StreamBuf> streams;
  WeightLookup weights{fp32 ? h->w32 : h->w};
  Launcher run{s, &h->launches};
  int rc = 0;
  // the split: this rank's band is latent rows [band0, band1) of `rows`; world == 1: the whole frame
  int rank, world;
  int rows = 0, band0 = 0, band1 = 0;
  const VaeSpLayout* lay = nullptr;   // null when planning
  int64_t halo_row_max = 0;           // the largest halo row of a chunk (T W C bf16), in bytes

  Run(ce_vae* h_, bool fp32_, int rank_, int world_, cudaStream_t s_ = nullptr) : h(h_), fp32(fp32_), s(s_), rank(rank_), world(world_) {}
  // a launching pass: the buffers go into `ws` as the planning pass `plan` measured them
  void bind(uint8_t* ws, const Run& plan) {
    dry = false;
    persist = Bump(ws);
    arena[0] = Bump(ws + plan.persist.bytes());
    arena[1] = Bump(ws + plan.persist.bytes() + plan.arena_bytes(0));
  }

  bool split() const { return world > 1; }
  int pair() const { return fp32 ? 2 : 1; }
  void set_band(int latent_rows) {
    rows = latent_rows;
    band0 = (int)((int64_t)rank * latent_rows / world);
    band1 = (int)((int64_t)(rank + 1) * latent_rows / world);
  }

  template <class T>
  T* take(size_t n) {
    T* p = arena[cur].take<T>((int64_t)n);
    arena_max[cur] = std::max(arena_max[cur], arena[cur].off);
    return p;
  }
  void next_block() {
    if (!fp32) return;
    cur ^= 1;
    arena[cur].off = 0;
  }
  void new_chunk() {
    arena[0].off = arena[1].off = 0;
    cur = 0;
  }
  int64_t arena_bytes(int i) const { return (arena_max[i] + 255) & ~int64_t(255); }
  int64_t workspace_bytes() const { return persist.bytes() + arena_bytes(0) + arena_bytes(1) + 256; }
  // a scratch activation: bf16, or fp32 values and (with `with_pair`) the pair a convolution reads
  Act act(int T, int H, int W, int C, bool with_pair = true) {
    Act a;
    a.T = T; a.H = H; a.W = W; a.C = C;
    if (!fp32) {
      a.p = take<bf16>(a.pixels() * C);
    } else {
      a.f = take<float>(a.pixels() * C);
      if (with_pair) a.p = take<bf16>(a.pixels() * 2 * C);
    }
    return a;
  }

  template <class Launch>
  void launch(Launch&& l) {
    if (!dry && !rc) rc = run(l);
  }
  void cuda(cudaError_t e) {
    if (e != cudaSuccess && !rc) rc = fail(CE_ERR_CUDA, cudaGetErrorString(e));
  }
  void copy(void* dst, const void* src, size_t bytes) {
    if (!dry && !rc) cuda(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, s));
  }

  // ---- streaming conv input buffers
  StreamBuf& stream(const std::string& name, int hist, int tcap, int H, int W_, int C, bool halo = false) {
    auto it = streams.find(name);
    if (it != streams.end()) return it->second;
    StreamBuf b;
    b.halo = halo && split();
    b.hist = hist; b.tcap = tcap; b.H = b.halo ? H + 2 : H; b.W = W_; b.C = C; b.pair = pair();
    const size_t elems = (size_t)(hist + tcap) * b.frame();
    b.p = persist.take<bf16>((int64_t)elems);
    // zero history = causal zero padding; split: also the halo rows past the global edge, which nothing writes
    const size_t zero = split() ? elems : (size_t)hist * b.frame();
    if (!dry && zero > 0) cuda(cudaMemsetAsync(b.p, 0, zero * 2, s));
    return streams.emplace(name, b).first->second;
  }
  Act chunk_of(StreamBuf& b, int T) {
    Act a;
    a.T = T; a.H = b.H; a.W = b.W; a.C = b.C;
    a.p = at(b.p, (size_t)b.hist * b.frame());
    if (T > b.tcap && !rc) rc = fail(CE_ERR_INVALID, "vae: chunk larger than the planned stream buffer");
    return a;
  }
  // history <- last `hist` frames of [history ; chunk of T frames]
  void push_history(StreamBuf& b, int T) {
    for (int i = 0; i < b.hist; ++i)   // ascending order: sources are always at or after the destination
      copy(at(b.p, i * b.frame()), at(b.p, (T + i) * b.frame()), b.frame() * 2);
  }

  // ---- the exchange between ranks
  uint8_t* region(int w) const { return h->sp.region[w]; }
  void barrier() { launch([&] { return launch_sp_barrier(h->sp, lay->flags, s); }); }
  void peer_copies(const SpCopy* jobs, int n) {
    if (n > 0) launch([&] { return launch_sp_copy(jobs, n, s); });
  }
  void copy_2d(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t height) {
    if (!dry && !rc) cuda(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, height, cudaMemcpyDeviceToDevice, s));
  }
  // A halo'd buffer holds T frames of band + 2 rows of W * C; rows 0 and band + 1 are the neighbours' edge rows.  The ones past the
  // global top and bottom are zero.
  void zero_edges(bf16* buf, int T, int band, int W, int C) {
    if (dry || rc) return;
    const size_t row = (size_t)W * C * 2, fr = (band + 2) * row;
    if (rank == 0) cuda(cudaMemset2DAsync(buf, fr, 0, row, T, s));
    if (rank == world - 1) cuda(cudaMemset2DAsync(reinterpret_cast<uint8_t*>(buf) + (band + 1) * row, fr, 0, row, T, s));
  }
  // The band rows of the halo'd buffer are written: store the first one into the rank above's "from below" slot and the last one into
  // the rank below's "from above" slot, barrier, then copy what the neighbours stored into rows 0 and band + 1.  Exchange i uses slot
  // set i mod 2, so a slot is rewritten only after every rank has passed the barrier that follows its unpacking.
  void halo_exchange(bf16* buf, int T, int band, int W, int C) {
    const int64_t row = (int64_t)W * C * 2, fr = (band + 2) * row;
    halo_row_max = std::max(halo_row_max, T * row);
    if (dry || rc) return;
    if (T * row > lay->halo_slot) {
      rc = fail(CE_ERR_INVALID, "vae sequence parallel: a halo row is larger than the region's slot");
      return;
    }
    const int set = (int)(h->sp.epoch & 1);
    auto slot = [&](int w, int below) { return region(w) + lay->halo + (2 * set + below) * lay->halo_slot; };
    uint8_t* b = reinterpret_cast<uint8_t*>(buf);
    SpCopy j[2];
    int n = 0;
    if (rank > 0) {
      j[n].src = b + row; j[n].dst = slot(rank - 1, 1); j[n].bytes = row; j[n].n0 = T; j[n].sp0 = fr; j[n].dp0 = row;
      ++n;
    }
    if (rank < world - 1) {
      j[n].src = b + band * row; j[n].dst = slot(rank + 1, 0); j[n].bytes = row; j[n].n0 = T; j[n].sp0 = fr; j[n].dp0 = row;
      ++n;
    }
    peer_copies(j, n);
    barrier();
    if (rank > 0) copy_2d(b, fr, slot(rank, 0), row, row, T);
    if (rank < world - 1) copy_2d(b + (band + 1) * row, fr, slot(rank, 1), row, row, T);
  }

  // ---- primitive ops: the only code that knows the precision
  // RMS_norm (+ SiLU) of x into y: bf16, or fp32 into y's fp32 values and / or its pair
  void rms(const Act& x, const std::string& gamma_name, const Act& y, bool silu) {
    if (fp32) {
      const float* g = weights.any<float>(gamma_name, x.C);
      launch([&] { return launch_rms_silu_cl_f32(x.f, g, y.f, y.p, x.pixels(), x.C, silu ? 1 : 0, s); });
      return;
    }
    const bf16* g = weights.any<bf16>(gamma_name, x.C);
    launch([&] { return launch_rms_silu_cl(x.p, g, y.p, x.pixels(), x.C, silu ? 1 : 0, s); });
  }
  // rms into the chunk y of a stream buffer; with halo rows one launch per frame (a frame's band rows are not next to the next frame's)
  void rms_into(const Act& x, const std::string& gamma_name, const StreamBuf& b, const Act& y, bool silu) {
    if (!b.halo) return rms(x, gamma_name, y, silu);
    for (int f = 0; f < x.T; ++f) {
      Act xf = x, yf = y;
      xf.T = 1; xf.p = at(x.p, f * x.frame());
      yf.p = at(y.p, f * (x.frame() + 2 * (size_t)x.W * x.C) + (size_t)x.W * x.C);
      rms(xf, gamma_name, yf, silu);
    }
  }
  // implicit-GEMM conv reading `in` = [Tin frames] (history included) -> out (bf16, or fp32 values and / or pair), plus resid's values;
  // with `planar` the output is stored planar into out.p (bf16) or out.f (fp32)
  void conv(const std::string& name, const bf16* in, int Tin, int Hin, int Win, int Cin, const Act& out, int kt, int kh, int kw, int st,
            int sh, int sw, int ph, int pw, const Act& resid = Act(), int split_time = 0, int t_base = 0, const Planar* planar = nullptr) {
    ConvArgs a;
    a.Cout = split_time ? out.C * 2 : out.C; a.Cin_pad = round_up(Cin, 64);
    // fp32: the weight's bf16 hi | hi | lo split (pack_parameter_fp32)
    a.w = weights.any<bf16>(name + ".weight", (int64_t)a.Cout * kt * kh * kw * a.Cin_pad * (fp32 ? 3 : 1));
    a.x = in; a.Tin = Tin; a.Hin = Hin; a.Win = Win; a.Cin = Cin;
    a.kt = kt; a.kh = kh; a.kw = kw; a.st = st; a.sh = sh; a.sw = sw; a.ph = ph; a.pw = pw;
    a.t_base = t_base;
    a.Tout = split_time ? out.T / 2 : out.T; a.Hout = out.H; a.Wout = out.W;
    a.split_time = split_time;
    if (planar) {
      a.planar_out = 1; a.clamp = planar->clamp; a.planar_T = planar->T; a.planar_t0 = planar->t0;
    }
    if (!fp32) {
      a.bias = weights.any<bf16>(name + ".bias", a.Cout);
      a.y = out.p; a.resid = resid.p;
      launch([&] { return launch_conv3d_cl(a, s); });
      return;
    }
    ConvF32 f;
    f.bias = weights.any<float>(name + ".bias", a.Cout);
    f.resid = resid.f; f.y = out.f; f.y_pair = out.p;
    launch([&] { return launch_conv3d_cl_f32(a, f, s); });
  }
  // streaming causal conv (kt = 3): x is already in the stream buffer's chunk region; halo rows replace the rows' zero padding
  void causal_conv(const std::string& name, StreamBuf& b, int T, const Act& out, int kh, const Act& resid = Act(), int split_time = 0,
                   const Planar* planar = nullptr) {
    conv(name, b.p, b.hist + T, b.H, b.W, b.C, out, 3, kh, kh, 1, 1, 1, b.halo ? 0 : kh / 2, kh / 2, resid, split_time, 0, planar);
    push_history(b, T);
    b.primed = true;
  }
  void gemm(const bf16* A, int lda, const bf16* Wt, int ldw, int M, int N, int K, bf16* out, int ldo, const bf16* bias, int epi = EPI_BIAS,
            const bf16* resid = nullptr, int ldr = 0) {
    if (!dry && !rc) rc = run_gemm(run, A, lda, Wt, ldw, M, N, K, out, ldo, bias, epi, resid, ldr);
  }
  // bf16 small-Cin conv: im2row + GEMM.  x addressed by strides (planar or channels-last); output row oh reads rows oh + dh - ph of x
  void small_conv(const std::string& name, const bf16* x, size_t sc, size_t st_, size_t sh, size_t sw, int Tin, int Hin, int Win, int Cin,
                  int t_base, int kt, int kh, bf16* out, int ldo, int Tout, int Hout, int ph, int Cout) {
    const int K = kt * kh * kh * Cin, Kpad = round_up(K, 8);
    bf16* A = take<bf16>((size_t)Tout * Hout * Win * Kpad);
    const bf16* w = weights.any<bf16>(name + ".weight", (int64_t)Cout * Kpad);
    const bf16* b = weights.any<bf16>(name + ".bias", Cout);
    launch([&] {
      return launch_im2row(x, sc, st_, sh, sw, Tin, Hin, Win, Cin, A, Kpad, Tout, Hout, Win, kt, kh, kh, ph, kh / 2, t_base, s);
    });
    gemm(A, Kpad, w, Kpad, Tout * Hout * Win, Cout, Kpad, out, ldo, b);
  }
  // the caller's planar input [C, pixels] as the stems read it: bf16 in place, fp32 as its pair [pixels, 2, Cp] in the persistent region
  const bf16* stem_input(const void* x, int C, int Cp, size_t pixels) {
    if (!fp32) return static_cast<const bf16*>(x);
    bf16* pair = persist.take<bf16>((int64_t)pixels * 2 * Cp);
    launch([&] { return launch_planar_to_pair(static_cast<const float*>(x), C, pixels, pair, Cp, s); });
    return pair;
  }
  // the caller's planar output: bf16 as a convolution's out.p, fp32 as its out.f
  Act caller_out(void* y, int T, int H, int W, int C) {
    Act a;
    a.T = T; a.H = H; a.W = W; a.C = C;
    if (fp32) a.f = static_cast<float*>(y);
    else a.p = static_cast<bf16*>(y);
    return a;
  }
  // nearest 2x upsample of x into scratch, as the convolution after it reads it (bf16, or the fp32 pair)
  bf16* upsample2x(const Act& x) {
    bf16* up = take<bf16>(x.pixels() * 4 * pair() * x.C);
    if (fp32) launch([&] { return launch_upsample2x_cl_f32(x.f, up, x.T, x.H, x.W, x.C, s); });
    else launch([&] { return launch_upsample2x_cl(x.p, up, x.T, x.H, x.W, x.C, s); });
    return up;
  }

  // encoder.conv1 (3x3x3 causal, Cin = 3) of chunk frames f0 .. into x, straight from the whole video (its own past frames are the
  // history).  bf16: im2row + GEMM over the planar video; split: the band's pixel rows and the rows around it, read from the row above
  // the band on (zero padding only at the global top and bottom).  fp32: the implicit conv on the video's pair, 3 channels padded to 8.
  void encoder_stem(const bf16* video, const Act& x, int T, int H, int Wd, int f0) {
    if (fp32) return conv("encoder.conv1", video, T, H, Wd, 8, x, 3, 3, 3, 1, 1, 1, 1, 1, Act(), 0, /*t_base=*/f0 - 2);
    const int skip = band0 > 0 ? 8 * band0 - 1 : 0;
    small_conv("encoder.conv1", at(video, (size_t)skip * Wd), (size_t)T * H * Wd, (size_t)H * Wd, (size_t)Wd, 1, T, H - skip, Wd, 3,
               /*t_base=*/f0 - 2, 3, 3, x.p, x.C, x.T, x.H, band0 > 0 ? 0 : 1, x.C);
  }
  // conv2 (1x1x1 on latent frame i of z [zc, Tl, h, w]) into decoder.conv1's stream buffer, then decoder.conv1 (3x3x3 causal) into a
  // new scratch activation of `top` channels.  bf16: both as im2row + GEMM; split: conv2 writes the band's rows and the halo rows
  // that exist, read from the whole z.  fp32: both implicit convs on the pair.
  Act decoder_stem(const bf16* z, int i, int Tl, int lh, int lw, int top) {
    const int zc = h->cfg.z_dim, a = band0, nb = band1 - band0;
    StreamBuf& s1 = stream("decoder.conv1", 2, 1, nb, lw, zc, true);
    Act x0 = chunk_of(s1, 1);
    if (fp32) {
      conv("conv2", z, Tl, lh, lw, zc, x0, 1, 1, 1, 1, 1, 1, 0, 0, Act(), 0, /*t_base=*/i);
      Act x = act(1, nb, lw, top);
      causal_conv("decoder.conv1", s1, 1, x, 3);
      return x;
    }
    const size_t zplane = (size_t)Tl * lh * lw;
    if (!s1.halo) {
      small_conv("conv2", z, zplane, (size_t)lh * lw, (size_t)lw, 1, Tl, lh, lw, zc, /*t_base=*/i, 1, 1, x0.p, zc, 1, lh, 0, zc);
    } else {
      const int lo = std::max(a - 1, 0), hi = std::min(a + nb + 1, lh);
      small_conv("conv2", at(z, (size_t)lo * lw), zplane, (size_t)lh * lw, (size_t)lw, 1, Tl, hi - lo, lw, zc, /*t_base=*/i, 1, 1,
                 at(x0.p, (size_t)(lo - a + 1) * lw * zc), zc, 1, hi - lo, 0, zc);
    }
    Act x = act(1, nb, lw, top);
    small_conv("decoder.conv1", s1.p, 1, (size_t)s1.H * lw * zc, (size_t)lw * zc, (size_t)zc, s1.hist + 1, s1.H, lw, zc, 0, 3, 3, x.p, top, 1,
               nb, s1.halo ? 0 : 1, top);
    push_history(s1, 1);
    return x;
  }
  // conv1 (1x1x1, 2z -> 2z) of the collected head outputs [P, 2z] (bf16, or the fp32 pair), then planar moments = mean | logvar.  bf16
  // runs it as a GEMM; split: each rank's band is gathered into every rank's moments.
  void encode_tail(const bf16* enc_out, void* moments, int Tl, int nb, int w) {
    const int zc = h->cfg.z_dim;
    const size_t P = (size_t)Tl * nb * w;
    if (fp32) {
      Act q = act(Tl, nb, w, 2 * zc, false);
      conv("conv1", enc_out, Tl, nb, w, 2 * zc, q, 1, 1, 1, 1, 1, 1, 0, 0);
      launch([&] { return launch_cl_to_planar_f32(q.f, 2 * zc, static_cast<float*>(moments), P, 2 * zc, s); });
      return;
    }
    bf16* q = take<bf16>(P * 2 * zc);
    const bf16* w1 = weights.any<bf16>("conv1.weight", (int64_t)4 * zc * zc);
    gemm(enc_out, 2 * zc, w1, 2 * zc, (int)P, 2 * zc, 2 * zc, q, 2 * zc, weights.any<bf16>("conv1.bias", 2 * zc));
    if (!split()) {
      launch([&] { return launch_cl_to_planar(q, 2 * zc, static_cast<bf16*>(moments), P, 2 * zc, s); });
      return;
    }
    bf16* band = take<bf16>(P * 2 * zc);   // the band's moments, planar
    launch([&] { return launch_cl_to_planar(q, 2 * zc, band, P, 2 * zc, s); });
    for (int t = 0; t < Tl; ++t) gather_moments(band, static_cast<bf16*>(moments), t, Tl, 2 * zc, w);
  }

  // ---- blocks
  // ResidualBlock.forward (wan2pt1.py:201-220).  halo_out (split only): the output feeds a stride-2 downsample, so it is written
  // with halo rows (one launch per frame) and its edge rows are exchanged.
  Act res_block(const std::string& n, const Act& x, int Cout, int tcap, bool halo_out = false) {
    next_block();
    StreamBuf& sa = stream(n + ".residual.2", 2, tcap, x.H, x.W, x.C, true);
    Act a_in = chunk_of(sa, x.T);
    rms_into(x, n + ".residual.0.gamma", sa, a_in, true);
    if (sa.halo) halo_exchange(a_in.p, x.T, x.H, x.W, x.C);
    Act t1 = act(x.T, x.H, x.W, Cout, false);
    causal_conv(n + ".residual.2", sa, x.T, t1, 3);
    StreamBuf& sb = stream(n + ".residual.6", 2, tcap, x.H, x.W, Cout, true);
    Act b_in = chunk_of(sb, x.T);
    rms_into(t1, n + ".residual.3.gamma", sb, b_in, true);
    if (sb.halo) halo_exchange(b_in.p, x.T, x.H, x.W, Cout);
    Act hres = x;
    if (x.C != Cout) {
      if (!dry && !x.p && !rc) rc = fail(CE_ERR_INVALID, "vae fp32: a shortcut input without its pair");
      hres = act(x.T, x.H, x.W, Cout, false);
      conv(n + ".shortcut", x.p, x.T, x.H, x.W, x.C, hres, 1, 1, 1, 1, 1, 1, 0, 0);
    }
    if (!(halo_out && split())) {
      Act out = act(x.T, x.H, x.W, Cout);
      causal_conv(n + ".residual.6", sb, x.T, out, 3, hres);
      return out;
    }
    Act out = act(x.T, x.H + 2, x.W, Cout);
    const size_t row = (size_t)x.W * Cout;
    for (int f = 0; f < x.T; ++f) {
      Act of = out, rf = hres;
      of.T = 1; of.H = x.H; of.p = at(out.p, f * out.frame() + row);
      rf.p = at(hres.p, f * x.H * row);
      conv(n + ".residual.6", sb.p, sb.hist + x.T, sb.H, sb.W, sb.C, of, 3, 3, 3, 1, 1, 1, 0, 1, rf, 0, f);
    }
    push_history(sb, x.T);
    sb.primed = true;
    zero_edges(out.p, x.T, x.H, x.W, Cout);
    halo_exchange(out.p, x.T, x.H, x.W, Cout);
    return out;
  }

  // AttentionBlock.forward (wan2pt1.py:240-259): per frame, single head of width C over H*W tokens.  Split (bf16): every rank stores
  // its band of the normalised frame into every rank's region, computes q|k and V^T of the whole frame and S, softmax, P.V, the
  // projection and the residual for its own rows.
  Act attn_block(const std::string& n, const Act& x) {
    next_block();
    Act xn = act(x.T, x.H, x.W, x.C, false);
    rms(x, n + ".norm.gamma", xn, false);
    Act out = act(x.T, x.H, x.W, x.C, false);
    if (fp32) attention_fp32(n, x, xn, out);
    else attention(n, x, xn, out);
    return out;
  }
  void attention(const std::string& n, const Act& x, const Act& xn, const Act& out) {
    const int C = x.C, P = rows * x.W, Ppad = round_up(P, 8);
    const int q0 = band0 * x.W, nq = x.H * x.W;
    GemmAttention a;
    a.wqk = weights.any<bf16>(n + ".to_qkv.weight", (int64_t)3 * C * C);
    a.bqk = weights.any<bf16>(n + ".to_qkv.bias", 3 * C);
    a.wv = a.wqk ? a.wqk + (size_t)2 * C * C : nullptr;
    a.bv = a.bqk ? a.bqk + 2 * C : nullptr;
    const bf16* wproj = weights.any<bf16>(n + ".proj.weight", (int64_t)C * C);
    const bf16* bproj = weights.any<bf16>(n + ".proj.bias", C);
    a.L = P; a.D = C; a.H = 1; a.dk = C; a.kpv = P; a.q0 = q0; a.nq = nq;
    a.sc.rule = SOFTMAX_SCALED;
    a.sc.scale = 1.0f / sqrtf((float)C);
    a.qk = take<bf16>((size_t)P * 2 * C);
    a.vT = take<bf16>((size_t)C * Ppad);
    a.S = take<float>((size_t)nq * Ppad);
    a.P = take<bf16>((size_t)nq * Ppad);
    a.out = take<bf16>((size_t)nq * C);
    a.ldo = C;
    for (int f = 0; f < x.T && !dry && !rc; ++f) {
      a.x = xn.p + (size_t)f * nq * C;
      if (split()) {
        const int set = (int)(h->sp.epoch & 1);
        SpCopy j[8];
        for (int w = 0; w < world; ++w) {
          j[w].src = a.x; j[w].dst = region(w) + lay->frame + set * lay->frame_bytes + (int64_t)q0 * C * 2; j[w].bytes = (int64_t)nq * C * 2;
        }
        peer_copies(j, world);
        barrier();
        a.x = reinterpret_cast<const bf16*>(region(rank) + lay->frame + set * lay->frame_bytes);
      }
      if (!rc) rc = gemm_attention(run, a);
      gemm(a.out, C, wproj, C, nq, C, C, out.p + (size_t)f * nq * C, C, bproj, EPI_BIAS_RESID, x.p + (size_t)f * nq * C, C);   // proj + identity
    }
  }
  void attention_fp32(const std::string& n, const Act& x, const Act& xn, const Act& out) {
    const int C = x.C, L = x.H * x.W, L8 = up8(L), Cp = up8(C);
    Lin32 qkv_w, proj_w;
    qkv_w.w = weights.any<float>(n + ".to_qkv.weight", (int64_t)3 * C * C);
    qkv_w.b = weights.any<float>(n + ".to_qkv.bias", 3 * C);
    proj_w.w = weights.any<float>(n + ".proj.weight", (int64_t)C * C);
    proj_w.b = weights.any<float>(n + ".proj.bias", C);
    float* qkv = take<float>((size_t)L * 3 * C);
    float* o = take<float>((size_t)L * 3 * C);   // attention output in columns [0, C) (Fp32Chain::attention's row stride is qkv's)
    Fp32Chain X{run, nullptr, nullptr, nullptr, nullptr, 6, nullptr};
    X.Ap = take<bf16>((size_t)split_elems(L, std::max(Cp, L8), 6));
    X.Wp = take<bf16>((size_t)std::max({split_elems(3 * C, C, 6), split_elems(L8, C, 6), split_elems(C, L8, 6)}));
    X.S = take<float>((size_t)L * L8);
    X.P = take<float>((size_t)L * L8);
    X.part = take<float>((size_t)L * std::max(3 * C, L8));
    const float scale = 1.0f / sqrtf((float)C);
    for (int f = 0; f < x.T && !dry && !rc; ++f) {
      const size_t off = (size_t)f * L * C;
      if ((rc = X.linear(xn.f + off, C, L, C, qkv_w, 3 * C, qkv, 3 * C, 0))) break;
      if ((rc = X.attention(qkv, qkv + C, qkv + 2 * C, o, 1, 1, L, L, 3 * C, C, scale))) break;
      if ((rc = X.linear(o, 3 * C, L, C, proj_w, C, out.f + off, C, 0))) break;
      rc = X.resid(out.f + off, x.f + off, L, C, nullptr, 0, L);
    }
  }

  // Resample upsample2d / upsample3d (wan2pt1.py:112-143)
  Act upsample(const std::string& n, Act x, bool temporal, int tcap_in) {
    next_block();
    const int C = x.C;
    if (temporal) {
      StreamBuf& st = stream(n + ".time_conv", 2, tcap_in, x.H, x.W, C);
      if (!st.primed) {
        st.primed = true;  // first chunk: "Rep" -- no temporal doubling, history stays zero (:116-120, 128-129)
      } else {
        copy(chunk_of(st, x.T).p, x.p, x.pixels() * pair() * C * 2);
        Act y = act(2 * x.T, x.H, x.W, C, false);
        causal_conv(n + ".time_conv", st, x.T, y, 1, Act(), /*split_time=*/1);
        x = y;
      }
    }
    if (!split()) {
      const bf16* up = upsample2x(x);
      Act out = act(x.T, 2 * x.H, 2 * x.W, C / 2);
      conv(n + ".resample.1", up, x.T, 2 * x.H, 2 * x.W, C, out, 1, 3, 3, 1, 1, 1, 1, 1);
      return out;
    }
    Act up = act(x.T, 2 * x.H + 2, 2 * x.W, C);   // halo'd: one launch per frame into the band rows
    for (int f = 0; f < x.T; ++f) {
      const bf16* xf = at(x.p, f * x.frame());
      bf16* uf = at(up.p, f * up.frame() + (size_t)2 * x.W * C);
      launch([&] { return launch_upsample2x_cl(xf, uf, 1, x.H, x.W, C, s); });
    }
    zero_edges(up.p, x.T, 2 * x.H, 2 * x.W, C);
    halo_exchange(up.p, x.T, 2 * x.H, 2 * x.W, C);
    Act out = act(x.T, 2 * x.H, 2 * x.W, C / 2);
    conv(n + ".resample.1", up.p, up.T, up.H, up.W, C, out, 1, 3, 3, 1, 1, 1, 0, 1);
    return out;
  }

  // Resample downsample2d / downsample3d (wan2pt1.py:145-159): ZeroPad2d(0,1,0,1) is the zero fill past the edge.  Split: x is
  // halo'd; ph = -1 skips its row above, and the row below the band (zero at the global bottom) is what ZeroPad2d(0,1,0,1) and the
  // stride-2 window read there.
  Act downsample(const std::string& n, const Act& x, bool temporal, int tcap_out_spatial) {
    next_block();
    const int C = x.C, band = split() ? x.H - 2 : x.H, ph = split() ? -1 : 0;
    const int Ho = (band + 1 - 3) / 2 + 1, Wo = (x.W + 1 - 3) / 2 + 1;
    if (!temporal) {
      Act out = act(x.T, Ho, Wo, C);
      conv(n + ".resample.1", x.p, x.T, x.H, x.W, C, out, 1, 3, 3, 1, 2, 2, ph, 0);
      return out;
    }
    StreamBuf& st = stream(n + ".time_conv", 1, tcap_out_spatial, Ho, Wo, C);
    Act sp = chunk_of(st, x.T);
    const bool first = !st.primed;
    if (first && fp32) sp.f = take<float>(sp.pixels() * C);
    conv(n + ".resample.1", x.p, x.T, x.H, x.W, C, sp, 1, 3, 3, 1, 2, 2, ph, 0);
    if (first) {  // first chunk passes through and becomes the history (:147-150)
      st.primed = true;
      Act out = sp;   // fp32: the chunk itself, whose pair nothing rewrites before the next chunk; bf16: a copy in scratch
      if (!fp32) {
        out = act(x.T, Ho, Wo, C);
        copy(out.p, sp.p, sp.pixels() * C * 2);
      }
      push_history(st, x.T);
      return out;
    }
    const int To = (1 + x.T - 3) / 2 + 1;
    Act out = act(To, Ho, Wo, C);
    conv(n + ".time_conv", st.p, 1 + x.T, Ho, Wo, C, out, 3, 1, 1, 2, 1, 1, 0, 0);
    push_history(st, x.T);
    return out;
  }

  // ---- gathering the outputs (split)
  // band = the decoder head's planar output [3, T, band rows, W] of this rank; store it into every rank's region video buffer
  // [3, video_frames, H, W], barrier, then copy the whole chunk into frames t0 .. t0 + T - 1 of the caller's video [3, T_px, H, W].
  void gather_video(const bf16* band, bf16* video, int T_px, int t0, int T, int H, int W) {
    if (dry || rc) return;
    const int64_t plane = (int64_t)H * W * 2, chan = lay->video_frames * plane;
    const int64_t r0 = (int64_t)band0 * 8 * W * 2, bytes = (int64_t)(band1 - band0) * 8 * W * 2;
    SpCopy j[8];
    for (int w = 0; w < world; ++w) {
      j[w].src = band; j[w].dst = region(w) + lay->video + r0; j[w].bytes = bytes;
      j[w].n0 = T; j[w].sp0 = bytes; j[w].dp0 = plane; j[w].n1 = 3; j[w].sp1 = T * bytes; j[w].dp1 = chan;
    }
    peer_copies(j, world);
    barrier();
    copy_2d(reinterpret_cast<uint8_t*>(video) + t0 * plane, (size_t)T_px * plane, region(rank) + lay->video, chan, T * plane, 3);
  }
  // band = this rank's moments [2 z_dim, Tl, band rows, w] (planar); latent frame t of every rank's band into every rank's region,
  // barrier, then the whole frame into moments [2 z_dim, Tl, h, w].
  void gather_moments(const bf16* band, bf16* moments, int t, int Tl, int Cm, int w) {
    if (dry || rc) return;
    const int set = (int)(h->sp.epoch & 1);
    const int nb = band1 - band0;
    const int64_t plane = (int64_t)rows * w * 2, bplane = (int64_t)nb * w * 2;
    SpCopy j[8];
    for (int r = 0; r < world; ++r) {
      j[r].src = reinterpret_cast<const uint8_t*>(band) + t * bplane;
      j[r].dst = region(r) + lay->moments + set * lay->moments_bytes + (int64_t)band0 * w * 2;
      j[r].bytes = bplane; j[r].n0 = Cm; j[r].sp0 = Tl * bplane; j[r].dp0 = plane;
    }
    peer_copies(j, world);
    barrier();
    copy_2d(reinterpret_cast<uint8_t*>(moments) + t * plane, (size_t)Tl * plane, region(rank) + lay->moments + set * lay->moments_bytes, plane,
            plane, Cm);
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
int run_decode(Run& R, const void* z, void* video, int Tl, int h, int w, int clamp) {
  const ce_vae_config& c = R.h->cfg;
  const int top = top_dim(c), zc = c.z_dim;
  const int T_px = 1 + 4 * (Tl - 1);
  const bf16* zin = R.stem_input(z, zc, zc, (size_t)Tl * h * w);
  R.set_band(h);
  std::vector<LayerSpec> layers = decoder_layers(c);
  int t_out = 0;
  for (int i = 0; i < Tl && !R.rc; ++i) {
    R.new_chunk();
    int cap = 1;  // frames a non-first chunk carries at the current depth (x2 after every upsample3d): stream capacity
    Act x = R.decoder_stem(zin, i, Tl, h, w, top);
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
    // head: RMS + SiLU + conv dim->3, planar clamped store straight into the output video (split: into a planar band [3, T, rows, W],
    // then gathered)
    StreamBuf& sh = R.stream("decoder.head.2", 2, cap, x.H, x.W, x.C, true);
    Act hin = R.chunk_of(sh, x.T);
    R.rms_into(x, "decoder.head.0.gamma", sh, hin, true);
    if (sh.halo) R.halo_exchange(hin.p, x.T, x.H, x.W, x.C);
    Act o = R.caller_out(video, x.T, x.H, x.W, 3);
    Planar pl{T_px, t_out, clamp};
    if (R.split()) {
      o.p = R.take<bf16>((size_t)3 * x.T * x.H * x.W);
      pl = Planar{x.T, 0, clamp};
    }
    R.causal_conv("decoder.head.2", sh, x.T, o, 3, Act(), 0, &pl);
    if (R.split()) R.gather_video(o.p, static_cast<bf16*>(video), T_px, t_out, x.T, 8 * h, x.W);
    t_out += x.T;
  }
  if (!R.rc && t_out != T_px) return fail(CE_ERR_INVALID, "vae decode: produced frame count mismatch");
  return R.rc;
}

// ---------------------------------------------------------------------------------------------- encode
// WanVAE_.encode (wan2pt1.py:502-533) + Encoder3d.forward (:315-357); video planar [3, T, H, W] -> moments planar [2 zc, Tl, H/8, W/8]
int run_encode(Run& R, const void* video, void* moments, int T, int H, int Wd) {
  const ce_vae_config& c = R.h->cfg;
  const int top = top_dim(c), zc = c.z_dim;
  const int Tl = 1 + (T - 1) / 4, h = H / 8, w = Wd / 8;
  const bf16* vin = R.stem_input(video, 3, 8, (size_t)T * H * Wd);
  R.set_band(h);
  const int nb = R.band1 - R.band0;   // the band's latent rows
  std::vector<LayerSpec> layers = encoder_layers(c);
  const size_t out_frame = (size_t)nb * w * 2 * zc * R.pair();
  bf16* enc_out = R.persist.take<bf16>((int64_t)(Tl * out_frame));  // head outputs of every chunk, channels-last (fp32: the pair)
  int t_lat = 0;
  for (int f0 = 0; f0 < T && !R.rc;) {
    const int Tc = f0 == 0 ? 1 : 4;
    R.new_chunk();
    int cap = 4;
    Act x = R.act(Tc, 8 * nb, Wd, c.dim);
    R.encoder_stem(vin, x, T, H, Wd, f0);
    for (size_t li = 0; li < layers.size(); ++li) {
      const LayerSpec& l = layers[li];
      const std::string n = "encoder.downsamples." + std::to_string(li);
      if (l.res) {
        x = R.res_block(n, x, l.cout, cap, li + 1 < layers.size() && !layers[li + 1].res);
      } else {
        x = R.downsample(n, x, l.mode == 1, cap);
        if (l.mode == 1) cap = cap > 1 ? cap / 2 : 1;
      }
    }
    x = R.res_block("encoder.middle.0", x, top, cap);
    x = R.attn_block("encoder.middle.1", x);
    x = R.res_block("encoder.middle.2", x, top, cap);
    StreamBuf& sh = R.stream("encoder.head.2", 2, cap, x.H, x.W, x.C, true);
    Act hin = R.chunk_of(sh, x.T);
    R.rms_into(x, "encoder.head.0.gamma", sh, hin, true);
    if (sh.halo) R.halo_exchange(hin.p, x.T, x.H, x.W, x.C);
    if (x.H != nb || x.W != w) return fail(CE_ERR_INVALID, "vae encode: spatial size mismatch (H, W must be multiples of 8)");
    Act o;
    o.T = x.T; o.H = x.H; o.W = x.W; o.C = 2 * zc;
    o.p = at(enc_out, t_lat * out_frame);
    R.causal_conv("encoder.head.2", sh, x.T, o, 3);
    t_lat += x.T;
    f0 += Tc;
  }
  if (!R.rc && t_lat != Tl) return fail(CE_ERR_INVALID, "vae encode: produced frame count mismatch");
  R.new_chunk();
  R.encode_tail(enc_out, moments, Tl, nb, w);
  return R.rc;
}

// One encode or decode: `R` plans (dry) or launches.  A planning pass leaves the first missing or mis-sized weight in R.weights.rc.
int walk(Run& R, bool decode, const void* in, void* out, int frames, int height, int width, int clamp) {
  return decode ? run_decode(R, in, out, frames, height, width, clamp) : run_encode(R, in, out, frames, height, width);
}

int check_geometry(const ce_vae* h, int T, int H, int W, bool decode) {
  CE_REQUIRE(h != nullptr, "vae: null handle");
  if (decode) {
    CE_REQUIRE(T >= 1 && H >= 1 && W >= 1, "vae decode: empty latent");
  } else {
    CE_REQUIRE(T >= 1 && (T - 1) % 4 == 0, "vae encode: frame count must be 1 + 4k (the reference fails otherwise)");
    CE_REQUIRE(H % 8 == 0 && W % 8 == 0 && H >= 8 && W >= 8, "vae encode: H, W must be multiples of 8");
  }
  if (h->sp.world > 1) {
    const int rows = decode ? H : H / 8;
    if (rows < h->sp.world)
      return fail(CE_ERR_INVALID, "vae sequence parallel: " + std::to_string(rows) + " latent rows cannot be split over " +
                                      std::to_string(h->sp.world) + " ranks (at least one row per rank)");
  }
  return CE_OK;
}

int count_temporal(const ce_vae_config& c) { return (c.temporal_downsample[0] != 0) + (c.temporal_downsample[1] != 0) + (c.temporal_downsample[2] != 0); }

// The peer region's layout for pixel geometry H x W.  The halo slot holds the largest halo row of any chunk: a planning pass of one
// 4-frame encode chunk and of one decode chunk past the first (later chunks have the same shapes) measures it.
int vae_sp_layout(ce_vae* h, int H, int W, int world, VaeSpLayout& L) {
  const ce_vae_config& c = h->cfg;
  const int lh = H / 8, lw = W / 8;
  Run enc(h, false, 0, world), dec(h, false, 0, world);
  CE_TRY(walk(enc, false, nullptr, nullptr, 5, H, W, 0));
  CE_TRY(walk(dec, true, nullptr, nullptr, 2, lh, lw, 0));
  auto al = [](int64_t v) { return (v + 1023) & ~int64_t(1023); };
  L = VaeSpLayout();
  L.flags = 0;
  L.halo = 1024;
  L.halo_slot = al(std::max(enc.halo_row_max, dec.halo_row_max));
  L.frame = L.halo + 4 * L.halo_slot;
  L.frame_bytes = al((int64_t)up8(lh * lw) * top_dim(c) * 2);
  L.video = L.frame + 2 * L.frame_bytes;
  L.video_frames = 1 << count_temporal(c);
  L.moments = L.video + al((int64_t)3 * L.video_frames * H * W * 2);
  L.moments_bytes = al((int64_t)2 * c.z_dim * lh * lw * 2);
  L.bytes = L.moments + 2 * L.moments_bytes;
  return CE_OK;
}

// One untiled encode or decode, bf16 or fp32, split over the configured ranks.  Every entry refuses in this order: the handle and
// the geometry; the precision's and the split's refusals; the planning pass, which checks every weight; with need != null, the
// answer to the workspace query; the device; the arguments; the split's capture and region checks, all before its first barrier;
// the workspace size.  The launch count restarts at zero.
int vae_call(ce_vae* h, bool decode, bool fp32, const void* in, void* out, int frames, int height, int width, int clamp, void* workspace,
             int64_t workspace_bytes, int64_t* need, void* stream) {
  CE_TRY(check_geometry(h, frames, height, width, decode));
  if (fp32 && h->sp.world > 1)
    return fail(CE_ERR_INVALID, "vae fp32: the VAE split over GPUs (ce_vae_sp_configure) is built for bf16 only; configure world = 1");
  CE_REQUIRE(!fp32 || !h->w32.empty(), "vae fp32: the handle has no fp32 weights (register them with ce_vae_set_weight_fp32)");
  Run plan(h, fp32, h->sp.rank, h->sp.world);
  CE_TRY(walk(plan, decode, nullptr, nullptr, frames, height, width, 0));
  CE_TRY(plan.weights.rc);
  if (need) {
    *need = plan.workspace_bytes();
    return CE_OK;
  }
  const std::string who = fp32 ? "vae fp32: " : "vae: ";
  CE_TRY(check_device());
  CE_REQUIRE(in && out && workspace, who + "null argument");
  CE_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, who + "workspace must be 256-byte aligned");
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  VaeSpLayout lay;
  if (plan.split()) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    CE_CHECK_CUDA(cudaStreamIsCapturing(s, &cs));
    CE_REQUIRE(cs == cudaStreamCaptureStatusNone, "vae sequence parallel: the stream is capturing (the split VAE cannot be captured)");
    const int H = decode ? 8 * height : height, W = decode ? 8 * width : width;
    CE_TRY(vae_sp_layout(h, H, W, h->sp.world, lay));
    if (lay.bytes > h->sp.region_bytes)
      return fail(CE_ERR_WORKSPACE, "vae sequence parallel: a " + std::to_string(H) + " x " + std::to_string(W) + " call needs a peer region of " +
                                        std::to_string(lay.bytes) + " bytes, the handle was configured with " +
                                        std::to_string(h->sp.region_bytes) + " (ce_vae_sp_region_bytes)");
  }
  const int64_t bytes = plan.workspace_bytes();
  if (bytes > workspace_bytes)
    return fail(CE_ERR_WORKSPACE, who + "workspace too small: need " + std::to_string(bytes) + " bytes, got " + std::to_string(workspace_bytes));
  Run R(h, fp32, h->sp.rank, h->sp.world, s);
  R.bind(reinterpret_cast<uint8_t*>(workspace), plan);
  R.lay = &lay;
  h->launches = 0;
  int rc = walk(R, decode, in, out, frames, height, width, clamp);
  if (!rc && R.split()) {   // nobody stores into a peer's region (next call) before the peer has read it
    R.barrier();
    rc = R.rc;
  }
  return rc;
}

int64_t workspace_query(ce_vae* h, bool decode, bool fp32, int frames, int height, int width) {
  int64_t need = -1;
  return vae_call(h, decode, fp32, nullptr, nullptr, frames, height, width, 0, nullptr, 0, &need, nullptr) ? -1 : need;
}

// ---------------------------------------------------------------------------------------------- tiled encode / decode
// diffusers AutoencoderKLWan.tiled_encode / tiled_decode: the frame is cut into overlapping tiles, each tile is a fresh untiled
// encode or decode (its own causal cache), and each result is blended with its blended upper and left neighbours (blend_v, then
// blend_h) and cropped to the stride.  Tiles are walked row-major in C; a tile is blended right after it is computed, which gives
// the same values as diffusers' blend-after-everything because a tile only reads neighbours that come before it.  What a later tile
// reads of a blended tile is kept, nothing else: the last blend_v rows of every tile of the previous and the current grid row (the
// strips) and the last blend_h columns of the previous and the current tile (the tails).

struct TileSpec {   // pixels, multiples of 8
  int min_h, min_w, stride_h, stride_w;
};

// The grid in latent units: tile (i, j) covers latent rows [i sh, i sh + min(mh, h - i sh)) and the matching columns.  A decode tile's
// input is those latents and its output 8x them in pixels; an encode tile's input is the pixels and its output the latents.
struct TileGrid {
  bool decode, fp32;
  int es;                        // element bytes
  int Cin, Tin, Cout, Tout;      // input [Cin, Tin, ...], output [Cout, Tout, ...]
  int h, w;                      // latent geometry
  int mh, mw, sh, sw;            // tile size and stride, latents
  int rows, cols;
  int in_f, out_f;               // input / output units per latent: (1, 8) decode, (8, 1) encode
  int bv, bw;                    // blend extents, output units
  int lat_h(int i) const { return std::min(mh, h - i * sh); }
  int lat_w(int j) const { return std::min(mw, w - j * sw); }
};

struct TileLayout {
  int64_t run_bytes = 0;
  uint8_t *run = nullptr, *stage = nullptr, *tile = nullptr, *strip[2] = {nullptr, nullptr}, *tail[2] = {nullptr, nullptr};
  int64_t strip_slot = 0;        // bytes of one tile's strip
  int64_t bytes = 0;
};

int tile_grid(const ce_vae* h, bool decode, bool fp32, int frames, int height, int width, const TileSpec& ts, TileGrid& g) {
  CE_TRY(check_geometry(h, frames, height, width, decode));
  if (h->sp.world > 1)
    return fail(CE_ERR_INVALID, "vae tiled: tiling is not built for the VAE split over GPUs (ce_vae_sp_configure); configure world = 1");
  CE_REQUIRE(ts.min_h >= 8 && ts.min_w >= 8 && ts.stride_h >= 8 && ts.stride_w >= 8 && ts.min_h % 8 == 0 && ts.min_w % 8 == 0 &&
                 ts.stride_h % 8 == 0 && ts.stride_w % 8 == 0,
             "vae tiled: tile sizes and strides must be positive multiples of 8 pixels");
  CE_REQUIRE(ts.stride_h <= ts.min_h && ts.stride_w <= ts.min_w, "vae tiled: a stride larger than the tile leaves pixels no tile covers");
  CE_REQUIRE(!fp32 || !h->w32.empty(), "vae tiled fp32: the handle has no fp32 weights (register them with ce_vae_set_weight_fp32)");
  g.decode = decode;
  g.fp32 = fp32;
  g.es = fp32 ? 4 : 2;
  const int zc = h->cfg.z_dim;
  g.h = decode ? height : height / 8;
  g.w = decode ? width : width / 8;
  g.mh = ts.min_h / 8; g.mw = ts.min_w / 8; g.sh = ts.stride_h / 8; g.sw = ts.stride_w / 8;
  g.rows = (g.h + g.sh - 1) / g.sh;
  g.cols = (g.w + g.sw - 1) / g.sw;
  g.in_f = decode ? 1 : 8;
  g.out_f = decode ? 8 : 1;
  g.Cin = decode ? zc : 3;
  g.Tin = frames;
  g.Cout = decode ? 3 : 2 * zc;
  g.Tout = decode ? 1 + 4 * (frames - 1) : 1 + (frames - 1) / 4;
  g.bv = (g.mh - g.sh) * g.out_f;
  g.bw = (g.mw - g.sw) * g.out_f;
  return CE_OK;
}

// Workspace: one tile's untiled run (the largest of the at most four tile shapes) | the staged input tile | the tile's output |
// two rows of strips | two tails.  Only the strips grow with the frame, by one tile's strip per tile column.
int tile_layout(ce_vae* h, const TileGrid& g, uint8_t* base, TileLayout& L) {
  L = TileLayout();
  for (int i : {0, g.rows - 1})
    for (int j : {0, g.cols - 1}) {
      int64_t need = 0;
      const int th = g.lat_h(i) * g.in_f, tw = g.lat_w(j) * g.in_f;
      CE_TRY(vae_call(h, g.decode, g.fp32, nullptr, nullptr, g.Tin, th, tw, 0, nullptr, 0, &need, nullptr));
      L.run_bytes = std::max(L.run_bytes, need);
    }
  const int64_t mh = std::min(g.mh, g.h), mw = std::min(g.mw, g.w);
  Bump b(base);
  L.run = b.take<uint8_t>(L.run_bytes);
  L.stage = b.take<uint8_t>((int64_t)g.Cin * g.Tin * mh * g.in_f * mw * g.in_f * g.es);
  L.tile = b.take<uint8_t>((int64_t)g.Cout * g.Tout * mh * g.out_f * mw * g.out_f * g.es);
  L.strip_slot = ((int64_t)g.Cout * g.Tout * std::min<int64_t>(g.bv, mh * g.out_f) * mw * g.out_f * g.es + 255) & ~int64_t(255);
  for (int k = 0; k < 2; ++k) L.strip[k] = b.take<uint8_t>(g.rows > 1 && g.bv > 0 ? g.cols * L.strip_slot : 0);
  for (int k = 0; k < 2; ++k)
    L.tail[k] = b.take<uint8_t>(g.cols > 1 ? (int64_t)g.Cout * g.Tout * mh * g.out_f * std::min<int64_t>(g.bw, mw * g.out_f) * g.es : 0);
  L.bytes = b.bytes() + 256;
  return CE_OK;
}

int run_tiled(ce_vae* h, bool decode, bool fp32, const void* in, void* out, int frames, int height, int width, const TileSpec& ts,
              int clamp, void* workspace, int64_t workspace_bytes, int64_t* need_out, void* stream) {
  TileGrid g;
  CE_TRY(tile_grid(h, decode, fp32, frames, height, width, ts, g));
  TileLayout L;
  CE_TRY(tile_layout(h, g, nullptr, L));
  if (need_out) {
    *need_out = L.bytes;
    return CE_OK;
  }
  CE_TRY(check_device());
  CE_REQUIRE(in && out && workspace, "vae tiled: null argument");
  CE_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "vae tiled: workspace must be 256-byte aligned");
  if (L.bytes > workspace_bytes)
    return fail(CE_ERR_WORKSPACE, "vae tiled: workspace too small: need " + std::to_string(L.bytes) + " bytes, got " + std::to_string(workspace_bytes));
  CE_TRY(tile_layout(h, g, reinterpret_cast<uint8_t*>(workspace), L));
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  Launcher launch{s, &h->launches};
  h->launches = 0;
  const int IH = g.h * g.in_f, IW = g.w * g.in_f;
  for (int i = 0; i < g.rows; ++i)
    for (int j = 0; j < g.cols; ++j) {
      const int lh = g.lat_h(i), lw = g.lat_w(j);
      const int ih = lh * g.in_f, iw = lw * g.in_f;
      // the tile's input, contiguous: [Cin, Tin, ih, iw] out of [Cin, Tin, IH, IW]
      cudaMemcpy3DParms p = {};
      p.srcPtr = make_cudaPitchedPtr(const_cast<void*>(in), (size_t)IW * g.es, (size_t)IW, (size_t)IH);
      p.srcPos = make_cudaPos((size_t)j * g.sw * g.in_f * g.es, (size_t)i * g.sh * g.in_f, 0);
      p.dstPtr = make_cudaPitchedPtr(L.stage, (size_t)iw * g.es, (size_t)iw, (size_t)ih);
      p.extent = make_cudaExtent((size_t)iw * g.es, (size_t)ih, (size_t)g.Cin * g.Tin);
      p.kind = cudaMemcpyDeviceToDevice;
      CE_CHECK_CUDA(cudaMemcpy3DAsync(&p, s));
      const int64_t launched = h->launches;   // vae_call counts the tile's launches from zero
      CE_TRY(vae_call(h, decode, fp32, L.stage, L.tile, g.Tin, ih, iw, 0, L.run, L.run_bytes, nullptr, stream));
      h->launches += launched;
      TileBlend b;
      b.fp32 = fp32;
      b.tile = L.tile; b.C = g.Cout; b.T = g.Tout; b.th = lh * g.out_f; b.tw = lw * g.out_f;
      if (i > 0 && g.bv > 0) {
        b.above = L.strip[(i - 1) & 1] + j * L.strip_slot;
        b.above_h = std::min(g.bv, g.lat_h(i - 1) * g.out_f);
      }
      if (j > 0 && g.bw > 0) {
        b.left = L.tail[(j - 1) & 1];
        b.left_w = std::min(g.bw, g.lat_w(j - 1) * g.out_f);
      }
      b.out = out; b.out_h = g.h * g.out_f; b.out_w = g.w * g.out_f;
      b.oy = i * g.sh * g.out_f; b.ox = j * g.sw * g.out_f; b.crop_h = g.sh * g.out_f; b.crop_w = g.sw * g.out_f;
      b.clamp = clamp;
      if (i + 1 < g.rows && g.bv > 0) {
        b.strip = L.strip[i & 1] + j * L.strip_slot;
        b.strip_h = std::min(g.bv, b.th);
      }
      if (j + 1 < g.cols && g.bw > 0) {
        b.tail = L.tail[j & 1];
        b.tail_w = std::min(g.bw, b.tw);
      }
      CE_TRY(launch([&] { return launch_tile_blend(b, s); }));
    }
  return CE_OK;
}

// The fields of a convolution's arguments that do not depend on its precision (bias, output and residual do).
ConvArgs conv_args(const ce_conv3d_args& c) {
  ConvArgs a;
  a.x = reinterpret_cast<const bf16*>(c.x); a.Tin = c.Tin; a.Hin = c.Hin; a.Win = c.Win; a.Cin = c.Cin;
  a.w = reinterpret_cast<const bf16*>(c.w); a.Cout = c.Cout; a.Cin_pad = c.Cin_pad;
  a.kt = c.kt; a.kh = c.kh; a.kw = c.kw; a.st = c.st; a.sh = c.sh; a.sw = c.sw; a.ph = c.ph; a.pw = c.pw;
  a.t_base = c.t_base;
  a.Tout = c.Tout; a.Hout = c.Hout; a.Wout = c.Wout;
  a.split_time = c.split_time;
  a.planar_out = c.planar_out; a.clamp = c.clamp; a.planar_T = c.planar_T; a.planar_t0 = c.planar_t0;
  return a;
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
  return workspace_query(h, decode != 0, false, frames, height, width);
}

int ce_vae_encode(ce_vae* h, const void* video, void* mean, int frames, int height, int width, void* workspace, int64_t workspace_bytes,
                  void* stream) {
  return vae_call(h, false, false, video, mean, frames, height, width, 0, workspace, workspace_bytes, nullptr, stream);
}

int ce_vae_decode(ce_vae* h, const void* z, void* video, int latent_frames, int latent_height, int latent_width, int clamp, void* workspace,
                  int64_t workspace_bytes, void* stream) {
  return vae_call(h, true, false, z, video, latent_frames, latent_height, latent_width, clamp, workspace, workspace_bytes, nullptr, stream);
}

int ce_vae_set_weight_fp32(ce_vae* h, const char* name, const void* ptr, int64_t numel) {
  CE_REQUIRE(h, "ce_vae_set_weight_fp32: null handle");
  return register_weight(h->w32, "ce_vae_set_weight_fp32", name, ptr, -1, numel);
}

int64_t ce_vae_workspace_bytes_fp32(ce_vae* h, int decode, int frames, int height, int width) {
  return workspace_query(h, decode != 0, true, frames, height, width);
}

int ce_vae_encode_fp32(ce_vae* h, const float* video, float* moments, int frames, int height, int width, void* workspace,
                       int64_t workspace_bytes, void* stream) {
  return vae_call(h, false, true, video, moments, frames, height, width, 0, workspace, workspace_bytes, nullptr, stream);
}

int ce_vae_decode_fp32(ce_vae* h, const float* z, float* video, int latent_frames, int latent_height, int latent_width, int clamp,
                       void* workspace, int64_t workspace_bytes, void* stream) {
  return vae_call(h, true, true, z, video, latent_frames, latent_height, latent_width, clamp, workspace, workspace_bytes, nullptr, stream);
}

int64_t ce_vae_last_launch_count(const ce_vae* h) { return h ? h->launches : 0; }

static int64_t tiled_bytes(ce_vae* h, bool fp32, int decode, int frames, int height, int width, int mh, int mw, int sh, int sw) {
  int64_t need = -1;
  return run_tiled(h, decode != 0, fp32, nullptr, nullptr, frames, height, width, TileSpec{mh, mw, sh, sw}, 0, nullptr, 0, &need, nullptr)
             ? -1
             : need;
}

int64_t ce_vae_workspace_bytes_tiled(ce_vae* h, int decode, int frames, int height, int width, int tile_min_height, int tile_min_width,
                                     int tile_stride_height, int tile_stride_width) {
  return tiled_bytes(h, false, decode, frames, height, width, tile_min_height, tile_min_width, tile_stride_height, tile_stride_width);
}

int64_t ce_vae_workspace_bytes_tiled_fp32(ce_vae* h, int decode, int frames, int height, int width, int tile_min_height, int tile_min_width,
                                          int tile_stride_height, int tile_stride_width) {
  return tiled_bytes(h, true, decode, frames, height, width, tile_min_height, tile_min_width, tile_stride_height, tile_stride_width);
}

int ce_vae_encode_tiled(ce_vae* h, const void* video, void* moments, int frames, int height, int width, int tile_min_height, int tile_min_width,
                        int tile_stride_height, int tile_stride_width, void* workspace, int64_t workspace_bytes, void* stream) {
  return run_tiled(h, false, false, video, moments, frames, height, width,
                   TileSpec{tile_min_height, tile_min_width, tile_stride_height, tile_stride_width}, 0, workspace, workspace_bytes, nullptr, stream);
}

int ce_vae_decode_tiled(ce_vae* h, const void* z, void* video, int latent_frames, int latent_height, int latent_width, int tile_min_height,
                        int tile_min_width, int tile_stride_height, int tile_stride_width, int clamp, void* workspace, int64_t workspace_bytes,
                        void* stream) {
  return run_tiled(h, true, false, z, video, latent_frames, latent_height, latent_width,
                   TileSpec{tile_min_height, tile_min_width, tile_stride_height, tile_stride_width}, clamp, workspace, workspace_bytes, nullptr,
                   stream);
}

int ce_vae_encode_tiled_fp32(ce_vae* h, const float* video, float* moments, int frames, int height, int width, int tile_min_height,
                             int tile_min_width, int tile_stride_height, int tile_stride_width, void* workspace, int64_t workspace_bytes,
                             void* stream) {
  return run_tiled(h, false, true, video, moments, frames, height, width,
                   TileSpec{tile_min_height, tile_min_width, tile_stride_height, tile_stride_width}, 0, workspace, workspace_bytes, nullptr, stream);
}

int ce_vae_decode_tiled_fp32(ce_vae* h, const float* z, float* video, int latent_frames, int latent_height, int latent_width, int tile_min_height,
                             int tile_min_width, int tile_stride_height, int tile_stride_width, int clamp, void* workspace,
                             int64_t workspace_bytes, void* stream) {
  return run_tiled(h, true, true, z, video, latent_frames, latent_height, latent_width,
                   TileSpec{tile_min_height, tile_min_width, tile_stride_height, tile_stride_width}, clamp, workspace, workspace_bytes, nullptr,
                   stream);
}

int ce_vae_tile_blend(const ce_vae_tile_blend_args* args, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  CE_REQUIRE(args != nullptr, "ce_vae_tile_blend: null args");
  TileBlend b;
  b.fp32 = args->fp32;
  b.tile = args->tile; b.C = args->C; b.T = args->T; b.th = args->th; b.tw = args->tw;
  b.above = args->above; b.above_h = args->above_h;
  b.left = args->left; b.left_w = args->left_w;
  b.out = args->out; b.out_h = args->out_h; b.out_w = args->out_w; b.oy = args->oy; b.ox = args->ox;
  b.crop_h = args->crop_h; b.crop_w = args->crop_w; b.clamp = args->clamp;
  b.strip = args->strip; b.strip_h = args->strip_h;
  b.tail = args->tail; b.tail_w = args->tail_w;
  return launch_tile_blend(b, reinterpret_cast<cudaStream_t>(stream));
}

int64_t ce_vae_sp_region_bytes(ce_vae* h, int height, int width, int world) {
  CE_REQUIRE(h, "ce_vae_sp_region_bytes: null handle");
  CE_REQUIRE(world >= 2 && world <= 8, "ce_vae_sp_region_bytes: world must be 2 to 8");
  CE_REQUIRE(height % 8 == 0 && width % 8 == 0 && height >= 8 && width >= 8, "ce_vae_sp_region_bytes: height, width must be multiples of 8");
  if (height / 8 < world)
    return fail(CE_ERR_INVALID, "ce_vae_sp_region_bytes: " + std::to_string(height / 8) + " latent rows cannot be split over " +
                                    std::to_string(world) + " ranks (at least one row per rank)");
  VaeSpLayout L;
  CE_TRY(vae_sp_layout(h, height, width, world, L));
  return L.bytes;
}

int ce_vae_sp_configure(ce_vae* h, int rank, int world, void* const* region_ptrs, int64_t region_bytes) {
  CE_REQUIRE(h, "ce_vae_sp_configure: null handle");
  return sp_configure(h->sp, "ce_vae_sp_configure", rank, world, region_ptrs, region_bytes);
}

int ce_vae_sp_host_barrier(ce_vae* h, int timeout_ms) { return sp_set_host_barrier(h ? &h->sp : nullptr, "ce_vae_sp_host_barrier", timeout_ms); }

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
  ConvArgs a = conv_args(*args);
  a.bias = reinterpret_cast<const bf16*>(args->bias);
  a.y = reinterpret_cast<bf16*>(args->y);
  a.resid = reinterpret_cast<const bf16*>(args->resid);
  return launch_conv3d_cl(a, reinterpret_cast<cudaStream_t>(stream));
}

int ce_conv3d_cl_ex_fp32(const ce_conv3d_args* args, void* y_pair, void* stream) {
  int rc = check_device();
  if (rc) return rc;
  CE_REQUIRE(args != nullptr, "ce_conv3d_cl_ex_fp32: null args");
  const ConvArgs a = conv_args(*args);
  ConvF32 f;
  f.bias = reinterpret_cast<const float*>(args->bias); f.resid = reinterpret_cast<const float*>(args->resid);
  f.y = reinterpret_cast<float*>(args->y); f.y_pair = reinterpret_cast<bf16*>(y_pair);
  return launch_conv3d_cl_f32(a, f, reinterpret_cast<cudaStream_t>(stream));
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
