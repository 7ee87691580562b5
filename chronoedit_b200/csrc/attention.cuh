// Interface of the wgmma attention forward (attention.cu).
#pragma once
#include "host_common.h"
#include "ptx.cuh"

namespace ce {

struct AttnArgs {
  int B = 0, H = 0, Lq = 0, Lk = 0, head_dim = 128;
  const bf16* q = nullptr;  // q[b, i, h*hd + d] at q + (b*Lq + i)*ldq + h*hd + d
  int ldq = 0;
  const bf16* k = nullptr;  // k[b, j, h*hd + d] at k + (b*Lk + j)*ldk + ...
  int ldk = 0;
  const bf16* v = nullptr;
  int ldv = 0;
  // optional SECOND key/value source (Lk2 > 0): out = bf16(attn(q,k,v)) + bf16(attn(q,k2,v2)), two independent softmaxes
  // in ONE launch (text + image cross-attention, transformer_chronoedit.py:84-104)
  const bf16* k2 = nullptr;
  int ldk2 = 0;
  const bf16* v2 = nullptr;
  int ldv2 = 0;
  int Lk2 = 0;
  bf16* out = nullptr;      // out[b, i, h*hd + d]
  int ldo = 0;
  float scale = 0.f;        // 1/sqrt(head_dim)
  long long* timing = nullptr;  // optional [16] device counters: phase cycles of thread 128 of block (0,0,0) (profiling aid)
  // sequence-parallel output scatter (csrc/dit.cu): when peer_rows > 0, query row i of sample b is stored at
  //   out_peer[i / peer_rows] + ((b * peer_rows + i % peer_rows) * ldo + h * head_dim + out_col0)
  // i.e. straight into the attention-output buffer of the rank that owns that token (its own pointer or a peer's, NVLink).
  bf16* out_peer[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  int peer_rows = 0;
  int out_col0 = 0;
  int accumulate = 0;       // 1: out = bf16(float(bf16(attn)) + float(out))   (image + text cross-attention sum)
};

// pipelined = false selects the serial schedule of the same kernel body (bit-identical output; a test and measurement aid).
int launch_attention(const AttnArgs& a, cudaStream_t stream, bool pipelined = true);

// The FP8 self-attention (attention.cu, DESIGN.md "FP8 attention"): Lq = Lk = L, head_dim 128, quantized operands.
struct AttnFp8Args {
  int B = 0, H = 0, L = 0;
  const uint8_t* q = nullptr;   // e4m3 q[b, i, h*128 + d] at q + (b*L + i)*ldqk + h*128 + d
  const uint8_t* k = nullptr;   // e4m3 k, same layout
  int ldqk = 0;                 // bytes, multiple of 16
  const float* q_scale = nullptr;   // q_scale[(b*L + i)*lds + h], one per (token, head)
  const float* k_scale = nullptr;   // the same for k
  int lds = 0;
  const uint8_t* vt = nullptr;  // e4m3 V^T [B, H, 128, Lpad]: channel rows, keys permuted within each 32-key group
  int Lpad = 0;                 // >= L, multiple of 32; keys [L, Lpad) are zero
  const float* v_scale = nullptr;   // [B, H*128], one per (sample, channel)
  bf16* out = nullptr;          // out[b, i, h*128 + c] at out + (b*L + i)*ldo + h*128 + c
  int ldo = 0;
  float scale = 0.f;            // 1/sqrt(head_dim)
};

int launch_attention_fp8(const AttnFp8Args& a, cudaStream_t stream);

}  // namespace ce
