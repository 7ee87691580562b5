// Interface of the HBM-bound row kernels of the DiT path (elementwise.cu).
#pragma once
#include "host_common.h"
#include "ptx.cuh"

namespace ce {

// Where the row kernels below take each row's statistics from.  p == nullptr: they reduce over the row themselves.  Otherwise from the
// epilogue of the GEMM that produced x (GemmArgs::stats_out, per-(row, N tile) partials, row r's at p + r * ld): `tiles` partials of
// width tile_n cover [0, D) of each matrix, and the kernels become streaming passes without a reduction or a barrier.  The RMSNorm
// reads only sums of squares (stats_mode 2) and does not use tile_n; the LayerNorm merges (mean, M2) pairs (stats_mode 1).
struct RowPartials {
  const float2* p = nullptr;
  int ld = 0, tiles = 0, tile_n = 0;
};

// y[row, :] = bf16( LN_fp32(x[row, :]) * (1 + scale[b, :]) + shift[b, :] )     (b = row / rows_per_batch)
//   scale/shift: fp32 [batches, mod_stride] or null (then the optional affine weight/bias, fp32 [D], is applied)
// FP32LayerNorm + adaLN modulate of transformer_chronoedit.py:279, 289, 460 and the affine norm2 of :284.
//   scale_is_1p: the `scale` table already holds (1 + scale) (ce_dit stores its modulation tables that way)
int launch_layernorm(const bf16* x, int ldx, bf16* y, int ldy, int rows, int D, float eps, const float* scale, const float* shift,
                     int mod_stride, int rows_per_batch, const float* weight, const float* bias, int scale_is_1p, const RowPartials& ps,
                     cudaStream_t stream);

// Sequence-parallel scatter of the normalised q | k (csrc/dit.cu): rows are the LOCAL tokens of this rank (rows_per_batch each,
// global token = tok0 + local index), RoPE uses the global token, and instead of being written back in place the vector of head h
// goes to the rank that owns head h:  dst[mat][h / heads_per_rank] + ((b * L_total + token) * (heads_per_rank * head_dim)
// + (h % heads_per_rank) * head_dim + offset inside the head).
// Only with partials: sequence parallelism requires D % 256 == 0, where the GEMM writes them.
struct SpScatter {
  bf16* dst[2][8];
  int world = 0;            // 0 = no scatter (in place)
  int heads_per_rank = 0;
  int L_total = 0;          // tokens per sample over all ranks
  int rows_per_batch = 0;   // local tokens per sample
  int tok0 = 0;             // first global token of this rank
};
// In place on x[rows, D] (leading dim ldx): diffusers RMSNorm across all heads (fp32 variance over D,
// y = bf16(bf16(x * rstd) * w)), then optionally interleaved-pair RoPE with cos/sin tables [L, hd/2] fp32
// (token = row % L).  transformer_chronoedit.py:62-65 and :71-79.
// `nmat` (1 or 2) matrices lie side by side in a row (q | k of the fused QKV output): matrix m starts at column m * D, uses weight m
// and, from partials, partials [m * tiles, (m + 1) * tiles).
int launch_rmsnorm_rope(bf16* x, int ldx, int rows, int D, float eps, const bf16* weight0, const bf16* weight1, int nmat,
                        const float* rope_cos, const float* rope_sin, int L, int head_dim, const RowPartials& ps, cudaStream_t stream,
                        const SpScatter* sp = nullptr);

// FP8 mode: per row m of x[rows, K] (K % 16 == 0), scale[m] = max_k |x[m,k]| / 448 (1 if that is 0) and
// q[m, k] = e4m3 bits of cvt.rn.satfinite(x[m,k] / scale[m]) (IEEE fp32 divisions).  One launch, HBM-bound.
int launch_quantize_rows_fp8(const bf16* x, int ldx, int rows, int K, uint8_t* q, int ldq, float* scale, cudaStream_t stream);

// FP8 self-attention, q | k: the same rule per (row, head) over 128 values.  x[rows, nh * 128] (leading dim ldx) -> q[rows, nh * 128]
// (ldq bytes) and scale[rows, nh].  For the fused QKV buffer nh = 2H covers q and k.  One warp per (row, head), HBM-bound.
int launch_quantize_heads_fp8(const bf16* x, int ldx, int rows, int nh, uint8_t* q, int ldq, float* scale, cudaStream_t stream);
// FP8 self-attention, v: one scale per (sample, channel), scale[b, c] = max_i |v[b, i, c]| / 448 (1 if that is 0), and
// vt[b, c / 128, c % 128, :] = e4m3(v[b, :, c] / scale[b, c]) transposed to keys-contiguous rows of Lpad bytes, the keys of each
// 32-key group at the positions the P V wgmma's A fragment wants (fp8_attention_key_order in transformer.py), keys >= L zero.
// v[b, i, c] at v + (b * L + i) * ldv + c, c < H * 128.  Two launches: the channel maxima, then transpose + quantize.
int launch_quantize_v_fp8(const bf16* v, int ldv, int B, int L, int H, uint8_t* vt, int Lpad, float* scale, cudaStream_t stream);

// Row softmax of the fp32 GEMM accumulators S [rows, lds] (rows = heads x Lq queries) into P [rows, ldp]: p = bf16(softmax_fp32(
// score)) over the keys j < cols, and 0 for the other columns up to ldp.  The score of key j in query row i of head h:
//   SOFTMAX_SCALED (VAE):  s * scale, exponentials with __expf
//   SOFTMAX_T5:    bf16(bf16(s) + bias[h, (j - i) + Lq - 1]); keys j >= valid are masked out (probability 0, as adding
//                  finfo(bf16).min does in the reference)
//   SOFTMAX_CLIP:  bf16(bf16(s) * scale)
enum SoftmaxRule { SOFTMAX_SCALED, SOFTMAX_T5, SOFTMAX_CLIP };
struct SoftmaxScores {
  SoftmaxRule rule = SOFTMAX_SCALED;
  float scale = 1.f;
  const bf16* bias = nullptr;   // T5: [heads, bias_ld]
  int bias_ld = 0, Lq = 0, valid = 0;
};
int launch_softmax_rows(const float* S, int lds, bf16* P, int ldp, int rows, int cols, const SoftmaxScores& sc, cudaStream_t stream);
// The fp32 validation forward's: P fp32 = softmax(s * scale) with expf.
int launch_softmax_rows_f32(const float* S, int lds, float* P, int ldp, int rows, int cols, float scale, cudaStream_t stream);

// patches[(b, tok - tok0), c*4 + dh*2 + dw] = x[b, c, f, 2i+dh, 2j+dw] for the tokens tok = (f, i, j) in [tok0, tok0 + ntok) of every
// sample   (im2row for the k=s=(1,2,2) patch-embedding conv, :368,429-430; a token range for sequence parallelism)
int launch_patchify(const bf16* x, bf16* patches, int B, int C, int T, int H, int W, int tok0, int ntok, cudaStream_t stream);
// out[b, c, f, 2i+dh, 2j+dw] = y[(b,f,i,j), (dh*2+dw)*C + c]       (unpatchify permute of :463-467)
int launch_unpatchify(const bf16* y, int ldy, bf16* out, int B, int C, int T, int H, int W, cudaStream_t stream);

// out[b, n] = act( sum_k x[b,k] * W[n,k] + bias[n] );  tiny-M Linear (time embedder / time_proj, :155-159).
//   w_is_bf16: weights/bias bf16 (else fp32); x is fp32; out fp32 (out_f32) and/or bf16 (out_bf16).
//   in_silu_bf16: the input is first mapped through bf16(SiLU(x)) (act_fn applied to the bf16 temb tensor).
//   act: 0 none, 1 SiLU on the output.  When out_bf16 is given the Linear result is rounded to bf16 first (and
//   out_f32, if also given, receives that rounded value).
int launch_small_linear(const float* x, int K, const void* W, const void* bias, int w_is_bf16, int N, int B,
                        int act, int in_silu_bf16, float* out_f32, bf16* out_bf16, cudaStream_t stream);

// emb[b, :] = [cos(t_b * f_i) | sin(t_b * f_i)], f_i = exp(-ln(10000) * i / half)   (diffusers Timesteps, flip_sin_to_cos)
int launch_timestep_sinusoid(const float* t, float* emb, int B, int dim, cudaStream_t stream);

// dst[b, :] = table[b % table_rows, :] + src[b, :] (fp32): scale_shift_table + temb (:274-276, :451)
//   plus_one_mask: bit c set -> chunk c is stored as 1 + value (the adaLN "scale" chunks)
int launch_add_table(const float* table, int table_rows, const bf16* src, int src_ld, float* dst, int B, int n,
                     int chunks, cudaStream_t stream, unsigned plus_one_mask = 0);

}  // namespace ce
