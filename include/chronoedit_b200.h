/*
 * chronoedit_b200 — C ABI of the H100-native ChronoEdit denoising hot path.
 *
 * The reference (nv-tlabs/ChronoEdit) has no FFI for this path: the boundary is two Python objects registered
 * into a diffusers pipeline (pipeline_chronoedit.py:175-183).  This header is the C-ABI underneath the Python
 * mirror classes in chronoedit_b200/ (INTEGRATION.md shows the ctypes binding); each entry point names the
 * reference interface it stands in for.
 *
 * Conventions
 *   - every pointer argument is a DEVICE pointer owned by the caller unless the name ends in _host;
 *   - activations / weights are bf16 unless stated; tensors are dense row-major in the layouts given;
 *   - `stream` is a cudaStream_t passed as void*; calls are asynchronous on it and never synchronise the device
 *     (the *_host variants synchronise `stream` before returning because they hand results back in host memory);
 *   - return value 0 = success, negative = failure (ce_last_error() holds the message of the calling thread's last
 *     failure); there is NO CPU fallback: on a machine without an sm_90 GPU every compute entry point fails;
 *   - one handle may be used from one thread at a time; distinct handles are independent.
 */
#ifndef CHRONOEDIT_B200_H_
#define CHRONOEDIT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CE_ABI_VERSION 1

int ce_abi_version(void);
const char* ce_last_error(void);
/* 0 iff the current CUDA device is sm_90 (H100). */
int ce_device_check(void);

/* ------------------------------------------------------------------------------------------------------------
 * DiT: ChronoEditTransformer3DModel  (chronoedit_diffusers/transformer_chronoedit.py:298-476)
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct ce_dit ce_dit;

typedef struct ce_dit_config {   /* = the @register_to_config arguments, transformer_chronoedit.py:342-360 */
  int32_t num_attention_heads;   /* 40 */
  int32_t attention_head_dim;    /* 128 (only value built) */
  int32_t in_channels;           /* 36 */
  int32_t out_channels;          /* 16 */
  int32_t text_dim;              /* 4096 */
  int32_t freq_dim;              /* 256 */
  int32_t ffn_dim;               /* 13824 */
  int32_t num_layers;            /* 40 */
  int32_t image_dim;             /* 1280; 0 = no image embedder / no added k,v projections */
  int32_t added_kv_proj_dim;     /* 5120 */
  int32_t rope_max_seq_len;      /* 1024 */
  int32_t rope_temporal_skip_len;/* 8 */
  float eps;                     /* 1e-6 */
  int32_t patch_t, patch_h, patch_w; /* (1,2,2) (only value built) */
} ce_dit_config;

/* ChronoEditTransformer3DModel.__init__ (:342-395).  No weights are allocated: the caller owns them. */
int ce_dit_create(const ce_dit_config* cfg, ce_dit** out);
void ce_dit_destroy(ce_dit* h);

/* Register one parameter by name (device pointer, kept alive by the caller until ce_dit_destroy).
 * Names are the reference state_dict's (e.g. "blocks.3.ffn.net.2.weight") except for the fused / stacked buffers the
 * Python mirror builds as views over the reference parameters:
 *   blocks.N.attn1.to_qkv.{weight,bias}      [3D,D] / [3D]   rows = to_q | to_k | to_v
 *   blocks.N.attn2.to_kv.{weight,bias}       [2D,D] / [2D]   rows = to_k | to_v
 *   blocks.N.attn2.add_kv_proj.{weight,bias} [2D,Da]/ [2D]   rows = add_k_proj | add_v_proj
 *   blocks.scale_shift_table                 [num_layers,6,D] fp32 (stack of blocks.N.scale_shift_table)
 *   patch_embedding.weight                   [D, Cin*pt*ph*pw] (the Conv3d weight, flattened)
 * dtype: 0 = bf16, 1 = fp32.  fp32 is required for (and only for) the reference's `_keep_in_fp32_modules`
 * (time_embedder, scale_shift_table, norm1/norm2/norm3 affine parameters, :338).
 * FP8 mode: dtype 2 = e4m3 (torch.float8_e4m3fn) for the six per-token block weights attn1.to_qkv, attn1.to_out.0,
 * attn2.to_q, attn2.to_out.0, ffn.net.0.proj and ffn.net.2, each with its fp32 per-output-channel scale registered as
 * "<name>.weight_scale" [N] (dtype 1): W ~ weight * weight_scale[n].  Either all six of every layer are e4m3 or none is;
 * ce_dit_weights_complete rejects a mixture.  Such a handle quantizes each of those GEMMs' activations per row on the
 * device (DESIGN.md, "FP8 mode"); sequence parallelism is not built for it. */
int ce_dit_set_weight(ce_dit* h, const char* name, const void* ptr, int dtype, int64_t numel);
/* 0 when every parameter the configuration needs has been registered; otherwise fails and names the first missing. */
int ce_dit_weights_complete(const ce_dit* h);

/* FP8 self-attention (DESIGN.md, "FP8 attention"), off by default: with enabled != 0 every block's self-attention quantizes q
 * and k per (token, head) and v per (sample, channel) to e4m3 on the device and runs on e4m3 wgmma.  Cross-attention, the
 * context cache and the weights are untouched; it works with bf16 and with FP8 weights.  ce_dit_workspace_bytes follows the
 * flag, so query it after setting it.  Sequence parallelism is refused while it is on. */
int ce_dit_set_attention_fp8(ce_dit* h, int enabled);

/* Run-time LoRA (DESIGN.md, "Run-time LoRA"): low-rank terms beside the block GEMMs, without touching the weights.  The tables
 * hold num_layers * CE_LORA_TARGETS entries, entry layer * CE_LORA_TARGETS + target, targets in this order:
 *   0 attn1.to_qkv   1 attn1.to_out.0   2 attn2.to_q   3 attn2.to_kv   4 attn2.add_kv_proj   5 attn2.to_out.0
 *   6 ffn.net.0.proj   7 ffn.net.2
 * Entry i: a_cat[i] [rank[i], K] bf16 (the stacked lora_A of every adapter on that GEMM) and b_cat[i] [N, rank[i]] bf16 (the
 * stacked lora_B, each adapter's columns pre-scaled by its scaling); the fused targets (0, 3, 4) stack their parts along N
 * (q | k | v, k | v), a part without an adapter holding zeros.  rank[i] % 8 == 0 (pad with zero rows / columns); 0 = no LoRA on
 * that GEMM.  The GEMM then computes base + bf16(bf16(x a_cat^T) b_cat^T), the term added in the epilogue before GELU, gate,
 * residual and the row statistics; an e4m3 weight keeps its FP8 rule for the base, the term reads the bf16 activations.
 * Pointers are the caller's (16-byte aligned device memory, kept alive while set).  n == 0 clears every entry.  Anything
 * invalid is refused before the handle changes.  ce_dit_workspace_bytes grows while a table is set (see there).  Refused at
 * forward time with sequence parallelism and by ce_dit_forward_fp32. */
#define CE_LORA_TARGETS 8
int ce_dit_set_lora(ce_dit* h, const void* const* a_cat, const void* const* b_cat, const int32_t* rank, int n);

/* Scratch bytes one forward needs for `batch` samples of latent geometry (frames, height, width) and text_len tokens.
 * A handle holding FP8 weights needs M * max(D, ffn_dim) bytes + M floats more (M = batch * tokens): the quantized rows.
 * With FP8 attention on: M * 2D bytes + M * 2H floats (q | k and their scales) + batch * D * Lpad bytes + batch * D floats
 * (V^T and its scales; Lpad = tokens rounded up to 32).
 * While a LoRA table is set (ce_dit_set_lora): Mx * R_max + Mx * max(3D, ffn_dim) bf16 more, the down-projection and the
 * low-rank term of one GEMM at a time (Mx = max(M, batch * text_len, batch * 257), R_max the largest rank of the table). */
int64_t ce_dit_workspace_bytes(const ce_dit* h, int batch, int frames, int height, int width, int text_len);

/* ChronoEditTransformer3DModel.forward (:397-476).
 *   hidden_states [B, in_channels, frames, height, width]   timestep [B] fp32 (the pipeline's int64 t cast to float, :155-157)
 *   encoder_hidden_states [B, text_len, text_dim]           encoder_hidden_states_image [B, 257, image_dim] or NULL
 *   sample (out) [B, out_channels, frames, height, width]
 * frames must be 2 or rope_temporal_skip_len (the reference asserts this, :205).
 * intermediates: optional; when non-NULL receives block 0's output [B*L, D] bf16 (parity tests). */
int ce_dit_forward(ce_dit* h, const void* hidden_states, const float* timestep, const void* encoder_hidden_states,
                   const void* encoder_hidden_states_image, void* sample, int batch, int frames, int height, int width,
                   int text_len, void* workspace, int64_t workspace_bytes, void* block0_out, void* stream);

/* The same forward with the STEP-INVARIANT context kept across calls: the text / image embedders (:147-165) and every block's
 * cross-attention K/V projections + RMSNorm (:52-60, :84-95) depend only on encoder_hidden_states[_image] and the weights, not
 * on the latents or the timestep, so within one edit they are the same at every denoising step.
 *   ctx_cache: device buffer of >= ce_dit_context_cache_bytes(h, batch, text_len) bytes owned by the caller, or NULL (= ce_dit_forward);
 *   ctx_reuse = 0: compute the context and leave it in ctx_cache;  ctx_reuse = 1: the cache already holds the context of THESE
 *   encoder states and weights (the caller's promise) -- the embedders and the 2 x num_layers K/V GEMMs are skipped.
 * The result is bit-identical either way (same kernels, same inputs).  Algorithmic FLOP counts in bench.py stay un-hoisted. */
int64_t ce_dit_context_cache_bytes(const ce_dit* h, int batch, int text_len);
int ce_dit_forward_ex(ce_dit* h, const void* hidden_states, const float* timestep, const void* encoder_hidden_states,
                      const void* encoder_hidden_states_image, void* sample, int batch, int frames, int height, int width,
                      int text_len, void* workspace, int64_t workspace_bytes, void* block0_out, void* ctx_cache,
                      int64_t ctx_cache_bytes, int ctx_reuse, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Sequence parallelism over the GPUs of one node for single-edit latency (SURVEY.md section 8(f) row 2; reference: the Ulysses /
 * xfuser path chronoedit_diffsynth/wan_video_new_chronoedit.py:330-355, 1448-1498 and the TE ring of
 * chronoedit/_src/networks/wan2pt1.py:352-353, 917-941).  One process per GPU, all weights on every rank, the tokens of the edit
 * split into `world` contiguous ranges.  The heads <-> tokens exchange around the self-attention is done by the producing kernels
 * themselves with stores into the consumer's memory over NVLink (csrc/seqpar.cuh); phases are ordered by a flag barrier in peer
 * memory.  Every rank passes the SAME full inputs and receives the same full sample, bit-identical to the single-GPU forward.
 *   region: one device buffer of ce_dit_sp_region_bytes(...) per rank, allocated with ce_ipc_alloc (zeroed), shared with the peers
 *   through ce_ipc_get_handle / ce_ipc_open (CUDA IPC; the 64-byte handles travel by any host channel, e.g. torch.distributed);
 *   region_ptrs[w] = address of rank w's region in THIS process (non-null, 256-byte aligned).  world = 1 switches it off; any
 *   other world outside 2..8 is refused, and so is a head count that world does not divide.
 * ------------------------------------------------------------------------------------------------------------ */
int64_t ce_dit_sp_region_bytes(const ce_dit* h, int batch, int frames, int height, int width, int world);
int ce_dit_sp_configure(ce_dit* h, int rank, int world, void* const* region_ptrs, int64_t region_bytes);

/* ------------------------------------------------------------------------------------------------------------
 * Batch split ("CFG parallelism") over the GPUs of one node: rank r of `world` computes samples [r B / world, (r + 1) B / world) of
 * each call's batch B through the unchanged forward, and every rank returns the full batch.  The samples never interact inside the
 * forward, so the only exchange is at its end: each rank stores its samples into every peer's region, one barrier, and copies the
 * other ranks' samples from its own region into the caller's buffer.  Every rank passes the SAME full inputs.  It composes with FP8
 * weights, FP8 attention and TeaCache (ce_dit_forward_cached ends in the same exchange), and with the token split (ce_dit_sp_*,
 * configured for the local batch B / world) as a grid: the token split runs on the rank's samples, the batch exchange follows.
 *   region: the flags block (1 KB, first), then two sample slots of [batch, out_channels, frames, height, width] bf16 (each rounded
 *   up to 1 KB) that alternate from call to call, so each call needs one barrier.  Any later call whose full sample fits a slot is
 *   accepted.  ce_dit_bp_region_bytes returns -1 for a world outside 2..8 or a batch it does not divide.
 *   ce_dit_bp_configure: as ce_dit_sp_configure (same refusals); world = 1 switches the split off.  Refused while the call-pair
 *   split below is configured.
 *   ce_dit_bp_host_barrier: the test aid of ce_dit_sp_host_barrier, for this group's barrier.
 * A split call refuses, before any launch: a batch the ranks do not divide (so the unchanged diffusers pipeline's batch-1 calls are
 * not split), a sample larger than a slot, block capture or block0_out, and a capturing stream.  ce_dit_forward_fp32 is refused.
 * ------------------------------------------------------------------------------------------------------------ */
int64_t ce_dit_bp_region_bytes(const ce_dit* h, int batch, int frames, int height, int width, int world);
int ce_dit_bp_configure(ce_dit* h, int rank, int world, void* const* region_ptrs, int64_t region_bytes);
int ce_dit_bp_host_barrier(ce_dit* h, int timeout_ms);

/* ------------------------------------------------------------------------------------------------------------
 * Call-pair split over two GPUs: the unchanged diffusers pipeline computes a CFG step as two batch-1 calls with the same latents and
 * timestep, one with the prompt and one with the negative prompt.  Rank 0 computes the first call, rank 1 the second, each with the
 * ordinary ce_dit_forward_ex (the token split underneath when configured); ce_dit_forward_ex itself does not look at this group.
 * After both, ce_dit_cp_exchange gives each rank the other's sample.
 *   region: the batch split's layout for one whole call: the flags block (1 KB, first), then two slots of [batch, out_channels,
 *   frames, height, width] bf16 (each rounded up to 1 KB) that alternate from pair to pair, so each pair needs one barrier.  A region
 *   sized for 8 latent frames serves temporal reasoning's cut to 2.  ce_dit_cp_region_bytes returns -1 for an invalid geometry.
 *   ce_dit_cp_configure: as ce_dit_bp_configure (same refusals), and a world other than 1 or 2 is refused; world = 1 switches it
 *   off.  Refused while the batch split is configured: the two CFG splits are exclusive.  The token split composes with either.
 *   ce_dit_cp_exchange: `own_sample` into the peer's slot of the current set; one barrier; the peer's sample from this rank's own slot
 *   into `other_sample`.  Three launches on `stream`, stream-ordered with the forward before and whatever reads the samples after.
 *   Refused before any launch: the group not configured, a sample larger than a slot, and a capturing stream.
 *   ce_dit_cp_host_barrier: the test aid of ce_dit_sp_host_barrier, for this group's barrier.
 * ------------------------------------------------------------------------------------------------------------ */
int64_t ce_dit_cp_region_bytes(const ce_dit* h, int batch, int frames, int height, int width);
int ce_dit_cp_configure(ce_dit* h, int rank, int world, void* const* region_ptrs, int64_t region_bytes);
int ce_dit_cp_exchange(ce_dit* h, const void* own_sample, void* other_sample, int batch, int frames, int height, int width, void* stream);
int ce_dit_cp_host_barrier(ce_dit* h, int timeout_ms);

int ce_ipc_alloc(int64_t bytes, void** ptr);
int ce_ipc_free(void* ptr);
int ce_ipc_get_handle(void* ptr, void* handle_out_64_bytes);
int ce_ipc_open(const void* handle_64_bytes, void** ptr);
int ce_ipc_close(void* ptr);

/* Parity aid: from now on every forward copies the output of block layers[i] ([B*L, D] bf16) to dst[i] (n = 0 clears). */
int ce_dit_set_capture(ce_dit* h, const int32_t* layers, void* const* dst, int n);

/* ------------------------------------------------------------------------------------------------------------
 * TeaCache (DESIGN.md, "TeaCache"; reference: chronoedit_diffsynth/wan_video_new_chronoedit.py:1190-1239, 1434-1492): skip every
 * block on a step whose timestep modulation moved little since the last computed step and add the residual the blocks produced
 * then.  The policy lives with the caller; these calls give it the three device pieces.  All three refuse sequence parallelism.
 *
 * ce_dit_teacache_probe: the time path alone (sinusoid, time embedder, time_proj) for `timestep` [B] fp32 into tproj_out [B, 6D] bf16,
 *   bit-identical to the forward's timestep_proj.  With prev_tproj (the [B, 6D] of an earlier call) non-NULL it also writes
 *   sums_out[0] = sum |bf16(tproj - prev)| and sums_out[1] = sum |prev| (fp32, a summation order fixed by B * 6D).  workspace:
 *   ce_dit_teacache_probe_bytes(h, batch) bytes.  Every buffer is a device buffer, 256-byte aligned.
 * ce_dit_set_residual_record: from now on every forward leaves residual = bf16(x_after_blocks - x_before_blocks) [B*L, D] bf16 in
 *   buf (x_before_blocks: the token stream right after the patch embedding).  The sample is unchanged.  A forward whose residual
 *   does not fit in `bytes` is refused.  buf = NULL switches it off.
 * ce_dit_forward_cached: the forward with the blocks replaced by x = bf16(x_before_blocks + residual), then the output head and
 *   unpatchify.  The geometry arguments and the workspace are those of ce_dit_forward_ex; the text and image embedders, the
 *   context cache and the blocks are not touched.
 * ------------------------------------------------------------------------------------------------------------ */
int64_t ce_dit_teacache_probe_bytes(const ce_dit* h, int batch);
int ce_dit_teacache_probe(ce_dit* h, const float* timestep, int batch, const void* prev_tproj, void* tproj_out, float* sums_out,
                          void* workspace, int64_t workspace_bytes, void* stream);
int ce_dit_set_residual_record(ce_dit* h, void* buf, int64_t bytes);
int ce_dit_forward_cached(ce_dit* h, const void* hidden_states, const float* timestep, const void* residual, int64_t residual_bytes,
                          void* sample, int batch, int frames, int height, int width, int text_len, void* workspace,
                          int64_t workspace_bytes, void* stream);

/* Same call with every tensor in (pinned) HOST memory: H2D copies of the inputs, forward, D2H of the sample, all on
 * `stream`, which is synchronised before returning.  `staging` is a device buffer of at least
 * ce_dit_host_staging_bytes(...) bytes.  This is the end-to-end ("e2e") path bench.py times. */
int64_t ce_dit_host_staging_bytes(const ce_dit* h, int batch, int frames, int height, int width, int text_len);
int ce_dit_forward_host(ce_dit* h, const void* hidden_states_host, const float* timestep_host,
                        const void* encoder_hidden_states_host, const void* encoder_hidden_states_image_host,
                        void* sample_host, int batch, int frames, int height, int width, int text_len, void* staging,
                        int64_t staging_bytes, void* workspace, int64_t workspace_bytes, void* stream);

/* The host-buffer call with the step-invariant context cache of ce_dit_forward_ex (device buffer, caller-owned).  The sample also
 * stays in `staging` at byte offset ce_dit_host_staging_sample_offset(...) (bf16 [B, out_channels, frames, height, width]) until
 * the next call, so that the scheduler step can consume it on the device without a second copy. */
int ce_dit_forward_host_ex(ce_dit* h, const void* hidden_states_host, const float* timestep_host,
                           const void* encoder_hidden_states_host, const void* encoder_hidden_states_image_host,
                           void* sample_host, int batch, int frames, int height, int width, int text_len, void* staging,
                           int64_t staging_bytes, void* workspace, int64_t workspace_bytes, void* ctx_cache,
                           int64_t ctx_cache_bytes, int ctx_reuse, void* stream);
int64_t ce_dit_host_staging_sample_offset(const ce_dit* h, int batch, int frames, int height, int width, int text_len);

/* VALIDATION mode: the same forward in fp32 -- fp32 inputs, fp32 parameters (registered under their REFERENCE names, unfused:
 * blocks.N.attn1.to_q.weight ..., blocks.N.scale_shift_table [6*D], scale_shift_table [2*D], patch_embedding.weight [D, Cin*4]),
 * fp32 residual stream, fp32 outputs.  Matrix products run on the same wgmma GEMM with every fp32 operand split into two bf16
 * terms (A_hi.W_hi + A_lo.W_hi + A_hi.W_lo, fp32 accumulate; csrc/dit_fp32.cu).  It exists so that north_star's
 * rtol 1e-3 / atol 1e-4 can be asserted end to end against the reference's fp32 run (tests/test_gpu_fp32_mode.py); it is about
 * 5-10x slower than the bf16 path and is not what bench.py measures.  block_out: optional, block 0's output [B*L, D] fp32. */
int ce_dit_set_weight_fp32(ce_dit* h, const char* name, const float* ptr, int64_t numel);
int64_t ce_dit_fp32_workspace_bytes(const ce_dit* h, int batch, int frames, int height, int width, int text_len);
int ce_dit_forward_fp32(ce_dit* h, const float* hidden_states, const float* timestep, const float* encoder_hidden_states,
                        const float* encoder_hidden_states_image, float* sample, int batch, int frames, int height, int width,
                        int text_len, void* workspace, int64_t workspace_bytes, float* block_out, void* stream);

/* Kernel launches issued by the last ce_dit_forward on this handle (bench.py's "gpu_launches"). */
int64_t ce_dit_last_launch_count(const ce_dit* h);

/* Device-side timing of the kernels of subsequent forwards: a CUDA event pair on the launch stream around every
 * launch (up to max_launches; later launches are not recorded).  ce_dit_profile_end waits for the last recorded event
 * and returns, per category c in {0: wgmma GEMM, 1: wgmma attention, 2: LayerNorm / RMSNorm row kernels,
 * 3: everything else}: total milliseconds, total algorithmic work (FLOPs for 0/1, bytes for 2) and launch count
 * (each array has 4 entries).  This is what bench.py's "roofline" object is computed from. */
int ce_dit_profile_begin(ce_dit* h, int max_launches);
int ce_dit_profile_end(ce_dit* h, double* ms_out, double* work_out, int64_t* count_out);

/* ------------------------------------------------------------------------------------------------------------
 * VAE: AutoencoderKLWan encode / decode as the pipeline uses them (pipeline_chronoedit.py:436-443, 776-781);
 * arithmetic = WanVAE_ of chronoedit/_src/tokenizers/wan2pt1.py:467-581 WITHOUT the latent mean/std (the pipeline applies
 * those itself, :427-445, :765-774).
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct ce_vae ce_vae;

typedef struct ce_vae_config {      /* _video_vae cfg, wan2pt1.py:597-605 */
  int32_t dim;                      /* 96 */
  int32_t z_dim;                    /* 16 */
  int32_t dim_mult[4];              /* 1,2,4,4 */
  int32_t num_res_blocks;           /* 2 */
  int32_t temporal_downsample[3];   /* 0,1,1 */
} ce_vae_config;

int ce_vae_create(const ce_vae_config* cfg, ce_vae** out);
void ce_vae_destroy(ce_vae* h);
/* Parameters by the in-tree twin's names (e.g. "decoder.upsamples.3.time_conv.weight"), all bf16, PRE-PACKED by the caller:
 *   convolution weights [Cout, Cin, kt, kh, kw] -> [Cout, taps, Cin_pad] with taps ordered (dt, dh, dw), Cin_pad = Cin rounded
 *     up to 64 (zero filled); the four small convolutions (encoder.conv1, decoder.conv1, conv1, conv2) -> [Cout, Kpad] with
 *     K = taps*Cin rounded up to 8;
 *   "*.gamma" [C]; attention "to_qkv.weight" [3C, C], "proj.weight" [C, C]; biases [Cout].
 * numel is checked against these sizes before anything is launched (ce_vae_workspace_bytes fails on a missing or mis-sized weight). */
int ce_vae_set_weight(ce_vae* h, const char* name, const void* ptr, int64_t numel);
/* decode != 0: (frames, height, width) is the LATENT geometry; else the PIXEL geometry. */
int64_t ce_vae_workspace_bytes(ce_vae* h, int decode, int frames, int height, int width);
/* video [3, frames, height, width] (planar, one sample, values in [-1,1], frames = 1+4k) -> posterior moments
 * [2*z_dim, 1+k, height/8, width/8]: channels [0,z) = mean (= AutoencoderKLWan.encode(x).latent_dist.mode()), [z,2z) = logvar */
int ce_vae_encode(ce_vae* h, const void* video, void* moments, int frames, int height, int width, void* workspace,
                  int64_t workspace_bytes, void* stream);
/* z [z_dim, Tl, h, w] -> video [3, 1+4(Tl-1), 8h, 8w]; clamp != 0 clamps to [-1,1] (= AutoencoderKLWan.decode(z)[0]) */
int ce_vae_decode(ce_vae* h, const void* z, void* video, int latent_frames, int latent_height, int latent_width, int clamp,
                  void* workspace, int64_t workspace_bytes, void* stream);
int64_t ce_vae_last_launch_count(const ce_vae* h);

/* The VAE in fp32, as the reference pipeline loads it (AutoencoderKLWan.from_pretrained(..., torch_dtype=torch.float32)): the calls
 * above with fp32 in and fp32 out, on parameters registered with ce_vae_set_weight_fp32 (a map of their own) under the same names:
 *   convolution weights [Cout, Cin, kt, kh, kw] fp32 -> [Cout, taps, Cin_pad / 64, 3, 64] bf16 with taps ordered (dt, dh, dw), Cin_pad
 *     = Cin rounded up to 64 (zero filled) and, per 64-channel block, hi = bf16(w), hi again, lo = bf16(w - hi) -- every convolution,
 *     the small ones included;
 *   "*.gamma" [C], biases [Cout], attention "to_qkv.weight" [3C, C] and "proj.weight" [C, C]: fp32 as they are.
 * Convolutions run on the wgmma implicit GEMM with both operands split into two bf16 terms (A_hi.W_hi + A_lo.W_hi + A_hi.W_lo, fp32
 * accumulation), the mid attention on 6-term split GEMMs with an fp32 softmax, everything else in fp32 (csrc/vae.cu).
 * Refused before any launch: a handle split over GPUs (ce_vae_sp_configure with world > 1), a handle without fp32 weights, a missing or
 * mis-sized weight, and a workspace smaller than ce_vae_workspace_bytes_fp32 or not 256-byte aligned.  ce_vae_workspace_bytes_fp32
 * returns -1 on any of the refusals it can see (geometry, split, weights). */
int ce_vae_set_weight_fp32(ce_vae* h, const char* name, const void* ptr, int64_t numel);
int64_t ce_vae_workspace_bytes_fp32(ce_vae* h, int decode, int frames, int height, int width);
int ce_vae_encode_fp32(ce_vae* h, const float* video, float* moments, int frames, int height, int width, void* workspace,
                       int64_t workspace_bytes, void* stream);
int ce_vae_decode_fp32(ce_vae* h, const float* z, float* video, int latent_frames, int latent_height, int latent_width, int clamp,
                       void* workspace, int64_t workspace_bytes, void* stream);

/* Tiled encode / decode (diffusers AutoencoderKLWan.tiled_encode / tiled_decode, what enable_tiling() switches on): the same inputs
 * and outputs as the calls above, computed tile by tile.  Tile sizes and strides are in pixels, multiples of 8, stride <= size.
 * Tiles start every stride (latent stride = stride / 8) and cover `size` (smaller at the right and bottom edges); each is a fresh
 * untiled encode or decode (its own causal cache, never clamped).  In grid order each result is blended in place with the blended
 * tile above (diffusers' blend_v over min(size - stride, both heights) rows) and then with the blended tile to its left (blend_h),
 * and its first stride x stride is written to the output (blend extents and crops in latent units when encoding, in pixels when
 * decoding).  clamp != 0 clamps the decoded pixels to [-1, 1] as they are written.
 * The workspace (ce_vae_workspace_bytes_tiled[_fp32], -1 on refusal) is one tile's untiled workspace plus the staged input and output
 * tile plus the last size - stride rows of every tile of two grid rows and the last size - stride columns of two tiles: it does not
 * grow with the height, and grows with the width by those rows only.  Refused before any launch: a handle split over GPUs
 * (ce_vae_sp_configure with world > 1), sizes or strides that are not positive multiples of 8, a stride larger than the size, and
 * everything the untiled call refuses. */
int64_t ce_vae_workspace_bytes_tiled(ce_vae* h, int decode, int frames, int height, int width, int tile_min_height, int tile_min_width,
                                     int tile_stride_height, int tile_stride_width);
int ce_vae_encode_tiled(ce_vae* h, const void* video, void* moments, int frames, int height, int width, int tile_min_height, int tile_min_width,
                        int tile_stride_height, int tile_stride_width, void* workspace, int64_t workspace_bytes, void* stream);
int ce_vae_decode_tiled(ce_vae* h, const void* z, void* video, int latent_frames, int latent_height, int latent_width, int tile_min_height,
                        int tile_min_width, int tile_stride_height, int tile_stride_width, int clamp, void* workspace, int64_t workspace_bytes,
                        void* stream);
int64_t ce_vae_workspace_bytes_tiled_fp32(ce_vae* h, int decode, int frames, int height, int width, int tile_min_height, int tile_min_width,
                                          int tile_stride_height, int tile_stride_width);
int ce_vae_encode_tiled_fp32(ce_vae* h, const float* video, float* moments, int frames, int height, int width, int tile_min_height,
                             int tile_min_width, int tile_stride_height, int tile_stride_width, void* workspace, int64_t workspace_bytes,
                             void* stream);
int ce_vae_decode_tiled_fp32(ce_vae* h, const float* z, float* video, int latent_frames, int latent_height, int latent_width, int tile_min_height,
                             int tile_min_width, int tile_stride_height, int tile_stride_width, int clamp, void* workspace,
                             int64_t workspace_bytes, void* stream);
/* Test aid: the blend launch of one tile.  Planar [C, T, rows, cols] tensors of one dtype (fp32 != 0: fp32, else bf16).  The tile
 * [C, T, th, tw] is blended with the last above_h rows of the blended tile above (above [C, T, above_h, tw]; extent min(above_h, th)),
 * then with the last left_w columns of the blended tile to its left (left [C, T, th, left_w]; extent min(left_w, tw)); null = none.
 * Its rows < crop_h and columns < crop_w go to out [C, T, out_h, out_w] at (oy, ox), clipped to out; the last strip_h rows to strip
 * [C, T, strip_h, tw] and the last tail_w columns to tail [C, T, th, tail_w] (null: not written). */
typedef struct ce_vae_tile_blend_args {
  int32_t fp32;
  const void* tile;
  int32_t C, T, th, tw;
  const void* above;
  int32_t above_h;
  const void* left;
  int32_t left_w;
  void* out;
  int32_t out_h, out_w, oy, ox, crop_h, crop_w, clamp;
  void* strip;
  int32_t strip_h;
  void* tail;
  int32_t tail_w;
} ce_vae_tile_blend_args;
int ce_vae_tile_blend(const ce_vae_tile_blend_args* args, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * The VAE split over the `world` ranks of a node (one process per GPU), for the latency of one edit: rank r encodes and
 * decodes latent rows [r h / world, (r + 1) h / world) (and the matching rows at every resolution), exchanges only the rows
 * that cross the band edges and the mid attention's input by peer stores into the other ranks' regions, and every rank
 * returns the full result, bit-identical to the single-GPU call.  Call ce_vae_encode / ce_vae_decode with the same full
 * inputs on every rank; ce_vae_workspace_bytes reports the band's need while the split is configured.
 *   ce_vae_sp_region_bytes: bytes of the peer region every rank needs for pixel geometry height x width (multiples of 8, at
 *     least `world` latent rows, world 2 to 8).  One region serves an encode of any 1 + 4k frames at height x width and a
 *     decode of any latent frame count at height / 8 x width / 8, and any smaller geometry whose need fits; -1 on refusal.
 *   ce_vae_sp_configure: region_ptrs[w] = rank w's region as seen from this process (ce_ipc_alloc / ce_ipc_open, 256-byte
 *     aligned).  world = 1 switches the split off; any other world outside 2..8 is refused.
 *   ce_vae_sp_host_barrier: as ce_dit_sp_host_barrier, for the VAE's barriers (a test aid: `world` handles of one process on
 *     one GPU play the ranks).
 * A call refuses, before any launch, fewer latent rows than ranks, a geometry whose need exceeds region_bytes and a capturing
 * stream.
 * ------------------------------------------------------------------------------------------------------------ */
int64_t ce_vae_sp_region_bytes(ce_vae* h, int height, int width, int world);
int ce_vae_sp_configure(ce_vae* h, int rank, int world, void* const* region_ptrs, int64_t region_bytes);
int ce_vae_sp_host_barrier(ce_vae* h, int timeout_ms);

/* ------------------------------------------------------------------------------------------------------------
 * Encoders in front of the loop (SURVEY.md section 8(f) row 3), once per edit:
 *   transformers.UMT5EncoderModel   -- pipeline_chronoedit.py:205-244  self.text_encoder(ids, mask).last_hidden_state
 *   transformers.CLIPVisionModel    -- pipeline_chronoedit.py:246-254  self.image_encoder(**image, output_hidden_states=True).hidden_states[-2]
 * Parameters are registered by their transformers state_dict names, bf16, with these host-side fusions:
 *   UMT5: "encoder.block.N.layer.0.SelfAttention.qk.weight" [2*H*d_kv, d_model] = rows of q | k;   "shared.weight" [vocab, d_model]
 *   CLIP: "vision_model.encoder.layers.N.self_attn.qk_proj.{weight,bias}" = q | k;  patch_embedding.weight flattened [D, 3*ps*ps] with K padded
 *         to a multiple of 8;  every LayerNorm additionally as fp32 "<name>.weight_f32" / "<name>.bias_f32" [D].
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct ce_encoder ce_encoder;
typedef struct ce_encoder_config {
  int32_t kind;          /* 0 = UMT5 text encoder, 1 = CLIP vision encoder */
  int32_t vocab_size;    /* UMT5: 256384 */
  int32_t d_model;       /* 4096 | 1280 */
  int32_t d_kv;          /* head dim: 64 | 80 */
  int32_t d_ff;          /* 10240 | 5120 */
  int32_t num_layers;    /* 24 | 32 */
  int32_t num_heads;     /* 64 | 16 */
  float eps;             /* 1e-6 | 1e-5 */
  int32_t image_size;    /* CLIP: 224 */
  int32_t patch_size;    /* CLIP: 14 */
  int32_t hidden_act;    /* CLIP: 0 = quick_gelu, 1 = gelu (erf) */
} ce_encoder_config;
int ce_encoder_create(const ce_encoder_config* cfg, ce_encoder** out);
void ce_encoder_destroy(ce_encoder* h);
int ce_encoder_set_weight(ce_encoder* h, const char* name, const void* ptr, int64_t numel);
int64_t ce_encoder_workspace_bytes(const ce_encoder* h, int batch, int seq_len);   /* CLIP: seq_len = 1 + (image_size/patch_size)^2 */
int64_t ce_encoder_last_launch_count(const ce_encoder* h);
/* input_ids [B, L] int64 (device); valid_len_host[b] = number of leading unmasked tokens (HOST array; the tokenizer pads on the right);
 * bias_tables [num_layers, H, 2L-1] bf16 (device): relative_attention_bias of layer l, head h at relative position (key - query) + L - 1
 * (the bucket function is host code, chronoedit_b200/encoders.py);  last_hidden_state [B, L, d_model] bf16.  L must be a multiple of 8. */
int ce_umt5_encode(ce_encoder* h, const int64_t* input_ids, const int32_t* valid_len_host, void* last_hidden_state, int batch,
                   int seq_len, const void* bias_tables, void* workspace, int64_t workspace_bytes, void* stream);
/* pixel_values [B, 3, S, S] bf16 -> hidden state after `layers_to_run` encoder layers [B, 1 + (S/ps)^2, d_model] bf16
 * (hidden_states[-2] = num_layers - 1 layers; 0 = the embeddings after pre_layrnorm). */
int ce_clip_vision_encode(ce_encoder* h, const void* pixel_values, void* out, int batch, int layers_to_run, void* workspace,
                          int64_t workspace_bytes, void* stream);
/* The CLIP call in fp32, as the reference CLI loads the image encoder (CLIPVisionModel.from_pretrained(..., torch_dtype=torch.float32)):
 * pixel_values [B, 3, S, S] fp32 -> out [B, 1 + (S/ps)^2, d_model] fp32, after `layers_to_run` encoder layers.  Parameters are
 * registered with ce_encoder_set_weight_fp32, fp32, under their transformers names UNFUSED ("...self_attn.q_proj.weight", the LayerNorms
 * without a suffix, "vision_model.embeddings.patch_embedding.weight" as it is, [D, 3, ps, ps]); post_layernorm is not read.  Products
 * run on the wgmma GEMM with every fp32 operand split into three bf16 terms (csrc/fp32_chain.cuh), within rtol 1e-3 / atol 1e-4 of
 * transformers' fp32 CLIPVisionModel at ViT-H/14 (tests/test_gpu_clip_fp32.py).
 * Refused before any launch: a UMT5 handle, a handle without fp32 weights, a missing or mis-sized weight, and a workspace smaller than
 * ce_clip_vision_fp32_workspace_bytes(h, batch) or not 256-byte aligned. */
int ce_encoder_set_weight_fp32(ce_encoder* h, const char* name, const float* ptr, int64_t numel);
int64_t ce_clip_vision_fp32_workspace_bytes(const ce_encoder* h, int batch);   /* -1 for a UMT5 handle or batch < 1 */
int ce_clip_vision_encode_fp32(ce_encoder* h, const float* pixel_values, float* out, int batch, int layers_to_run, void* workspace,
                               int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Individual hot-path operators (used by the handles above; exported for operator-level parity tests / profiling)
 * ------------------------------------------------------------------------------------------------------------ */

/* One channels-last convolution on the wgmma implicit-GEMM kernel (CausalConv3d / Conv2d of wan2pt1.py:42-60, 98-110):
 *   y[to,oh,ow,n] = bias[n] + sum W[n,(dt,dh,dw),c] * x[t_base + to*st + dt, oh*sh + dh - ph, ow*sw + dw - pw, c]
 * x [Tin,Hin,Win,Cin], w packed [Cout, taps, Cin_pad64], y [Tout,Hout,Wout,Cout] (split_time: [2*Tout,...,Cout/2]),
 * resid optional (same geometry as y). */
int ce_conv3d_cl_bf16(const void* x, int Tin, int Hin, int Win, int Cin, const void* w, const void* bias, int Cout, int kt,
                      int kh, int kw, int st, int sh, int sw, int ph, int pw, int t_base, void* y, int Tout, int Hout, int Wout,
                      const void* resid, int split_time, void* stream);

/* out[M,N] = epilogue(A[M,K] x W[N,K]^T + bias): one nn.Linear (+ fused elementwise tail).
 * epilogue: 0 bias | 1 bias+GELU(tanh) | 2 bias+GELU(erf) | 3 bias, gate*y + resid (fp32) | 4 bias, y + resid
 * out_f32 (optional, [M,N]): acc + bias in fp32 before any rounding. */
int ce_linear_bf16(const void* A, int lda, const void* W, int ldw, const void* bias, void* out, int ldo, float* out_f32,
                   int M, int N, int K, int epilogue, const void* resid, int ldr, const float* gate, int gate_stride,
                   int rows_per_batch, void* stream);

/* F.scaled_dot_product_attention (non-causal, no mask, head_dim 128) on [B, L, H*128]-strided q/k/v
 * (transformer_chronoedit.py:91-99).  accumulate=1 adds into `out` in bf16 (text + image cross-attention, :103-104). */
int ce_attention_bf16(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, void* out, int ldo, int B,
                      int H, int Lq, int Lk, float scale, int accumulate, void* stream);

/* Profiling aid: subsequent ce_attention_bf16 calls record, for the first consumer thread of block 0, into `buf` (device,
 * 16 x int64) the cycles of three phases summed over the key tiles, and [3] the key tiles walked; NULL stops.
 * Pipelined schedule (the default): [0] up to S_j's result (waits for K_j, V_{j-1} and the issue turn, issue of S_j and
 * P_{j-1} V_{j-1}, wait for S_j), [1] the softmax of tile j, [2] the wait for P_{j-1} V_{j-1} plus the rescale of o.
 * Serial schedule (version 1 below): [0] S = Q K^T incl. the wait for K, [1] the softmax, [2] P V incl. the wait for V. */
int ce_debug_attention_timing(long long* buf);

/* Test and measurement aid: the schedule of the bf16 attention kernel for later ce_attention_bf16 / ce_attention_dual_bf16
 * calls in this process.  0 and -1 (the default): the pipelined schedule, S of key tile j and P V of tile j-1 issued together
 * and the softmax of tile j run under that P V.  1: the serial schedule (S, softmax, P V per tile) of the same kernel body,
 * with bit-identical output.  Every other version is rejected.  The DiT forward always runs the pipelined schedule. */
int ce_debug_attention_kernel(int version);

/* Cross-attention with TWO key/value sources in one launch: out = bf16(SDPA(q,k,v)) + bf16(SDPA(q,k2,v2)) — the text and
 * image streams of ChronoEditAttnProcessor2_0 (transformer_chronoedit.py:84-104). */
int ce_attention_dual_bf16(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, const void* k2, int ldk2,
                           const void* v2, int ldv2, void* out, int ldo, int B, int H, int Lq, int Lk, int Lk2, float scale,
                           void* stream);

/* FP32LayerNorm (+ adaLN modulate or affine) over the last dim of x[rows, D] -> y (bf16). (:279, :284, :289, :460) */
int ce_layernorm_bf16(const void* x, int ldx, void* y, int ldy, int rows, int D, float eps, const float* scale,
                      const float* shift, int mod_stride, int rows_per_batch, const float* weight, const float* bias,
                      void* stream);

/* diffusers RMSNorm across heads, then optional interleaved RoPE, in place (:62-65, :71-79).
 * rope_cos / rope_sin: fp32 [L, head_dim/2] or NULL. */
int ce_rmsnorm_rope_bf16(void* x, int ldx, int rows, int D, float eps, const void* weight, const float* rope_cos,
                         const float* rope_sin, int L, int head_dim, void* stream);

/* ChronoEditRotaryPosEmbed.forward (:168-213) as fp32 cos/sin tables [L, head_dim/2] written to HOST arrays. */
int ce_rope_table_host(int head_dim, int frames, int height_patches, int width_patches, int max_seq_len,
                       int temporal_skip_len, float theta, float* cos_out_host, float* sin_out_host);

/* ------------------------------------------------------------------------------------------------------------
 * Test aid: the sequence-parallel forward on ONE GPU.  With timeout_ms > 0 the barriers between the phases of the exchange
 * (ce_dit_sp_configure) launch no kernel: each one synchronises the rank's stream, then its thread waits until the threads of
 * all `world` handles of this process configured with the same region table (same region_ptrs[0]) have arrived.  So `world`
 * handles driven from `world` host threads, each on its own stream, with ordinary device allocations as regions, run the same
 * kernels, address arithmetic and peer stores as `world` GPUs, and no kernel ever spins on another rank's progress.  A wait
 * longer than timeout_ms fails with an error naming the rank and the barrier, and every later barrier of that group fails at
 * once (configure again to start over).  The mode is refused while the stream is capturing a graph.  0 (the default) restores
 * the device barrier.  The setting survives ce_dit_sp_configure.  The single-GPU forward is unaffected.
 * ------------------------------------------------------------------------------------------------------------ */
int ce_dit_sp_host_barrier(ce_dit* h, int timeout_ms);

/* ------------------------------------------------------------------------------------------------------------
 * Test aids: the DiT's fused-statistics path, one operator at a time.  When D % 256 == 0 the GEMM that writes a
 * row also writes per-(row, N tile) statistics of the values it stored, and the LayerNorm / RMSNorm that follows
 * merges those partials instead of reducing over the row.  Not needed to run the model.
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct ce_linear_args {
  const void* A;           /* [M, lda] bf16 */
  int32_t lda;
  const void* W;           /* [N, ldw] bf16 (nn.Linear weight) */
  int32_t ldw;
  int32_t M, N, K;         /* N % 8 == 0 */
  void* out;               /* [M, ldo] bf16 (may be NULL when out_f32 is given and stats_mode == 0) */
  int32_t ldo;
  float* out_f32;          /* optional [M, ld_f32]: acc + bias in fp32 before any rounding */
  int32_t ld_f32;          /* 0 = N */
  const void* bias;        /* [N] bf16 or NULL */
  const void* bias_row;    /* [M] bf16 or NULL: added per output row */
  int32_t epilogue;        /* as ce_linear_bf16 */
  const void* resid;       /* [M, ldr] bf16, epilogues 3 and 4 */
  int32_t ldr;
  const float* gate;       /* [batches, gate_stride] fp32, epilogue 3; batch = row / rows_per_batch */
  int32_t gate_stride;
  int32_t rows_per_batch;
  float* stats_out;        /* optional [M, stats_ld] pairs of floats, one per (row, N tile) of the stored bf16 output: */
  int32_t stats_ld;        /*   stats_mode 1: (mean, M2 = sum (y - mean)^2) over the tile's columns  */
  int32_t stats_mode;      /*   stats_mode 2: (sum y^2, 0);  tile width 256 if N >= 256, else 128 if N >= 128, else 64 */
  int32_t group_m;         /* M tiles per rasterisation group; 0 = default.  Results do not depend on it. */
} ce_linear_args;

/* out = epilogue(A x W^T + bias) with every option of the DiT's GEMM, including the row statistics. */
int ce_linear_ex_bf16(const ce_linear_args* args, void* stream);

/* FP8 mode's GEMM: base.A [M, lda] and base.W [N, ldw] hold e4m3 (lda, ldw, K multiples of 16); the accumulator is
 * y = (sum_k A W) * a_scale[m] * w_scale[n] (fp32 [M] and [N], w_scale 8-byte aligned), then every epilogue option of
 * `base` applies to y as ce_linear_ex_bf16 applies it to A x W^T (out_f32 receives y + bias). */
typedef struct ce_linear_fp8_args {
  ce_linear_args base;
  const float* a_scale;
  const float* w_scale;
} ce_linear_fp8_args;
int ce_linear_fp8_ex(const ce_linear_fp8_args* args, void* stream);

/* The two GEMMs above with run-time LoRA's epilogue addend: term [M, ldt] bf16 (ldt % 8 == 0, ldt >= N, 16-byte aligned) is
 * added as y = bf16(bf16(acc + bias) + term) before GELU, gate, residual and the row statistics.  out_f32 is refused. */
int ce_linear_lora_bf16(const ce_linear_args* args, const void* term, int ldt, void* stream);
int ce_linear_lora_fp8(const ce_linear_fp8_args* args, const void* term, int ldt, void* stream);

/* Per-row e4m3 quantization of x [rows, K] bf16 (K % 16 == 0, ldx % 8 == 0, ldq % 16 == 0): scale[m] = max_k |x| / 448
 * (1 for a zero row), q[m, k] = e4m3 bits of cvt.rn.satfinite(x / scale[m]), the division in IEEE fp32. */
int ce_quantize_rows_fp8(const void* x, int ldx, int rows, int K, void* q, int ldq, float* scale, void* stream);

/* FP8 attention, q | k: the rule of ce_quantize_rows_fp8 per (row, head) over 128 values.  x [rows, heads * 128] bf16 (ldx % 8)
 * -> q [rows, heads * 128] e4m3 (ldq bytes, % 16) and scale [rows, heads] fp32. */
int ce_quantize_heads_fp8(const void* x, int ldx, int rows, int heads, void* q, int ldq, float* scale, void* stream);
/* FP8 attention, v [B, L, H * 128] bf16 (row stride ldv): scale [B, H * 128] = max over the sample's tokens |v| / 448 (1 if 0);
 * vt [B, H, 128, Lpad] e4m3 = v / scale transposed, keys contiguous (Lpad >= L, % 32), the keys of every 32-key group stored in
 * the order fp8_attention_key_order() of chronoedit_b200/transformer.py gives, keys >= L zero.  Two launches. */
int ce_quantize_v_fp8(const void* v, int ldv, int B, int L, int H, void* vt, int Lpad, float* scale, void* stream);
/* FP8 self-attention on the quantizers' outputs: q, k [B*L, ldqk bytes] e4m3 (head h at column h * 128), q_scale / k_scale
 * [(b*L + i) * lds + h], vt / v_scale as ce_quantize_v_fp8 writes them; out [B*L, ldo] bf16, head h at column h * 128.
 * out = bf16((sum_j P^ v^) v_scale / sum_j P^) with P^ = e4m3(256 exp2((q^ k^ q_scale k_scale) scale log2e - running max)). */
int ce_attention_fp8(const void* q, const void* k, int ldqk, const float* q_scale, const float* k_scale, int lds, const void* vt, int Lpad,
                     const float* v_scale, void* out, int ldo, int B, int H, int L, float scale, void* stream);

/* FP32LayerNorm (+ modulate or affine) like ce_layernorm_bf16, with the row statistics merged from `tiles` stats_mode-1
 * partials of width tile_n covering [0, D) (stats [rows, stats_ld] float pairs).  scale_is_1p: `scale` holds 1 + scale.
 * stats == NULL: the kernel reduces over each row itself, as ce_layernorm_bf16 does (stats_ld, tiles, tile_n are ignored). */
int ce_layernorm_stats_bf16(const void* x, int ldx, void* y, int ldy, int rows, int D, float eps, const float* scale,
                            const float* shift, int mod_stride, int rows_per_batch, const float* weight, const float* bias,
                            int scale_is_1p, const float* stats, int stats_ld, int tiles, int tile_n, void* stream);

/* RMSNorm across heads (+ optional RoPE) like ce_rmsnorm_rope_bf16, in place on nmat (1 or 2) matrices of width D side by
 * side in x (q | k): matrix m starts at column m * D, uses weight m and the stats_mode-2 partials [m * tiles, (m+1) * tiles).
 * stats == NULL: the kernel reduces over each row of each matrix itself, as ce_rmsnorm_rope_bf16 does (stats_ld and tiles
 * are ignored). */
int ce_rmsnorm_rope_stats_bf16(void* x, int ldx, int rows, int D, float eps, const void* weight0, const void* weight1, int nmat,
                               const float* rope_cos, const float* rope_sin, int L, int head_dim, const float* stats,
                               int stats_ld, int tiles, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Test aids: the VAE and encoder operators, one at a time, each with the argument checks of the model's own launches.
 * Channels-last tensors are [T, H, W, C] bf16.  Not needed to run the model.
 * ------------------------------------------------------------------------------------------------------------ */

/* RMS_norm (+ SiLU) over the channels of x [pixels, C] -> y (C % 8 == 0, C <= 512), with the reference's bf16 rounding points:
 * n = bf16(||x||), y = bf16(bf16(bf16(x / max(n, 1e-12)) * sqrt(C)) * gamma[c]), then y = bf16(silu(y)) when apply_silu != 0. */
int ce_rms_silu_cl_bf16(const void* x, const void* gamma, void* y, int64_t pixels, int C, int apply_silu, void* stream);

/* Nearest 2x spatial upsample: y [T, 2H, 2W, C] from x [T, H, W, C], C % 8 == 0. */
int ce_upsample2x_cl_bf16(const void* x, void* y, int T, int H, int W, int C, void* stream);

/* im2row of a stride-1 convolution: A [Tout*Hout*Wout, Kpad] (16-byte aligned) with
 *   A[(to,oh,ow), ((dt*kh + dh)*kw + dw)*Cin + c] = x[c*sc + ti*st + hi*sh + wi*sw],  ti = t_base + to + dt, hi = oh + dh - ph,
 *   wi = ow + dw - pw,
 * zero where (ti, hi, wi) lies outside [0,Tin) x [0,Hin) x [0,Win) and in the columns K = kt*kh*kw*Cin .. Kpad-1
 * (Kpad % 8 == 0, Kpad >= K).  Strides are in elements, so x may be planar [Cin, Tin, Hin, Win] or channels-last. */
int ce_im2row_bf16(const void* x, int64_t sc, int64_t st, int64_t sh, int64_t sw, int Tin, int Hin, int Win, int Cin, void* A, int Kpad,
                   int Tout, int Hout, int Wout, int kt, int kh, int kw, int ph, int pw, int t_base, void* stream);

/* The convolution of ce_conv3d_cl_bf16 with every option of the VAE's launches. */
typedef struct ce_conv3d_args {
  const void* x;                 /* [Tin, Hin, Win, Cin] */
  int32_t Tin, Hin, Win, Cin;    /* Cin % 8 == 0 */
  const void* w;                 /* [Cout, kt*kh*kw, Cin_pad] */
  const void* bias;              /* [Cout] or NULL */
  int32_t Cout, Cin_pad;         /* Cin_pad % 64 == 0, Cin_pad >= Cin */
  int32_t kt, kh, kw;
  int32_t st, sh, sw;            /* sh, sw in {1, 2} */
  int32_t ph, pw;
  int32_t t_base;                /* first input frame of output frame 0 */
  void* y;                       /* [Tout, Hout, Wout, Cout] (split_time: [2*Tout, Hout, Wout, Cout/2]; planar_out: see below) */
  int32_t Tout, Hout, Wout;
  const void* resid;             /* optional, same layout as y: y = bf16(bf16(conv) + resid) */
  int32_t split_time;            /* 1: channel n goes to frame 2*to + n / (Cout/2), channel n % (Cout/2); Cout % 16 == 0 */
  int32_t planar_out;            /* 1: y is planar [Cout, planar_T, Hout, Wout] and output frame to is stored at planar_t0 + to, */
  int32_t clamp;                 /*    clamped to [-1, 1] when clamp != 0 (the decoder head); no resid or split_time with it */
  int32_t planar_T, planar_t0;
} ce_conv3d_args;
int ce_conv3d_cl_ex_bf16(const ce_conv3d_args* args, void* stream);
/* The fp32 VAE's convolution with the same arguments, read as: x the split pair [Tin, Hin, Win, 2, Cin] bf16 (hi = bf16(v) then
 * lo = bf16(v - hi) for each pixel's channels), w packed as for ce_vae_set_weight_fp32, bias [Cout] fp32, resid fp32 in y's layout,
 * y fp32 (or NULL when only y_pair is wanted; not with planar_out), y_pair optional: the split pair of y [frames, Hout, Wout, 2, C]. */
int ce_conv3d_cl_ex_fp32(const ce_conv3d_args* args, void* y_pair, void* stream);

/* Multi-head self-attention composed of GEMMs over one sequence of L tokens, as the VAE mid-block (H = 1, dk = D) and both
 * encoders run it; I = H * dk, L8 = L rounded up to 8.
 *   q | k = x Wqk^T + bqk -> qk [L, 2I];  V^T = Wv x^T + bv -> vT [I, L8];  S_h = q_h k_h^T (fp32) -> S [H, L, L8];
 *   P = bf16(softmax over keys j < L of the rule's score) -> P [H, L, L8], zero in columns L .. L8-1;
 *   out[:, h*dk : (h+1)*dk] = bf16(P_h[:, 0:kpv] V_h) -> out [L, ldo].
 * Score of key j in query row i of head h:
 *   rule 0 (VAE):  S * scale;  rule 2 (CLIP):  bf16(bf16(S) * scale);
 *   rule 1 (UMT5): bf16(bf16(S) + bias[h * bias_ld + (j - i) + L - 1]) over the keys j < valid only (1 <= valid; bias_ld >= 2L - 1).
 * The caller owns every buffer: x with L8 readable rows of D (rows L .. L8-1 only reach columns of V^T that P.V does not sum
 * over, or multiply zeros of P), qk [L8, 2I] (rows L .. L8-1 are read, never written), vT [I, L8], S [H, L, L8] fp32,
 * P [H, L, L8], out [L, ldo].  kpv in [L, L8]: the keys P.V sums over (L8 only when V^T is finite there). */
typedef struct ce_gemm_attention_args {
  const void* x;                 /* [L8, D] */
  int32_t D, L, H, dk, kpv;      /* D, dk % 8 == 0 */
  const void* wqk;               /* [2I, D] = rows of Wq | Wk */
  const void* bqk;               /* [2I] or NULL */
  const void* wv;                /* [I, D] */
  const void* bv;                /* [I] or NULL */
  int32_t rule;                  /* 0 scaled (VAE), 1 T5 (UMT5), 2 CLIP */
  float scale;
  const void* bias;              /* rule 1: [H, bias_ld] bf16 */
  int32_t bias_ld, valid;
  void* qk;
  void* vT;
  float* S;
  void* P;
  void* out;
  int32_t ldo;                   /* % 8 == 0, >= I */
} ce_gemm_attention_args;
int ce_gemm_attention_bf16(const ce_gemm_attention_args* args, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Sampling glue either side of the DiT call (SURVEY.md section 8(f) row 1): one launch per denoising step for
 *   noise = uncond + g*(cond - uncond)                                   chronoedit_diffusers/pipeline_chronoedit.py:736
 *   FlowUniPCMultistepScheduler.step: x0 conversion, UniC corrector, UniP predictor (solver_order 2, bh2, predict_x0,
 *   flow_prediction, lower_order_final)                                  chronoedit/_src/models/fm_solvers_unipc.py:670-756
 *   channels [0, c_lat) of the next cat([latents, condition], 1).to(bf16) pipeline_chronoedit.py:712
 * Every intermediate is rounded to the tensor dtype exactly where the reference's separate torch kernels round, so the
 * result is bit-identical to running the reference on CUDA.  The scalar coefficients are the caller's business (the Python
 * mirror chronoedit_b200/scheduler.py computes them with the same fp32 CPU tensor ops as the reference, :418-447, :565-620);
 * divisions by r_k arrive as the fp32 reciprocal because that is how torch's CUDA `tensor / scalar` evaluates.
 * ------------------------------------------------------------------------------------------------------------ */
#define CE_DTYPE_F32 0
#define CE_DTYPE_BF16 1

typedef struct ce_unipc_step_args {
  int32_t sample_dtype;          /* dtype of sample / last_sample / m_prev* / outputs: CE_DTYPE_F32 | CE_DTYPE_BF16 */
  int32_t model_dtype;           /* dtype of cond / uncond; (f32,f32) (f32,bf16) (bf16,bf16) are built */
  int64_t n;                     /* elements of the latent [B, c_lat, T, H, W] */
  const void* cond;              /* model output (conditional) */
  const void* uncond;            /* model output (unconditional) or NULL: no guidance */
  float guidance;
  float sigma;                   /* sigmas[step_index]: x0 = sample - sigma * v                       (:340-341) */
  const void* sample;            /* x_t */
  const void* last_sample;       /* sample before the previous predictor; corrector only                (:567) */
  const void* m_prev;            /* model_outputs[-1] before this call (x0 prediction of the previous step) or NULL */
  const void* m_prev2;           /* model_outputs[-2] before this call or NULL */
  int32_t use_corrector;         /* step_index > 0 and last_sample is set                               (:701-705) */
  int32_t c_order;               /* 1 | 2: this_order of the previous step */
  float c_x, c_m0, c_bh;         /* sigma_t/sigma_s0, alpha_t*h_phi_1, alpha_t*B_h at (step_index, step_index-1) */
  float c_inv_rk, c_rho0, c_rho1;/* order 2: 1/r_k and solve(R, b) cast to the sample dtype; order 1 uses 0.5 */
  int32_t p_order;               /* 1 | 2: min(2, steps - step_index, lower_order_nums + 1)             (:729-737) */
  float p_x, p_m0, p_bh;         /* the same three scalars at (step_index+1, step_index) */
  float p_inv_rk;                /* order 2 */
  float p_zero;                  /* order 1: alpha_t*B_h*0, still subtracted by the reference (sign of zero) */
  void* x0_out;                  /* -> model_outputs[-1] */
  void* corrected_out;           /* -> last_sample (written only when use_corrector) */
  void* prev_sample_out;         /* -> returned sample */
  void* model_input_out;         /* optional bf16 [B, c_total, inner]: channels [0, c_lat) <- prev_sample; NULL = skip */
  int64_t inner;                 /* T*H*W */
  int32_t c_lat, c_total;        /* 16, 36 */
} ce_unipc_step_args;

int ce_unipc_step(const ce_unipc_step_args* args, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CHRONOEDIT_B200_H_ */
