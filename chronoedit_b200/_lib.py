"""ctypes binding of libchronoedit_b200.so (the C ABI declared in include/chronoedit_b200.h).

There is no CPU or PyTorch fallback: if the shared library is missing this module raises, and every compute
entry point fails on a machine without an sm_90 GPU.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libchronoedit_b200.so")


class CEError(RuntimeError):
    pass


class VAEConfigC(ctypes.Structure):
    _fields_ = [("dim", c_int32), ("z_dim", c_int32), ("dim_mult", c_int32 * 4), ("num_res_blocks", c_int32),
                ("temporal_downsample", c_int32 * 3)]


class DiTConfigC(ctypes.Structure):
    _fields_ = [
        ("num_attention_heads", c_int32), ("attention_head_dim", c_int32), ("in_channels", c_int32),
        ("out_channels", c_int32), ("text_dim", c_int32), ("freq_dim", c_int32), ("ffn_dim", c_int32),
        ("num_layers", c_int32), ("image_dim", c_int32), ("added_kv_proj_dim", c_int32),
        ("rope_max_seq_len", c_int32), ("rope_temporal_skip_len", c_int32), ("eps", c_float),
        ("patch_t", c_int32), ("patch_h", c_int32), ("patch_w", c_int32),
    ]


class EncoderConfigC(ctypes.Structure):   # ce_encoder_config
    _fields_ = [("kind", c_int32), ("vocab_size", c_int32), ("d_model", c_int32), ("d_kv", c_int32), ("d_ff", c_int32),
                ("num_layers", c_int32), ("num_heads", c_int32), ("eps", c_float), ("image_size", c_int32), ("patch_size", c_int32),
                ("hidden_act", c_int32)]


class UniPCStepArgsC(ctypes.Structure):   # ce_unipc_step_args (field order = include/chronoedit_b200.h)
    _fields_ = [
        ("sample_dtype", c_int32), ("model_dtype", c_int32), ("n", c_int64), ("cond", c_void_p), ("uncond", c_void_p),
        ("guidance", c_float), ("sigma", c_float), ("sample", c_void_p), ("last_sample", c_void_p), ("m_prev", c_void_p),
        ("m_prev2", c_void_p), ("use_corrector", c_int32), ("c_order", c_int32), ("c_x", c_float), ("c_m0", c_float),
        ("c_bh", c_float), ("c_inv_rk", c_float), ("c_rho0", c_float), ("c_rho1", c_float), ("p_order", c_int32),
        ("p_x", c_float), ("p_m0", c_float), ("p_bh", c_float), ("p_inv_rk", c_float), ("p_zero", c_float),
        ("x0_out", c_void_p), ("corrected_out", c_void_p), ("prev_sample_out", c_void_p), ("model_input_out", c_void_p),
        ("inner", c_int64), ("c_lat", c_int32), ("c_total", c_int32),
    ]


class LinearArgsC(ctypes.Structure):   # ce_linear_args (field order = include/chronoedit_b200.h)
    _fields_ = [
        ("A", c_void_p), ("lda", c_int32), ("W", c_void_p), ("ldw", c_int32), ("M", c_int32), ("N", c_int32), ("K", c_int32),
        ("out", c_void_p), ("ldo", c_int32), ("out_f32", c_void_p), ("ld_f32", c_int32), ("bias", c_void_p), ("bias_row", c_void_p),
        ("epilogue", c_int32), ("resid", c_void_p), ("ldr", c_int32), ("gate", c_void_p), ("gate_stride", c_int32),
        ("rows_per_batch", c_int32), ("stats_out", c_void_p), ("stats_ld", c_int32), ("stats_mode", c_int32), ("group_m", c_int32),
    ]


class LinearFp8ArgsC(ctypes.Structure):   # ce_linear_fp8_args
    _fields_ = [("base", LinearArgsC), ("a_scale", c_void_p), ("w_scale", c_void_p)]


class Conv3dArgsC(ctypes.Structure):   # ce_conv3d_args
    _fields_ = [
        ("x", c_void_p), ("Tin", c_int32), ("Hin", c_int32), ("Win", c_int32), ("Cin", c_int32), ("w", c_void_p), ("bias", c_void_p),
        ("Cout", c_int32), ("Cin_pad", c_int32), ("kt", c_int32), ("kh", c_int32), ("kw", c_int32), ("st", c_int32), ("sh", c_int32),
        ("sw", c_int32), ("ph", c_int32), ("pw", c_int32), ("t_base", c_int32), ("y", c_void_p), ("Tout", c_int32), ("Hout", c_int32),
        ("Wout", c_int32), ("resid", c_void_p), ("split_time", c_int32), ("planar_out", c_int32), ("clamp", c_int32),
        ("planar_T", c_int32), ("planar_t0", c_int32),
    ]


class GemmAttentionArgsC(ctypes.Structure):   # ce_gemm_attention_args
    _fields_ = [
        ("x", c_void_p), ("D", c_int32), ("L", c_int32), ("H", c_int32), ("dk", c_int32), ("kpv", c_int32), ("wqk", c_void_p),
        ("bqk", c_void_p), ("wv", c_void_p), ("bv", c_void_p), ("rule", c_int32), ("scale", c_float), ("bias", c_void_p),
        ("bias_ld", c_int32), ("valid", c_int32), ("qk", c_void_p), ("vT", c_void_p), ("S", c_void_p), ("P", c_void_p),
        ("out", c_void_p), ("ldo", c_int32),
    ]


class TileBlendArgsC(ctypes.Structure):   # ce_vae_tile_blend_args
    _fields_ = [
        ("fp32", c_int32), ("tile", c_void_p), ("C", c_int32), ("T", c_int32), ("th", c_int32), ("tw", c_int32), ("above", c_void_p),
        ("above_h", c_int32), ("left", c_void_p), ("left_w", c_int32), ("out", c_void_p), ("out_h", c_int32), ("out_w", c_int32),
        ("oy", c_int32), ("ox", c_int32), ("crop_h", c_int32), ("crop_w", c_int32), ("clamp", c_int32), ("strip", c_void_p),
        ("strip_h", c_int32), ("tail", c_void_p), ("tail_w", c_int32),
    ]


# name -> (restype, argtypes); every symbol include/chronoedit_b200.h declares
SIGNATURES = {
    "ce_abi_version": (c_int, []),
    "ce_last_error": (c_char_p, []),
    "ce_device_check": (c_int, []),
    "ce_unipc_step": (c_int, [POINTER(UniPCStepArgsC), c_void_p]),
    "ce_dit_create": (c_int, [POINTER(DiTConfigC), POINTER(c_void_p)]),
    "ce_dit_destroy": (None, [c_void_p]),
    "ce_dit_set_weight": (c_int, [c_void_p, c_char_p, c_void_p, c_int, c_int64]),
    "ce_dit_weights_complete": (c_int, [c_void_p]),
    "ce_dit_workspace_bytes": (c_int64, [c_void_p, c_int, c_int, c_int, c_int, c_int]),
    "ce_dit_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                               c_int, c_void_p, c_int64, c_void_p, c_void_p]),
    "ce_dit_context_cache_bytes": (c_int64, [c_void_p, c_int, c_int]),
    "ce_dit_forward_ex": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                  c_int, c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_int, c_void_p]),
    "ce_dit_sp_region_bytes": (c_int64, [c_void_p, c_int, c_int, c_int, c_int, c_int]),
    "ce_dit_sp_configure": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int64]),
    "ce_dit_sp_host_barrier": (c_int, [c_void_p, c_int]),
    "ce_dit_bp_region_bytes": (c_int64, [c_void_p, c_int, c_int, c_int, c_int, c_int]),
    "ce_dit_bp_configure": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int64]),
    "ce_dit_bp_host_barrier": (c_int, [c_void_p, c_int]),
    "ce_dit_cp_region_bytes": (c_int64, [c_void_p, c_int, c_int, c_int, c_int]),
    "ce_dit_cp_configure": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int64]),
    "ce_dit_cp_exchange": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "ce_dit_cp_host_barrier": (c_int, [c_void_p, c_int]),
    "ce_ipc_alloc": (c_int, [c_int64, POINTER(c_void_p)]),
    "ce_ipc_free": (c_int, [c_void_p]),
    "ce_ipc_get_handle": (c_int, [c_void_p, c_void_p]),
    "ce_ipc_open": (c_int, [c_void_p, POINTER(c_void_p)]),
    "ce_ipc_close": (c_int, [c_void_p]),
    "ce_dit_set_capture": (c_int, [c_void_p, c_void_p, c_void_p, c_int]),
    "ce_dit_teacache_probe_bytes": (c_int64, [c_void_p, c_int]),
    "ce_dit_teacache_probe": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p]),
    "ce_dit_set_residual_record": (c_int, [c_void_p, c_void_p, c_int64]),
    "ce_dit_forward_cached": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                      c_void_p, c_int64, c_void_p]),
    "ce_dit_host_staging_bytes": (c_int64, [c_void_p, c_int, c_int, c_int, c_int, c_int]),
    "ce_dit_forward_host": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                    c_int, c_int, c_void_p, c_int64, c_void_p, c_int64, c_void_p]),
    "ce_dit_forward_host_ex": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                       c_int, c_int, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_int, c_void_p]),
    "ce_dit_host_staging_sample_offset": (c_int64, [c_void_p, c_int, c_int, c_int, c_int, c_int]),
    "ce_dit_set_weight_fp32": (c_int, [c_void_p, c_char_p, c_void_p, c_int64]),
    "ce_dit_fp32_workspace_bytes": (c_int64, [c_void_p, c_int, c_int, c_int, c_int, c_int]),
    "ce_dit_forward_fp32": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                    c_void_p, c_int64, c_void_p, c_void_p]),
    "ce_dit_last_launch_count": (c_int64, [c_void_p]),
    "ce_dit_profile_begin": (c_int, [c_void_p, c_int]),
    "ce_dit_profile_end": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "ce_encoder_create": (c_int, [POINTER(EncoderConfigC), POINTER(c_void_p)]),
    "ce_encoder_destroy": (None, [c_void_p]),
    "ce_encoder_set_weight": (c_int, [c_void_p, c_char_p, c_void_p, c_int64]),
    "ce_encoder_workspace_bytes": (c_int64, [c_void_p, c_int, c_int]),
    "ce_encoder_last_launch_count": (c_int64, [c_void_p]),
    "ce_umt5_encode": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int64, c_void_p]),
    "ce_clip_vision_encode": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int64, c_void_p]),
    "ce_encoder_set_weight_fp32": (c_int, [c_void_p, c_char_p, c_void_p, c_int64]),
    "ce_clip_vision_fp32_workspace_bytes": (c_int64, [c_void_p, c_int]),
    "ce_clip_vision_encode_fp32": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int64, c_void_p]),
    "ce_vae_create": (c_int, [c_void_p, POINTER(c_void_p)]),
    "ce_vae_destroy": (None, [c_void_p]),
    "ce_vae_set_weight": (c_int, [c_void_p, c_char_p, c_void_p, c_int64]),
    "ce_vae_workspace_bytes": (c_int64, [c_void_p, c_int, c_int, c_int, c_int]),
    "ce_vae_encode": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_int64, c_void_p]),
    "ce_vae_decode": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int64, c_void_p]),
    "ce_vae_last_launch_count": (c_int64, [c_void_p]),
    "ce_vae_set_weight_fp32": (c_int, [c_void_p, c_char_p, c_void_p, c_int64]),
    "ce_vae_workspace_bytes_fp32": (c_int64, [c_void_p, c_int, c_int, c_int, c_int]),
    "ce_vae_encode_fp32": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_int64, c_void_p]),
    "ce_vae_decode_fp32": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int64, c_void_p]),
    "ce_vae_workspace_bytes_tiled": (c_int64, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int]),
    "ce_vae_encode_tiled": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int64,
                                    c_void_p]),
    "ce_vae_decode_tiled": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                    c_int64, c_void_p]),
    "ce_vae_workspace_bytes_tiled_fp32": (c_int64, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int]),
    "ce_vae_encode_tiled_fp32": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                         c_int64, c_void_p]),
    "ce_vae_decode_tiled_fp32": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                         c_void_p, c_int64, c_void_p]),
    "ce_vae_tile_blend": (c_int, [POINTER(TileBlendArgsC), c_void_p]),
    "ce_vae_sp_region_bytes": (c_int64, [c_void_p, c_int, c_int, c_int]),
    "ce_vae_sp_configure": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int64]),
    "ce_vae_sp_host_barrier": (c_int, [c_void_p, c_int]),
    "ce_conv3d_cl_bf16": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                  c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    "ce_linear_bf16": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int,
                               c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p]),
    "ce_attention_bf16": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_int,
                                  c_int, c_int, c_float, c_int, c_void_p]),
    "ce_debug_attention_kernel": (c_int, [c_int]),
    "ce_debug_attention_timing": (c_int, [c_void_p]),
    "ce_attention_dual_bf16": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int,
                                       c_int, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "ce_layernorm_bf16": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_int,
                                  c_int, c_void_p, c_void_p, c_void_p]),
    "ce_rmsnorm_rope_bf16": (c_int, [c_void_p, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p, c_int,
                                     c_int, c_void_p]),
    "ce_rope_table_host": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p]),
    "ce_linear_ex_bf16": (c_int, [POINTER(LinearArgsC), c_void_p]),
    "ce_linear_fp8_ex": (c_int, [POINTER(LinearFp8ArgsC), c_void_p]),
    "ce_linear_lora_bf16": (c_int, [POINTER(LinearArgsC), c_void_p, c_int, c_void_p]),
    "ce_linear_lora_fp8": (c_int, [POINTER(LinearFp8ArgsC), c_void_p, c_int, c_void_p]),
    "ce_dit_set_lora": (c_int, [c_void_p, POINTER(c_void_p), POINTER(c_void_p), POINTER(c_int32), c_int]),
    "ce_quantize_rows_fp8": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "ce_dit_set_attention_fp8": (c_int, [c_void_p, c_int]),
    "ce_quantize_heads_fp8": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "ce_quantize_v_fp8": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "ce_attention_fp8": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int,
                                 c_int, c_int, c_int, c_float, c_void_p]),
    "ce_layernorm_stats_bf16": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_int,
                                        c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p]),
    "ce_rmsnorm_rope_stats_bf16": (c_int, [c_void_p, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                           c_int, c_int, c_void_p, c_int, c_int, c_void_p]),
    "ce_rms_silu_cl_bf16": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p]),
    "ce_upsample2x_cl_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "ce_im2row_bf16": (c_int, [c_void_p, c_int64, c_int64, c_int64, c_int64, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, c_int,
                               c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "ce_conv3d_cl_ex_bf16": (c_int, [POINTER(Conv3dArgsC), c_void_p]),
    "ce_conv3d_cl_ex_fp32": (c_int, [POINTER(Conv3dArgsC), c_void_p, c_void_p]),
    "ce_gemm_attention_bf16": (c_int, [POINTER(GemmAttentionArgsC), c_void_p]),
}

_lib = None


def lib() -> ctypes.CDLL:
    """Load (once) and return the shared library with typed signatures."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise CEError(
                f"{LIB_PATH} is missing: build it with `python -m chronoedit_b200.build` (or __graft_entry__.build()). "
                "chronoedit_b200 has no CPU / PyTorch fallback.")
        l = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)  # AttributeError = header and library out of sync
            fn.restype = res
            fn.argtypes = args
        if l.ce_abi_version() != 1:
            raise CEError(f"ABI version mismatch: library reports {l.ce_abi_version()}, binding expects 1")
        _lib = l
    return _lib


def check(rc: int) -> None:
    if rc != 0:
        msg = lib().ce_last_error()
        raise CEError(f"chronoedit_b200 error {rc}: {msg.decode() if msg else '?'}")


def ptr(t) -> c_void_p:
    """Device (or host) data pointer of a torch tensor as c_void_p; None -> NULL."""
    if t is None:
        return c_void_p(0)
    return c_void_p(t.data_ptr())


def current_stream() -> c_void_p:
    import torch

    return c_void_p(torch.cuda.current_stream().cuda_stream)
