"""H100-native drop-in for `ChronoEditTransformer3DModel`.

Host-side mirror of /root/reference/chronoedit_diffusers/transformer_chronoedit.py:298-476: same constructor
arguments, same parameter names (so a diffusers checkpoint / `state_dict` loads unchanged), same
`forward(hidden_states, timestep, encoder_hidden_states, encoder_hidden_states_image=None, return_dict=True,
attention_kwargs=None)` signature and return types, `.config`, `.dtype`, `from_pretrained`.  All arithmetic happens in
libchronoedit_b200.so (hand-written sm_90a kernels) through the C ABI of include/chronoedit_b200.h; PyTorch only
owns the memory and the stream.  There is no PyTorch fallback path.
"""
from __future__ import annotations

import contextlib
import json
import math
import os
from dataclasses import dataclass
from typing import Any, Dict, Optional, Tuple, Union

import torch
import torch.nn as nn

from . import _lib
from . import teacache as _tc
from ._checkpoint import load_safetensors
from ._lib import CEError, DiTConfigC, check, current_stream, ptr

# reference `_keep_in_fp32_modules` (transformer_chronoedit.py:338)
KEEP_FP32 = ("time_embedder", "scale_shift_table", "norm1", "norm2", "norm3")
# Run-time LoRA (set_adapters): block linear layer -> (ce_dit_set_lora target, part of the fused GEMM's N, parts).  The fused QKV
# and context K | V GEMMs stack their layers' rows, so an adapter's lora_B lands at rows [part * N, (part + 1) * N) of the target.
LORA_TARGETS = {"attn1.to_q": (0, 0, 3), "attn1.to_k": (0, 1, 3), "attn1.to_v": (0, 2, 3), "attn1.to_out.0": (1, 0, 1),
                "attn2.to_q": (2, 0, 1), "attn2.to_k": (3, 0, 2), "attn2.to_v": (3, 1, 2), "attn2.add_k_proj": (4, 0, 2),
                "attn2.add_v_proj": (4, 1, 2), "attn2.to_out.0": (5, 0, 1), "ffn.net.0.proj": (6, 0, 1), "ffn.net.2": (7, 0, 1)}
LORA_NUM_TARGETS = 8

# The FP8 mode's weights: the six per-token GEMMs of every block (attn1.to_qkv is the fused to_q | to_k | to_v).  The patch
# embedding, the condition embedders, proj_out and the step-invariant cross-attention K/V projections stay bf16.
FP8_LINEARS = ("attn1.to_q", "attn1.to_k", "attn1.to_v", "attn1.to_out.0", "attn2.to_q", "attn2.to_out.0", "ffn.net.0.proj",
               "ffn.net.2")


def quantize_fp8_rows(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The FP8 mode's quantization rule, one scale per row of `x` (an output channel of a weight, a token of an activation):
    s = max_k |x[row, k]| / 448 in fp32 (1 if that maximum is 0) and q = e4m3(clamp(x / s, -448, 448)), rounded to nearest-even.
    Returns (q as torch.float8_e4m3fn, s as fp32).  The same on CPU and CUDA, and what the device computes for every FP8
    GEMM's activations (ce_quantize_rows_fp8)."""
    x = x.float()
    amax = x.abs().amax(dim=-1)
    # a tensor divisor: torch's CUDA division by a Python scalar multiplies by its reciprocal, which is not the IEEE quotient
    s = torch.where(amax == 0, torch.ones_like(amax), amax / torch.full_like(amax, 448.0))
    q = (x / s.unsqueeze(-1)).clamp(-448, 448).to(torch.float8_e4m3fn)
    return q, s


def quantize_fp8_heads(x: torch.Tensor, head_dim: int = 128) -> Tuple[torch.Tensor, torch.Tensor]:
    """The FP8 attention's rule for q and k: `quantize_fp8_rows` per (token, head), over the head_dim values of each head.
    x [..., heads * head_dim] -> (q [..., heads * head_dim] float8_e4m3fn, s [..., heads] fp32).  What ce_quantize_heads_fp8
    computes, bit for bit."""
    *lead, n = x.shape
    q, s = quantize_fp8_rows(x.reshape(-1, head_dim))
    return q.reshape(*lead, n), s.reshape(*lead, n // head_dim)


def quantize_fp8_channels(v: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The FP8 attention's rule for v [B, L, C]: one scale per (sample, channel) over the sample's tokens, i.e.
    `quantize_fp8_rows(v[b].T)` for every sample.  Returns (v^T [B, C, L] float8_e4m3fn, keys in order, and s [B, C] fp32).
    One sample's scales never depend on another sample."""
    return quantize_fp8_rows(v.transpose(1, 2))


def fp8_attention_key_order() -> torch.Tensor:
    """Key (0..31) held at position p of every 32-key group of the device's V^T rows (ce_quantize_v_fp8): the order in which the
    S accumulator's registers already are the 8-bit A fragment of the P V wgmma (DESIGN.md, "FP8 attention").
    `stored[..., 32 g + p] = vt[..., 32 g + order[p]]`."""
    p = torch.arange(32)
    return 16 * (p // 16) + 8 * ((p % 4) // 2) + 2 * ((p % 16) // 4) + p % 2


def _cond_entry(entries: list, slots: int, txt_in, img_in, new) -> Tuple[Dict[str, Any], bool]:
    """(entry, hit) of the LRU cache, least recently used first, that the context cache and the TeaCache states share.  A hit needs
    the SAME conditioning tensor objects the entry holds, at the same in-place versions: the unchanged pipeline passes the same
    `prompt_embeds` / `negative_prompt_embeds` / `image_embeds` at every step (pipeline_chronoedit.py:715-735).  A miss appends
    `new(evicted)` plus the key; `evicted` (the LRU entry when all `slots` are taken, else None) is dropped once `new` returned."""
    ver = lambda t: None if t is None else t._version
    for i, e in enumerate(entries):
        if e["txt"] is txt_in and e["img"] is img_in and e["txt_v"] == ver(txt_in) and e["img_v"] == ver(img_in):
            entries.append(entries.pop(i))   # by position, since list.remove would compare the entries' tensors with ==
            return e, True
    full = len(entries) >= slots
    e = dict(new(entries[0] if full else None), txt=txt_in, img=img_in, txt_v=ver(txt_in), img_v=ver(img_in))
    if full:
        del entries[0]
    entries.append(e)
    return e, False


@dataclass
class Transformer2DModelOutput:
    """Same shape as diffusers.models.modeling_outputs.Transformer2DModelOutput."""

    sample: torch.Tensor


class _Config(dict):
    """Attribute + item access, like diffusers' FrozenDict config."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e


class _P(nn.Module):
    """Parameter holder (weight[, bias]) — shapes/names follow the reference module tree; no forward."""

    def __init__(self, weight_shape, bias_shape=None, dtype=torch.bfloat16, device=None):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(weight_shape, dtype=dtype, device=device), requires_grad=False)
        if bias_shape is not None:
            self.bias = nn.Parameter(torch.empty(bias_shape, dtype=dtype, device=device), requires_grad=False)


class _GELU(nn.Module):
    def __init__(self, din, dout, dtype, device):
        super().__init__()
        self.proj = _P((dout, din), (dout,), dtype, device)


class _FeedForward(nn.Module):
    def __init__(self, din, inner, dout, dtype, device):
        super().__init__()
        self.net = nn.ModuleList([_GELU(din, inner, dtype, device), nn.Identity(), _P((dout, inner), (dout,), dtype, device)])


class _Attention(nn.Module):
    def __init__(self, dim, added_kv_proj_dim, dtype, device):
        super().__init__()
        self.norm_q = _P((dim,), None, dtype, device)
        self.norm_k = _P((dim,), None, dtype, device)
        self.to_q = _P((dim, dim), (dim,), dtype, device)
        self.to_k = _P((dim, dim), (dim,), dtype, device)
        self.to_v = _P((dim, dim), (dim,), dtype, device)
        if added_kv_proj_dim is not None:
            self.add_k_proj = _P((dim, added_kv_proj_dim), (dim,), dtype, device)
            self.add_v_proj = _P((dim, added_kv_proj_dim), (dim,), dtype, device)
            self.norm_added_k = _P((dim,), None, dtype, device)
        self.to_out = nn.ModuleList([_P((dim, dim), (dim,), dtype, device), nn.Identity()])


class _Block(nn.Module):
    def __init__(self, dim, ffn_dim, added_kv_proj_dim, dtype, device):
        super().__init__()
        self.attn1 = _Attention(dim, None, dtype, device)
        self.attn2 = _Attention(dim, added_kv_proj_dim, dtype, device)
        self.norm2 = _P((dim,), (dim,), torch.float32, device)
        self.ffn = _FeedForward(dim, ffn_dim, dim, dtype, device)
        self.scale_shift_table = nn.Parameter(torch.empty(1, 6, dim, dtype=torch.float32, device=device), requires_grad=False)


class _TimestepEmbedding(nn.Module):
    def __init__(self, freq_dim, dim, device):
        super().__init__()
        self.linear_1 = _P((dim, freq_dim), (dim,), torch.float32, device)
        self.linear_2 = _P((dim, dim), (dim,), torch.float32, device)


class _TextProjection(nn.Module):
    def __init__(self, din, dim, dtype, device):
        super().__init__()
        self.linear_1 = _P((dim, din), (dim,), dtype, device)
        self.linear_2 = _P((dim, dim), (dim,), dtype, device)


class _ImageEmbedding(nn.Module):
    def __init__(self, din, dout, dtype, device):
        super().__init__()
        self.norm1 = _P((din,), (din,), torch.float32, device)
        self.ff = _FeedForward(din, din, dout, dtype, device)
        self.norm2 = _P((dout,), (dout,), torch.float32, device)


class _ConditionEmbedder(nn.Module):
    def __init__(self, dim, freq_dim, text_dim, image_dim, dtype, device):
        super().__init__()
        self.time_embedder = _TimestepEmbedding(freq_dim, dim, device)
        self.time_proj = _P((6 * dim, dim), (6 * dim,), dtype, device)
        self.text_embedder = _TextProjection(text_dim, dim, dtype, device)
        if image_dim is not None:
            self.image_embedder = _ImageEmbedding(image_dim, dim, dtype, device)


class ChronoEditTransformer3DModel(nn.Module):
    """See module docstring.  Constructor arguments = transformer_chronoedit.py:342-360."""

    config_name = "config.json"

    def __init__(
        self,
        patch_size: Tuple[int, int, int] = (1, 2, 2),
        num_attention_heads: int = 40,
        attention_head_dim: int = 128,
        in_channels: int = 16,
        out_channels: int = 16,
        text_dim: int = 4096,
        freq_dim: int = 256,
        ffn_dim: int = 13824,
        num_layers: int = 40,
        cross_attn_norm: bool = True,
        qk_norm: Optional[str] = "rms_norm_across_heads",
        eps: float = 1e-6,
        image_dim: Optional[int] = None,
        added_kv_proj_dim: Optional[int] = None,
        rope_max_seq_len: int = 1024,
        rope_temporal_skip_len: int = 8,
        *,
        torch_dtype: torch.dtype = torch.bfloat16,
        device: Optional[Union[str, torch.device]] = None,
        cache_context: bool = False,
        use_cuda_graph: bool = False,
    ) -> None:
        super().__init__()
        if torch_dtype != torch.bfloat16:
            raise CEError("chronoedit_b200 computes in bf16 (fp32 for the reference's _keep_in_fp32_modules); "
                          f"torch_dtype={torch_dtype} is not built")
        if tuple(patch_size) != (1, 2, 2) or attention_head_dim != 128:
            raise CEError("only patch_size (1,2,2) and attention_head_dim 128 are built")
        if not cross_attn_norm or qk_norm != "rms_norm_across_heads":
            raise CEError("only cross_attn_norm=True, qk_norm='rms_norm_across_heads' (the ChronoEdit configuration) is built")
        if (image_dim is None) != (added_kv_proj_dim is None):
            raise CEError("image_dim and added_kv_proj_dim must be given together (I2V configuration)")
        out_channels = out_channels or in_channels
        self.config = _Config(
            patch_size=tuple(patch_size), num_attention_heads=num_attention_heads, attention_head_dim=attention_head_dim,
            in_channels=in_channels, out_channels=out_channels, text_dim=text_dim, freq_dim=freq_dim, ffn_dim=ffn_dim,
            num_layers=num_layers, cross_attn_norm=cross_attn_norm, qk_norm=qk_norm, eps=eps, image_dim=image_dim,
            added_kv_proj_dim=added_kv_proj_dim, rope_max_seq_len=rope_max_seq_len,
            rope_temporal_skip_len=rope_temporal_skip_len)
        dim = num_attention_heads * attention_head_dim
        dt = torch_dtype
        self.patch_embedding = _P((dim, in_channels) + tuple(patch_size), (dim,), dt, device)
        self.condition_embedder = _ConditionEmbedder(dim, freq_dim, text_dim, image_dim, dt, device)
        self.blocks = nn.ModuleList([_Block(dim, ffn_dim, added_kv_proj_dim, dt, device) for _ in range(num_layers)])
        self.proj_out = _P((out_channels * math.prod(patch_size), dim), (out_channels * math.prod(patch_size),), dt, device)
        self.scale_shift_table = nn.Parameter(torch.empty(1, 2, dim, dtype=torch.float32, device=device), requires_grad=False)
        self._handle = None
        self._packed = False
        self._pack_keepalive: Dict[str, torch.Tensor] = {}
        self._workspaces: Dict[Tuple, torch.Tensor] = {}
        self.last_block0: Optional[torch.Tensor] = None
        # opt-in hoisting of the step-invariant context (text / image embedders, cross-attention K/V of all blocks): see
        # `ce_dit_forward_ex` in include/chronoedit_b200.h.  Up to `_ctx_slots` (prompt, negative prompt) entries, LRU.
        self.cache_context = bool(cache_context)
        # opt-in CUDA-graph replay of the forward (SURVEY 2.3 X5): the ~590 launches of a forward are captured once per
        # (geometry, context slot) and replayed; inputs are staged into fixed device buffers, the result is returned from one.
        self.use_cuda_graph = bool(use_cuda_graph)
        self._graphs: Dict[Tuple, Dict[str, Any]] = {}
        self._ctx_slots = 2
        self._ctx_cache: list = []   # entries: dict(txt=, img=, txt_v=, img_v=, shape=, buf=)
        self._lora_adapters: Dict[str, Dict[str, torch.Tensor]] = {}
        # run-time LoRA (set_adapters): the active set [(name, weight)] in activation order, the on / off switch, and what the
        # handle holds: key (set, scale, device) of the packed tables, the tables {(layer, target): (A_cat, B_raw, col_scale, B_cat)}
        self._lora_set: list = []
        self._lora_on = True
        self._lora_gen = 0      # bumped whenever a loaded adapter's content may have changed: part of the tables' key
        self._lora_scale = 1.0  # the last attention_kwargs["scale"]: forward_host, which takes none, keeps it
        self._lora_key = None
        self._lora_tables: Dict[Tuple[int, int], Tuple[torch.Tensor, ...]] = {}
        self.last_captures: Dict[int, torch.Tensor] = {}
        self._fp8 = False
        self._fp8_attention = False
        # opt-in TeaCache (enable_teacache): settings, per-conditioning states, the probe's buffers and the per-call records
        self._teacache: Optional[Dict[str, Any]] = None
        self._tc_slots = 2
        self._tc_states: list = []   # entries: dict(txt=, img=, txt_v=, img_v=, slot=, policy=, prev=, spare=, resid=, geom=)
        self._tc_next_slot = 0
        self._tc_probe: Dict[str, Any] = {}
        self._tc_records: list = []
        # the splits over GPUs, set by chronoedit_b200.parallel: the token split, the batch split, the call pair and its open first call
        self._sp_state: Optional[Dict[str, Any]] = None
        self._bp_state: Optional[Dict[str, Any]] = None
        self._cp_state: Optional[Dict[str, Any]] = None
        self._cp_pair: Optional[Dict[str, Any]] = None

    # ------------------------------------------------------------------------------------------ plumbing
    @property
    def dtype(self) -> torch.dtype:
        return torch.bfloat16

    @property
    def device(self) -> torch.device:
        return self.patch_embedding.weight.device

    def _invalidate(self, kind: str) -> None:
        """Drop what a change of `kind` makes stale.
        "results": the weights, the adapters or this rank's share of a call's samples changed, so what was computed from them
            is stale: the context cache's K/V, the TeaCache states (their residuals) and the captured graphs.
        "layout": the launch sequence or its scratch changed: the workspaces and the captured graphs (which hold their addresses).
        "storage": the parameters are new tensors, maybe on another device, so the fused device buffers must be rebuilt (`_packed`)
            and the TeaCache probe's buffers reallocated; drops both of the above."""
        assert kind in ("results", "layout", "storage"), kind
        if kind == "storage":
            self._packed = False
            self._tc_probe = {}
        if kind != "layout":
            self._ctx_cache = []
            self._tc_states = []
        if kind != "results":
            self._workspaces = {}
        self._graphs = {}

    def _apply(self, fn, *a, **k):
        # .to()/.cuda()/.cpu() re-allocate parameters: the fused device buffers must be rebuilt
        self._invalidate("storage")
        if self._lora_key is not None:   # the packed LoRA tables are rebuilt on the new device (or cleared from the handle)
            self._lora_key = ("moved",)
        self._lora_tables = {}
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        if self._fp8:
            raise CEError("load_state_dict after enable_fp8(): the FP8 block weights are quantized from the bf16 ones; load the "
                          "checkpoint (and fuse any LoRA) first, then call enable_fp8()")
        self._invalidate("storage" if assign else "results")
        return super().load_state_dict(state_dict, strict=strict, assign=assign)

    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                _lib.lib().ce_dit_destroy(self._handle)
        except Exception:
            pass

    def _cfg_c(self) -> DiTConfigC:
        c = self.config
        return DiTConfigC(
            c.num_attention_heads, c.attention_head_dim, c.in_channels, c.out_channels, c.text_dim, c.freq_dim, c.ffn_dim,
            c.num_layers, c.image_dim or 0, c.added_kv_proj_dim or 0, c.rope_max_seq_len, c.rope_temporal_skip_len, c.eps,
            *c.patch_size)

    def _ensure_handle(self):
        if self._handle is None:
            h = _lib.c_void_p()
            cfg = self._cfg_c()
            check(_lib.lib().ce_dit_create(_lib.ctypes.byref(cfg), _lib.ctypes.byref(h)))
            check(_lib.lib().ce_dit_set_attention_fp8(h, int(self._fp8_attention)))
            self._handle = h
        return self._handle

    # ------------------------------------------------------------------------------------------ FP8 mode
    @property
    def fp8_enabled(self) -> bool:
        return self._fp8

    @torch.no_grad()
    def enable_fp8(self) -> None:
        """Opt-in FP8 mode (DESIGN.md, "FP8 mode"): the six per-token GEMMs of every block run as e4m3 wgmma with one scale per
        output channel (weights, quantized here by `quantize_fp8_rows`) and one per token (activations, quantized on the device
        before each GEMM).  Each of those layers then holds buffers `weight_fp8` (float8_e4m3fn, [N, K]) and `weight_scale`
        (fp32, [N]) instead of its bf16 `weight`, whose storage is released.  One-way; works on CPU or CUDA, and the buffers
        follow .to() / .cpu().  Call it after loading the checkpoint and fusing any LoRA: both raise afterwards."""
        if self._fp8:
            return
        for blk in self.blocks:
            for name in FP8_LINEARS:
                holder = blk.get_submodule(name)
                q, s = quantize_fp8_rows(holder.weight.data)
                del holder.weight
                holder.register_buffer("weight_fp8", q)
                holder.register_buffer("weight_scale", s)
        self._fp8 = True
        self._pack_keepalive = {}   # the fused bf16 QKV buffers
        self._invalidate("storage")

    @property
    def fp8_attention_enabled(self) -> bool:
        return self._fp8_attention

    def enable_fp8_attention(self, enabled: bool = True) -> None:
        """Opt-in FP8 self-attention (DESIGN.md, "FP8 attention"): every block's self-attention quantizes q and k per (token, head)
        and v per (sample, channel) to e4m3 on the device and runs on e4m3 wgmma.  Cross-attention stays bf16.  Reversible
        (`enable_fp8_attention(False)`), touches no weight, independent of `enable_fp8()`; it survives .to(), load_state_dict
        and fuse_lora.  Toggling drops captured CUDA graphs and workspaces; the context cache stays valid."""
        enabled = bool(enabled)
        if enabled == self._fp8_attention:
            return
        if self._handle is not None:
            check(_lib.lib().ce_dit_set_attention_fp8(self._handle, int(enabled)))
        self._fp8_attention = enabled
        self._invalidate("layout")

    # ------------------------------------------------------------------------------------------ fp32 validation mode
    @torch.no_grad()
    def enable_fp32_validation(self, state_dict_fp32: Dict[str, torch.Tensor]) -> None:
        """Register an fp32 copy of every parameter (reference names, e.g. the reference model's own fp32 state dict) for
        `forward_fp32`.  The bf16 parameters of this module are untouched."""
        dev = self.device
        if dev.type != "cuda":
            raise CEError("fp32 validation mode needs the module on a CUDA (sm_90) device; there is no CPU path")
        L = _lib.lib()
        self._ensure_handle()
        own = {n for n, _ in self.named_parameters()}
        missing = sorted(own - set(state_dict_fp32))
        if missing:
            raise CEError(f"enable_fp32_validation: state dict lacks {len(missing)} parameters, first: {missing[0]}")
        keep = {}
        for n in own:
            t = state_dict_fp32[n].detach().to(device=dev, dtype=torch.float32).contiguous()
            keep[n] = t
            check(L.ce_dit_set_weight_fp32(self._handle, n.encode(), ptr(t), t.numel()))
        self._fp32_keepalive = keep

    @torch.no_grad()
    def forward_fp32(self, hidden_states: torch.Tensor, timestep: torch.Tensor, encoder_hidden_states: torch.Tensor,
                     encoder_hidden_states_image: Optional[torch.Tensor] = None, return_block0: bool = False):
        """VALIDATION mode (include/chronoedit_b200.h, ce_dit_forward_fp32): fp32 in, fp32 weights, fp32 out, every matrix product
        on the wgmma GEMM with split-bf16 operands.  Meets rtol 1e-3 / atol 1e-4 against the reference's fp32 run end to end
        (tests/test_gpu_fp32_mode.py); far slower than forward() and not part of any benchmark."""
        if not getattr(self, "_fp32_keepalive", None):
            raise CEError("call enable_fp32_validation(fp32_state_dict) first")
        self._refuse_cp("forward_fp32")
        if self._lora_active():
            raise CEError("forward_fp32 is not built for run-time LoRA (set_adapters): call disable_lora() first")
        self._check_inputs(hidden_states, timestep, encoder_hidden_states, encoder_hidden_states_image)
        dev = self.device
        B, C, T, H, W = hidden_states.shape
        x, t, txt, img = self._to_device(torch.float32, hidden_states, timestep, encoder_hidden_states, encoder_hidden_states_image)
        L = _lib.lib()
        Lt = txt.shape[1]
        n = L.ce_dit_fp32_workspace_bytes(self._handle, B, T, H, W, Lt)
        if n < 0:
            raise CEError("fp32 validation mode: unsupported geometry")
        ws = torch.empty(n, dtype=torch.uint8, device=dev)
        out = torch.empty(B, self.config.out_channels, T, H, W, dtype=torch.float32, device=dev)
        b0 = None
        if return_block0:
            b0 = torch.empty(B * T * (H // 2) * (W // 2), self.config.num_attention_heads * self.config.attention_head_dim,
                             dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            check(L.ce_dit_forward_fp32(self._handle, ptr(x), ptr(t), ptr(txt), ptr(img), ptr(out), B, T, H, W, Lt, ptr(ws), ws.numel(),
                                        ptr(b0), current_stream()))
        return (out, b0) if return_block0 else out

    @torch.no_grad()
    def pack_weights(self) -> None:
        """Build the fused buffers the kernels read (QKV / KV rows stacked, scale_shift_tables stacked) and register
        every parameter with the C handle.  The reference parameters become VIEWS of the fused buffers, so no memory
        is duplicated and later in-place updates (e.g. a fused LoRA) are seen by the kernels.  Called lazily by
        forward(); call it again after replacing parameter tensors."""
        L = _lib.lib()
        dev = self.device
        if dev.type != "cuda":
            raise CEError("ChronoEditTransformer3DModel must live on a CUDA (sm_90) device; there is no CPU path")
        for n, p in self.named_parameters():
            want = torch.float32 if any(k in n for k in KEEP_FP32) else torch.bfloat16
            if p.dtype != want:
                p.data = p.data.to(want)
        for n, b in self.named_buffers():
            want = torch.float8_e4m3fn if n.endswith(".weight_fp8") else torch.float32
            if b.dtype != want:
                raise CEError(f"FP8 buffer {n} has dtype {b.dtype}, expected {want} (was the module cast with .to(dtype)?)")
        self._ensure_handle()
        keep: Dict[str, torch.Tensor] = {}

        def fuse(prefix, holders, attr):
            parts = [getattr(m, attr) for m in holders]
            fused = torch.cat([p.data for p in parts], dim=0).contiguous()
            off = 0
            for p in parts:
                n0 = p.shape[0]
                p.data = fused[off: off + n0]
                off += n0
            keep[prefix + "." + attr] = fused
            return fused

        def reg(name, t):
            t = t.contiguous() if not t.is_contiguous() else t
            keep[name] = t
            code = {torch.bfloat16: 0, torch.float32: 1, torch.float8_e4m3fn: 2}[t.dtype]
            check(L.ce_dit_set_weight(self._handle, name.encode(), ptr(t), code, t.numel()))

        fused_names = set()
        for i, blk in enumerate(self.blocks):
            p = f"blocks.{i}."
            qkv = [blk.attn1.to_q, blk.attn1.to_k, blk.attn1.to_v]
            if self._fp8:   # e4m3 weight under the bf16 name, scales beside it
                reg(p + "attn1.to_qkv.weight", fuse(p + "attn1.to_qkv", qkv, "weight_fp8"))
                reg(p + "attn1.to_qkv.weight_scale", fuse(p + "attn1.to_qkv", qkv, "weight_scale"))
            for attr in ("weight", "bias"):
                if attr == "bias" or not self._fp8:
                    reg(p + "attn1.to_qkv." + attr, fuse(p + "attn1.to_qkv", qkv, attr))
                reg(p + "attn2.to_kv." + attr, fuse(p + "attn2.to_kv", [blk.attn2.to_k, blk.attn2.to_v], attr))
                if self.config.image_dim is not None:
                    reg(p + "attn2.add_kv_proj." + attr, fuse(p + "attn2.add_kv_proj", [blk.attn2.add_k_proj, blk.attn2.add_v_proj], attr))
            fused_names.update(p + s for s in ("attn1.to_q.", "attn1.to_k.", "attn1.to_v.", "attn2.to_k.", "attn2.to_v.",
                                               "attn2.add_k_proj.", "attn2.add_v_proj."))
        table = torch.cat([blk.scale_shift_table.data for blk in self.blocks], dim=0).contiguous()  # [layers, 6, D]
        for i, blk in enumerate(self.blocks):
            blk.scale_shift_table.data = table[i: i + 1]
        reg("blocks.scale_shift_table", table)
        for n, p in self.named_parameters():
            if any(n.startswith(f) for f in fused_names) or (n.startswith("blocks.") and n.endswith("scale_shift_table")):
                continue
            reg(n, p.data)
        for n, b in self.named_buffers():   # FP8 mode: weight_fp8 / weight_scale of the unfused block GEMMs
            if not any(n.startswith(f) for f in fused_names):
                reg(n[: -len("_fp8")] if n.endswith(".weight_fp8") else n, b)
        check(L.ce_dit_weights_complete(self._handle))
        self._pack_keepalive = keep
        if self._packed:   # a re-pack: what was computed from the replaced tensors is stale (an unpacked model has nothing cached)
            self._invalidate("results")
        self._packed = True

    # ------------------------------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(
        self,
        hidden_states: torch.Tensor,
        timestep: torch.LongTensor,
        encoder_hidden_states: torch.Tensor,
        encoder_hidden_states_image: Optional[torch.Tensor] = None,
        return_dict: bool = True,
        attention_kwargs: Optional[Dict[str, Any]] = None,
        return_block0: bool = False,
        capture_layers: Optional[Tuple[int, ...]] = None,
    ) -> Union[Transformer2DModelOutput, Tuple[torch.Tensor]]:
        # attention_kwargs["scale"] only matters for un-fused PEFT LoRA layers (transformer_chronoedit.py:406-419): it multiplies
        # every active adapter's scaling (PEFT's scale_lora_layers).  With no adapter active at run time the reference warns and
        # ignores it (:416-419), and so does this mirror.
        lora_scale = 1.0 if attention_kwargs is None else float(attention_kwargs.get("scale", 1.0))
        if lora_scale != 1.0 and not self._lora_active():
            import warnings

            warnings.warn("Passing `scale` via `attention_kwargs` when not using the PEFT backend is ineffective "
                          "(LoRA must be fused with fuse_lora(lora_scale=...) before inference).")
        self._refuse_token_split(lora=self._lora_active())
        dev = self.device
        self._check_inputs(hidden_states, timestep, encoder_hidden_states, encoder_hidden_states_image)
        B, C, T, H, W = hidden_states.shape
        if self._teacache is not None:
            if return_block0 or capture_layers:
                raise CEError("return_block0 / capture_layers are not available while TeaCache is on (a skipped step runs no "
                              "blocks): call disable_teacache() first")
            self._refuse_token_split(teacache=True)
        cp = self._cp_state
        role, pair = self._cp_role(hidden_states, timestep, encoder_hidden_states_image, return_block0, capture_layers) if cp else (0, None)
        computes = not cp or role == cp["rank"]
        self._lora_scale = lora_scale
        self._lora_sync(lora_scale)
        x, t, txt, img = self._to_device(torch.bfloat16, hidden_states, timestep, encoder_hidden_states, encoder_hidden_states_image)
        out = torch.empty(B, self.config.out_channels, T, H, W, dtype=torch.bfloat16, device=dev)
        L_tok = T * (H // 2) * (W // 2)
        Dm = self.config.num_attention_heads * self.config.attention_head_dim
        b0 = torch.empty(B * L_tok, Dm, dtype=torch.bfloat16, device=dev) if return_block0 else None
        caps: Dict[int, torch.Tensor] = {}
        if capture_layers:
            caps = {int(l): torch.empty(B * L_tok, Dm, dtype=torch.bfloat16, device=dev) for l in capture_layers}
        # (no graph replay in sequence-parallel or batch-split mode: the peer barrier's epoch is a launch argument and must advance
        # every forward)
        # (no graph replay with TeaCache either: each call chooses between two launch sequences after a device-to-host read)
        # (nor with run-time LoRA: a set change moves the tables the captured launches would read)
        # (a call of a CFG pair that the other rank computes runs no forward and touches no per-conditioning state)
        if not computes:
            pass
        elif self._teacache is not None:
            self._teacache_forward(x, t, txt, img, out, encoder_hidden_states, encoder_hidden_states_image)
        elif (self.use_cuda_graph and not caps and b0 is None and not self._sp_state and not self._bp_state and not cp
              and not self._lora_active()):
            out = self._graphed_forward(x, t, txt, img, encoder_hidden_states, encoder_hidden_states_image)
        else:
            self._native_forward(x, t, txt, img, out, b0, caps, encoder_hidden_states, encoder_hidden_states_image)
        if cp:
            out = self._cp_finish(role, pair, computes, out, hidden_states, timestep, encoder_hidden_states_image)
        self.last_block0 = b0
        self.last_captures = caps
        if not return_dict:
            return (out,)
        return Transformer2DModelOutput(sample=out)

    def _local_samples(self, B: int) -> Tuple[int, int]:
        """(first, count) of the samples of a B-sample call this handle computes: its share under the batch split
        (parallel.enable_cfg_parallel), else all of them.  The workspace, the context cache and the TeaCache buffers are sized by
        `count`.  A batch the ranks do not divide is left whole here, for the forward to refuse."""
        st = self._bp_state
        if not st or B % st["world"]:
            return 0, B
        n = B // st["world"]
        return st["rank"] * n, n

    def _check_inputs(self, hidden_states, timestep, encoder_hidden_states, encoder_hidden_states_image, host: bool = False,
                      out: Optional[torch.Tensor] = None) -> None:
        """Refuse inputs whose extents disagree with the model, from tensor metadata alone.  The C library works out every extent
        from the config and (B, T, H, W, Lt), so it cannot see a tensor that is too small.  With `host` (forward_host, whose C call
        copies the inputs and the sample itself) the tensors must also be on the CPU: the timestep of any dtype, the others
        contiguous bf16, and `out`, when given, of the sample's shape."""
        c = self.config
        if hidden_states.dim() != 5:
            raise CEError("hidden_states must be [B, C, T, H, W]")
        B, C, T, H, W = hidden_states.shape
        if C != c.in_channels:
            raise CEError(f"hidden_states has {C} channels, model expects {c.in_channels}")
        img = encoder_hidden_states_image
        if (img is None) != (c.image_dim is None):
            raise CEError("encoder_hidden_states_image must be passed iff the model was built with image_dim")
        if timestep.numel() not in (1, B):
            raise CEError(f"timestep has {timestep.numel()} elements, expected 1 or B = {B}")
        txt = encoder_hidden_states
        for name, tns, dim in (("encoder_hidden_states", txt, c.text_dim), ("encoder_hidden_states_image", img, c.image_dim)):
            if tns is not None and (tns.dim() != 3 or tns.shape[0] != B or tns.shape[2] != dim):
                raise CEError(f"{name} must be [B, tokens, {dim}] with B = {B}, got {list(tns.shape)}")
        if img is not None and img.shape[1] != 257:
            raise CEError("encoder_hidden_states_image must have 257 tokens (transformer_chronoedit.py:53)")
        if not host:
            return
        if timestep.device.type != "cpu":
            raise CEError(f"forward_host expects a CPU timestep, got one on {timestep.device}")
        for name, tns in (("hidden_states", hidden_states), ("encoder_hidden_states", txt), ("encoder_hidden_states_image", img),
                          ("out", out)):
            if tns is not None and (tns.device.type != "cpu" or tns.dtype != torch.bfloat16 or not tns.is_contiguous()):
                raise CEError(f"forward_host expects contiguous CPU bf16 tensors: {name} is {tns.dtype} on {tns.device}"
                              + ("" if tns.is_contiguous() else ", not contiguous"))
        if out is not None and tuple(out.shape) != (B, c.out_channels, T, H, W):
            raise CEError(f"out must be [B, out_channels, T, H, W] = {[B, c.out_channels, T, H, W]}, got {list(out.shape)}")

    def _to_device(self, dtype, hidden_states, timestep, encoder_hidden_states, encoder_hidden_states_image):
        """The checked inputs as the C forward reads them: contiguous on the module's device in `dtype`, the timestep fp32 [B]."""
        cast = lambda a: None if a is None else a.to(device=self.device, dtype=dtype).contiguous()
        t = timestep.to(device=self.device, dtype=torch.float32).reshape(-1).expand(hidden_states.shape[0]).contiguous()
        return cast(hidden_states), t, cast(encoder_hidden_states), cast(encoder_hidden_states_image)

    def _refuse_token_split(self, lora: bool = False, teacache: bool = False) -> None:
        """Under the token split (parallel.enable_sequence_parallel): refuse run-time LoRA when `lora`, TeaCache when `teacache`."""
        if self._sp_state and lora:
            raise CEError("run-time LoRA (set_adapters) is not built for sequence parallelism: call disable_lora() or disable the "
                          "sequence-parallel mode first")
        if self._sp_state and teacache:
            raise CEError("TeaCache is not built for sequence parallelism: disable one of the two")

    def _refuse_cp(self, who: str) -> None:
        if self._cp_state:
            raise CEError(f"{who} is not available with the call-pair split (parallel.enable_cfg_parallel_calls pairs the calls of "
                          "forward()): call parallel.disable_cfg_parallel_calls first")

    def _cp_role(self, hidden_states, timestep, img_in, return_block0, capture_layers) -> Tuple[int, Optional[Dict[str, Any]]]:
        """Call-pair split (parallel.enable_cfg_parallel_calls): (role of this call, the open pair's record for role 1).  Role 0 is
        the first call of a pair (the prompt, computed by rank 0), role 1 the second (the negative prompt, computed by rank 1).  Every
        refusal comes before any launch.  A second call that does not pair with the first (by object identity and in-place version,
        so no host sync) drops the pair and raises: every rank sees the same calls, so every rank raises at the same call and no rank
        waits at the exchange's barrier."""
        if return_block0 or capture_layers:
            raise CEError("return_block0 / capture_layers are not available with the call-pair split (each rank computes one call "
                          "of a pair): call parallel.disable_cfg_parallel_calls first")
        if self.device.type == "cuda" and torch.cuda.is_current_stream_capturing():
            raise CEError("call-pair split: the stream is capturing (the exchange's barrier epoch advances every pair, so it cannot "
                          "be replayed from a graph)")
        pair = self._cp_pair
        if pair is None:
            return 0, None
        self._cp_pair = None
        same = (hidden_states is pair["x"] and hidden_states._version == pair["x_v"] and tuple(hidden_states.shape) == pair["x_shape"]
                and timestep is pair["t"] and timestep._version == pair["t_v"] and tuple(timestep.shape) == pair["t_shape"]
                and img_in is pair["img"])
        if not same:
            raise CEError("call-pair split: this call does not pair with the previous one.  The second call of a CFG pair must pass "
                          "the same hidden_states and timestep tensors, unchanged, and the same encoder_hidden_states_image as the "
                          "first: the mode needs classifier-free guidance (guidance_scale > 1, two transformer calls per step).  The "
                          "open pair is dropped; the next call starts a new one")
        return 1, pair

    def _cp_finish(self, role, pair, computes, out, hidden_states, timestep, img_in) -> torch.Tensor:
        """Call-pair split, after this rank's forward (when it computes this call).  Role 0: rank 1 fills its sample with bf16 NaN
        (0xFFFF) on the stream, and the pair is opened holding the sample.  Role 1: ce_dit_cp_exchange swaps the two samples, so
        rank 1's role-0 sample, still held by the caller, receives the prompt call's result in place, and rank 0 returns the
        negative-prompt call's.  Everything is stream-ordered: the guidance combine that follows on the current stream sees both."""
        if role == 0:
            if not computes:
                out.view(torch.int16).fill_(-1)
            self._cp_pair = dict(x=hidden_states, x_v=hidden_states._version, x_shape=tuple(hidden_states.shape), t=timestep,
                                 t_v=timestep._version, t_shape=tuple(timestep.shape), img=img_in, out0=out)
            return out
        out0 = pair["out0"]
        self._native_cp_exchange(*((out, out0) if computes else (out0, out)))
        return out

    def _native_cp_exchange(self, own, other) -> None:
        """ce_dit_cp_exchange on the current stream: `own` into the peer's slot, one barrier, the peer's sample into `other`."""
        B, _, T, H, W = own.shape
        with torch.cuda.device(self.device):
            check(_lib.lib().ce_dit_cp_exchange(self._ensure_handle(), ptr(own), ptr(other), B, T, H, W, current_stream()))

    def _ensure_packed(self) -> None:
        if not self._packed:
            self.pack_weights()

    @contextlib.contextmanager
    def _pre_launch(self, shape, Lt: int, cond=None):
        """Around every native forward's C call: packs the weights if needed and yields this rank's workspace for a forward of
        `shape` (B, C, T, H, W) with Lt text tokens and the context-cache slot (buffer, reuse flag) of `cond` = (txt_in, img_in, txt,
        img), (None, 0) without.  A slot the call was to fill is dropped if the body raises: it is unfilled or only partly filled."""
        self._ensure_packed()
        B, _, T, H, W = shape
        key = (self._local_samples(B)[1], T, H, W, Lt, str(self.device))
        ws = self._workspaces.get(key)
        if ws is None:
            n = _lib.lib().ce_dit_workspace_bytes(self._handle, *key[:5])
            if n < 0:
                check(-1)
            # one live geometry at a time keeps the footprint bounded; graphs captured on the old workspace go with it
            self._invalidate("layout")
            ws = self._workspaces[key] = torch.empty(n, dtype=torch.uint8, device=self.device)
        ctx_buf, ctx_reuse = self._context_slot(*cond) if cond is not None and self.cache_context else (None, 0)
        try:
            yield ws, ctx_buf, ctx_reuse
        except BaseException:
            self._drop_unfilled(ctx_buf, ctx_reuse)
            raise

    def _forward_ex(self, x, t, txt, img, out, b0, ws, ctx_buf, ctx_reuse) -> None:
        """ce_dit_forward_ex on the current stream, the one call of it the eager forward and the graph capture share."""
        B, _, T, H, W = x.shape
        with torch.cuda.device(self.device):
            self._check_forward(_lib.lib().ce_dit_forward_ex(
                self._handle, ptr(x), ptr(t), ptr(txt), ptr(img), ptr(out), B, T, H, W, txt.shape[1], ptr(ws), ws.numel(), ptr(b0),
                ptr(ctx_buf), ctx_buf.numel() if ctx_buf is not None else 0, ctx_reuse, current_stream()), ctx_buf, ctx_reuse)

    def _native_forward(self, x, t, txt, img, out, b0, caps, txt_in, img_in) -> None:
        """The one place the DiT forward reaches the C ABI (ce_dit_forward_ex).  x [B,C,T,H,W] bf16, t [B] fp32, txt / img bf16,
        all contiguous on the module's device; `out` (and the optional block captures) are written in place."""
        L = _lib.lib()
        with self._pre_launch(x.shape, txt.shape[1], (txt_in, img_in, txt, img)) as (ws, ctx_buf, ctx_reuse):
            if caps:
                lay = (_lib.c_int32 * len(caps))(*caps.keys())
                dst = (_lib.c_void_p * len(caps))(*[v.data_ptr() for v in caps.values()])
                check(L.ce_dit_set_capture(self._handle, lay, dst, len(caps)))
            try:
                self._forward_ex(x, t, txt, img, out, b0, ws, ctx_buf, ctx_reuse)
            finally:
                if caps:
                    check(L.ce_dit_set_capture(self._handle, None, None, 0))

    def _graphed_forward(self, x, t, txt, img, txt_in, img_in) -> torch.Tensor:
        """Replay (or, the second time a configuration is seen, capture) the forward as one CUDA graph.  A configuration = geometry +
        the context-cache slot in use (its buffer address is baked into the captured launches).  The first call of a configuration
        runs eagerly: it packs weights, builds RoPE tables, opts kernels into their shared-memory sizes and fills the context cache
        -- none of which may happen during capture.  Inputs are copied into fixed staging tensors; the returned sample is a fresh
        tensor (a copy out of the graph's fixed output buffer)."""
        with self._pre_launch(x.shape, txt.shape[1], (txt_in, img_in, txt, img)) as (ws, ctx_buf, ctx_reuse):
            key = (tuple(x.shape), tuple(txt.shape), None if img is None else tuple(img.shape),
                   None if ctx_buf is None else ctx_buf.data_ptr())
            B, _, T, H, W = x.shape
            g = self._graphs.get(key)
            if g is None or (self.cache_context and not ctx_reuse):
                # eager: first sight of this configuration, or the context has to be (re)computed into the slot
                out = torch.empty(B, self.config.out_channels, T, H, W, dtype=torch.bfloat16, device=self.device)
                self._forward_ex(x, t, txt, img, out, None, ws, ctx_buf, ctx_reuse)
                if g is None:
                    self._graphs[key] = {"graph": None}
                return out
            if g["graph"] is None:   # second sight: capture (with ctx_reuse = 1 when the context cache is on)
                st = {"x": x.clone(), "t": t.clone(), "txt": txt.clone(), "img": None if img is None else img.clone(),
                      "out": torch.empty(B, self.config.out_channels, T, H, W, dtype=torch.bfloat16, device=self.device)}
                torch.cuda.synchronize(self.device)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    self._forward_ex(st["x"], st["t"], st["txt"], st["img"], st["out"], None, ws, ctx_buf, ctx_reuse)
                g.update(st)
                g["graph"] = graph
            g["x"].copy_(x)
            g["t"].copy_(t)
            if not self.cache_context:   # with the context cache the captured launches do not read the encoder states at all
                g["txt"].copy_(txt)
                if img is not None:
                    g["img"].copy_(img)
            g["graph"].replay()
            return g["out"].clone()

    def _context_slot(self, txt_in, img_in, txt, img):
        """(cache buffer, reuse flag) for these encoder states: an entry of the conditioning-keyed LRU (`_cond_entry`).  A new entry
        takes over the evicted one's buffer when it is large enough."""
        def new(old):
            n = _lib.lib().ce_dit_context_cache_bytes(self._handle, self._local_samples(txt.shape[0])[1], txt.shape[1])
            if n < 0:
                check(-1)
            if old is not None and old["buf"].numel() >= n and old["buf"].device == self.device:
                return dict(buf=old["buf"])
            return dict(buf=torch.empty(n, dtype=torch.uint8, device=self.device))

        e, hit = _cond_entry(self._ctx_cache, self._ctx_slots, txt_in, img_in, new)
        return e["buf"], int(hit)

    def _check_forward(self, rc, ctx_buf, ctx_reuse) -> None:
        """check(rc) of a forward call: a failed call drops the context-cache slot it was to fill (it may have stopped part way)."""
        if rc != 0:
            self._drop_unfilled(ctx_buf, ctx_reuse)
        check(rc)

    def _drop_unfilled(self, ctx_buf, ctx_reuse) -> None:
        if ctx_buf is not None and not ctx_reuse:
            self._ctx_cache = [e for e in self._ctx_cache if e["buf"] is not ctx_buf]

    def clear_context_cache(self) -> None:
        self._ctx_cache = []

    # ------------------------------------------------------------------------------------------ TeaCache
    def enable_teacache(self, tea_cache_l1_thresh: float, num_inference_steps: int,
                        tea_cache_model_id: str = _tc.DEFAULT_MODEL_ID) -> None:
        """Opt-in TeaCache (DESIGN.md, "TeaCache"), the reference DiffSynth pipeline's `tea_cache_l1_thresh` /
        `tea_cache_model_id`: on a step whose timestep modulation moved little since the last computed step, skip every block
        and add the residual the blocks produced then.  One state per conditioning (the same encoder_hidden_states /
        encoder_hidden_states_image objects at the same version), so the pipeline's cond and uncond calls are kept apart.
        `num_inference_steps` must be the schedule's length: the first and last step of it always compute.  Drops earlier
        states.  Not available with sequence parallelism, return_block0 or capture_layers; CUDA-graph replay is not used."""
        _tc.coefficients(tea_cache_model_id)   # raises on an unknown id, listing the supported ones
        if int(num_inference_steps) < 1:
            raise ValueError("num_inference_steps must be >= 1")
        self._refuse_token_split(teacache=True)
        self._teacache = dict(thresh=float(tea_cache_l1_thresh), steps=int(num_inference_steps), model_id=tea_cache_model_id)
        self.reset_teacache()

    def disable_teacache(self) -> None:
        """Back to the plain forward.  The call records stay readable until the next enable_teacache / reset_teacache."""
        self._teacache = None
        self._tc_states = []

    def reset_teacache(self) -> None:
        """Forget every conditioning's state and the call records: the next call of each conditioning is step 0."""
        self._tc_states = []
        self._tc_records = []
        self._tc_next_slot = 0

    @property
    def teacache_enabled(self) -> bool:
        return self._teacache is not None

    @property
    def teacache_records(self) -> Tuple["_tc.Record", ...]:
        """One record per forward since enable_teacache / reset_teacache: (slot, step, rel, acc, computed)."""
        return tuple(self._tc_records)

    def _teacache_state(self, txt_in, img_in) -> Dict[str, Any]:
        """The state of this conditioning: an entry of the conditioning-keyed LRU (`_cond_entry`) of up to `_tc_slots` states.  A
        new state starts at step 0."""
        def new(_):
            c = self._teacache
            self._tc_next_slot += 1
            return dict(slot=self._tc_next_slot - 1, policy=_tc.TeaCacheState(c["steps"], c["thresh"], c["model_id"]), prev=None,
                        spare=None, resid=None, geom=None)

        return _cond_entry(self._tc_states, self._tc_slots, txt_in, img_in, new)[0]

    def _teacache_forward(self, x, t, txt, img, out, txt_in, img_in) -> None:
        """One TeaCache call: the probe (time path, and the two sums against the previous call's modulation when the rule
        evaluates rel), one 8-byte device-to-host read, the rule, then either the forward with the residual recorded or the
        forward without blocks.  A call whose geometry differs from the stored residual's computes (see DESIGN.md).  Under the batch
        split the rule sees only this rank's samples: the probe takes their timesteps, and the modulation and the residual are theirs."""
        B, _, T, H, W = x.shape
        D = self.config.num_attention_heads * self.config.attention_head_dim
        bp = self._bp_state
        if bp and B % bp["world"]:   # before the probe's launches; the forward itself would refuse it too
            raise CEError(f"batch split: a batch of {B} does not divide over {bp['world']} ranks.  Only a call that carries the whole CFG "
                          "pair is split: the unchanged diffusers pipeline's batch-1 calls are not split.  Run the pair as one batch-2 call")
        s0, B = self._local_samples(B)
        st = self._teacache_state(txt_in, img_in)
        pol: _tc.TeaCacheState = st["policy"]
        if st["spare"] is None or st["spare"].numel() != B * 6 * D:
            st["spare"] = torch.empty(B * 6 * D, dtype=torch.bfloat16, device=self.device)
        cur = st["spare"]
        prev = st["prev"] if st["prev"] is not None and st["prev"].numel() == cur.numel() else None
        sums = self._native_probe(t[s0: s0 + B], prev if pol.needs_rel() else None, cur)
        rel = None if sums is None else _tc.rel_from_sums(sums[0], sums[1], B * 6 * D)
        st["prev"], st["spare"] = cur, st["prev"]   # prev = t_mod on every call, skipped or not
        geom = (x.shape[0], s0, B, T, H, W)   # the rank's share too: a residual of other samples is not reused
        step, computed = pol.decide(rel, force_compute=st["geom"] != geom)
        if computed:
            if st["geom"] != geom:
                st["resid"] = torch.empty(B * (T * (H // 2) * (W // 2)) * D, dtype=torch.bfloat16, device=self.device)
                st["geom"] = None
            self._native_teacache_forward(x, t, txt, img, out, txt_in, img_in, st["resid"], True)
            st["geom"] = geom
        else:
            self._native_teacache_forward(x, t, txt, img, out, txt_in, img_in, st["resid"], False)
        self._tc_records.append(_tc.Record(st["slot"], step, rel, pol.acc, computed))

    def _native_probe(self, t, prev, cur):
        """ce_dit_teacache_probe: the timestep modulation of t into `cur` ([B * 6D] bf16); with `prev` also the two sums, read
        back through pinned memory (the only device-to-host read of a TeaCache call).  Returns (sum |cur - prev|, sum |prev|)
        or None."""
        self._ensure_packed()
        L = _lib.lib()
        B = t.numel()
        pr = self._tc_probe
        if pr.get("batch") != B:
            n = L.ce_dit_teacache_probe_bytes(self._handle, B)
            if n < 0:
                check(-1)
            pr.update(batch=B, ws=torch.empty(n, dtype=torch.uint8, device=self.device),
                      sums=torch.empty(64, dtype=torch.float32, device=self.device))
            if "host" not in pr:
                pr["host"] = torch.empty(2, dtype=torch.float32).pin_memory()
                pr["event"] = torch.cuda.Event()
        with torch.cuda.device(self.device):
            check(L.ce_dit_teacache_probe(self._handle, ptr(t), B, ptr(prev), ptr(cur), ptr(pr["sums"] if prev is not None else None),
                                          ptr(pr["ws"]), pr["ws"].numel(), current_stream()))
            if prev is None:
                return None
            pr["host"].copy_(pr["sums"][:2], non_blocking=True)
            pr["event"].record()
        pr["event"].synchronize()
        s0, s1 = pr["host"].tolist()
        return s0, s1

    def _native_teacache_forward(self, x, t, txt, img, out, txt_in, img_in, resid, record: bool) -> None:
        """record: the full forward (ce_dit_forward_ex, context cache as configured) leaving bf16(x_after_blocks -
        x_before_blocks) in `resid`.  Otherwise ce_dit_forward_cached: x_before_blocks + resid, then the output head."""
        L = _lib.lib()
        if record:
            check(L.ce_dit_set_residual_record(self._handle, ptr(resid), resid.numel() * 2))
            try:
                self._native_forward(x, t, txt, img, out, None, {}, txt_in, img_in)
            finally:
                check(L.ce_dit_set_residual_record(self._handle, None, 0))
            return
        B, _, T, H, W = x.shape
        Lt = txt.shape[1]
        with self._pre_launch(x.shape, Lt) as (ws, _, _), torch.cuda.device(self.device):
            check(L.ce_dit_forward_cached(self._handle, ptr(x), ptr(t), ptr(resid), resid.numel() * 2, ptr(out), B, T, H, W, Lt,
                                          ptr(ws), ws.numel(), current_stream()))

    @torch.no_grad()
    def forward_host(self, hidden_states: torch.Tensor, timestep: torch.Tensor, encoder_hidden_states: torch.Tensor,
                     encoder_hidden_states_image: Optional[torch.Tensor], out: Optional[torch.Tensor] = None,
                     return_device_sample: bool = False):
        """End-to-end variant: all tensors are (pinned) HOST bf16/fp32 tensors; H2D, forward and D2H happen inside the
        C-ABI call (ce_dit_forward_host_ex).  Returns the host sample tensor (and, with `return_device_sample`, a view of the same
        sample still on the device -- valid until the next forward_host call -- for the scheduler step)."""
        self._refuse_cp("forward_host")
        self._refuse_token_split(lora=self._lora_active())
        self._check_inputs(hidden_states, timestep, encoder_hidden_states, encoder_hidden_states_image, host=True, out=out)
        self._lora_sync(self._lora_scale)   # no attention_kwargs here: the scale of the last forward() call
        B, C, T, H, W = hidden_states.shape
        Lt = encoder_hidden_states.shape[1]
        t = timestep.to(torch.float32).reshape(-1).expand(B).contiguous()   # the C call copies B timesteps
        L = _lib.lib()
        cond = (encoder_hidden_states, encoder_hidden_states_image, encoder_hidden_states, encoder_hidden_states_image)
        with self._pre_launch(hidden_states.shape, Lt, cond) as (ws, ctx_buf, ctx_reuse):
            n = L.ce_dit_host_staging_bytes(self._handle, B, T, H, W, Lt)
            st = self._workspaces.get("staging")
            if st is None or st.numel() < n:
                st = torch.empty(n, dtype=torch.uint8, device=self.device)
                self._workspaces["staging"] = st
            if out is None:
                out = torch.empty(B, self.config.out_channels, T, H, W, dtype=torch.bfloat16).pin_memory()
            with torch.cuda.device(self.device):
                self._check_forward(L.ce_dit_forward_host_ex(
                    self._handle, ptr(hidden_states), ptr(t), ptr(encoder_hidden_states), ptr(encoder_hidden_states_image), ptr(out),
                    B, T, H, W, Lt, ptr(st), st.numel(), ptr(ws), ws.numel(), ptr(ctx_buf),
                    ctx_buf.numel() if ctx_buf is not None else 0, ctx_reuse, current_stream()), ctx_buf, ctx_reuse)
        if not return_device_sample:
            return out
        off = L.ce_dit_host_staging_sample_offset(self._handle, B, T, H, W, Lt)
        dev_sample = st[off: off + out.numel() * 2].view(torch.bfloat16).view(out.shape)
        return out, dev_sample

    def launches_per_forward(self) -> int:
        return int(_lib.lib().ce_dit_last_launch_count(self._handle)) if self._handle else 0

    # ------------------------------------------------------------------------------------------ LoRA
    # (original Wan module name -> diffusers name): the pairs of the reference's own converters -- per-block modules
    # chronoedit/_src/models/utils.py:112-212, non-block modules :214-290; the diffusers-side names are those of
    # chronoedit_diffsynth/wan_video_dit_chronoedit.py:439-496 read right to left.
    _WAN_TO_DIFFUSERS = (("self_attn.q", "attn1.to_q"), ("self_attn.k", "attn1.to_k"), ("self_attn.v", "attn1.to_v"),
                         ("self_attn.o", "attn1.to_out.0"), ("cross_attn.q", "attn2.to_q"), ("cross_attn.k_img", "attn2.add_k_proj"),
                         ("cross_attn.v_img", "attn2.add_v_proj"), ("cross_attn.k", "attn2.to_k"), ("cross_attn.v", "attn2.to_v"),
                         ("cross_attn.o", "attn2.to_out.0"), ("ffn.0", "ffn.net.0.proj"), ("ffn.2", "ffn.net.2"))
    _WAN_TO_DIFFUSERS_GLOBAL = {
        "time_embedding.0": "condition_embedder.time_embedder.linear_1", "time_embedding.2": "condition_embedder.time_embedder.linear_2",
        "text_embedding.0": "condition_embedder.text_embedder.linear_1", "text_embedding.2": "condition_embedder.text_embedder.linear_2",
        "time_projection.1": "condition_embedder.time_proj", "head.head": "proj_out",
        "img_emb.proj.1": "condition_embedder.image_embedder.ff.net.0.proj", "img_emb.proj.3": "condition_embedder.image_embedder.ff.net.2",
    }

    def _parse_lora(self, lora_state_dict: Dict[str, torch.Tensor], adapter_name: Optional[str]):
        """Pass 1 of fuse_lora: key grammar, name mapping, presence of both factors, shapes.  Nothing is modified here, so a bad
        file leaves the model untouched.  Returns [(parameter, A, B, alpha or None, module name)]; for a block weight that
        enable_fp8() replaced, the parameter is its `weight_fp8` buffer (run-time LoRA reads its shape only)."""
        params = dict(self.named_parameters())
        params.update({n[: -len("_fp8")]: b for n, b in self.named_buffers() if n.endswith(".weight_fp8")})
        pairs: Dict[str, Dict[str, torch.Tensor]] = {}
        for key, val in lora_state_dict.items():
            k = key
            for pre in ("transformer.", "diffusion_model."):
                if k.startswith(pre):
                    k = k[len(pre):]
            if k.endswith((".diff", ".diff_b")) or ".lora_B." in k and k.endswith(".bias"):
                raise CEError(f"fuse_lora: '{key}' is a weight/bias delta, not a low-rank pair; not supported")
            k = k.replace(".lora_down.", ".lora_A.").replace(".lora_up.", ".lora_B.")
            kind = None
            for tag, nm in ((".lora_A.", "A"), (".lora_B.", "B")):
                if tag in k and k.endswith(".weight"):
                    mod, rest = k.split(tag, 1)
                    seg = rest[: -len("weight")].strip(".")       # "" or the PEFT adapter segment ("default", ...)
                    if seg and adapter_name is not None and seg != adapter_name:
                        kind = "skip"   # another adapter's weights
                    elif "." in seg:
                        raise CEError(f"fuse_lora: unrecognised key '{key}'")
                    else:
                        kind = nm
                    break
            if kind is None and k.endswith(".alpha"):
                mod, kind = k[: -len(".alpha")], "alpha"
            if kind is None:
                raise CEError(f"fuse_lora: unrecognised key '{key}'")
            if kind == "skip":
                continue
            if mod in self._WAN_TO_DIFFUSERS_GLOBAL:
                mod = self._WAN_TO_DIFFUSERS_GLOBAL[mod]
            else:
                for wan, dif in self._WAN_TO_DIFFUSERS:
                    if mod.endswith("." + wan):
                        mod = mod[: -len(wan)] + dif
                        break
            if kind in pairs.setdefault(mod, {}):
                raise CEError(f"fuse_lora: '{mod}' has more than one {kind} entry (several adapters in one file? pass adapter_name)")
            pairs[mod][kind] = val
        plan = []
        for mod, d in pairs.items():
            if "A" not in d or "B" not in d:
                raise CEError(f"fuse_lora: '{mod}' needs both lora_A and lora_B")
            w = params.get(mod + ".weight")
            if w is None:
                raise CEError(f"fuse_lora: no parameter '{mod}.weight' in this model")
            A, B = d["A"], d["B"]
            r = A.shape[0]
            if A.dim() != 2 or B.dim() != 2 or A.shape != (r, w.shape[1]) or B.shape != (w.shape[0], r):
                raise CEError(f"fuse_lora: shapes of '{mod}' do not match: A {tuple(A.shape)} B {tuple(B.shape)} W {tuple(w.shape)}")
            plan.append((w, A, B, float(d["alpha"]) if "alpha" in d else None, mod))
        return plan

    def load_lora_adapter(self, state_dict: Dict[str, torch.Tensor], prefix: Optional[str] = "transformer", network_alphas=None,
                          adapter_name: Optional[str] = None, **unused) -> None:
        """diffusers `PeftAdapterMixin.load_lora_adapter` as `WanLoraLoaderMixin.load_lora_weights` calls it
        (run_inference_diffusers.py:371): keep the adapter's factors (validated now) until `fuse_lora` merges them."""
        if prefix:
            sub = {k[len(prefix) + 1:]: v for k, v in state_dict.items() if k.startswith(prefix + ".")}
            state_dict = sub or {k: v for k, v in state_dict.items() if not k.startswith(("text_encoder.", "vae."))}
        name = adapter_name or f"default_{len(self._lora_adapters)}"
        self._parse_lora(state_dict, None)   # fail now, not at fuse time
        self._lora_adapters[name] = dict(state_dict)
        self._lora_gen += 1   # the name may be in the active set with other content: the packed tables are stale

    def unload_lora(self) -> None:
        self._lora_adapters.clear()
        self._lora_gen += 1
        if self._lora_set:
            self._lora_set = []
            self._invalidate("results")

    @torch.no_grad()
    def fuse_lora(self, *args, **kwargs) -> int:
        """`pipe.load_lora_weights(path); pipe.fuse_lora(lora_scale=s)` (run_inference_diffusers.py:369-376) for this module:
        W += (B @ A) * (s * alpha / r), in place and in the weight dtype, which is PEFT's merge arithmetic.  The kernels see
        the result without repacking because the fused QKV buffers are views of the same storage.

        Two call styles: diffusers' `fuse_lora(lora_scale, safe_fusing=False, adapter_names=None)` merges the adapters handed over
        by `load_lora_adapter`; `fuse_lora(state_dict, lora_scale=s)` merges a state dict directly.  Keys: diffusers / PEFT style
        `[transformer.]blocks.N.attn1.to_q.lora_A[.adapter].weight` (+ `lora_B`, optional `.alpha`), or the original Wan style the
        in-tree loader converts (`[diffusion_model.]blocks.N.self_attn.q.lora_down|lora_A.weight`, `lora_up|lora_B`, `.alpha`, and
        the non-block modules time_embedding / text_embedding / time_projection / head.head / img_emb.proj;
        chronoedit/_src/models/utils.py:66-290, wan_t2v_model.py:385-391).  `diff` / `diff_b` entries (norm / bias deltas the
        reference converter drops or treats as lora_bias) are rejected.  Everything is validated BEFORE the first weight is
        touched.  One-time weight preparation with torch matmuls; not on the per-step path.  Returns the number of weights updated."""
        if self._fp8:
            raise CEError("fuse_lora after enable_fp8(): fuse the LoRA into the bf16 weights first, then call enable_fp8()")
        if self._lora_active():
            raise CEError("fuse_lora while adapters are active at run time (set_adapters): merging a run-time set into the weights "
                          "is not built; call disable_lora() or delete_adapters(...) first")
        lora_state_dict = kwargs.pop("lora_state_dict", None)
        if args and isinstance(args[0], dict):        # fuse_lora(state_dict[, lora_scale])
            lora_state_dict, args = args[0], args[1:]
        lora_scale = kwargs.pop("lora_scale", args[0] if len(args) > 0 else 1.0)
        safe_fusing = bool(kwargs.pop("safe_fusing", args[1] if len(args) > 1 else False))
        adapter_names = kwargs.pop("adapter_names", args[2] if len(args) > 2 else None)
        adapter_name = kwargs.pop("adapter_name", None)
        if kwargs:
            raise TypeError(f"fuse_lora: unexpected arguments {sorted(kwargs)}")
        if lora_state_dict is not None:
            plans = [self._parse_lora(lora_state_dict, adapter_name)]
        else:
            names = list(self._lora_adapters) if adapter_names is None else list(adapter_names)
            missing = [n for n in names if n not in self._lora_adapters]
            if missing or not names:
                raise CEError(f"fuse_lora: no loaded adapter named {missing or '(none loaded)'}")
            plans = [self._parse_lora(self._lora_adapters[n], None) for n in names]
        n = 0
        deltas = []
        for plan in plans:
            for w, A, B, alpha, _ in plan:
                A, B = A.to(w.device, w.dtype), B.to(w.device, w.dtype)
                r = A.shape[0]
                delta = (B @ A) * (float(lora_scale) * (alpha if alpha is not None else float(r)) / r)   # peft get_delta_weight
                if safe_fusing and not torch.isfinite(delta).all():
                    raise CEError("fuse_lora(safe_fusing=True): non-finite values in the LoRA delta; nothing was fused")
                deltas.append((w, delta))
        for w, delta in deltas:
            w.data += delta
            n += 1
        if lora_state_dict is None:
            self._lora_adapters.clear()   # merged: a second fuse_lora must not add them again
            self._lora_set = []           # and a (switched-off) run-time set of them is gone with them
            self._lora_gen += 1
        self._invalidate("results")
        return n

    # ------------------------------------------------------------------------------------------ run-time LoRA
    # diffusers' PEFT names (PeftAdapterMixin), so pipe.set_adapters(...) reaches this module unchanged.  DESIGN.md, "Run-time LoRA".
    def set_adapters(self, adapter_names, weights=None) -> None:
        """Run the adapters `adapter_names` (loaded with load_lora_adapter) beside the block GEMMs, without touching the weights:
        each linear layer an adapter covers computes base + bf16(bf16(x A^T) B^T) * weight * alpha / r, summed over the set.
        `weights` is one number for all or one per adapter (default 1; None in a list means 1, as in diffusers).  Everything is validated before anything changes: an
        unknown name, and an adapter on a module other than a block linear layer (LORA_TARGETS; merge those with fuse_lora), are
        refused.  The factors are packed once, on the module's device, in bf16.  Works with FP8 weights and FP8 attention, the
        context cache, TeaCache, the batch and call-pair splits and forward_host; not with sequence parallelism or forward_fp32.
        A new set drops the context cache, the TeaCache states and captured CUDA graphs; graphs are not replayed while a set is
        active.  An empty list clears the set."""
        names = [adapter_names] if isinstance(adapter_names, str) else list(adapter_names)
        if weights is None:
            ws = [1.0] * len(names)
        elif isinstance(weights, (int, float)):
            ws = [float(weights)] * len(names)
        else:
            ws = list(weights)
            if len(ws) != len(names):
                raise ValueError(f"set_adapters: {len(names)} adapters but {len(ws)} weights")
            if not all(w is None or isinstance(w, (int, float)) for w in ws):
                raise CEError("set_adapters: per-block weight dicts are not built; pass one number (or None for 1) per adapter")
            ws = [1.0 if w is None else float(w) for w in ws]
        missing = [n for n in names if n not in self._lora_adapters]
        if missing:
            raise CEError(f"set_adapters: no loaded adapter named {missing}; loaded: {sorted(self._lora_adapters)}")
        if len(set(names)) != len(names):
            raise CEError(f"set_adapters: an adapter is named twice in {names}")
        for n in names:
            self._lora_entries(n)
        self._refuse_token_split(lora=bool(names))
        self._lora_set = list(zip(names, ws))
        self._lora_on = True
        self._invalidate("results")
        if self.device.type == "cuda":
            self._lora_sync(self._lora_scale)

    def disable_lora(self) -> None:
        """Switch the active set off (the forward is the plain one again); enable_lora() switches it back on."""
        self._lora_on = False
        self._invalidate("results")

    def enable_lora(self) -> None:
        self._lora_on = True
        self._invalidate("results")

    def delete_adapters(self, adapter_names) -> None:
        """Drop loaded adapters, and take them out of the active set."""
        names = [adapter_names] if isinstance(adapter_names, str) else list(adapter_names)
        missing = [n for n in names if n not in self._lora_adapters]
        if missing:
            raise CEError(f"delete_adapters: no loaded adapter named {missing}")
        for n in names:
            del self._lora_adapters[n]
        self._lora_gen += 1
        kept = [(n, w) for n, w in self._lora_set if n not in names]
        if kept != self._lora_set:
            self._lora_set = kept
            self._invalidate("results")

    def active_adapters(self) -> list:
        """The names of the set chosen with set_adapters, in activation order (also while disable_lora() has it off)."""
        return [n for n, _ in self._lora_set]

    def _lora_active(self) -> bool:
        return self._lora_on and bool(self._lora_set)

    def _lora_entries(self, name):
        """[(layer, target, part, A, B, alpha or None)] of a loaded adapter; refuses a module that is not a block linear layer."""
        out = []
        for _, A, B, alpha, mod in self._parse_lora(self._lora_adapters[name], None):
            head, _, sub = mod.partition(".")
            layer, _, sub = sub.partition(".")
            if head != "blocks" or not layer.isdigit() or sub not in LORA_TARGETS:
                raise CEError(f"set_adapters: adapter '{name}' has a LoRA on '{mod}', which is not a block linear layer.  Run-time "
                              f"LoRA covers {', '.join(LORA_TARGETS)} of every block; merge an adapter on other modules into the "
                              "weights with fuse_lora instead")
            target, part, _ = LORA_TARGETS[sub]
            out.append((int(layer), target, part, A, B, alpha))
        return out

    @torch.no_grad()
    def _lora_pack(self) -> Dict[Tuple[int, int], Tuple[torch.Tensor, ...]]:
        """The active set as ce_dit_set_lora tables, on the module's device: per (layer, target) A_cat [R, K] (every adapter's
        lora_A stacked in activation order, R padded to 8 with zero rows), B_raw [N, R] (lora_B at its part's rows, zeros
        elsewhere) and col_scale [R] fp32 (weight * alpha / r of the column's adapter)."""
        groups: Dict[Tuple[int, int], list] = {}
        for name, weight in self._lora_set:
            for layer, target, part, A, B, alpha in self._lora_entries(name):
                r = A.shape[0]
                groups.setdefault((layer, target), []).append((part, A, B, weight * (alpha / r if alpha is not None else 1.0)))
        parts_of = {t: p for t, _, p in LORA_TARGETS.values()}
        dev = self.device
        tables = {}
        for (layer, target), ents in groups.items():
            R = sum(A.shape[0] for _, A, _, _ in ents)
            Rp = (R + 7) // 8 * 8
            K, Np = ents[0][1].shape[1], ents[0][2].shape[0]
            a_cat = torch.zeros(Rp, K, dtype=torch.bfloat16, device=dev)
            b_raw = torch.zeros(Np * parts_of[target], Rp, dtype=torch.bfloat16, device=dev)
            col_scale = torch.zeros(Rp, dtype=torch.float32, device=dev)
            c = 0
            for part, A, B, scaling in ents:
                r = A.shape[0]
                a_cat[c: c + r] = A.to(device=dev, dtype=torch.bfloat16)
                b_raw[part * Np: (part + 1) * Np, c: c + r] = B.to(device=dev, dtype=torch.bfloat16)
                col_scale[c: c + r] = scaling
                c += r
            tables[(layer, target)] = (a_cat, b_raw, col_scale)
        return tables

    @torch.no_grad()
    def _lora_sync(self, scale: float) -> None:
        """Bring the handle's LoRA tables to the active set at `scale` (attention_kwargs["scale"]).  Nothing happens while they are
        current, so the per-step path does no work for them; a new set packs the factors, a new scale only rescales B_cat
        = bf16(B_raw * col_scale * scale) on the device.  Any change drops the workspaces and what was computed with the old tables."""
        want = self._lora_active()
        key = (self._lora_gen, tuple(self._lora_set), str(self.device), float(scale)) if want else None
        if key == self._lora_key:
            return
        L = _lib.lib()
        h = self._ensure_handle()
        if want:
            old = self._lora_key
            if not (self._lora_tables and old and old[:3] == key[:3]):
                self._lora_tables = {k: v[:3] for k, v in self._lora_pack().items()}
            self._lora_tables = {k: (a, b, cs, (b.float() * (cs * key[3])).to(torch.bfloat16).contiguous())
                                 for k, (a, b, cs, *_) in self._lora_tables.items()}
            n = self.config.num_layers * LORA_NUM_TARGETS
            a_p, b_p, r_p = (_lib.c_void_p * n)(), (_lib.c_void_p * n)(), (_lib.c_int32 * n)()
            for (layer, target), (a, _, _, b) in self._lora_tables.items():
                i = layer * LORA_NUM_TARGETS + target
                a_p[i], b_p[i], r_p[i] = a.data_ptr(), b.data_ptr(), a.shape[0]
            check(L.ce_dit_set_lora(h, a_p, b_p, r_p, n))
        else:
            check(L.ce_dit_set_lora(h, None, None, None, 0))
            self._lora_tables = {}
        self._lora_key = key
        self._invalidate("results")   # what was computed with the old tables
        self._invalidate("layout")    # their scratch is part of the workspace

    # ------------------------------------------------------------------------------------------ loading
    @classmethod
    def from_config(cls, config: Dict[str, Any], **kw) -> "ChronoEditTransformer3DModel":
        fields = ("patch_size", "num_attention_heads", "attention_head_dim", "in_channels", "out_channels", "text_dim", "freq_dim",
                  "ffn_dim", "num_layers", "cross_attn_norm", "qk_norm", "eps", "image_dim", "added_kv_proj_dim",
                  "rope_max_seq_len", "rope_temporal_skip_len")
        return cls(**{k: config[k] for k in fields if k in config}, **kw)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path: str, subfolder: Optional[str] = None,
                        torch_dtype: torch.dtype = torch.bfloat16, device: Optional[Union[str, torch.device]] = None,
                        **unused) -> "ChronoEditTransformer3DModel":
        """Load a diffusers-format checkpoint directory (config.json + diffusion_pytorch_model*.safetensors), the layout
        `run_inference_diffusers.py:349-353` reads.  Local paths only (no hub download)."""
        root = os.path.join(pretrained_model_name_or_path, subfolder) if subfolder else pretrained_model_name_or_path
        with open(os.path.join(root, cls.config_name)) as f:
            cfg = json.load(f)
        model = cls.from_config(cfg, torch_dtype=torch_dtype, device=device or "cpu")
        # `_keys_to_ignore_on_load_unexpected` (transformer_chronoedit.py:339)
        load_safetensors(model, root, "diffusion_pytorch_model", skip=lambda k: "norm_added_q" in k)
        return model
