"""H100-native drop-ins for the two encoders the pipeline runs once per edit (SURVEY.md section 8(f) row 3):

    transformers.UMT5EncoderModel   `self.text_encoder(input_ids, attention_mask).last_hidden_state`   pipeline_chronoedit.py:205-244
    transformers.CLIPVisionModel    `self.image_encoder(**image, output_hidden_states=True).hidden_states[-2]`     :246-254

Same constructor configuration fields, same parameter names as the transformers modules (their `state_dict()` loads unchanged),
same call surface as far as the pipeline touches it.  All arithmetic runs in libchronoedit_b200.so (`ce_umt5_encode`,
`ce_clip_vision_encode`: wgmma GEMMs + row kernels, csrc/encoders.cu); PyTorch owns memory and streams.  No CPU path.

`from_pretrained` reads a local transformers-format directory (config.json + model.safetensors or its sharded index).  CLIP also runs
in fp32 (`torch_dtype=torch.float32`, `ce_clip_vision_encode_fp32`), as the reference CLI loads it
(run_inference_diffusers.py:333-337); the text encoder is bf16 only, as the pipeline loads it.
"""
from __future__ import annotations

import json
import math
import os
from types import SimpleNamespace
from typing import Dict, Optional

import torch
import torch.nn as nn

from . import _lib
from ._checkpoint import load_safetensors
from ._lib import CEError, EncoderConfigC, check, current_stream, ptr


class _Cfg(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e


def _reg(mod: nn.Module, dotted: str, shape, dtype=torch.bfloat16, device=None) -> None:
    parts = dotted.split(".")
    for part in parts[:-1]:
        if not hasattr(mod, part):
            mod.add_module(part, nn.Module())
        mod = getattr(mod, part)
    mod.register_parameter(parts[-1], nn.Parameter(torch.empty(shape, dtype=dtype, device=device), requires_grad=False))


def _read_config(pretrained_model_name_or_path: str, subfolder: Optional[str], fields) -> tuple:
    root = os.path.join(pretrained_model_name_or_path, subfolder) if subfolder else pretrained_model_name_or_path
    with open(os.path.join(root, "config.json")) as f:
        cfg = json.load(f)
    return root, {k: cfg[k] for k in fields if k in cfg}


class _Base(nn.Module):
    def __init__(self):
        super().__init__()
        self._fp32 = False
        self._handle = None
        self._packed = False
        self._keep: Dict[str, torch.Tensor] = {}
        self._ws: Optional[torch.Tensor] = None

    @property
    def dtype(self) -> torch.dtype:
        return torch.float32 if self._fp32 else torch.bfloat16

    @property
    def device(self) -> torch.device:
        return next(self.parameters()).device

    def _apply(self, fn, *a, **k):
        self._packed = False
        return super()._apply(fn, *a, **k)

    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                _lib.lib().ce_encoder_destroy(self._handle)
        except Exception:
            pass

    def _create(self, cfg: EncoderConfigC) -> None:
        if self._handle is None:
            h = _lib.c_void_p()
            check(_lib.lib().ce_encoder_create(_lib.ctypes.byref(cfg), _lib.ctypes.byref(h)))
            self._handle = h

    def _set(self, name: str, t: torch.Tensor) -> None:
        t = t.contiguous()
        self._keep[name] = t
        set_weight = _lib.lib().ce_encoder_set_weight_fp32 if self._fp32 else _lib.lib().ce_encoder_set_weight
        check(set_weight(self._handle, name.encode(), ptr(t), t.numel()))

    def _workspace(self, B: int, L: int) -> torch.Tensor:
        if self._fp32:
            n = _lib.lib().ce_clip_vision_fp32_workspace_bytes(self._handle, B)
        else:
            n = _lib.lib().ce_encoder_workspace_bytes(self._handle, B, L)
        if n < 0:
            check(-1)
        if self._ws is None or self._ws.numel() < n or self._ws.device != self.device:
            self._ws = torch.empty(n, dtype=torch.uint8, device=self.device)
        return self._ws

    def launches(self) -> int:
        return int(_lib.lib().ce_encoder_last_launch_count(self._handle)) if self._handle else 0


class UMT5EncoderModel(_Base):
    """transformers.UMT5EncoderModel (google/umt5-xxl: d_model 4096, 64 heads x 64, d_ff 10240, 24 layers, gated GELU, 32 relative
    position buckets per layer, max distance 128; chronoedit/_src/modules/umt5.py:480-489 has the same hyper-parameters)."""

    def __init__(self, vocab_size: int = 256384, d_model: int = 4096, d_kv: int = 64, d_ff: int = 10240, num_layers: int = 24, num_heads: int = 64,
                 relative_attention_num_buckets: int = 32, relative_attention_max_distance: int = 128, layer_norm_epsilon: float = 1e-6,
                 feed_forward_proj: str = "gated-gelu", *, device=None, **unused):
        super().__init__()
        if feed_forward_proj != "gated-gelu":
            raise CEError("only the gated-GELU feed-forward of UMT5 is built")
        self.config = _Cfg(vocab_size=vocab_size, d_model=d_model, d_kv=d_kv, d_ff=d_ff, num_layers=num_layers, num_heads=num_heads,
                           relative_attention_num_buckets=relative_attention_num_buckets,
                           relative_attention_max_distance=relative_attention_max_distance, layer_norm_epsilon=layer_norm_epsilon,
                           feed_forward_proj=feed_forward_proj)
        inner = num_heads * d_kv
        _reg(self, "shared.weight", (vocab_size, d_model), device=device)
        for l in range(num_layers):
            p = f"encoder.block.{l}.layer."
            for n in ("q", "k", "v"):
                _reg(self, p + f"0.SelfAttention.{n}.weight", (inner, d_model), device=device)
            _reg(self, p + "0.SelfAttention.o.weight", (d_model, inner), device=device)
            _reg(self, p + "0.SelfAttention.relative_attention_bias.weight", (relative_attention_num_buckets, num_heads), device=device)
            _reg(self, p + "0.layer_norm.weight", (d_model,), device=device)
            _reg(self, p + "1.DenseReluDense.wi_0.weight", (d_ff, d_model), device=device)
            _reg(self, p + "1.DenseReluDense.wi_1.weight", (d_ff, d_model), device=device)
            _reg(self, p + "1.DenseReluDense.wo.weight", (d_model, d_ff), device=device)
            _reg(self, p + "1.layer_norm.weight", (d_model,), device=device)
        _reg(self, "encoder.final_layer_norm.weight", (d_model,), device=device)
        self._bias_tables: Dict[int, torch.Tensor] = {}

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        sd = {k: v for k, v in state_dict.items() if k != "encoder.embed_tokens.weight"}   # tied to shared.weight in transformers
        self._packed = False
        return super().load_state_dict(sd, strict=strict, assign=assign)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path: str, subfolder: Optional[str] = None, torch_dtype: Optional[torch.dtype] = None,
                        device=None, **unused) -> "UMT5EncoderModel":
        """`UMT5EncoderModel.from_pretrained(model_id, subfolder="text_encoder")` for a LOCAL transformers-format directory (config.json +
        model.safetensors or model.safetensors.index.json).  bf16 only: the pipeline runs the text encoder in its own bf16."""
        if torch_dtype not in (None, torch.bfloat16):
            raise CEError(f"UMT5EncoderModel: torch_dtype {torch_dtype} is not built; the text encoder runs in bf16 only")
        fields = ("vocab_size", "d_model", "d_kv", "d_ff", "num_layers", "num_heads", "relative_attention_num_buckets",
                  "relative_attention_max_distance", "layer_norm_epsilon", "feed_forward_proj")
        root, cfg = _read_config(pretrained_model_name_or_path, subfolder, fields)
        model = cls(**cfg, device=device or "cpu")
        load_safetensors(model, root, "model", skip=lambda k: k == "encoder.embed_tokens.weight")   # tied to shared.weight
        return model

    # T5 bucket function (transformers UMT5Attention._relative_position_bucket, bidirectional), host code
    def _bucket(self, rel: torch.Tensor) -> torch.Tensor:
        nb = self.config.relative_attention_num_buckets // 2
        out = (rel > 0).to(torch.long) * nb
        rel = rel.abs()
        max_exact = nb // 2
        is_small = rel < max_exact
        large = max_exact + (torch.log(rel.float() / max_exact) / math.log(self.config.relative_attention_max_distance / max_exact)
                             * (nb - max_exact)).to(torch.long)
        large = torch.min(large, torch.full_like(large, nb - 1))
        return out + torch.where(is_small, rel, large)

    @torch.no_grad()
    def _pack(self) -> None:
        if self.device.type != "cuda":
            raise CEError("UMT5EncoderModel must live on a CUDA (sm_90) device; there is no CPU path")
        c = self.config
        self._create(EncoderConfigC(0, c.vocab_size, c.d_model, c.d_kv, c.d_ff, c.num_layers, c.num_heads, c.layer_norm_epsilon, 0, 0, 0))
        self._keep = {}
        params = dict(self.named_parameters())
        for n, p in params.items():
            if p.dtype != torch.bfloat16:
                p.data = p.data.to(torch.bfloat16)
        for l in range(c.num_layers):
            p = f"encoder.block.{l}.layer.0.SelfAttention."
            self._set(p + "qk.weight", torch.cat([params[p + "q.weight"].data, params[p + "k.weight"].data], dim=0))
        for n, prm in params.items():
            if n.endswith(("SelfAttention.q.weight", "SelfAttention.k.weight", "relative_attention_bias.weight")):
                continue
            self._set(n, prm.data)
        self._bias_tables = {}
        self._packed = True

    def _bias(self, L: int) -> torch.Tensor:
        t = self._bias_tables.get(L)
        if t is None:
            c = self.config
            rel = torch.arange(-(L - 1), L, device=self.device)            # key - query = -(L-1) .. L-1
            bucket = self._bucket(rel)                                      # [2L-1]
            tabs = []
            for l in range(c.num_layers):
                w = dict(self.named_parameters())[f"encoder.block.{l}.layer.0.SelfAttention.relative_attention_bias.weight"].data   # [buckets, H]
                tabs.append(w[bucket].t().contiguous())                     # [H, 2L-1]
            t = torch.stack(tabs).contiguous().to(torch.bfloat16)
            self._bias_tables = {L: t}
        return t

    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None, **unused):
        if not self._packed:
            self._pack()
        B, L = input_ids.shape
        if L % 8 != 0:
            raise CEError("UMT5EncoderModel: sequence length must be a multiple of 8 (the pipeline pads to max_sequence_length=512)")
        ids = input_ids.to(device=self.device, dtype=torch.int64).contiguous()
        if attention_mask is None:
            valid = [L] * B
        else:
            m = attention_mask.to("cpu").to(torch.bool)
            valid = m.sum(dim=1).tolist()
            for b in range(B):
                if not bool(m[b, : valid[b]].all()) or valid[b] == 0:
                    raise CEError("UMT5EncoderModel: attention_mask must be a non-empty prefix of ones (right padding, as the tokenizer call "
                                  "at pipeline_chronoedit.py:221-229 produces)")
        vl = (_lib.c_int32 * B)(*[int(v) for v in valid])
        out = torch.empty(B, L, self.config.d_model, dtype=torch.bfloat16, device=self.device)
        ws = self._workspace(B, L)
        bias = self._bias(L)
        with torch.cuda.device(self.device):
            check(_lib.lib().ce_umt5_encode(self._handle, ptr(ids), vl, ptr(out), B, L, ptr(bias), ptr(ws), ws.numel(), current_stream()))
        return SimpleNamespace(last_hidden_state=out)


class _LazyHiddenStates:
    """`hidden_states` of CLIPVisionModel(..., output_hidden_states=True): entry i = output after i encoder layers (0 = embeddings after
    pre_layrnorm).  Only the entry that is asked for is computed (the pipeline reads [-2])."""

    def __init__(self, model: "CLIPVisionModel", pixel_values: torch.Tensor):
        self._m, self._px = model, pixel_values
        self._n = model.config.num_hidden_layers + 1

    def __len__(self):
        return self._n

    def __getitem__(self, i: int) -> torch.Tensor:
        if i < 0:
            i += self._n
        if not 0 <= i < self._n:
            raise IndexError(i)
        return self._m._encode(self._px, i)


class CLIPVisionModel(_Base):
    """transformers.CLIPVisionModel (ViT-H/14: hidden 1280, 32 layers, 16 heads x 80, MLP 5120, 224 px / patch 14 -> 257 tokens;
    chronoedit/_src/modules/clip.py:312-319)."""

    def __init__(self, hidden_size: int = 1280, intermediate_size: int = 5120, num_hidden_layers: int = 32, num_attention_heads: int = 16,
                 image_size: int = 224, patch_size: int = 14, hidden_act: str = "gelu", layer_norm_eps: float = 1e-5, num_channels: int = 3, *,
                 torch_dtype: Optional[torch.dtype] = None, device=None, **unused):
        super().__init__()
        if hidden_act not in ("gelu", "quick_gelu") or num_channels != 3 or hidden_size % num_attention_heads:
            raise CEError("CLIPVisionModel: hidden_act must be gelu or quick_gelu, 3 input channels")
        if torch_dtype not in (None, torch.bfloat16, torch.float32):
            raise CEError(f"CLIPVisionModel: torch_dtype {torch_dtype} is not built; use torch.bfloat16 or torch.float32")
        self._fp32 = torch_dtype == torch.float32
        dt = self.dtype
        self.config = _Cfg(hidden_size=hidden_size, intermediate_size=intermediate_size, num_hidden_layers=num_hidden_layers,
                           num_attention_heads=num_attention_heads, image_size=image_size, patch_size=patch_size, hidden_act=hidden_act,
                           layer_norm_eps=layer_norm_eps, num_channels=num_channels)
        D, F = hidden_size, intermediate_size
        n_pos = 1 + (image_size // patch_size) ** 2
        vm = "vision_model."
        _reg(self, vm + "embeddings.class_embedding", (D,), dtype=dt, device=device)
        _reg(self, vm + "embeddings.patch_embedding.weight", (D, 3, patch_size, patch_size), dtype=dt, device=device)
        _reg(self, vm + "embeddings.position_embedding.weight", (n_pos, D), dtype=dt, device=device)
        for n in ("pre_layrnorm", "post_layernorm"):
            _reg(self, vm + n + ".weight", (D,), dtype=dt, device=device)
            _reg(self, vm + n + ".bias", (D,), dtype=dt, device=device)
        for l in range(num_hidden_layers):
            p = vm + f"encoder.layers.{l}."
            for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
                _reg(self, p + f"self_attn.{n}.weight", (D, D), dtype=dt, device=device)
                _reg(self, p + f"self_attn.{n}.bias", (D,), dtype=dt, device=device)
            for n in ("layer_norm1", "layer_norm2"):
                _reg(self, p + n + ".weight", (D,), dtype=dt, device=device)
                _reg(self, p + n + ".bias", (D,), dtype=dt, device=device)
            _reg(self, p + "mlp.fc1.weight", (F, D), dtype=dt, device=device)
            _reg(self, p + "mlp.fc1.bias", (F,), dtype=dt, device=device)
            _reg(self, p + "mlp.fc2.weight", (D, F), dtype=dt, device=device)
            _reg(self, p + "mlp.fc2.bias", (D,), dtype=dt, device=device)

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        sd = {k: v for k, v in state_dict.items() if not k.endswith("position_ids")}   # non-parameter buffer of older transformers
        self._packed = False
        return super().load_state_dict(sd, strict=strict, assign=assign)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path: str, subfolder: Optional[str] = None, torch_dtype: Optional[torch.dtype] = None,
                        device=None, **unused) -> "CLIPVisionModel":
        """`CLIPVisionModel.from_pretrained(model_id, subfolder="image_encoder", torch_dtype=torch.float32)` (run_inference_diffusers.py:333-337)
        for a LOCAL transformers-format directory (config.json + model.safetensors or model.safetensors.index.json).  torch_dtype as the
        constructor takes it: None or torch.bfloat16 gives the bf16 encoder, torch.float32 the fp32 one."""
        fields = ("hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads", "image_size", "patch_size", "hidden_act",
                  "layer_norm_eps", "num_channels")
        root, cfg = _read_config(pretrained_model_name_or_path, subfolder, fields)
        model = cls(**cfg, torch_dtype=torch_dtype, device=device or "cpu")
        load_safetensors(model, root, "model", skip=lambda k: k.endswith("position_ids"))   # buffer of older transformers
        return model

    @torch.no_grad()
    def _pack(self) -> None:
        if self.device.type != "cuda":
            raise CEError("CLIPVisionModel must live on a CUDA (sm_90) device; there is no CPU path")
        c = self.config
        self._create(EncoderConfigC(1, 0, c.hidden_size, c.hidden_size // c.num_attention_heads, c.intermediate_size, c.num_hidden_layers,
                                    c.num_attention_heads, c.layer_norm_eps, c.image_size, c.patch_size, 1 if c.hidden_act == "gelu" else 0))
        self._keep = {}
        params = dict(self.named_parameters())
        if self._fp32:   # the parameters as they are, under their own names (post_layernorm is not read)
            for n, p in params.items():
                if p.dtype != torch.float32:
                    p.data = p.data.float()
                if "post_layernorm" not in n:
                    self._set(n, p.data)
            self._packed = True
            return
        for n, p in params.items():
            if p.dtype != torch.bfloat16:
                p.data = p.data.to(torch.bfloat16)
        vm = "vision_model."
        K = 3 * c.patch_size * c.patch_size
        Kp = (K + 7) // 8 * 8
        pe = torch.zeros(c.hidden_size, Kp, dtype=torch.bfloat16, device=self.device)
        pe[:, :K] = params[vm + "embeddings.patch_embedding.weight"].data.reshape(c.hidden_size, K)
        self._set(vm + "embeddings.patch_embedding.weight", pe)
        self._set(vm + "embeddings.class_embedding", params[vm + "embeddings.class_embedding"].data)
        self._set(vm + "embeddings.position_embedding.weight", params[vm + "embeddings.position_embedding.weight"].data)
        ln_names = [vm + "pre_layrnorm"] + [vm + f"encoder.layers.{l}.{n}" for l in range(c.num_hidden_layers) for n in ("layer_norm1", "layer_norm2")]
        for n in ln_names:   # torch.nn.LayerNorm computes in fp32 from the bf16 parameters
            self._set(n + ".weight_f32", params[n + ".weight"].data.float())
            self._set(n + ".bias_f32", params[n + ".bias"].data.float())
        for l in range(c.num_hidden_layers):
            p = vm + f"encoder.layers.{l}."
            self._set(p + "self_attn.qk_proj.weight", torch.cat([params[p + "self_attn.q_proj.weight"].data, params[p + "self_attn.k_proj.weight"].data], 0))
            self._set(p + "self_attn.qk_proj.bias", torch.cat([params[p + "self_attn.q_proj.bias"].data, params[p + "self_attn.k_proj.bias"].data], 0))
            for n in ("self_attn.v_proj.weight", "self_attn.v_proj.bias", "self_attn.out_proj.weight", "self_attn.out_proj.bias", "mlp.fc1.weight",
                      "mlp.fc1.bias", "mlp.fc2.weight", "mlp.fc2.bias"):
                self._set(p + n, params[p + n].data)
        self._packed = True

    @torch.no_grad()
    def _encode(self, pixel_values: torch.Tensor, layers_to_run: int) -> torch.Tensor:
        if not self._packed:
            self._pack()
        c = self.config
        B = pixel_values.shape[0]
        if tuple(pixel_values.shape[1:]) != (3, c.image_size, c.image_size):
            raise CEError(f"CLIPVisionModel expects pixel_values [B, 3, {c.image_size}, {c.image_size}]")
        px = pixel_values.to(device=self.device, dtype=self.dtype).contiguous()
        L = 1 + (c.image_size // c.patch_size) ** 2
        out = torch.empty(B, L, c.hidden_size, dtype=self.dtype, device=self.device)
        ws = self._workspace(B, L)
        encode = _lib.lib().ce_clip_vision_encode_fp32 if self._fp32 else _lib.lib().ce_clip_vision_encode
        with torch.cuda.device(self.device):
            check(encode(self._handle, ptr(px), ptr(out), B, int(layers_to_run), ptr(ws), ws.numel(), current_stream()))
        return out

    @torch.no_grad()
    def forward(self, pixel_values: torch.Tensor, output_hidden_states: bool = False, **unused):
        hs = _LazyHiddenStates(self, pixel_values)
        if not output_hidden_states:
            raise CEError("CLIPVisionModel mirror: the pipeline reads hidden_states[-2] (pass output_hidden_states=True); the pooled output / "
                          "post_layernorm head is not built")
        return SimpleNamespace(hidden_states=hs)
