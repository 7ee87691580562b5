"""Restatement of the reference's TeaCache rule and of a DiT forward under a given skip schedule -- TEST INFRASTRUCTURE ONLY
(oracle/__init__.py).

Restates `TeaCache` of /root/reference/chronoedit_diffsynth/wan_video_new_chronoedit.py:1190-1239 as a function of the sequence
of timestep modulations t_mod ([B, 6, D], the diffusers model's timestep_proj) and its use in `model_fn_wan_video` (:1434-1438,
:1454-1455, :1491-1492): a computed call stores residual = x_after_blocks - x_before_blocks, a skipped call replaces the
blocks by x_before_blocks + residual, and the output head runs either way.

Pinning: tests/golden/make_golden_teacache.py runs the UNMODIFIED reference class (taken from the reference file with `ast`) on
t_mod sequences from `time_modulation` and stores its decisions and accumulators under tests/golden/teacache_*;
tests/test_teacache_cpu.py requires `rule` to reproduce them.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from . import dit_oracle as D

Tensor = torch.Tensor


def time_modulation(sd: Dict[str, Tensor], cfg: D.DiTConfig, timestep: Tensor, dtype: torch.dtype = torch.bfloat16) -> Tensor:
    """t_mod [B, 6, D]: the condition embedder's time path (transformer_chronoedit.py:147-159), temb cast to `dtype`."""
    p = "condition_embedder."
    t = D.timestep_sinusoid(timestep, cfg.freq_dim)
    w1 = sd[p + "time_embedder.linear_1.weight"]
    t = t.to(w1.dtype)
    temb = F.linear(F.silu(F.linear(t, w1, sd[p + "time_embedder.linear_1.bias"])),
                    sd[p + "time_embedder.linear_2.weight"], sd[p + "time_embedder.linear_2.bias"]).to(dtype)
    tproj = F.linear(F.silu(temb), sd[p + "time_proj.weight"], sd[p + "time_proj.bias"])
    return tproj.unflatten(1, (6, -1))


def rel_l1(t_mod: Tensor, prev: Tensor) -> float:
    """The reference's relative L1 distance (:1222), in the tensors' own dtype and device semantics."""
    return ((t_mod - prev).abs().mean() / prev.abs().mean()).cpu().item()


def rule(t_mods: Sequence[Tensor], rel_l1_thresh: float, num_inference_steps: int, coefficients: Sequence[float]) -> List[dict]:
    """The decisions of one TeaCache object over successive calls with t_mods[0], t_mods[1], ... (the step counter wraps at
    num_inference_steps).  Per call: step, rel (None on the first and last step), acc after the call, computed."""
    poly = np.poly1d(coefficients)
    step, acc, prev, out = 0, 0, None, []
    for t_mod in t_mods:
        rel = None
        if step == 0 or step == num_inference_steps - 1:
            computed, acc = True, 0
        else:
            rel = rel_l1(t_mod, prev)
            acc += poly(rel)
            if acc < rel_l1_thresh:
                computed = False
            else:
                computed, acc = True, 0
        out.append(dict(step=step, rel=rel, acc=float(acc), computed=computed))
        prev = t_mod
        step += 1
        if step == num_inference_steps:
            step = 0
    return out


def forward_parts(sd: Dict[str, Tensor], cfg: D.DiTConfig, hidden_states: Tensor, timestep: Tensor, encoder_hidden_states: Tensor,
                  encoder_hidden_states_image: Optional[Tensor] = None, residual: Optional[Tensor] = None):
    """dit_oracle.dit_forward split around the blocks.  residual None: the blocks run and (sample, x_before_blocks,
    x_after_blocks) is returned.  Otherwise the blocks are replaced by x_before_blocks + residual (a skipped TeaCache call) and
    (sample, x_before_blocks, that sum) is returned.  Token streams are [B, L, D]."""
    T, Hh, Ww = hidden_states.shape[2:]
    x = F.conv3d(hidden_states, sd["patch_embedding.weight"], sd["patch_embedding.bias"], stride=cfg.patch_size)
    x0 = x.flatten(2).transpose(1, 2)
    if residual is None:
        temb, tproj, text, image = D.condition_embedder(sd, cfg, timestep, encoder_hidden_states, encoder_hidden_states_image)
        temb6 = tproj.unflatten(1, (6, -1))
        ctx = text if image is None else torch.concat([image, text], dim=1)
        freqs = D.rope_table(cfg, T, Hh, Ww).to(hidden_states.device)
        x = x0
        for i in range(cfg.num_layers):
            x = D.block(sd, i, cfg, x, ctx, temb6, freqs)
    else:
        temb = time_embedding(sd, cfg, timestep, x0.dtype)
        x = x0 + residual
    return head(sd, cfg, x, temb, (T, Hh, Ww)), x0, x


def head(sd: Dict[str, Tensor], cfg: D.DiTConfig, x: Tensor, temb: Tensor, thw) -> Tensor:
    """The output head (transformer_chronoedit.py:451-467): modulated norm_out, proj_out and unpatchify of x [B, L, D]."""
    B = x.shape[0]
    pt, ph, pw = cfg.patch_size
    ppf, pph, ppw = thw[0] // pt, thw[1] // ph, thw[2] // pw
    shift, scale = (sd["scale_shift_table"] + temb.unsqueeze(1)).chunk(2, dim=1)
    x = (D._fp32_layer_norm(x.float(), None, None, cfg.eps) * (1 + scale) + shift).type_as(x)
    x = F.linear(x, sd["proj_out.weight"], sd["proj_out.bias"])
    x = x.reshape(B, ppf, pph, ppw, pt, ph, pw, -1).permute(0, 7, 1, 4, 2, 5, 3, 6)
    return x.flatten(6, 7).flatten(4, 5).flatten(2, 3)


def time_embedding(sd: Dict[str, Tensor], cfg: D.DiTConfig, timestep: Tensor, dtype: torch.dtype) -> Tensor:
    """temb [B, D] of the condition embedder (transformer_chronoedit.py:153-157), cast to `dtype`."""
    p = "condition_embedder."
    t = D.timestep_sinusoid(timestep, cfg.freq_dim).to(sd[p + "time_embedder.linear_1.weight"].dtype)
    return F.linear(F.silu(F.linear(t, sd[p + "time_embedder.linear_1.weight"], sd[p + "time_embedder.linear_1.bias"])),
                    sd[p + "time_embedder.linear_2.weight"], sd[p + "time_embedder.linear_2.bias"]).to(dtype)


class ScheduledTransformer:
    """The oracle transformer surface of pipeline_oracle.OracleTransformer, run under a given skip schedule: `computed[k]` says
    whether the k-th call runs the blocks.  Residuals are kept per conditioning (the encoder_hidden_states object), as the
    reference keeps one TeaCache per conditioning."""

    def __init__(self, sd: Dict[str, Tensor], cfg: D.DiTConfig, dtype: torch.dtype, computed: Sequence[bool]):
        from types import SimpleNamespace

        self.sd, self.cfg, self.dtype = sd, cfg, dtype
        self.config = SimpleNamespace(patch_size=cfg.patch_size)
        self.computed = list(computed)
        self.calls = 0
        self._resid: Dict[int, Tensor] = {}

    def __call__(self, hidden_states, timestep, encoder_hidden_states, encoder_hidden_states_image=None, attention_kwargs=None,
                 return_dict=True):
        from types import SimpleNamespace

        k = id(encoder_hidden_states)
        if self.computed[self.calls]:
            out, x0, xl = forward_parts(self.sd, self.cfg, hidden_states, timestep, encoder_hidden_states, encoder_hidden_states_image)
            self._resid[k] = xl - x0
        else:
            out, _, _ = forward_parts(self.sd, self.cfg, hidden_states, timestep, encoder_hidden_states, encoder_hidden_states_image,
                                      residual=self._resid[k])
        self.calls += 1
        return (out,) if not return_dict else SimpleNamespace(sample=out)
