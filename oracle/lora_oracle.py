"""Run-time LoRA's rule (DESIGN.md, "Run-time LoRA") on top of the DiT oracle: PEFT's unfused LoRA forward,

    base   = F.linear(x, W, b)                                     (or the rule `inner` applies, e.g. the FP8 mode's)
    result = base + sum_i bf16(bf16(bf16(x A_i^T) B_i^T) * scaling_i)     in the dtype of x, over the adapters in order

for the linear layers an adapter covers.  TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

from . import dit_oracle as O

Adapters = Dict[str, List[Tuple[torch.Tensor, torch.Tensor, float]]]   # module name -> [(A [r, K], B [N, r], scaling)]


def lora_term(x: torch.Tensor, A: torch.Tensor, B: torch.Tensor, scaling: float) -> torch.Tensor:
    """One adapter's addend, PEFT's `lora_B(lora_A(x)) * scaling` with the factors in the dtype of x."""
    return F.linear(F.linear(x, A.to(x.dtype)), B.to(x.dtype)) * scaling


class _LoraF:
    """Stands in for torch.nn.functional inside the oracle: F.linear on a weight an adapter covers adds the LoRA terms."""

    def __init__(self, terms, inner=None):
        self.terms = terms   # id(weight tensor) -> [(A, B, scaling)]
        self.inner = inner if inner is not None else F

    def __getattr__(self, name):
        return getattr(F, name)

    def linear(self, x, w, b=None):
        y = self.inner.linear(x, w, b)
        for A, B, s in self.terms.get(id(w), ()):
            y = y + lora_term(x, A, B, s)
        return y


def dit_forward(sd: Dict[str, torch.Tensor], cfg: O.DiTConfig, adapters: Adapters, *inputs, inner=None) -> torch.Tensor:
    """dit_oracle.dit_forward with the adapters' terms on the linear layers they name, in the dtype of `inputs`.  `inner`
    (optional) replaces F.linear for the base product, as the FP8 tests' emulation does."""
    terms = {}
    for mod, lst in adapters.items():
        w = sd[mod + ".weight"]
        if any(v is w for k, v in sd.items() if k != mod + ".weight"):
            raise ValueError(f"{mod}.weight is shared with another entry of the state dict: its id would not name it alone")
        terms[id(w)] = lst
    saved = O.F
    O.F = _LoraF(terms, inner)
    try:
        with torch.no_grad():
            return O.dit_forward(sd, cfg, *inputs)
    finally:
        O.F = saved


def adapters_of(entries: List[Tuple[Dict[str, torch.Tensor], float]], scale: float = 1.0,
                device: Optional[torch.device] = None) -> Adapters:
    """Adapters from [(lora state dict with diffusers keys `[transformer.]<module>.lora_A.weight` / `lora_B` / `alpha`, weight)]
    in activation order: scaling = weight * scale * alpha / r (alpha = r when absent), as PEFT's set_adapters and
    scale_lora_layers give it."""
    out: Adapters = {}
    for sd, weight in entries:
        mods = {}
        for k, v in sd.items():
            k = k[len("transformer."):] if k.startswith("transformer.") else k
            for tag, kind in ((".lora_A.weight", "A"), (".lora_B.weight", "B"), (".alpha", "alpha")):
                if k.endswith(tag):
                    mods.setdefault(k[: -len(tag)], {})[kind] = v
        for mod, d in mods.items():
            r = d["A"].shape[0]
            alpha = float(d["alpha"]) if "alpha" in d else float(r)
            A, B = d["A"], d["B"]
            if device is not None:
                A, B = A.to(device), B.to(device)
            out.setdefault(mod, []).append((A, B, weight * scale * alpha / r))
    return out
