"""TeaCache policy: which denoising steps may skip the DiT blocks (DESIGN.md, "TeaCache").

Restates the rule of the reference's DiffSynth pipeline, `TeaCache.check` in
/root/reference/chronoedit_diffsynth/wan_video_new_chronoedit.py:1190-1239.  One `TeaCacheState` exists per conditioning.  On
each call it receives `rel`, the relative L1 change of the timestep modulation since the previous call:

    rel = (t_mod - prev).abs().mean() / prev.abs().mean()        (bf16 tensors, .item() to a Python float)

Step 0 and step num_inference_steps - 1 always compute and reset the accumulator.  Every other step adds poly(rel) (numpy
poly1d, float64) to it and skips when the sum is still below the threshold; a computed step resets it.  The step counter
wraps at num_inference_steps.

The device computes only the two fp32 sums; `rel_from_sums` rounds them the way torch's CUDA bf16 mean and division do.  This
module is pure host code: no torch operation runs here.
"""
from __future__ import annotations

import struct
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence

# Rescale polynomials, highest power first, as np.poly1d takes them: wan_video_new_chronoedit.py:1200-1205.
COEFFICIENTS: Dict[str, List[float]] = {
    "Wan2.1-T2V-1.3B": [-5.21862437e+04, 9.23041404e+03, -5.28275948e+02, 1.36987616e+01, -4.99875664e-02],
    "Wan2.1-T2V-14B": [-3.03318725e+05, 4.90537029e+04, -2.65530556e+03, 5.87365115e+01, -3.15583525e-01],
    "Wan2.1-I2V-14B-480P": [2.57151496e+05, -3.54229917e+04, 1.40286849e+03, -1.35890334e+01, 1.32517977e-01],
    "Wan2.1-I2V-14B-720P": [8.10705460e+03, 2.13393892e+03, -3.72934672e+02, 1.66203073e+01, -4.17769401e-02],
}
DEFAULT_MODEL_ID = "Wan2.1-I2V-14B-720P"   # ChronoEdit is built on Wan2.1-I2V-14B-720P


def coefficients(model_id: str) -> List[float]:
    if model_id not in COEFFICIENTS:
        raise ValueError(f"{model_id} is not a supported TeaCache model id. Please choose a valid model id in "
                         f"({', '.join(COEFFICIENTS)}).")
    return list(COEFFICIENTS[model_id])


def poly(coeffs: Sequence[float], x: float) -> float:
    """np.poly1d(coeffs)(x) for a Python float: Horner's rule in float64, the same operations numpy performs."""
    y = 0.0
    for c in coeffs:
        y = y * x + c
    return y


def _f32(x: float) -> float:
    return struct.unpack("<f", struct.pack("<f", x))[0]


def _bf16(x: float) -> float:
    """Round an fp32 value to bf16 (nearest, ties to even), as float -> at::BFloat16 does."""
    u = struct.unpack("<I", struct.pack("<f", _f32(x)))[0]
    if (u & 0x7F800000) == 0x7F800000 and (u & 0x7FFFFF):   # NaN stays NaN
        return float("nan")
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return struct.unpack("<f", struct.pack("<I", u))[0]


def rel_from_sums(sum_abs_diff: float, sum_abs_prev: float, n: int) -> float:
    """`((a - b).abs().mean() / b.abs().mean()).item()` for bf16 CUDA tensors of n elements, from the fp32 sums of |bf16(a - b)|
    and |b|.  ATen's CUDA mean multiplies the fp32 sum by the fp32 factor 1 / n and rounds the product to bf16; the bf16
    quotient is computed in fp32 and rounded to bf16."""
    factor = _f32(1.0 / _f32(float(n)))
    num = _bf16(_f32(_f32(sum_abs_diff) * factor))
    den = _bf16(_f32(_f32(sum_abs_prev) * factor))
    return _bf16(_f32(num / den)) if den != 0.0 else (float("nan") if num == 0.0 else float("inf"))


@dataclass(frozen=True)
class Record:
    """One call of a TeaCache state: which conditioning slot, the step (before the increment), rel (None on a step that does
    not evaluate it), the accumulator after the call, and whether the blocks ran."""
    slot: int
    step: int
    rel: Optional[float]
    acc: float
    computed: bool


class TeaCacheState:
    """The per-conditioning state machine of the reference's `TeaCache.check`, driven by rel values instead of tensors."""

    def __init__(self, num_inference_steps: int, rel_l1_thresh: float, model_id: str = DEFAULT_MODEL_ID):
        if num_inference_steps < 1:
            raise ValueError("num_inference_steps must be >= 1")
        self.num_inference_steps = int(num_inference_steps)
        self.rel_l1_thresh = float(rel_l1_thresh)
        self.coefficients = coefficients(model_id)
        self.step = 0
        self.acc = 0.0

    def needs_rel(self) -> bool:
        """Whether this call evaluates rel (every step except the first and the last of the schedule)."""
        return not (self.step == 0 or self.step == self.num_inference_steps - 1)

    def decide(self, rel: Optional[float], force_compute: bool = False):
        """One call: returns (step, computed).  `rel` is read only when needs_rel().  force_compute, or rel None on such a step,
        makes the call compute and reset the accumulator: the mirror does this when the stored residual has another geometry,
        or when the batch changed so that rel cannot be formed."""
        step = self.step
        if not self.needs_rel():
            computed = True
            self.acc = 0.0
        else:
            if rel is not None:
                self.acc += poly(self.coefficients, float(rel))
            if rel is not None and self.acc < self.rel_l1_thresh and not force_compute:
                computed = False
            else:
                computed = True
                self.acc = 0.0
        self.step += 1
        if self.step == self.num_inference_steps:
            self.step = 0
        return step, computed
