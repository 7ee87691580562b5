#!/usr/bin/env python
"""Golden fixtures for the TeaCache rule, recorded from the UNMODIFIED reference class in this container.

    python tests/golden/make_golden_teacache.py    # writes tests/golden/teacache_tmod.safetensors + TEACACHE_MANIFEST.json

Source of truth executed here (never copied): the `TeaCache` class of
/root/reference/chronoedit_diffsynth/wan_video_new_chronoedit.py (:1190-1239), taken out of the file with `ast` and executed
on its own (the file's other imports are not needed by the class).  Its inputs are timestep modulations from the oracle's time
path (oracle/teacache_oracle.time_modulation) on seeded weights of the 2-layer test configuration, over the UniPC timesteps of
a 50-step shift-5 and an 8-step shift-2 schedule.  Each sequence is fed twice in a row, so the step counter's wrap is
recorded too.  The oracle restatement must reproduce every decision and accumulator or generation aborts."""
from __future__ import annotations

import ast
import json
import os
import sys

import numpy as np
import torch
from safetensors.torch import save_file

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import dit_oracle as D, ref_loader, teacache_oracle as TC, unipc_oracle as U  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
SCHEDULES = {"s50_shift5": (50, 5.0), "s8_shift2": (8, 2.0)}
THRESHOLDS = (0.1, 0.15, 0.2, 0.25, 0.3)
CFG = D.DiTConfig.tiny()


def reference_teacache_class():
    path = os.path.join(ref_loader.REFERENCE_ROOT, "chronoedit_diffsynth", "wan_video_new_chronoedit.py")
    src = open(path).read()
    node = next(n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == "TeaCache")
    ns = {"np": np, "torch": torch, "WanModel": object}
    exec(compile(ast.Module(body=[node], type_ignores=[]), path, "exec"), ns)
    return ns["TeaCache"]


def tmod_sequence(n_steps: int, shift: float) -> torch.Tensor:
    """[n_steps, 1, 6, D] bf16: the time path at every timestep of the schedule (bf16 weights, as the pipeline runs)."""
    sd = {k: (v if "time_embedder" in k else v.to(torch.bfloat16)) for k, v in D.random_state_dict(CFG, seed=31).items()}
    # a larger time_proj bias brings the step-to-step change of random weights (rel ~ 0.2) down to rel ~ 0.01, where the 720P
    # polynomial adds about 0.1 per step and thresholds 0.1 to 0.3 give a mix of computed and skipped calls
    b = "condition_embedder.time_proj.bias"
    sd[b] = (sd[b].float() * 20).to(torch.bfloat16)
    _, timesteps = U.flow_sigmas(n_steps, shift)
    return torch.stack([TC.time_modulation(sd, CFG, t.reshape(1).float()) for t in timesteps])


def main():
    assert ref_loader.reference_available(), "needs /root/reference"
    TeaCache = reference_teacache_class()
    coeffs = TeaCache(1, 0.1, "Wan2.1-I2V-14B-720P").coefficients_dict
    tensors, cases = {}, {}
    for name, (n, shift) in SCHEDULES.items():
        seq = tmod_sequence(n, shift)
        tensors[name] = seq.contiguous()
        calls = list(seq) + list(seq)   # twice: the counter wraps at n
        for model_id in coeffs:
            for thresh in THRESHOLDS if model_id == "Wan2.1-I2V-14B-720P" else (0.2,):
                tc = TeaCache(n, thresh, model_id)
                computed, acc = [], []
                for t_mod in calls:
                    x = torch.zeros(1, 4, 8)
                    skip = tc.check(None, x, t_mod)
                    if not skip:
                        tc.store(x)
                    computed.append(not skip)
                    acc.append(float(tc.accumulated_rel_l1_distance))
                got = TC.rule(calls, thresh, n, coeffs[model_id])
                assert [g["computed"] for g in got] == computed and [g["acc"] for g in got] == acc, (name, model_id, thresh)
                cases[f"{name}/{model_id}/{thresh}"] = dict(schedule=name, steps=n, model_id=model_id, thresh=thresh, computed=computed,
                                                            acc=acc)
                print(f"{name} {model_id} {thresh}: {sum(not c for c in computed)} of {len(computed)} calls skipped")
    save_file(tensors, os.path.join(OUT, "teacache_tmod.safetensors"))
    with open(os.path.join(OUT, "TEACACHE_MANIFEST.json"), "w") as f:
        json.dump(dict(source="chronoedit_diffsynth/wan_video_new_chronoedit.py:1190-1239 (TeaCache, executed unmodified)",
                       coefficients=coeffs, cases=cases), f, indent=1)


if __name__ == "__main__":
    main()
