#!/usr/bin/env python
"""bench.py's flagship configuration (14B, 720p, 2 latent frames, batch-2 CFG DiT call + fused UniPC step per denoising step) in
one numeric mode per invocation, for comparing the opt-in FP8 mode against bf16:

    python scripts/bench_fp8.py --mode bf16|fp8 [--attention bf16|fp8] [--steps 4] [--warmup 2] [--layers 40]

--attention fp8 also switches the self-attention to FP8 (enable_fp8_attention); its quantizers count as row kernels.

Prints one JSON line: steps/s (CUDA events over the timed steps), the ce_dit_profile split by class from a separate profiled
pass (GEMM / attention / row kernels, the FP8 row quantization counted as row kernels), the device bytes of the DiT's
parameters and buffers, and the card's name, power limit and clocks read in the same process.  Run the two modes alternately
to see the spread: other work shares the machine.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (configuration, inputs and weight initialisation of the flagship workload)

CLASSES = ("gemm", "attention", "rows", "other")


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    vals = [v.strip() for v in r.stdout.splitlines()[0].split(",")] if r.returncode == 0 and r.stdout else []
    return dict(zip(("gpu", "power_limit", "max_sm_clock", "sm_clock", "mem_clock"), vals))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", choices=("bf16", "fp8"), required=True)
    ap.add_argument("--attention", choices=("bf16", "fp8"), default="bf16")
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--layers", type=int, default=40)
    args = ap.parse_args()

    import torch

    import chronoedit_b200 as ce
    from chronoedit_b200 import _lib
    from chronoedit_b200.scheduler import FlowUniPCMultistepScheduler

    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8.py measures on an H100; there is no CPU measurement")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model = ce.ChronoEditTransformer3DModel(**bench.model_config(args.layers), device=dev, cache_context=True)
    bench.init_weights_(model, seed=0)
    if args.mode == "fp8":
        model.enable_fp8()
    if args.attention == "fp8":
        model.enable_fp8_attention()
    model.pack_weights()
    torch.cuda.synchronize()
    weight_bytes = sum(t.numel() * t.element_size() for t in list(model.parameters()) + list(model.buffers()))

    g = torch.Generator(device="cpu").manual_seed(42)
    F, H, W = bench.FRAMES, bench.LAT_H, bench.LAT_W
    latents = torch.randn(1, 16, F, H, W, generator=g)
    cond = torch.randn(1, 20, F, H, W, generator=g)
    cond[:, :4] = 0
    cond[:, :4, 0] = 1
    text = torch.randn(2, bench.TEXT_LEN, 4096, generator=g)
    text[0, 120:] = 0
    text[1, 40:] = 0
    img = torch.randn(1, 257, 1280, generator=g).expand(2, -1, -1).contiguous()
    d_lat = latents.to(dev, torch.bfloat16)
    d_in = torch.cat([d_lat, cond.to(dev, torch.bfloat16)], dim=1).contiguous()
    d_text, d_img = text.to(dev, torch.bfloat16), img.to(dev, torch.bfloat16)
    sched = FlowUniPCMultistepScheduler(num_train_timesteps=1000, shift=1, use_dynamic_shifting=False)

    def step():
        nonlocal d_lat
        if sched.step_index is None or sched.step_index >= 50:
            sched.set_timesteps(50, device=dev, shift=5.0)
        t = sched.timesteps[sched.step_index or 0]
        out = model(d_in.expand(2, -1, -1, -1, -1), t.expand(2), d_text, d_img, return_dict=False)[0]
        d_lat = sched.step_cfg(out[0:1], out[1:2], bench.GUIDANCE, t, d_lat, model_input_out=d_in)

    for _ in range(args.warmup):
        step()
    model.clear_context_cache()   # the timed steps are the first steps of an edit, as in bench.py
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    info = gpu_info()   # clocks right after the timed steps

    # profiled pass: per-launch events, kept out of the timing above
    L = _lib.lib()
    _lib.check(L.ce_dit_profile_begin(model._handle, 1200 * args.steps))
    for _ in range(args.steps):
        step()
    torch.cuda.synchronize()
    pms, work, cnt = (ctypes.c_double * 4)(), (ctypes.c_double * 4)(), (ctypes.c_int64 * 4)()
    _lib.check(L.ce_dit_profile_end(model._handle, pms, work, cnt))
    total = sum(pms)
    split = {c: {"ms_per_step": round(pms[i] / args.steps, 2), "share": round(pms[i] / total, 3), "launches_per_step": cnt[i] // args.steps}
             for i, c in enumerate(CLASSES)}
    split["gemm"]["tflops"] = round(work[0] / (pms[0] / 1000.0) / 1e12, 1) if pms[0] else None
    split["rows"]["GBps"] = round(work[2] / (pms[2] / 1000.0) / 1e9, 1) if pms[2] else None
    attn = {"attention": args.attention} if args.attention != "bf16" else {}
    print(json.dumps({"mode": args.mode, **attn, "layers": args.layers, "steps": args.steps, "steps_per_s": round(args.steps / (ms / 1000.0), 4),
                      "ms_per_step": round(ms / args.steps, 1), "profile": split, "device_weight_bytes": weight_bytes, **info}), flush=True)


if __name__ == "__main__":
    main()
