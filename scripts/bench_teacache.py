#!/usr/bin/env python
"""TeaCache on bench.py's flagship configuration (14B, 720p, 5 pixel frames = 2 latent frames, batch-2 CFG DiT call and the
fused UniPC step, 50-step schedule with shift 5):

    python scripts/bench_teacache.py [--layers 40] [--rounds 5] [--thresholds 0.1 0.2 0.3]

Prints one JSON line with the card's name and power limit and:
  * ms per computed forward (the forward with the residual recorded) against the plain forward, in alternating rounds;
  * ms per skipped forward (patch embedding + residual, output head);
  * the GPU idle gap around the decision read: from the end of one forward to the start of the next, with the probe and its
    8-byte device-to-host read in between;
  * the 50-step loop time and the skip count with TeaCache off and at each threshold.
The weights are random: the timestep modulation of random time-embedding weights moves differently from a trained model's, so
the skip counts say nothing about a real checkpoint.  What transfers is the speed model
computed x ms_computed + skipped x ms_skipped (+ one probe per call).
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import bench  # noqa: E402  (configuration, inputs and weight initialisation of the flagship workload)
from bench_fp8 import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--thresholds", type=float, nargs="*", default=[0.1, 0.2, 0.3])
    args = ap.parse_args()

    import torch

    import chronoedit_b200 as ce
    from chronoedit_b200.scheduler import FlowUniPCMultistepScheduler

    if not torch.cuda.is_available():
        raise SystemExit("bench_teacache.py measures on an H100; there is no CPU measurement")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model = ce.ChronoEditTransformer3DModel(**bench.model_config(args.layers), device=dev, cache_context=True)
    bench.init_weights_(model, seed=0)
    model.pack_weights()

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
    d_text, d_img = text.to(dev, torch.bfloat16), img.to(dev, torch.bfloat16)
    d_cond = cond.to(dev, torch.bfloat16)

    def ev():
        return torch.cuda.Event(enable_timing=True)

    # ---- one forward of each kind, alternated
    d_in = torch.cat([latents.to(dev, torch.bfloat16), d_cond], dim=1).expand(2, -1, -1, -1, -1).contiguous()
    t = torch.full((2,), 500.0, device=dev)
    out = torch.empty(2, 16, F, H, W, dtype=torch.bfloat16, device=dev)
    D = model.config.num_attention_heads * model.config.attention_head_dim
    resid = torch.empty(2 * F * (H // 2) * (W // 2) * D, dtype=torch.bfloat16, device=dev)
    kinds = {
        "plain": lambda: model._native_forward(d_in, t, d_text, d_img, out, None, {}, d_text, d_img),
        "computed": lambda: model._native_teacache_forward(d_in, t, d_text, d_img, out, d_text, d_img, resid, True),
        "skipped": lambda: model._native_teacache_forward(d_in, t, d_text, d_img, out, d_text, d_img, resid, False),
    }
    times = {k: [] for k in kinds}
    for k in kinds:   # warm-up, fills the context cache
        kinds[k]()
    for _ in range(args.rounds):
        for k, fn in kinds.items():
            a, b = ev(), ev()
            a.record()
            fn()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b))

    # ---- the gap around the decision read: end of a forward -> probe -> read -> start of the next forward
    cur = torch.empty(2 * 6 * D, dtype=torch.bfloat16, device=dev)
    prev = torch.empty_like(cur)
    model._native_probe(t, None, prev)
    gaps = []
    for _ in range(args.rounds):
        kinds["skipped"]()
        a, b = ev(), ev()
        a.record()
        model._native_probe(t, prev, cur)
        b.record()
        kinds["skipped"]()
        b.synchronize()
        gaps.append(a.elapsed_time(b) * 1000.0)

    # ---- the 50-step loop
    sched = FlowUniPCMultistepScheduler(num_train_timesteps=1000, shift=1, use_dynamic_shifting=False)

    def loop(thresh):
        if thresh is None:
            model.disable_teacache()
        else:
            model.enable_teacache(thresh, num_inference_steps=args.steps)
        model.clear_context_cache()
        sched.set_timesteps(args.steps, device=dev, shift=5.0)
        lat = latents.to(dev, torch.bfloat16)
        x_in = torch.cat([lat, d_cond], dim=1).contiguous()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for ts in sched.timesteps:
            o = model(x_in.expand(2, -1, -1, -1, -1), ts.expand(2), d_text, d_img, return_dict=False)[0]
            lat = sched.step_cfg(o[0:1], o[1:2], bench.GUIDANCE, ts, lat, model_input_out=x_in)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1000.0
        skipped = sum(not r.computed for r in model.teacache_records) if thresh is not None else 0
        return {"threshold": thresh or 0.0, "loop_ms": round(ms, 1), "forwards": args.steps, "skipped": skipped}

    loops = [loop(None)] + [loop(th) for th in args.thresholds]
    model.disable_teacache()
    med = lambda v: sorted(v)[len(v) // 2]
    print(json.dumps({
        "layers": args.layers, "rounds": args.rounds, "geometry": [2, F, H, W],
        "ms_plain": round(med(times["plain"]), 2), "ms_computed": round(med(times["computed"]), 2),
        "ms_skipped": round(med(times["skipped"]), 3), "ms_all": {k: [round(x, 2) for x in v] for k, v in times.items()},
        "probe_read_gap_us": round(med(gaps), 1), "loops": loops,
        "note": "random weights: skip counts do not predict a trained checkpoint's", **gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
