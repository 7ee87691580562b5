#!/usr/bin/env python
"""Run-time LoRA (set_adapters) at bench.py's size: ms per DiT step with no adapter, one adapter and two stacked adapters, at ranks
32 and 64, in bf16 and with FP8 weights + FP8 attention, plus the time of set_adapters itself.

    python scripts/bench_lora.py [--layers 40] [--steps 4]

A step is one forward of the CFG pair as one batch-2 call, as bench.py's loop runs it: ChronoEdit-14B, 720p, bench.py's latent
frames, random weights and random adapters on all twelve block linear layers, context cache on.  Prints one JSON line with the card's
name and power limit."""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MODULES = ("attn1.to_q", "attn1.to_k", "attn1.to_v", "attn1.to_out.0", "attn2.to_q", "attn2.to_k", "attn2.to_v", "attn2.to_out.0",
           "attn2.add_k_proj", "attn2.add_v_proj", "ffn.net.0.proj", "ffn.net.2")


def random_lora(model, rank, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    sd = {}
    for i, blk in enumerate(model.blocks):
        for mod in MODULES:
            holder = blk.get_submodule(mod)
            w = holder.weight if hasattr(holder, "weight") else holder.weight_fp8
            N, K = w.shape
            sd[f"blocks.{i}.{mod}.lora_A.weight"] = (torch.randn(rank, K, generator=g, device=dev) / K ** 0.5).bfloat16()
            sd[f"blocks.{i}.{mod}.lora_B.weight"] = (torch.randn(N, rank, generator=g, device=dev) * 0.1 / rank ** 0.5).bfloat16()
    return sd


def main():
    import bench
    import chronoedit_b200 as ce
    from scripts.bench_cfg_parallel import card

    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=40)
    ap.add_argument("--steps", type=int, default=4)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    T, H, W = bench.FRAMES, bench.LAT_H, bench.LAT_W
    g = torch.Generator(device=dev).manual_seed(7)
    x = torch.randn(2, 36, T, H, W, generator=g, device=dev).bfloat16()
    txt = torch.randn(2, bench.TEXT_LEN, 4096, generator=g, device=dev).bfloat16()
    img = torch.randn(2, 257, 1280, generator=g, device=dev).bfloat16()
    t = torch.full((2,), 500.0, device=dev)

    def timed(model, n):
        model(x, t, txt, img, return_dict=False)     # warm-up: workspaces, context cache
        model(x, t, txt, img, return_dict=False)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            model(x, t, txt, img, return_dict=False)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    results = {}
    for mode in ("bf16", "fp8+fp8_attention"):
        model = ce.ChronoEditTransformer3DModel(**bench.model_config(args.layers), device=dev, cache_context=True)
        bench.init_weights_(model, seed=0)
        if mode != "bf16":
            model.enable_fp8()
            model.enable_fp8_attention()
        model.pack_weights()
        r = {"none": timed(model, args.steps)}
        for rank in (32, 64):
            model.load_lora_adapter(random_lora(model, rank, 1, dev), prefix=None, adapter_name=f"a{rank}")
            model.load_lora_adapter(random_lora(model, rank, 2, dev), prefix=None, adapter_name=f"b{rank}")
            for names in ([f"a{rank}"], [f"a{rank}", f"b{rank}"]):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                model.set_adapters(names, [1.0, 0.6][: len(names)])
                torch.cuda.synchronize()
                set_ms = (time.perf_counter() - t0) * 1e3
                r[f"rank{rank}_x{len(names)}"] = {"ms_per_step": timed(model, args.steps), "set_adapters_ms": set_ms}
            model.delete_adapters([f"a{rank}", f"b{rank}"])
        r["none_after"] = timed(model, args.steps)
        results[mode] = r
        del model
        torch.cuda.empty_cache()
    name, limit = card()
    print(json.dumps({"workload": f"ChronoEdit-14B ({args.layers} layers), batch-2 forward of latent [2,36,{T},{H},{W}], "
                                  "adapters on the 12 block linear layers of every block",
                      "card": name, "power_limit_and_max_sm_clock": limit, "results": results}), flush=True)


if __name__ == "__main__":
    main()
