#!/usr/bin/env python
"""The CLIP image encoder at ViT-H/14 (1280 wide, 32 layers, 16 heads x 80, 224 px -> 257 tokens): ms per
`hidden_states[-2]` call in bf16 and in fp32 (as the reference CLI loads it), at batch 1 and 2, with the launches of one call.

    python scripts/bench_clip.py [--iters 10] [--warmup 3]

Random weights; CUDA events around `iters` back-to-back calls after `warmup` calls of the same shape.  The pipeline runs the
encoder once per edit, so these are per-edit costs.  Prints one JSON line with the card's name and power limit."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

VIT_H = dict(hidden_size=1280, intermediate_size=5120, num_hidden_layers=32, num_attention_heads=16, image_size=224, patch_size=14,
             hidden_act="gelu")


def main():
    import chronoedit_b200 as ce
    from scripts.bench_cfg_parallel import card

    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.manual_seed(0)
    sd = {k: torch.randn(v.shape) * (0.02 if v.dim() == 2 else 0.1) for k, v in ce.CLIPVisionModel(**VIT_H, device="meta").state_dict().items()}
    for k in sd:
        if "norm" in k and k.endswith("weight"):
            sd[k] += 1.0
    px = torch.randn(2, 3, 224, 224, device=dev)
    res = {}
    for label, dtype in (("bf16", None), ("fp32", torch.float32)):
        m = ce.CLIPVisionModel(**VIT_H, torch_dtype=dtype)
        m.load_state_dict(sd)
        m = m.to(dev)
        for B in (1, 2):
            x = px[:B].contiguous()
            call = lambda: m(pixel_values=x, output_hidden_states=True).hidden_states[-2]
            for _ in range(args.warmup):
                call()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                call()
            e1.record()
            torch.cuda.synchronize()
            res[f"{label}_b{B}_ms"] = round(e0.elapsed_time(e1) / args.iters, 3)
            res[f"{label}_b{B}_launches"] = m.launches()
        del m
        torch.cuda.empty_cache()
    name, limit = card()
    print(json.dumps({"bench": "clip_vit_h", "gpu": name, "power_limit_and_max_sm_clock": limit, "iters": args.iters, "warmup": args.warmup,
                      **res}), flush=True)


if __name__ == "__main__":
    main()
