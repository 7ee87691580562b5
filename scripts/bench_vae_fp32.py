#!/usr/bin/env python
"""The Wan2.1 VAE (96..384 channels) at 720p in bf16 and in fp32 (as the reference pipeline's example loads it): ms per encode of 5
frames and per decode of 5 and 29 frames (2 and 8 latent frames; temporal reasoning decodes 29), with the max / mean error of each
against the fp32 oracle (oracle/vae_oracle.py on the GPU, TF32 off) and the launches of one call.

    python scripts/bench_vae_fp32.py [--iters 3] [--warmup 1]

Random fp32 weights (the bf16 VAE gets them rounded); CUDA events around `iters` back-to-back calls after `warmup` calls of the same
shape.  The pipeline runs one encode and one decode per edit, so these are per-edit costs.  Prints one JSON line with the card's name
and power limit."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    from chronoedit_b200.autoencoder import AutoencoderKLWan
    from oracle import vae_oracle as V
    from scripts.bench_cfg_parallel import card

    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = V.VAEConfig.wan21()
    sd = V.random_state_dict(cfg, seed=41)
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    g = torch.Generator(device="cpu").manual_seed(42)
    inputs = {"encode_5f": (torch.rand(1, 3, 5, 720, 1280, generator=g) * 2 - 1).to(dev),
              "decode_5f": torch.randn(1, 16, 2, 90, 160, generator=g).to(dev),
              "decode_29f": torch.randn(1, 16, 8, 90, 160, generator=g).to(dev)}
    refs = {k: (V.vae_encode(sd_dev, cfg, x) if k.startswith("encode") else V.vae_decode(sd_dev, cfg, x)) for k, x in inputs.items()}
    torch.cuda.synchronize()
    res = {}
    for label, dtype in (("bf16", torch.bfloat16), ("fp32", torch.float32)):
        m = AutoencoderKLWan(torch_dtype=dtype)
        m.load_state_dict({k: v.to(dtype) for k, v in sd.items()})
        m = m.to(dev)
        for what, x in inputs.items():
            call = (lambda: m.encode(x).latent_dist.mode()) if what.startswith("encode") else (lambda: m.decode(x, return_dict=False)[0])
            for _ in range(args.warmup):
                out = call()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                out = call()
            e1.record()
            torch.cuda.synchronize()
            err = (out.float() - refs[what]).abs()
            res[f"{label}_{what}_ms"] = round(e0.elapsed_time(e1) / args.iters, 2)
            res[f"{label}_{what}_max_err"] = float(f"{err.max().item():.3g}")
            res[f"{label}_{what}_mean_err"] = float(f"{err.mean().item():.3g}")
            res[f"{label}_{what}_launches"] = m.launches()
            del out, err
        del m
        torch.cuda.empty_cache()
    name, limit = card()
    print(json.dumps({"bench": "vae_720p", "gpu": name, "power_limit_and_max_sm_clock": limit, "iters": args.iters, "warmup": args.warmup,
                      **res}), flush=True)


if __name__ == "__main__":
    main()
