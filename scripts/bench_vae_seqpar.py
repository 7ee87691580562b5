#!/usr/bin/env python
"""Latency of the VAE of ONE edit split over the GPUs of a node by row bands (parallel.enable_vae_sequence_parallel).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node W --master-addr 127.0.0.1 scripts/bench_vae_seqpar.py [--reps 3]

Workloads, at 720p with the Wan2.1 VAE (random weights, synthetic inputs): the edit's bookends (encode 5 frames, decode 2 latent
frames) and temporal reasoning's (encode 29 frames, decode 8 latent frames, then their first and last).  Prints one JSON line: ms per
call with the rows split over W ranks next to the single-GPU call measured in the same run on the same card (every rank runs it, the
slowest rank counts), whether every rank's result is bit-identical to the single-GPU one, and the peer region's bytes."""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    from chronoedit_b200 import parallel
    from chronoedit_b200.autoencoder import AutoencoderKLWan

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--height", type=int, default=720)
    ap.add_argument("--width", type=int, default=1280)
    args = ap.parse_args()
    rank, local, world = int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    H, W = args.height, args.width
    vae = AutoencoderKLWan(device=dev)
    g = torch.Generator(device=dev).manual_seed(7)   # same seed on every rank: identical weights without a broadcast
    with torch.no_grad():
        for n, p in vae.named_parameters():
            if n.endswith("gamma"):
                p.normal_(0, 0.1, generator=g).add_(1.0)
            elif n.endswith("bias"):
                p.normal_(0, 0.02, generator=g)
            else:
                p.normal_(0, p[0].numel() ** -0.5, generator=g)
    gi = torch.Generator(device=dev).manual_seed(11)
    z8 = torch.randn(1, 16, 8, H // 8, W // 8, generator=gi, device=dev).bfloat16()
    calls = {
        "encode_5f": lambda: vae.encode(v5).latent_dist.mode(),
        "decode_2lat": lambda: vae.decode(z8[:, :, :2].contiguous(), return_dict=False)[0],
        "encode_29f": lambda: vae.encode(v29).latent_dist.mode(),
        "decode_8lat": lambda: vae.decode(z8, return_dict=False)[0],
        "decode_first_last": lambda: vae.decode(z8[:, :, [0, -1]].contiguous(), return_dict=False)[0],
    }
    v5 = (torch.rand(1, 3, 5, H, W, generator=gi, device=dev) * 2 - 1).bfloat16()
    v29 = (torch.rand(1, 3, 29, H, W, generator=gi, device=dev) * 2 - 1).bfloat16()

    def timed(fn):
        out = fn().clone()   # warm-up (workspace, modules)
        dist.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = torch.tensor([e0.elapsed_time(e1) / args.reps], device=dev)
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms), out

    single = {k: timed(fn) for k, fn in calls.items()}
    region = parallel.enable_vae_sequence_parallel(vae, H, W)
    split = {k: timed(fn) for k, fn in calls.items()}
    parallel.disable_vae_sequence_parallel(vae)
    same = torch.tensor([int(all(torch.equal(split[k][1], single[k][1]) for k in calls))], device=dev)
    dist.all_reduce(same, op=dist.ReduceOp.MIN)
    if rank == 0:
        props = torch.cuda.get_device_properties(dev)
        line = {"world": world, "geometry": f"{H}x{W}", "gpu": props.name, "region_bytes": region, "bit_identical": bool(same.item()),
                "single_gpu_ms": {k: round(v[0], 2) for k, v in single.items()},
                "split_ms": {k: round(v[0], 2) for k, v in split.items()}}
        print(json.dumps(line), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
