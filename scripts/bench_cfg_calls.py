#!/usr/bin/env python
"""The unchanged pipeline's CFG pair split by calls over two GPUs (parallel.enable_cfg_parallel_calls): one denoising step in the
pipeline's order -- the prompt call, the negative-prompt call with the same latents and timestep (both batch 1), the guidance combine
-- timed with the split and on one GPU.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node W --master-addr 127.0.0.1 scripts/bench_cfg_calls.py \
        [--mode bf16|fp8] [--latent-frames 2] [--layers 40] [--steps 6]

W = 2 splits the pair; W = 1 (or a plain `python scripts/bench_cfg_calls.py`) takes the single-GPU column only.  Workload = bench.py's:
ChronoEdit-14B, 720p, bench.py's latent frames, random weights, context cache on.  --mode fp8 is FP8 weights plus FP8 attention.
Prints one JSON line with ms per step for the split and for one GPU in the same run, the card's name and power limit, and whether
every rank's combined prediction was bit-identical to the single-GPU step."""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import bench
    import chronoedit_b200 as ce
    from chronoedit_b200 import parallel
    from scripts.bench_cfg_parallel import card

    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="bf16", choices=["bf16", "fp8"])
    ap.add_argument("--latent-frames", type=int, default=bench.FRAMES, choices=[2, 8])
    ap.add_argument("--layers", type=int, default=40)
    ap.add_argument("--steps", type=int, default=6)
    args = ap.parse_args()
    distributed = "RANK" in os.environ
    rank, local, world = (int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])) if distributed else (0, 0, 1)
    if world > 2:
        raise SystemExit("the call-pair split runs on 2 ranks (the grid with the token split is not timed here)")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if distributed:
        dist.init_process_group("nccl", device_id=dev)

    model = ce.ChronoEditTransformer3DModel(**bench.model_config(args.layers), device=dev, cache_context=True)
    bench.init_weights_(model, seed=0)          # same seed on every rank: identical weights without a broadcast
    if args.mode == "fp8":
        model.enable_fp8()
        model.enable_fp8_attention()
    model.pack_weights()
    T, H, W = args.latent_frames, bench.LAT_H, bench.LAT_W
    g = torch.Generator(device=dev).manual_seed(7)
    x = torch.randn(1, 36, T, H, W, generator=g, device=dev).bfloat16()
    prompt = torch.randn(1, bench.TEXT_LEN, 4096, generator=g, device=dev).bfloat16()
    prompt[:, 120:] = 0
    negative = torch.randn(1, bench.TEXT_LEN, 4096, generator=g, device=dev).bfloat16()
    negative[:, 40:] = 0
    img = torch.randn(1, 257, 1280, generator=g, device=dev).bfloat16()
    t = torch.full((1,), 500.0, device=dev)

    def step():
        noise_pred = model(hidden_states=x, timestep=t, encoder_hidden_states=prompt, encoder_hidden_states_image=img, return_dict=False)[0]
        noise_uncond = model(hidden_states=x, timestep=t, encoder_hidden_states=negative, encoder_hidden_states_image=img,
                             return_dict=False)[0]
        return noise_uncond + 5.0 * (noise_pred - noise_uncond)

    def timed(n):
        step()                                   # warm-up (context cache, workspaces)
        step()
        if distributed:
            dist.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            out = step()
        e1.record()
        torch.cuda.synchronize()
        ms = torch.tensor([e0.elapsed_time(e1) / n], device=dev)
        if distributed:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms), out

    single_ms, single = timed(args.steps)        # every rank runs both calls by itself
    split_ms, same, region = None, True, 0
    if world == 2:
        region = parallel.enable_cfg_parallel_calls(model, 1, T, H, W)
        split_ms, out = timed(args.steps)
        same = torch.equal(out, single)
        parallel.disable_cfg_parallel_calls(model)
    if distributed:
        flag = torch.tensor([int(same)], device=dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        same = bool(flag.item())
    name, limit = card()
    if rank == 0:
        print(json.dumps({
            "workload": f"ChronoEdit-14B ({args.layers} layers), latent [1,36,{T},{H},{W}] = {T * (H // 2) * (W // 2)} tokens, one step "
                        f"of the unchanged pipeline: prompt call + negative-prompt call + guidance combine, mode {args.mode}",
            "world": world, "card": name, "power_limit_and_max_sm_clock": limit,
            "ms_per_step_single_gpu": single_ms, "ms_per_step_split": split_ms,
            "speedup": None if split_ms is None else single_ms / split_ms, "bit_identical_on_all_ranks": same,
            "peer_region_bytes_per_rank": region}), flush=True)
    if distributed:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
