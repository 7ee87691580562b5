#!/usr/bin/env python
"""The CFG pair of one edit split over GPUs (parallel.enable_cfg_parallel): prompt and negative prompt of bench.py's batch-2 forward,
one half per rank, optionally with the tokens of each half split further (--token-ranks, the grid).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node W --master-addr 127.0.0.1 scripts/bench_cfg_parallel.py \
        [--mode bf16|fp8|fp8-attn] [--token-ranks N] [--latent-frames 2] [--layers 40] [--steps 6]

W = 2 splits the pair; W = 2 N with --token-ranks N > 1 runs the grid (the pair over 2 ranks, the tokens of each half over N).  With
W = 1 only the single-GPU numbers are taken.  Workload = bench.py's: ChronoEdit-14B, 720p, bench.py's latent frames, random weights.
Prints one JSON line with ms per DiT forward of the pair for the split and for the single-GPU batch-2 forward in the same run, the
single-GPU batch-1 forward (the work one rank of the split does, without the exchange), the card's name and power limit, and whether
every rank's output was bit-identical to the single-GPU forward.  --mode fp8 is FP8 weights plus FP8 attention (bench_fp8.py's fastest
mode); fp8-attn is FP8 attention alone."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    """(name, power limit) of the current GPU, read in the same run as the numbers."""
    name = torch.cuda.get_device_name()
    try:
        idx = torch.cuda.current_device()
        q = subprocess.run(["nvidia-smi", f"--id={idx}", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        limit = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def main():
    import bench
    import chronoedit_b200 as ce
    from chronoedit_b200 import parallel

    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="bf16", choices=["bf16", "fp8", "fp8-attn"])
    ap.add_argument("--token-ranks", type=int, default=1, help="ranks per half of the pair for the token split (grid when > 1)")
    ap.add_argument("--latent-frames", type=int, default=bench.FRAMES, choices=[2, 8])
    ap.add_argument("--layers", type=int, default=40)
    ap.add_argument("--steps", type=int, default=6)
    args = ap.parse_args()
    rank, local, world = int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    N = args.token_ranks
    if world > 1 and world != 2 * N:
        raise SystemExit(f"--token-ranks {N} needs {2 * N} processes, got {world}")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    # every rank creates every group, in the same order: token groups {0..N-1}, {N..2N-1}; pair groups {j, j + N}
    token_group = pair_group = None
    if world > 1 and N > 1:
        tgs = [dist.new_group(list(range(i * N, (i + 1) * N))) for i in range(2)]
        pgs = [dist.new_group([j, j + N]) for j in range(N)]
        token_group, pair_group = tgs[rank // N], pgs[rank % N]

    model = ce.ChronoEditTransformer3DModel(**bench.model_config(args.layers), device=dev, cache_context=True)
    bench.init_weights_(model, seed=0)          # same seed on every rank: identical weights without a broadcast
    if args.mode == "fp8":
        model.enable_fp8()
    if args.mode in ("fp8", "fp8-attn"):
        model.enable_fp8_attention()
    model.pack_weights()
    T, H, W = args.latent_frames, bench.LAT_H, bench.LAT_W
    g = torch.Generator(device=dev).manual_seed(7)
    x = torch.randn(2, 36, T, H, W, generator=g, device=dev).bfloat16()
    text = torch.randn(2, bench.TEXT_LEN, 4096, generator=g, device=dev).bfloat16()
    text[0, 120:] = 0
    text[1, 40:] = 0
    img = torch.randn(1, 257, 1280, generator=g, device=dev).bfloat16().expand(2, -1, -1).contiguous()
    t = torch.full((2,), 500, device=dev)

    def timed(n, *inp):
        model(*inp, return_dict=False)        # warm-up (context cache, workspaces)
        model(*inp, return_dict=False)
        dist.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            out = model(*inp, return_dict=False)[0]
        e1.record()
        torch.cuda.synchronize()
        ms = torch.tensor([e0.elapsed_time(e1) / n], device=dev)
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms), out

    half = (x[:1].contiguous(), t[:1].contiguous(), text[:1].contiguous(), img[:1].contiguous())
    b1_ms, _ = timed(args.steps, *half)                 # what one rank of the pair split computes, without the exchange
    model.clear_context_cache()
    single_ms, single = timed(args.steps, x, t, text, img)   # every rank runs the whole pair by itself
    split_ms, same, region = None, True, 0
    if world > 1:
        if N > 1:
            region += parallel.enable_sequence_parallel(model, 1, T, H, W, group=token_group)
        region += parallel.enable_cfg_parallel(model, 2, T, H, W, group=pair_group)
        split_ms, out = timed(args.steps, x, t, text, img)
        same = torch.equal(out, single)
        parallel.disable_cfg_parallel(model)
        parallel.disable_sequence_parallel(model)
    flag = torch.tensor([int(same)], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    name, limit = card()
    if rank == 0:
        print(json.dumps({
            "workload": f"ChronoEdit-14B ({args.layers} layers), latent [2,36,{T},{H},{W}] = {T * (H // 2) * (W // 2)} tokens x CFG pair, "
                        f"one DiT forward, mode {args.mode}",
            "world": world, "token_ranks": N if world > 1 else 1, "card": name, "power_limit_and_max_sm_clock": limit,
            "ms_per_step_single_gpu_batch2": single_ms, "ms_per_step_single_gpu_batch1": b1_ms,
            "ms_per_step_split": split_ms, "speedup": None if split_ms is None else single_ms / split_ms,
            "batch1_over_batch2": b1_ms / single_ms, "bit_identical_on_all_ranks": bool(flag.item()),
            "peer_region_bytes_per_rank": region}), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
