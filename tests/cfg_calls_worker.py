"""Worker of tests/test_gpu_cfg_calls.py (run under torchrun, two processes, one per GPU): the call-pair split of an 8-step
pipeline-order loop with FP8 weights, FP8 attention and TeaCache must give, on both ranks, the single-GPU loop's combined noise
predictions bit for bit, and each rank's TeaCache records must be the single-GPU records of the conditioning it computes."""
import dataclasses
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import chronoedit_b200 as ce
    from chronoedit_b200 import parallel
    from tests.test_gpu_cfg_calls_one_gpu import _loop, _loop_inputs

    rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    heads, latent = 4, (2, 32, 32)
    m = ce.ChronoEditTransformer3DModel(num_attention_heads=heads, in_channels=36, out_channels=16, ffn_dim=1024, num_layers=2, image_dim=1280,
                                        added_kv_proj_dim=heads * 128, device=dev, cache_context=True)
    g = torch.Generator(device=dev).manual_seed(1234)          # same seed on every rank: identical weights
    for n, p in m.named_parameters():
        if ".norm" in n and n.endswith("weight"):
            p.data.normal_(0, 0.1, generator=g).add_(1.0)
        else:
            p.data.normal_(0, 0.03, generator=g)
    m.enable_fp8()
    m.enable_fp8_attention()
    m.enable_teacache(1e9, num_inference_steps=8)
    inp = _loop_inputs(latent, dev, seed=99, steps=8)
    single = _loop(m, inp)
    single_records = m.teacache_records
    m.reset_teacache()
    parallel.enable_cfg_parallel_calls(m, 1, *latent)
    split = _loop(m, inp)
    torch.cuda.synchronize()
    records = m.teacache_records
    parallel.disable_cfg_parallel_calls(m)
    same = all(torch.equal(a, b) for a, b in zip(split, single))
    want = [dataclasses.replace(e, slot=0) for e in single_records if e.slot == rank]
    same_records = list(records) == want
    skipped = sum(not e.computed for e in records)
    print(f"rank {rank}: FP8 + FP8 attention + TeaCache, 8 steps: call-pair split == single-GPU: {same}, records equal: {same_records} "
          f"({skipped} of {len(records)} calls skipped)", flush=True)
    ok = same and same_records and skipped > 0
    flag = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.destroy_process_group()
    sys.exit(0 if int(flag.item()) == 1 and world == 2 else 1)


if __name__ == "__main__":
    main()
