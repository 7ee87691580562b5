"""Worker of tests/test_gpu_cfg_parallel.py (run under torchrun, one process per GPU): the batch-split DiT forward with FP8 weights and
FP8 attention must return, on every rank, the single-GPU forward of the full batch bit for bit."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import chronoedit_b200 as ce
    from chronoedit_b200 import parallel

    rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    ok = True
    heads, (T, H, W) = 4, (2, 32, 32)
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
    for B in (world, 2 * world):
        gi = torch.Generator(device=dev).manual_seed(99 + B)
        x = torch.randn(B, 36, T, H, W, generator=gi, device=dev).bfloat16()
        text = torch.randn(B, 512, 4096, generator=gi, device=dev).bfloat16()
        img = torch.randn(B, 257, 1280, generator=gi, device=dev).bfloat16()
        t = torch.tensor([900 - 37 * b for b in range(B)], device=dev)
        single = m(x, t, text, img, return_dict=False)[0].clone()
        parallel.enable_cfg_parallel(m, B, T, H, W)
        for it in range(3):
            out = m(x, t, text, img, return_dict=False)[0]
            torch.cuda.synchronize()
            same = torch.equal(out, single)
            print(f"rank {rank}: FP8 + FP8 attention B={B} iter {it}: batch split == single-GPU: {same}"
                  + ("" if same else f"  max|diff|={float((out.float() - single.float()).abs().max()):.4g}"), flush=True)
            ok = ok and same
        parallel.disable_cfg_parallel(m)
        ok = ok and torch.equal(m(x, t, text, img, return_dict=False)[0], single)
    flag = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.destroy_process_group()
    sys.exit(0 if int(flag.item()) == 1 else 1)


if __name__ == "__main__":
    main()
