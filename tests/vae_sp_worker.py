"""Worker of tests/test_gpu_vae_seqpar.py (run under torchrun, one process per GPU): the split VAE's encode and decode must be
bit-identical to the single-GPU call on every rank."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from chronoedit_b200 import parallel
    from chronoedit_b200.autoencoder import AutoencoderKLWan

    rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    ok = True
    for dim, (H, W) in ((32, (88, 56)), (96, (128, 96))):
        m = AutoencoderKLWan(base_dim=dim, device=dev)
        g = torch.Generator(device=dev).manual_seed(1234)          # same seed on every rank: identical weights
        with torch.no_grad():
            for n, p in m.named_parameters():
                if n.endswith("gamma"):
                    p.normal_(0, 0.1, generator=g).add_(1.0)
                elif n.endswith("bias"):
                    p.normal_(0, 0.05, generator=g)
                else:
                    p.normal_(0, p[0].numel() ** -0.5, generator=g)
        gi = torch.Generator(device=dev).manual_seed(99)
        video = (torch.rand(1, 3, 9, H, W, generator=gi, device=dev) * 2 - 1).bfloat16()
        z = torch.randn(1, 16, 3, H // 8, W // 8, generator=gi, device=dev).bfloat16()
        mu1 = m.encode(video).latent_dist.mode().clone()
        dec1 = m.decode(z, return_dict=False)[0].clone()
        parallel.enable_vae_sequence_parallel(m, H, W)
        for it in range(2):
            mu = m.encode(video).latent_dist.mode()
            dec = m.decode(z, return_dict=False)[0]
            torch.cuda.synchronize()
            same = torch.equal(mu, mu1) and torch.equal(dec, dec1)
            print(f"rank {rank}: dim={dim} {H}x{W} iter {it}: split == single-GPU: {same}", flush=True)
            ok = ok and same
        parallel.disable_vae_sequence_parallel(m)
        ok = ok and torch.equal(m.decode(z, return_dict=False)[0], dec1)
        del m
    flag = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.destroy_process_group()
    sys.exit(0 if int(flag.item()) == 1 else 1)


if __name__ == "__main__":
    main()
