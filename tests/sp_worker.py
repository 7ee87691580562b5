"""Worker of tests/test_gpu_seqpar.py (run under torchrun, one process per GPU): the split DiT forward and the split VAE's encode and
decode must be bit-identical to the single-GPU calls on every rank.  Arguments: the checks to run, "dit" and / or "vae" (none: both)."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def check_dit(rank, world, dev):
    import chronoedit_b200 as ce
    from chronoedit_b200 import parallel

    ok = True
    # (heads, dim = heads*128, latent T, H, W): 512 tokens (256 per rank at world 2) and 1920 tokens (960 per rank: query tiles of 128 rows
    # straddle the rank boundary), batch 2
    for heads, (T, H, W), B in ((2, (2, 32, 32), 1), (4, (2, 48, 40), 2), (8, (8, 24, 20), 1)):
        if heads % world or (T * (H // 2) * (W // 2)) % world:
            continue
        m = ce.ChronoEditTransformer3DModel(num_attention_heads=heads, in_channels=36, out_channels=16, ffn_dim=1024, num_layers=2, image_dim=1280,
                                            added_kv_proj_dim=heads * 128, device=dev)
        g = torch.Generator(device=dev).manual_seed(1234)          # same seed on every rank: identical weights
        for n, p in m.named_parameters():
            if ".norm" in n and n.endswith("weight"):
                p.data.normal_(0, 0.1, generator=g).add_(1.0)
            else:
                p.data.normal_(0, 0.03, generator=g)
        gi = torch.Generator(device=dev).manual_seed(99)
        x = torch.randn(B, 36, T, H, W, generator=gi, device=dev).bfloat16()
        text = torch.randn(B, 512, 4096, generator=gi, device=dev).bfloat16()
        img = torch.randn(B, 257, 1280, generator=gi, device=dev).bfloat16()
        t = torch.full((B,), 613, device=dev)
        single = m(x, t, text, img, return_dict=False)[0].clone()
        parallel.enable_sequence_parallel(m, B, T, H, W)
        for it in range(3):
            out = m(x, t, text, img, return_dict=False)[0]
            torch.cuda.synchronize()
            same = torch.equal(out, single)
            print(f"rank {rank}: heads={heads} latent=({T},{H},{W}) B={B} iter {it}: sequence-parallel == single-GPU: {same}"
                  + ("" if same else f"  max|diff|={float((out.float() - single.float()).abs().max()):.4g}"), flush=True)
            ok = ok and same
        parallel.disable_sequence_parallel(m)
        again = m(x, t, text, img, return_dict=False)[0]
        ok = ok and torch.equal(again, single)
        del m
    return ok


def check_vae(rank, world, dev):
    from chronoedit_b200 import parallel
    from chronoedit_b200.autoencoder import AutoencoderKLWan

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
    return ok


def main():
    checks = {"dit": check_dit, "vae": check_vae}
    names = sys.argv[1:] or list(checks)
    assert all(n in checks for n in names), f"usage: sp_worker.py [dit] [vae]; got {names}"
    rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    ok = True
    for n in names:
        ok = checks[n](rank, world, dev) and ok
    flag = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.destroy_process_group()
    sys.exit(0 if int(flag.item()) == 1 else 1)


if __name__ == "__main__":
    main()
