#!/usr/bin/env python
"""The Wan2.1 VAE (96..384 channels) untiled and tiled (enable_tiling() with diffusers' default 256 px tiles at a 192 px stride), in
bf16 and fp32: ms and workspace bytes of an encode of 5 frames and of decodes of 2 / 5 / 8 latent frames (5 / 17 / 29 pixel frames)
at 720 x 1280, 1056 x 1584 (the upscaler example) and 2160 x 3840.  An untiled call whose workspace does not fit beside its input
and output in the free device memory is reported by its workspace bytes only.  Then, in a profiled run of its own, the blend
launches' share of a tiled decode's kernel time and their bandwidth against the data sheet's 3.35 TB/s.

    python scripts/bench_vae_tiling.py [--iters 1] [--warmup 1] [--sizes 720x1280,1056x1584,2160x3840] [--dtypes bf16,fp32]

Random weights; CUDA events around `iters` back-to-back calls after `warmup` calls of the same shape (no warm-up at 2160 x 3840,
where one call takes seconds and every kernel has been loaded by the smaller sizes).  Prints one JSON line per measurement and a
last line with the card's name and power limit."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

TILES = (256, 256, 192, 192)
OPS = (("encode_5f", False, 5), ("decode_2l", True, 2), ("decode_5l", True, 5), ("decode_8l", True, 8))


def blend_bytes(decode, frames, H, W, es, z_dim=16, tiles=TILES):
    """Bytes the blend launches of one tiled call read and write: the tile, the rows of the strip above and the columns of the tail to
    the left that it blends with; the crop, the strip and the tail it stores (csrc/vae.cu run_tiled)."""
    mh, mw, sh, sw = (t // 8 for t in tiles)
    h, w = H // 8, W // 8
    f = 8 if decode else 1
    C, T = (3, 1 + 4 * (frames - 1)) if decode else (2 * z_dim, 1 + (frames - 1) // 4)
    bv, bw = (mh - sh) * f, (mw - sw) * f
    rows, cols = -(-h // sh), -(-w // sw)
    total = 0
    for i in range(rows):
        for j in range(cols):
            th, tw = min(mh, h - i * sh) * f, min(mw, w - j * sw) * f
            n = th * tw                                                       # the tile
            if i > 0:
                n += min(bv, min(mh, h - (i - 1) * sh) * f, th) * tw          # strip rows read
            if j > 0:
                n += th * min(bw, min(mw, w - (j - 1) * sw) * f, tw)          # tail columns read
            n += min(sh * f, th) * min(sw * f, tw)                            # crop
            n += (min(bv, th) * tw if i + 1 < rows else 0) + (th * min(bw, tw) if j + 1 < cols else 0)
            total += n * C * T * es
    return total


def main():
    from chronoedit_b200 import _lib
    from chronoedit_b200.autoencoder import AutoencoderKLWan
    from oracle import vae_oracle as V
    from scripts.bench_cfg_parallel import card

    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=1)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sizes", default="720x1280,1056x1584,2160x3840")
    ap.add_argument("--dtypes", default="bf16,fp32")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg = V.VAEConfig.wan21()
    sd = V.random_state_dict(cfg, seed=41)
    sizes = [tuple(int(v) for v in s.split("x")) for s in args.sizes.split(",")]
    L = _lib.lib()
    name, limit = card()
    for label in args.dtypes.split(","):
        dtype = {"bf16": torch.bfloat16, "fp32": torch.float32}[label]
        es = 2 if dtype == torch.bfloat16 else 4
        m = AutoencoderKLWan(torch_dtype=dtype, clamp_output=False)
        m.load_state_dict({k: v.to(dtype) for k, v in sd.items()})
        m = m.to(dev)
        m.pack_weights()
        ws_fn = L.ce_vae_workspace_bytes_fp32 if dtype == torch.float32 else L.ce_vae_workspace_bytes
        ws_tiled_fn = L.ce_vae_workspace_bytes_tiled_fp32 if dtype == torch.float32 else L.ce_vae_workspace_bytes_tiled
        for H, W in sizes:
            g = torch.Generator(device="cpu").manual_seed(42)
            for what, decode, frames in OPS:
                geo = (frames, H // 8, W // 8) if decode else (frames, H, W)
                x = (torch.randn(1, 16, *geo, generator=g) if decode else torch.rand(1, 3, *geo, generator=g) * 2 - 1).to(dev, dtype)
                out_bytes = (3 * (1 + 4 * (frames - 1)) * H * W if decode else 32 * (1 + (frames - 1) // 4) * (H // 8) * (W // 8)) * es
                for tiled in (False, True):
                    ws = (ws_tiled_fn(m._handle, int(decode), *geo, *TILES) if tiled else ws_fn(m._handle, int(decode), *geo))
                    rec = {"dtype": label, "size": f"{H}x{W}", "op": what, "tiled": tiled, "workspace_bytes": ws,
                           "blend_bytes": blend_bytes(decode, frames, H, W, es) if tiled else 0}
                    m._ws = None
                    torch.cuda.empty_cache()
                    if ws + out_bytes + (2 << 30) > torch.cuda.mem_get_info()[0]:
                        rec["ms"] = "does not fit"
                        print(json.dumps(rec), flush=True)
                        continue
                    if tiled:
                        m.enable_tiling(*TILES)
                    else:
                        m.disable_tiling()
                    call = (lambda: m.decode(x, return_dict=False)[0]) if decode else (lambda: m.encode(x).latent_dist.mode())
                    for _ in range(args.warmup if H * W < 2160 * 3840 else 0):
                        call()
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.iters):
                        out = call()
                    e1.record()
                    torch.cuda.synchronize()
                    rec["ms"] = round(e0.elapsed_time(e1) / args.iters, 2)
                    rec["launches"] = m.launches()
                    del out
                    print(json.dumps(rec), flush=True)
                del x
        # the blend launches' share of a tiled 720p decode of 5 latent frames, from the kernel trace of one call
        H, W, frames = 720, 1280, 5
        m.enable_tiling(*TILES)
        z = torch.randn(1, 16, frames, H // 8, W // 8, generator=torch.Generator().manual_seed(43)).to(dev, dtype)
        m.decode(z, return_dict=False)
        torch.cuda.synchronize()
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            m.decode(z, return_dict=False)
            torch.cuda.synchronize()
        total = blend = 0.0
        n_blend = 0
        for ev in prof.key_averages():
            t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            if t <= 0:
                continue
            total += t
            if "tile_blend_kernel" in ev.key:
                blend += t
                n_blend += ev.count
        nbytes = blend_bytes(True, frames, H, W, es)
        print(json.dumps({"dtype": label, "profile": "tiled decode 5 latent frames 720x1280", "blend_launches": n_blend,
                          "blend_us": round(blend, 1), "kernel_us": round(total, 1), "blend_share": round(blend / total, 5) if total else None,
                          "blend_bytes": nbytes, "blend_GBps": round(nbytes / (blend * 1e-6) / 1e9, 1) if blend else None,
                          "blend_share_of_3350GBps": round(nbytes / (blend * 1e-6) / 3.35e12, 3) if blend else None}), flush=True)
        del m, z
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "vae_tiling", "gpu": name, "power_limit_and_max_sm_clock": limit, "tiles": TILES, "iters": args.iters,
                      "warmup": args.warmup}), flush=True)


if __name__ == "__main__":
    main()
