"""Host checks of the VAE split over ranks (ce_vae_sp_*) that need no GPU: the peer region's size against a restatement of its layout,
and the refusals of the C entry points and of the Python plumbing."""
import ctypes

import pytest

from oracle.vae_oracle import VAEConfig


def halo_row_bytes(cfg, H, W):
    """The largest halo row of any chunk, in bytes: T frames x width x channels of every buffer that feeds a convolution with three
    kernel rows (both residual convolutions, the stride-2 downsample, the conv after an upsample, the heads).  Encode: a 4-frame chunk;
    decode: a chunk past the first (the one the temporal upsamples double)."""
    dims = [cfg.dim * m for m in (1,) + tuple(cfg.dim_mult)]
    top, nrb, td = dims[-1], cfg.num_res_blocks, list(cfg.temperal_downsample)
    rows = []
    T, w = 4, W
    for i in range(4):
        cin = dims[i]
        for _ in range(nrb):
            rows += [T * w * cin, T * w * dims[i + 1]]
            cin = dims[i + 1]
        if i != 3:
            rows.append(T * w * dims[i + 1])
            w = (w + 1 - 3) // 2 + 1
            if td[i]:
                T = (1 + T - 3) // 2 + 1
    rows += [T * w * top] * 5                      # middle.0, middle.2 (two each), head
    ddims = [top] + [cfg.dim * m for m in reversed(cfg.dim_mult)]
    T, w = 1, W // 8
    rows += [T * w * top] * 4
    for i in range(4):
        cin = ddims[i] // 2 if i >= 1 else ddims[i]
        for _ in range(nrb + 1):
            rows += [T * w * cin, T * w * ddims[i + 1]]
            cin = ddims[i + 1]
        if i != 3:
            if td[2 - i]:
                T *= 2
            w *= 2
            rows.append(T * w * ddims[i + 1])
    rows.append(T * w * ddims[4])
    return 2 * max(rows)


def vae_sp_layout(cfg, H, W):
    """Restatement of vae_sp_layout (csrc/vae.cu): byte offsets of a rank's peer region for pixel geometry H x W.  Sub-buffers start at
    multiples of 1024 bytes."""
    al = lambda v: (v + 1023) & ~1023
    h, w = H // 8, W // 8
    top = cfg.dim * cfg.dim_mult[-1]
    lay = {"flags": 0, "halo": 1024, "halo_slot": al(halo_row_bytes(cfg, H, W))}
    lay["frame"] = lay["halo"] + 4 * lay["halo_slot"]
    lay["frame_bytes"] = al((h * w + 7) // 8 * 8 * top * 2)
    lay["video"] = lay["frame"] + 2 * lay["frame_bytes"]
    lay["video_frames"] = 2 ** sum(bool(t) for t in cfg.temperal_downsample)
    lay["moments"] = lay["video"] + al(3 * lay["video_frames"] * H * W * 2)
    lay["moments_bytes"] = al(2 * cfg.z_dim * h * w * 2)
    lay["bytes"] = lay["moments"] + 2 * lay["moments_bytes"]
    return lay


def _handle(cfg):
    from chronoedit_b200 import _lib

    L = _lib.lib()
    c = _lib.VAEConfigC(cfg.dim, cfg.z_dim, (_lib.c_int32 * 4)(*cfg.dim_mult), cfg.num_res_blocks,
                        (_lib.c_int32 * 3)(*[int(b) for b in cfg.temperal_downsample]))
    h = ctypes.c_void_p()
    _lib.check(L.ce_vae_create(ctypes.byref(c), ctypes.byref(h)))
    return L, h


CONFIGS = {"tiny": VAEConfig.tiny(32), "wan21": VAEConfig.wan21(), "two_res": VAEConfig(dim=48, num_res_blocks=1)}


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_region_bytes_match_the_layout(name):
    cfg = CONFIGS[name]
    L, h = _handle(cfg)
    try:
        for H, W in ((64, 64), (64, 48), (128, 96), (720, 1280), (480, 832)):
            for world in range(2, 9):
                if H // 8 < world:
                    continue
                assert L.ce_vae_sp_region_bytes(h, H, W, world) == vae_sp_layout(cfg, H, W)["bytes"], (H, W, world)
    finally:
        L.ce_vae_destroy(h)


def test_region_bytes_refusals():
    L, h = _handle(CONFIGS["tiny"])
    try:
        for args, msg in (((64, 64, 1), b"world must be 2 to 8"), ((64, 64, 9), b"world must be 2 to 8"),
                          ((32, 48, 5), b"4 latent rows cannot be split over 5 ranks"), ((60, 64, 2), b"multiples of 8")):
            assert L.ce_vae_sp_region_bytes(h, *args) < 0
            assert msg in L.ce_last_error(), (args, L.ce_last_error())
        assert L.ce_vae_sp_region_bytes(None, 64, 64, 2) < 0
    finally:
        L.ce_vae_destroy(h)


def test_configure_refusals():
    L, h = _handle(CONFIGS["tiny"])
    try:
        good = (ctypes.c_void_p * 2)(4096, 8192)
        for rank, world, table, n in ((2, 2, good, 1 << 20), (-1, 2, good, 1 << 20), (0, 9, (ctypes.c_void_p * 9)(*[4096] * 9), 1 << 20),
                                      (0, 2, None, 1 << 20), (0, 2, good, 0), (0, 0, good, 1 << 20)):
            assert L.ce_vae_sp_configure(h, rank, world, table, n) != 0
            assert b"ce_vae_sp_configure: arguments" in L.ce_last_error()
        for table in ((ctypes.c_void_p * 2)(4096, None), (ctypes.c_void_p * 2)(4096, 8192 + 16)):
            assert L.ce_vae_sp_configure(h, 0, 2, table, 1 << 20) != 0
            assert b"256-byte aligned" in L.ce_last_error()
        assert L.ce_vae_sp_configure(None, 0, 1, None, 0) != 0
        assert L.ce_vae_sp_configure(h, 0, 1, None, 0) == 0   # world 1: off, whatever else is passed
    finally:
        L.ce_vae_destroy(h)


def test_host_barrier_arguments():
    L, h = _handle(CONFIGS["tiny"])
    try:
        assert L.ce_vae_sp_host_barrier(h, -1) != 0 and b"ce_vae_sp_host_barrier: arguments" in L.ce_last_error()
        assert L.ce_vae_sp_host_barrier(None, 100) != 0
        assert L.ce_vae_sp_host_barrier(h, 100) == 0
        assert L.ce_vae_sp_host_barrier(h, 0) == 0   # back to the device barrier
    finally:
        L.ce_vae_destroy(h)


def test_enable_needs_a_process_group():
    import torch.distributed as dist

    import chronoedit_b200 as ce
    from chronoedit_b200 import parallel
    from chronoedit_b200.autoencoder import AutoencoderKLWan

    assert not dist.is_initialized()
    vae = AutoencoderKLWan(base_dim=32)
    with pytest.raises(ce.CEError, match="initialised torch.distributed process group"):
        parallel.enable_vae_sequence_parallel(vae, 64, 64)
    parallel.disable_vae_sequence_parallel(vae)   # nothing to release
