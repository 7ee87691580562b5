"""The tiled VAE on the GPU (enable_tiling): the blend launch bit for bit against the oracle's blend, the mirror's tiled encode and
decode against the fp32 oracle's tiled rule (bf16: the acceptance rule of test_gpu_vae.py; fp32: rtol 1e-3 / atol 1e-4 as the fp32
VAE is held), a one-tile grid against the untiled call, the workspace, and the unchanged pipeline with tiling and slicing on.
Tiles of 64 px with a 48 px stride over 200 x 328 px give a ragged grid of 5 x 7 tiles quickly.  Each comparison prints one JSON
line."""
import ctypes
import json

import pytest
import torch

from tests import vae_tiling_oracle as VT

gpu = pytest.mark.gpu
TILES = (64, 64, 48, 48)
H, W = 200, 328


def _report(**kw):
    print(json.dumps(kw))


def _configs():
    from oracle import vae_oracle as V

    return {"tiny": V.VAEConfig.tiny(32), "wan21": V.VAEConfig.wan21()}


def _vae(cfg, sd, dtype):
    from chronoedit_b200.autoencoder import AutoencoderKLWan

    m = AutoencoderKLWan(base_dim=cfg.dim, z_dim=cfg.z_dim, dim_mult=tuple(cfg.dim_mult), num_res_blocks=cfg.num_res_blocks,
                         temperal_downsample=tuple(cfg.temperal_downsample), torch_dtype=dtype, clamp_output=False)
    m.load_state_dict({k: v.to(dtype) for k, v in sd.items()}, strict=True)
    return m.cuda()


def _inputs(frames, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(1, 3, frames, H, W, generator=g) * 2 - 1
    z = torch.randn(1, 16, 1 + (frames - 1) // 4, H // 8, W // 8, generator=g)
    return x.cuda(), z.cuda()


# ---------------------------------------------------------------------------------------------------------------- the blend launch
@gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("layout", ["aligned", "ragged"])
def test_blend_launch_matches_the_oracle(dtype, layout):
    """A 3 x 3 grid of random tiles (ragged edges; odd widths force the scalar path) walked as the C tile loop walks it: each tile
    blended against the strip of the tile above and the tail of the tile to its left, both written by earlier launches."""
    import chronoedit_b200._lib as L

    heights, widths, ev, eh, crop = ((40, 40, 17), (40, 40, 16), 16, 16, 24) if layout == "aligned" else \
        ((40, 40, 17), (41, 41, 9), 13, 11, 27)
    g = torch.Generator().manual_seed(11)
    C, T = 3, 5
    grid = [[(torch.randn(1, C, T, hh, ww, generator=g) * 2).to(dtype) for ww in widths] for hh in heights]
    want = VT.blend_grid([[t.clone() for t in row] for row in grid], ev, eh, crop, crop, 10 ** 6, 10 ** 6).cuda()
    out = torch.full(want.shape[1:], float("nan"), dtype=dtype, device="cuda")
    strips, tails = {}, {}
    for i, hh in enumerate(heights):
        for j, ww in enumerate(widths):
            tile = grid[i][j][0].cuda().contiguous()
            a = L.TileBlendArgsC(fp32=int(dtype == torch.float32), tile=tile.data_ptr(), C=C, T=T, th=hh, tw=ww,
                                 out=out.data_ptr(), out_h=out.shape[2], out_w=out.shape[3], oy=i * crop, ox=j * crop, crop_h=crop,
                                 crop_w=crop)
            if i > 0:
                a.above, a.above_h = strips[i - 1, j].data_ptr(), strips[i - 1, j].shape[2]
            if j > 0:
                a.left, a.left_w = tails[i, j - 1].data_ptr(), tails[i, j - 1].shape[3]
            strips[i, j] = torch.empty(C, T, min(ev, hh), ww, dtype=dtype, device="cuda")
            tails[i, j] = torch.empty(C, T, hh, min(eh, ww), dtype=dtype, device="cuda")
            a.strip, a.strip_h = strips[i, j].data_ptr(), strips[i, j].shape[2]
            a.tail, a.tail_w = tails[i, j].data_ptr(), tails[i, j].shape[3]
            L.check(L.lib().ce_vae_tile_blend(ctypes.byref(a), L.current_stream()))
    torch.cuda.synchronize()
    assert torch.equal(out, want[0]), (out.float() - want[0].float()).abs().max()


# ---------------------------------------------------------------------------------------------------------------- the mirror
def _oracle(sd, cfg, what, x, dtype):
    s = {k: v.to(device="cuda", dtype=dtype) for k, v in sd.items()}
    x = x.to(dtype)
    return (VT.vae_encode_tiled(s, cfg, x, TILES) if what == "encode" else VT.vae_decode_tiled(s, cfg, x, TILES)).float()


def _call(m, what, x):
    return m.encode(x).latent_dist.mode() if what == "encode" else m.decode(x, return_dict=False)[0]


@gpu
@pytest.mark.parametrize("name,frames", [("tiny", 1), ("tiny", 5), ("tiny", 9), ("wan21", 1), ("wan21", 5), ("wan21", 9)])
def test_tiled_bf16_matches_the_tiled_oracle(name, frames):
    from oracle import vae_oracle as V

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = _configs()[name]
    sd = V.random_state_dict(cfg, seed=41)
    x, z = _inputs(frames, seed=42 + frames)
    m = _vae(cfg, sd, torch.bfloat16)
    m.enable_tiling(*TILES)
    for what, inp in (("encode", x), ("decode", z)):
        got = _call(m, what, inp).float()
        assert m.launches() > 0
        ref32, ref16 = _oracle(sd, cfg, what, inp, torch.float32), _oracle(sd, cfg, what, inp, torch.bfloat16)
        assert got.shape == ref32.shape and torch.isfinite(got).all()
        e_ref, e_our = (ref16 - ref32).abs(), (got - ref32).abs()
        _report(case=f"{name}_{frames}f", out=what, ours_mean=e_our.mean().item(), ref_bf16_mean=e_ref.mean().item(),
                ours_max=e_our.max().item(), ref_bf16_max=e_ref.max().item())
        assert e_our.mean() <= 1.25 * e_ref.mean(), f"{what}: mean err {e_our.mean():.3g} vs the oracle's bf16 {e_ref.mean():.3g}"
        assert e_our.max() <= 2.0 * e_ref.max(), f"{what}: max err {e_our.max():.3g} vs the oracle's bf16 {e_ref.max():.3g}"


@gpu
@pytest.mark.parametrize("name,frames", [("tiny", 9), ("wan21", 5)])
def test_tiled_fp32_matches_the_tiled_oracle(name, frames):
    from oracle import vae_oracle as V

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = _configs()[name]
    sd = V.random_state_dict(cfg, seed=43)
    x, z = _inputs(frames, seed=44)
    m = _vae(cfg, sd, torch.float32)
    m.enable_tiling(*TILES)
    for what, inp in (("encode", x), ("decode", z)):
        got = _call(m, what, inp)
        ref = _oracle(sd, cfg, what, inp, torch.float32)
        assert got.dtype == torch.float32 and got.shape == ref.shape
        e = (got - ref).abs()
        _report(case=f"fp32_{name}_{frames}f", out=what, max_err=e.max().item(), mean_err=e.mean().item())
        assert torch.allclose(got, ref, rtol=1e-3, atol=1e-4), e.max()


@gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_one_tile_grid_is_the_untiled_call(dtype):
    """Tiles as large as the frame: the tiled entry points return the untiled call's bits (the untiled decode without its clamp)."""
    from oracle import vae_oracle as V

    cfg = _configs()["tiny"]
    m = _vae(cfg, V.random_state_dict(cfg, seed=45), dtype)
    x, z = (t.to(dtype) for t in _inputs(5, seed=46))
    m.enable_tiling(H, W, H, W)
    moments = lambda: torch.full((1, 2 * cfg.z_dim, 2, H // 8, W // 8), float("nan"), dtype=dtype, device="cuda")
    video = lambda: torch.full((1, 3, 5, H, W), float("nan"), dtype=dtype, device="cuda")
    for decode, inp, alloc, untiled in ((False, x, moments, m._native_encode), (True, z, video, m._native_decode)):
        ref, got = alloc(), alloc()
        untiled(inp, ref)   # the mirror was built with clamp_output=False
        m._native_tiled(inp, got, decode=decode)
        assert torch.equal(got, ref)


@gpu
def test_tiled_workspace_is_bounded_by_the_tile():
    """Wan2.1 widths, default tiles: the tiled workspace does not grow with the height, grows with the width by the blend strips only,
    and is far below the untiled workspace at 720p."""
    from oracle import vae_oracle as V

    import chronoedit_b200._lib as L

    cfg = _configs()["wan21"]
    m = _vae(cfg, V.random_state_dict(cfg, seed=47), torch.bfloat16)
    m.pack_weights()
    lib, hd, tiles = L.lib(), m._handle, VT.DEFAULT_TILES
    rep = {}
    for decode, T, geo in ((0, 5, lambda a, b: (a, b)), (1, 2, lambda a, b: (a // 8, b // 8))):
        t720 = lib.ce_vae_workspace_bytes_tiled(hd, decode, T, *geo(720, 1280), *tiles)
        t2160 = lib.ce_vae_workspace_bytes_tiled(hd, decode, T, *geo(2160, 1280), *tiles)
        t4k = lib.ce_vae_workspace_bytes_tiled(hd, decode, T, *geo(2160, 3840), *tiles)
        u720 = lib.ce_vae_workspace_bytes(hd, decode, T, *geo(720, 1280))
        rep["decode" if decode else "encode"] = {"tiled_720p": t720, "tiled_2160x1280": t2160, "tiled_2160x3840": t4k, "untiled_720p": u720}
        assert 0 < t720 == t2160 < u720
        assert t720 < t4k < t720 + (64 << 20)   # the strips of 13 more tile columns: tens of MB at most
    _report(workspace=rep)


# ---------------------------------------------------------------------------------------------------------------- the pipeline
@gpu
def test_pipeline_with_tiling_and_slicing():
    """The unchanged pipeline's edit (oracle/pipeline_oracle.py harness) with pipe.vae.enable_tiling() and enable_slicing(): the CUDA
    mirrors against the oracle pipeline with the same tiled rule, as test_gpu_pipeline.py holds them."""
    import chronoedit_b200 as ce
    from chronoedit_b200.autoencoder import AutoencoderKLWan
    from oracle import cases, pipeline_cases as PC

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda", 0)
    case = PC.PIPELINE_CASES["edit_5f"]
    dsd, vsd = PC.weights()
    cfg = PC.DIT_CFG
    tr = ce.ChronoEditTransformer3DModel(
        patch_size=cfg.patch_size, num_attention_heads=cfg.num_attention_heads, attention_head_dim=cfg.attention_head_dim,
        in_channels=cfg.in_channels, out_channels=cfg.out_channels, text_dim=cfg.text_dim, freq_dim=cfg.freq_dim, ffn_dim=cfg.ffn_dim,
        num_layers=cfg.num_layers, eps=cfg.eps, image_dim=cfg.image_dim, added_kv_proj_dim=cfg.added_kv_proj_dim, cache_context=True)
    tr.load_state_dict(cases.to_bf16_state(dsd))
    vc = PC.VAE_CFG
    vae = AutoencoderKLWan(base_dim=vc.dim, z_dim=vc.z_dim, dim_mult=tuple(vc.dim_mult), num_res_blocks=vc.num_res_blocks,
                           temperal_downsample=tuple(vc.temperal_downsample))
    vae.load_state_dict({k: v.to(torch.bfloat16) for k, v in vsd.items()})
    vae.enable_tiling(*TILES)
    vae.enable_slicing()
    tr, vae = tr.to(dev), vae.to(dev)
    ours = PC.run_oracle_pipeline(case, torch.bfloat16, device=dev, transformer=tr, vae=vae,
                                  scheduler=ce.FlowUniPCMultistepScheduler(shift=case.sched_shift)).float()

    def oracle(dtype):
        v = VT.TiledOracleVAE({k: t.to(dev, dtype) for k, t in vsd.items()}, vc, dtype, TILES)
        out = PC.run_oracle_pipeline(case, dtype, device=dev, vae=v).float()
        assert v.tiled_calls >= 2   # the condition video's encode and the decode
        return out

    ref16, ref32 = oracle(torch.bfloat16), oracle(torch.float32)
    torch.cuda.synchronize()
    assert ours.shape == ref32.shape and torch.isfinite(ours).all()
    e_ref, e_our = (ref16 - ref32).abs(), (ours - ref32).abs()
    _report(case="pipeline_edit_5f_tiled", ours_mean=e_our.mean().item(), ref_bf16_mean=e_ref.mean().item(), ours_max=e_our.max().item(),
            ref_bf16_max=e_ref.max().item())
    assert e_our.mean() <= 1.25 * e_ref.mean()
    assert e_our.max() <= 2.0 * e_ref.max() + 1e-3
