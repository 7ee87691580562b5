"""Host checks of the tiled VAE (enable_tiling / enable_slicing) that need no GPU: the blend rule against a literal transcription of
diffusers' blend_v / blend_h and against the rounding the device kernel implements, tiled = untiled when one tile covers the frame,
the mirror's switches and trigger conditions, the C library's refusals, and the tiled workspace's dependence on the frame size."""
import ctypes

import pytest
import torch

from oracle import vae_oracle as V
from tests import vae_tiling_oracle as VT


class _DiffusersBlend:
    """diffusers 0.35.2 AutoencoderKLWan.blend_v / blend_h, as methods, transcribed line by line."""

    def blend_v(self, a, b, blend_extent):
        blend_extent = min(a.shape[-2], b.shape[-2], blend_extent)
        for y in range(blend_extent):
            b[:, :, :, y, :] = a[:, :, :, -blend_extent + y, :] * (1 - y / blend_extent) + b[:, :, :, y, :] * (
                y / blend_extent
            )
        return b

    def blend_h(self, a, b, blend_extent):
        blend_extent = min(a.shape[-1], b.shape[-1], blend_extent)
        for x in range(blend_extent):
            b[:, :, :, :, x] = a[:, :, :, :, -blend_extent + x] * (1 - x / blend_extent) + b[:, :, :, :, x] * (
                x / blend_extent
            )
        return b


def _ragged_grid(dtype, seed, heights=(40, 40, 17), widths=(40, 40, 9), C=3, T=5):
    g = torch.Generator().manual_seed(seed)
    return [[(torch.randn(1, C, T, hh, ww, generator=g) * 2).to(dtype) for ww in widths] for hh in heights]


def _closed_form(a, b, k, e):
    """One blend step with the rounding the device kernel implements: fp32 weights from Python floats, each product rounded to the
    tile's dtype, then the sum rounded."""
    wa, wb = torch.tensor(1 - k / e, dtype=torch.float32), torch.tensor(k / e, dtype=torch.float32)
    pa, pb = (a.float() * wa).to(a.dtype).float(), (b.float() * wb).to(a.dtype).float()
    return (pa + pb).to(a.dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_blend_matches_diffusers_transcription(dtype):
    ref = _DiffusersBlend()
    for seed, (ev, eh) in enumerate(((16, 16), (64, 8), (3, 40))):
        ours, theirs = _ragged_grid(dtype, seed), _ragged_grid(dtype, seed)
        out = VT.blend_grid(ours, ev, eh, 24, 24, 10 ** 6, 10 ** 6)
        result_rows = []
        for i, row in enumerate(theirs):
            result_row = []
            for j, tile in enumerate(row):
                if i > 0:
                    tile = ref.blend_v(theirs[i - 1][j], tile, ev)
                if j > 0:
                    tile = ref.blend_h(row[j - 1], tile, eh)
                result_row.append(tile[:, :, :, :24, :24])
            result_rows.append(torch.cat(result_row, dim=-1))
        want = torch.cat(result_rows, dim=3)
        assert out.dtype == dtype and torch.equal(out, want)
        for i in range(len(ours)):   # every tile, tails included, as diffusers leaves it
            for j in range(len(ours[0])):
                assert torch.equal(ours[i][j], theirs[i][j])


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_blend_rounding_is_the_kernels(dtype):
    """blend_v / blend_h as torch evaluates them equal the per-element expression csrc/vae_kernels.cu implements."""
    g = torch.Generator().manual_seed(7)
    a = (torch.randn(1, 2, 3, 21, 13, generator=g) * 3).to(dtype)
    b0 = (torch.randn(1, 2, 3, 17, 13, generator=g) * 3).to(dtype)
    e = 16
    got = VT.blend_v(a, b0.clone(), e)
    want = b0.clone()
    for y in range(e):
        want[:, :, :, y, :] = _closed_form(a[:, :, :, -e + y, :], b0[:, :, :, y, :], y, e)
    assert torch.equal(got, want)
    a = (torch.randn(1, 2, 3, 9, 40, generator=g) * 3).to(dtype)
    b0 = (torch.randn(1, 2, 3, 9, 11, generator=g) * 3).to(dtype)
    got = VT.blend_h(a, b0.clone(), 64)   # extent clipped to b's 11 columns
    want = b0.clone()
    for x in range(11):
        want[..., x] = _closed_form(a[..., -11 + x], b0[..., x], x, 11)
    assert torch.equal(got, want)


def test_one_tile_equals_untiled():
    cfg = V.VAEConfig.tiny(32)
    sd = V.random_state_dict(cfg, seed=3)
    g = torch.Generator().manual_seed(4)
    x = torch.rand(1, 3, 5, 32, 48, generator=g) * 2 - 1
    z = torch.randn(1, cfg.z_dim, 2, 4, 6, generator=g)
    for tiles in ((32, 48, 32, 48), (64, 64, 48, 48), (256, 256, 192, 192)):
        assert torch.equal(VT.vae_encode_tiled(sd, cfg, x, tiles), V.vae_encode(sd, cfg, x))
        assert torch.equal(VT.vae_decode_tiled(sd, cfg, z, tiles), V.vae_decode(sd, cfg, z, clamp=False))


def test_tiled_grid_covers_the_frame():
    """A ragged multi-tile grid gives the untiled shapes, and tiles really were blended (the result differs from untiled)."""
    cfg = V.VAEConfig.tiny(32)
    sd = V.random_state_dict(cfg, seed=5)
    g = torch.Generator().manual_seed(6)
    z = torch.randn(1, cfg.z_dim, 1, 9, 13, generator=g)
    out = VT.vae_decode_tiled(sd, cfg, z, (32, 48, 24, 32))
    ref = V.vae_decode(sd, cfg, z, clamp=False)
    assert out.shape == ref.shape and not torch.equal(out, ref)
    x = torch.rand(1, 3, 1, 72, 104, generator=g) * 2 - 1
    mu = VT.vae_encode_tiled(sd, cfg, x, (32, 48, 24, 32))
    assert mu.shape == V.vae_encode(sd, cfg, x).shape


def _mirror(**kw):
    from chronoedit_b200.autoencoder import AutoencoderKLWan

    return AutoencoderKLWan(base_dim=32, **kw)


def test_mirror_switches_follow_diffusers():
    m = _mirror()
    assert (m.use_tiling, m.use_slicing) == (False, False)
    assert m._tiles() == VT.DEFAULT_TILES
    m.enable_tiling()
    assert m.use_tiling and m._tiles() == (256, 256, 192, 192)
    m.enable_tiling(tile_sample_min_height=128, tile_sample_stride_width=96)
    assert m._tiles() == (128, 256, 192, 96)
    m.enable_tiling(64, 64, 48, 48)
    assert m._tiles() == (64, 64, 48, 48)
    m.disable_tiling()
    assert not m.use_tiling and m._tiles() == (64, 64, 48, 48)   # the sizes stay, as in diffusers
    m.enable_slicing()
    assert m.use_slicing and not m.use_tiling
    m.disable_slicing()
    assert not m.use_slicing


def test_mirror_trigger_conditions():
    m = _mirror()
    assert not m._tiled_encode(1024, 1024) and not m._tiled_decode(128, 128)   # tiling off
    m.enable_tiling()
    assert not m._tiled_encode(256, 256) and m._tiled_encode(256, 264) and m._tiled_encode(264, 8)
    assert not m._tiled_decode(32, 32) and m._tiled_decode(32, 33) and m._tiled_decode(33, 1)
    m.enable_tiling(64, 128, 48, 96)
    assert m._tiled_encode(72, 128) and not m._tiled_encode(64, 128) and m._tiled_encode(64, 136)
    assert m._tiled_decode(9, 16) and not m._tiled_decode(8, 16) and m._tiled_decode(8, 17)
    for H, W in ((64, 128), (72, 128), (64, 136)):
        assert m._tiled_encode(H, W) == VT.tiles_encode(m._tiles(), H, W)
        assert m._tiled_decode(H // 8, W // 8) == VT.tiles_decode(m._tiles(), H // 8, W // 8)


def test_mirror_refuses_tiling_under_the_split_before_the_input():
    from chronoedit_b200._lib import CEError

    m = _mirror()
    m.enable_tiling(64, 64, 48, 48)
    m._sp_state = {"world": 2}
    x = torch.empty(1, 3, 5, 128, 128, device="meta")   # any read of it would fail differently
    with pytest.raises(CEError, match="not built for the VAE split"):
        m.encode(x)
    with pytest.raises(CEError, match="not built for the VAE split"):
        m.decode(torch.empty(1, 16, 2, 16, 16, device="meta"))


# ------------------------------------------------------------------------------------------------------------- the C library
def _handle_with_weights(cfg, fp32=False):
    """A VAE handle whose weights are registered with their packed sizes at fake addresses: enough for the host-side planning."""
    from chronoedit_b200 import _lib
    from chronoedit_b200.autoencoder import _param_shapes, pack_parameter, pack_parameter_fp32

    L = _lib.lib()
    c = _lib.VAEConfigC(cfg.dim, cfg.z_dim, (_lib.c_int32 * 4)(*cfg.dim_mult), cfg.num_res_blocks,
                        (_lib.c_int32 * 3)(*[int(b) for b in cfg.temperal_downsample]))
    h = ctypes.c_void_p()
    _lib.check(L.ce_vae_create(ctypes.byref(c), ctypes.byref(h)))
    shapes = _param_shapes(cfg.dim, cfg.z_dim, tuple(cfg.dim_mult), cfg.num_res_blocks, tuple(cfg.temperal_downsample))
    for name, shape in shapes.items():
        t = (pack_parameter_fp32 if fp32 else pack_parameter)(name, torch.zeros(shape))
        _lib.check((L.ce_vae_set_weight_fp32 if fp32 else L.ce_vae_set_weight)(h, name.encode(), ctypes.c_void_p(1 << 20), t.numel()))
    return L, h


def test_refusals_before_any_launch():
    L, h = _handle_with_weights(V.VAEConfig.tiny(32))
    try:
        for tiles, msg in (((64, 64, 72, 48), b"stride larger than the tile"), ((64, 64, 48, 44), b"multiples of 8"),
                           ((0, 64, 48, 48), b"multiples of 8")):
            assert L.ce_vae_workspace_bytes_tiled(h, 0, 5, 128, 128, *tiles) == -1
            assert msg in L.ce_last_error(), (tiles, L.ce_last_error())
            assert L.ce_vae_decode_tiled(h, ctypes.c_void_p(16), ctypes.c_void_p(16), 2, 16, 16, *tiles, 0, ctypes.c_void_p(256), 1 << 40,
                                         None) != 0
            assert msg in L.ce_last_error()
        regions = (ctypes.c_void_p * 2)(4096, 8192)
        assert L.ce_vae_sp_configure(h, 0, 2, regions, 1 << 30) == 0
        for fn, args in ((L.ce_vae_encode_tiled, (5, 128, 128, 64, 64, 48, 48)), (L.ce_vae_decode_tiled, (2, 16, 16, 64, 64, 48, 48, 0))):
            assert fn(h, ctypes.c_void_p(16), ctypes.c_void_p(16), *args, ctypes.c_void_p(256), 1 << 40, None) != 0
            assert b"not built for the VAE split" in L.ce_last_error()
        assert L.ce_vae_workspace_bytes_tiled(h, 1, 2, 16, 16, 64, 64, 48, 48) == -1
        assert L.ce_vae_sp_configure(h, 0, 1, None, 0) == 0
        assert L.ce_vae_workspace_bytes_tiled(h, 1, 2, 16, 16, 64, 64, 48, 48) > 0
    finally:
        L.ce_vae_destroy(h)


def _strip_bytes(Cout, Tout, tiles, es, decode):
    """One tile's strip: the last min - stride rows (latents when encoding) of the blended output tile, 256-byte aligned."""
    mh, mw, sh, sw = tiles
    rows, width = (mh - sh, mw) if decode else (mh // 8 - sh // 8, mw // 8)
    return (Cout * Tout * rows * width * es + 255) // 256 * 256


@pytest.mark.parametrize("fp32", [False, True])
def test_workspace_grows_with_the_width_by_the_strips_only(fp32):
    cfg = V.VAEConfig.tiny(32)
    L, h = _handle_with_weights(cfg, fp32)
    ws_tiled = L.ce_vae_workspace_bytes_tiled_fp32 if fp32 else L.ce_vae_workspace_bytes_tiled
    ws = L.ce_vae_workspace_bytes_fp32 if fp32 else L.ce_vae_workspace_bytes
    es = 4 if fp32 else 2
    tiles = (256, 256, 192, 192)
    try:
        for decode, T, Tout, Cout in ((1, 2, 5, 3), (0, 5, 2, 2 * cfg.z_dim)):
            geo = (lambda H, W: (H // 8, W // 8)) if decode else (lambda H, W: (H, W))
            n720 = ws_tiled(h, decode, T, *geo(720, 1280), *tiles)
            assert n720 > 0 and n720 == ws_tiled(h, decode, T, *geo(2160, 1280), *tiles)   # not with the height
            n4k = ws_tiled(h, decode, T, *geo(2160, 3840), *tiles)
            cols = lambda W: -(-(W // 8) // 24)
            assert n4k - n720 == 2 * (cols(3840) - cols(1280)) * _strip_bytes(Cout, Tout, tiles, es, decode)
            assert n720 < ws(h, decode, T, *geo(720, 1280))
    finally:
        L.ce_vae_destroy(h)
