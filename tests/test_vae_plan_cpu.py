"""The VAE's planning pass without a GPU: the workspace every entry point asks for, pinned for the fp32, tiled and split plans
(the bf16 untiled sizes are pinned in test_weight_checks_cpu.VAE_SIZES).  A handle with its weights registered at fake
addresses is enough, since planning only measures the bump allocators and looks the weights up."""
import ctypes

import pytest

from oracle import vae_oracle as V
from tests.test_vae_tiling_cpu import _handle_with_weights
from tests.test_weight_checks_cpu import VAE_GEOMETRIES
from tests.vae_tiling_oracle import DEFAULT_TILES

CONFIGS = {"tiny": V.VAEConfig.tiny(32), "wan21": V.VAEConfig.wan21()}

# (decode, frames, height, width, tiles): encode 5 frames / decode 2 latent frames of 200 x 328 and of 720 x 1280
TILED_GEOMETRIES = [(0, 5, 200, 328, (64, 64, 48, 48)), (1, 2, 25, 41, (64, 64, 48, 48)), (0, 5, 720, 1280, DEFAULT_TILES),
                    (1, 2, 90, 160, DEFAULT_TILES)]
# (world, rank) of the split; each plans an encode of 5 x 64 x 64 and a decode of 2 x 8 x 8
SPLITS = [(2, 0), (2, 1), (4, 0), (4, 3)]

SIZES = {
    "tiny": {
        "fp32": [956416, 12933376, 13133056, 6077696, 34488576, 11402035456, 1192704, 18992896, 18994432, 9620224, 50647296,
                 15037747456],
        "tiled": [22790656, 34523648, 370541056, 558268928],
        "tiled_fp32": [34816512, 51884544, 557056512, 830145024],
        "split": [(12013824, 18117632), (12013824, 18117632), (6369536, 9629184), (6369536, 9629184)],
        "region": [271360, 271360],
    },
    "wan21": {
        "fp32": [6402048, 38295808, 38495488, 21701888, 102121728, 23950541056, 7114496, 56962816, 56964352, 32386816, 151900416,
                 35150745856],
        "tiled": [62210560, 102156800, 1001259520, 1640399360],
        "tiled_fp32": [102449664, 153137664, 1639186944, 2450194944],
        "split": [(33124608, 54162432), (33124608, 54162432), (17649920, 28790272), (17649920, 28790272)],
        "region": [599040, 599040],
    },
}


@pytest.mark.parametrize("config", list(CONFIGS))
def test_fp32_workspace_sizes(config):
    L, h = _handle_with_weights(CONFIGS[config], fp32=True)
    try:
        assert [L.ce_vae_workspace_bytes_fp32(h, *g) for g in VAE_GEOMETRIES] == SIZES[config]["fp32"]
        assert [L.ce_vae_workspace_bytes_tiled_fp32(h, d, t, H, W, *ts) for d, t, H, W, ts in TILED_GEOMETRIES] == \
            SIZES[config]["tiled_fp32"]
    finally:
        L.ce_vae_destroy(h)


@pytest.mark.parametrize("config", list(CONFIGS))
def test_tiled_workspace_sizes(config):
    L, h = _handle_with_weights(CONFIGS[config])
    try:
        assert [L.ce_vae_workspace_bytes_tiled(h, d, t, H, W, *ts) for d, t, H, W, ts in TILED_GEOMETRIES] == SIZES[config]["tiled"]
    finally:
        L.ce_vae_destroy(h)


@pytest.mark.parametrize("config", list(CONFIGS))
def test_split_workspace_and_region_sizes(config):
    L, h = _handle_with_weights(CONFIGS[config])
    try:
        got = []
        for world, rank in SPLITS:
            regions = (ctypes.c_void_p * world)(*[4096 * (w + 1) for w in range(world)])
            assert L.ce_vae_sp_configure(h, rank, world, regions, 1 << 30) == 0
            got.append((L.ce_vae_workspace_bytes(h, 0, 5, 64, 64), L.ce_vae_workspace_bytes(h, 1, 2, 8, 8)))
        assert got == SIZES[config]["split"]
        assert [L.ce_vae_sp_region_bytes(h, 64, 64, world) for world in (2, 4)] == SIZES[config]["region"]
    finally:
        L.ce_vae_destroy(h)
