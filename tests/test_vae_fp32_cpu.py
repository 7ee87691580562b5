"""CPU tests of the fp32 VAE: `torch_dtype=torch.float32` builds and loads fp32 parameters and reports them, the dtypes and the
split over GPUs that are not built for it are refused before anything runs, and the fp32 C entry points check every weight by
name and element count before the first launch."""
import ctypes
import json
import os

import pytest
import torch
from safetensors.torch import save_file

from chronoedit_b200 import _lib as L
from oracle import vae_oracle as V

CE_ERR_NO_DEVICE = -3
CE_ERR_MISSING_WEIGHT = -4


def _fp32_weights(cfg, seed=5):
    """Random fp32 weights, most of which bf16 cannot represent."""
    sd = V.random_state_dict(cfg, seed=seed)
    assert all(v.dtype == torch.float32 for v in sd.values())
    return sd


def _vae(cfg, **kw):
    from chronoedit_b200.autoencoder import AutoencoderKLWan

    return AutoencoderKLWan(base_dim=cfg.dim, z_dim=cfg.z_dim, dim_mult=tuple(cfg.dim_mult), num_res_blocks=cfg.num_res_blocks,
                            temperal_downsample=tuple(cfg.temperal_downsample), **kw)


def test_fp32_vae_keeps_fp32_parameters():
    cfg = V.VAEConfig.tiny(32)
    sd = _fp32_weights(cfg)
    m = _vae(cfg, torch_dtype=torch.float32)
    assert m.dtype == torch.float32
    assert all(p.dtype == torch.float32 for p in m.parameters())
    m.load_state_dict(sd, strict=True)
    own = dict(m.named_parameters())
    assert any(not torch.equal(v, v.bfloat16().float()) for v in sd.values()), "the weights must not be bf16 values"
    for k, v in sd.items():
        assert torch.equal(own[k].data, v), k
    # the bf16 default is unchanged
    b = _vae(cfg)
    assert b.dtype == torch.bfloat16 and all(p.dtype == torch.bfloat16 for p in b.parameters())


def test_from_pretrained_fp32_keeps_the_checkpoint_values(tmp_path):
    from chronoedit_b200.autoencoder import AutoencoderKLWan

    cfg = V.VAEConfig.tiny(32)
    twin = _fp32_weights(cfg)
    kmap = AutoencoderKLWan.diffusers_key_map(cfg.dim, cfg.z_dim, tuple(cfg.dim_mult), cfg.num_res_blocks, tuple(cfg.temperal_downsample))
    vae_dir = tmp_path / "ckpt" / "vae"
    os.makedirs(vae_dir)
    with open(vae_dir / "config.json", "w") as f:
        json.dump({"_class_name": "AutoencoderKLWan", "base_dim": cfg.dim, "z_dim": cfg.z_dim, "dim_mult": list(cfg.dim_mult),
                   "num_res_blocks": cfg.num_res_blocks, "attn_scales": [], "temperal_downsample": list(cfg.temperal_downsample),
                   "dropout": 0.0}, f)
    save_file({d: twin[t].contiguous() for d, t in kmap.items()}, str(vae_dir / "diffusion_pytorch_model.safetensors"))
    m = AutoencoderKLWan.from_pretrained(str(tmp_path / "ckpt"), subfolder="vae", torch_dtype=torch.float32)
    assert m.dtype == torch.float32
    own = dict(m.named_parameters())
    for k, v in twin.items():
        assert own[k].dtype == torch.float32 and torch.equal(own[k].data, v), k
    # the same checkpoint in bf16 is rounded, as before
    b = AutoencoderKLWan.from_pretrained(str(tmp_path / "ckpt"), subfolder="vae", torch_dtype=torch.bfloat16)
    assert b.dtype == torch.bfloat16
    assert all(torch.equal(p.data, twin[k].bfloat16()) for k, p in b.named_parameters())


@pytest.mark.parametrize("dtype", [torch.float16, torch.float64])
def test_other_dtypes_are_refused(dtype):
    from chronoedit_b200 import CEError

    with pytest.raises(CEError, match="bf16"):
        _vae(V.VAEConfig.tiny(32), torch_dtype=dtype)


def test_the_split_over_gpus_refuses_an_fp32_vae():
    """Refused by dtype before any process group, region or launch is touched."""
    from chronoedit_b200 import CEError, parallel

    m = _vae(V.VAEConfig.tiny(32), torch_dtype=torch.float32)
    with pytest.raises(CEError, match="fp32"):
        parallel.enable_vae_sequence_parallel(m, 64, 64)
    with pytest.raises(CEError, match="fp32"):
        parallel.configure_vae_sequence_parallel(m, 0, [0, 0], 1 << 20, {})
    m._sp_state = {"world": 2}   # a split configured some other way: encode / decode refuse before the input is touched
    with pytest.raises(CEError, match="split over GPUs"):
        m.encode(torch.zeros(1, 3, 1, 16, 16))
    with pytest.raises(CEError, match="split over GPUs"):
        m.decode(torch.zeros(1, 16, 1, 2, 2))


def test_pack_parameter_fp32_layout():
    """Convolution weights become [Cout, taps, Cin_pad / 64, 3, 64] bf16 with hi | hi | lo per 64-channel block."""
    from chronoedit_b200.autoencoder import pack_parameter_fp32

    g = torch.Generator().manual_seed(0)
    w = torch.randn(5, 70, 3, 1, 1, generator=g)
    p = pack_parameter_fp32("x.time_conv.weight", w)
    assert p.dtype == torch.bfloat16 and p.shape == (5, 3 * 128 * 3)
    p = p.reshape(5, 3, 2, 3, 64)
    full = torch.zeros(5, 3, 128)
    full[:, :, :70] = w[:, :, :, 0, 0].permute(0, 2, 1)
    full = full.reshape(5, 3, 2, 64)
    assert torch.equal(p[:, :, :, 0], full.bfloat16()) and torch.equal(p[:, :, :, 1], full.bfloat16())
    assert torch.equal(p[:, :, :, 2], (full - full.bfloat16().float()).bfloat16())
    assert (full - p[:, :, :, 0].float() - p[:, :, :, 2].float()).abs().max() <= 2.0 ** -16 * full.abs().max()
    # gammas, biases and the attention's matrices stay fp32
    assert pack_parameter_fp32("a.residual.0.gamma", torch.ones(8, 1, 1, 1)).dtype == torch.float32
    q = pack_parameter_fp32("a.middle.1.to_qkv.weight", torch.ones(24, 8, 1, 1))
    assert q.dtype == torch.float32 and q.shape == (24, 8)


# ---------------------------------------------------------------------------------------------------------------------- C ABI
class Fake:
    """One aligned host address: the handle only keeps pointers, and nothing here dereferences them."""

    def __init__(self):
        self._buf = torch.zeros(64, dtype=torch.uint8)
        self.ptr = ctypes.c_void_p((self._buf.data_ptr() + 15) & ~15)


FAKE = Fake()
no_device = pytest.mark.skipif(L.lib().ce_device_check() == 0, reason="a complete weight set would launch on fake host pointers")


def _handle_with(weights):
    """A tiny fp32 VAE handle with `weights` (name -> element count) registered on a fake pointer."""
    m = _vae(V.VAEConfig.tiny(32), torch_dtype=torch.float32)
    h = m._ensure_handle()
    for k, n in weights.items():
        assert L.lib().ce_vae_set_weight_fp32(h, k.encode(), FAKE.ptr, n) == 0
    return m, h


def _packed_sizes():
    from chronoedit_b200.autoencoder import pack_parameter_fp32

    cfg = V.VAEConfig.tiny(32)
    return {k: pack_parameter_fp32(k, torch.zeros(s)).numel() for k, s in V.param_shapes(cfg).items()}


def _error():
    return (L.lib().ce_last_error() or b"").decode()


def test_fp32_abi_checks_every_weight_before_a_launch():
    lib = L.lib()
    sizes = _packed_sizes()
    m, h = _handle_with(sizes)
    assert lib.ce_vae_workspace_bytes_fp32(h, 0, 5, 32, 48) > 0
    assert lib.ce_vae_workspace_bytes_fp32(h, 1, 2, 4, 6) > 0
    # the bf16 entry points do not see the fp32 weights
    assert lib.ce_vae_workspace_bytes(h, 1, 2, 4, 6) == -1
    for name in ("encoder.conv1.weight", "decoder.middle.1.to_qkv.weight", "decoder.head.2.bias", "conv1.weight",
                 "encoder.downsamples.2.resample.1.weight", "decoder.upsamples.3.time_conv.weight"):
        m, h = _handle_with({**sizes, name: sizes[name] - 1})
        decode = not name.startswith("encoder") and name != "conv1.weight"
        assert lib.ce_vae_workspace_bytes_fp32(h, int(decode), 5 if not decode else 2, 32 if not decode else 4, 48 if not decode else 6) == -1
        assert name in _error()
        out = torch.zeros(16)
        rc = (lib.ce_vae_decode_fp32(h, FAKE.ptr, L.ptr(out), 2, 4, 6, 0, FAKE.ptr, 1 << 40, None) if decode else
              lib.ce_vae_encode_fp32(h, FAKE.ptr, L.ptr(out), 5, 32, 48, FAKE.ptr, 1 << 40, None))
        assert rc == CE_ERR_MISSING_WEIGHT and name in _error()
        m, h = _handle_with({k: v for k, v in sizes.items() if k != name})
        assert lib.ce_vae_workspace_bytes_fp32(h, int(decode), 5 if not decode else 2, 32 if not decode else 4, 48 if not decode else 6) == -1
        assert name in _error()


def test_fp32_abi_refusals():
    lib = L.lib()
    m, h = _handle_with({})
    assert lib.ce_vae_set_weight_fp32(h, b"conv1.bias", None, 32) != 0
    assert lib.ce_vae_set_weight_fp32(None, b"conv1.bias", FAKE.ptr, 32) != 0
    assert lib.ce_vae_workspace_bytes_fp32(h, 1, 1, 2, 2) == -1   # no fp32 weights at all
    assert "ce_vae_set_weight_fp32" in _error()
    assert lib.ce_vae_workspace_bytes_fp32(None, 1, 1, 2, 2) == -1
    m, h = _handle_with(_packed_sizes())
    assert lib.ce_vae_workspace_bytes_fp32(h, 0, 4, 32, 48) == -1   # frames must be 1 + 4k
    assert lib.ce_vae_workspace_bytes_fp32(h, 0, 5, 30, 48) == -1   # H, W multiples of 8


@no_device
def test_fp32_abi_complete_set_reaches_the_device_check():
    m, h = _handle_with(_packed_sizes())
    out = torch.zeros(16)
    assert L.lib().ce_vae_decode_fp32(h, FAKE.ptr, L.ptr(out), 2, 4, 6, 0, FAKE.ptr, 1 << 40, None) == CE_ERR_NO_DEVICE
    assert L.lib().ce_conv3d_cl_ex_fp32(None, None, None) == CE_ERR_NO_DEVICE
