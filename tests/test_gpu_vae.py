"""Parity of the VAE path on the GPU: the wgmma implicit-GEMM convolution against torch's fp32 conv3d on the same
bf16 inputs, and full encode / decode against the golden fixtures recorded from the UNMODIFIED reference VAE
(chronoedit/_src/tokenizers/wan2pt1.py) — same acceptance rule as the DiT (tests/test_gpu_dit.py): our bf16 result must
be as close to the reference's fp32 result as the reference's own bf16 run is."""
import json
import os

import pytest
import torch
import torch.nn.functional as F
from safetensors.torch import load_file

gpu = pytest.mark.gpu


def _L():
    import chronoedit_b200._lib as L

    return L


def run_conv(Cin, Cout, T, H, W, k, stride=(1, 1, 1), pad=(0, 0), hist=0, resid=False, split_time=False, seed=0):
    """x channels-last [hist+T, H, W, Cin]; reference = F.conv3d on the NCTHW view with explicit spatial zero padding."""
    from chronoedit_b200.autoencoder import pack_parameter

    L = _L()
    lib = L.lib()
    g = torch.Generator(device="cpu").manual_seed(seed)
    kt, kh, kw = k
    st, sh, sw = stride
    ph, pw = pad
    Tin = hist + T
    x = torch.randn(Tin, H, W, Cin, generator=g).bfloat16().cuda()
    w = (torch.randn(Cout, Cin, kt, kh, kw, generator=g) / (Cin * kt * kh * kw) ** 0.5).bfloat16().cuda()
    b = (0.1 * torch.randn(Cout, generator=g)).bfloat16().cuda()
    xn = x.permute(3, 0, 1, 2)[None].float()                       # [1, Cin, Tin, H, W]
    if sh == 2:   # ZeroPad2d((0,1,0,1)) + stride-2 conv (wan2pt1.py:106-110)
        xp = F.pad(xn, (0, 1, 0, 1))
    else:
        xp = F.pad(xn, (pw, pw, ph, ph))
    ref = F.conv3d(xp, w.float(), b.float(), stride=(st, sh, sw))  # [1, Cout, Tout, Hout, Wout]
    _, _, Tout, Hout, Wout = ref.shape
    ref = ref[0].permute(1, 2, 3, 0)                               # [Tout, Hout, Wout, Cout]
    ref = ref.bfloat16().float()
    c_store = Cout // 2 if split_time else Cout
    if split_time:  # channels [0,C) -> even frames, [C,2C) -> odd frames (wan2pt1.py:137-139)
        ref = torch.stack((ref[..., :c_store], ref[..., c_store:]), dim=1).reshape(2 * Tout, Hout, Wout, c_store)
    r = None
    if resid:
        r = torch.randn(ref.shape, generator=g).bfloat16().cuda()
        ref = ref + r.float().cpu().cuda()
    y = torch.zeros(ref.shape, dtype=torch.bfloat16, device="cuda")
    wp = pack_parameter("layer.weight", w)
    L.check(lib.ce_conv3d_cl_bf16(L.ptr(x), Tin, H, W, Cin, L.ptr(wp), L.ptr(b), Cout, kt, kh, kw, st, sh, sw, ph, pw, 0, L.ptr(y), Tout, Hout,
                                  Wout, L.ptr(r), int(split_time), L.current_stream()))
    torch.cuda.synchronize()
    err = (y.float() - ref).abs()
    tol = 2.0 ** -7 * ref.abs() + 2.0 ** -8 * ref.abs().mean()
    bad = (err > tol).float().mean().item()
    assert torch.isfinite(y.float()).all()
    assert bad < 2e-3, f"conv Cin={Cin} Cout={Cout} k={k} stride={stride}: {bad * 100:.3f}% beyond 1 bf16 ulp, max err {err.max().item():.4g}"
    assert (err.mean() / ref.abs().mean()).item() < 3e-3


@gpu
@pytest.mark.parametrize("Cin,Cout", [(96, 96), (192, 384), (384, 192), (32, 64), (64, 32)])
def test_conv_causal_3x3x3(Cin, Cout):
    run_conv(Cin, Cout, T=2, H=19, W=37, k=(3, 3, 3), pad=(1, 1), hist=2, seed=Cin + Cout)


@gpu
def test_conv_pointwise_and_residual():
    run_conv(192, 384, T=3, H=16, W=24, k=(1, 1, 1), seed=1)
    run_conv(96, 96, T=1, H=24, W=40, k=(3, 3, 3), pad=(1, 1), hist=2, resid=True, seed=2)


@gpu
def test_conv_spatial_3x3_and_head():
    run_conv(384, 192, T=2, H=20, W=28, k=(1, 3, 3), pad=(1, 1), seed=3)          # Resample conv2d after upsample
    run_conv(96, 3, T=4, H=16, W=32, k=(3, 3, 3), pad=(1, 1), hist=2, seed=4)     # decoder head (Cout = 3)


@gpu
def test_conv_time_conv_split():
    run_conv(384, 768, T=2, H=9, W=13, k=(3, 1, 1), hist=2, split_time=True, seed=5)   # upsample3d time_conv + frame interleave


@gpu
def test_conv_strided():
    run_conv(96, 96, T=2, H=32, W=48, k=(1, 3, 3), stride=(1, 2, 2), seed=6)       # downsample conv2d (ZeroPad2d(0,1,0,1), stride 2)
    run_conv(96, 96, T=1, H=31, W=45, k=(1, 3, 3), stride=(1, 2, 2), seed=7)       # odd sizes
    run_conv(192, 192, T=4, H=8, W=12, k=(3, 1, 1), stride=(2, 1, 1), hist=1, seed=8)  # downsample3d time_conv


def _build_vae(case):
    import chronoedit_b200 as ce
    from chronoedit_b200.autoencoder import AutoencoderKLWan
    from oracle import cases

    cfg = case.cfg
    m = AutoencoderKLWan(base_dim=cfg.dim, z_dim=cfg.z_dim, dim_mult=tuple(cfg.dim_mult), num_res_blocks=cfg.num_res_blocks,
                         temperal_downsample=tuple(cfg.temperal_downsample), clamp_output=False)
    sd = {k: v.to(torch.bfloat16) for k, v in cases.vae_weights(case).items()}
    m.load_state_dict(sd, strict=True)
    return m.cuda()


@gpu
@pytest.mark.parametrize("name", ["tiny_5f", "tiny_9f", "tiny_1f", "wan_5f_64"])
def test_vae_matches_reference(name, golden_dir):
    from oracle import cases

    case = cases.VAE_CASES[name]
    gold = load_file(os.path.join(golden_dir, f"vae_{name}.safetensors"))
    man = json.load(open(os.path.join(golden_dir, "MANIFEST.json")))["cases"][f"vae_{name}"]
    video, z = cases.vae_inputs(case)
    assert abs(cases.checksum(torch.cat([video.flatten(), z.flatten()])) - man["inputs_checksum"]) <= 1e-6 * abs(man["inputs_checksum"])
    m = _build_vae(case)
    mu = m.encode(video.cuda()).latent_dist.mode().float().cpu()
    dec = m.decode(z.cuda(), return_dict=False)[0].float().cpu()
    torch.cuda.synchronize()
    assert m.launches() > 0
    for got, key in ((mu, "mu"), (dec, "dec")):
        ref32, ref16 = gold[f"{key}_fp32"], gold[f"{key}_bf16"].float()
        assert got.shape == ref32.shape, (got.shape, ref32.shape)
        assert torch.isfinite(got).all()
        e_ref = (ref16 - ref32).abs()
        e_our = (got - ref32).abs()
        assert e_our.mean() <= 1.25 * e_ref.mean(), f"{key}: mean err {e_our.mean():.3g} vs reference's own bf16 error {e_ref.mean():.3g}"
        assert e_our.max() <= 2.0 * e_ref.max(), f"{key}: max err {e_our.max():.3g} vs reference's own bf16 error {e_ref.max():.3g}"


@gpu
def test_vae_decode_clamps_and_streams():
    """diffusers clamps decode output; and decoding Tl frames must equal decoding the same stream frame by frame is NOT
    required (the cache is per call) -- but the first pixel frame depends only on latent frame 0 (causality)."""
    from oracle import cases

    case = cases.VAE_CASES["tiny_9f"]
    _, z = cases.vae_inputs(case)
    m = _build_vae(case)
    full = m.decode(z.cuda(), return_dict=False)[0]
    first = m.decode(z[:, :, :1].cuda(), return_dict=False)[0]
    assert torch.equal(full[:, :, :1], first), "decode is not causal in time"
    m.clamp_output = True
    assert m.decode((3 * z).cuda(), return_dict=False)[0].abs().max() <= 1.0
