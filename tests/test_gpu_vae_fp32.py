"""The fp32 VAE on the GPU: its split-bf16 convolution against F.conv3d in fp64 within a bound derived from the split rule, encode
and decode within rtol 1e-3 / atol 1e-4 of the unmodified reference's fp32 run (the golden fixtures) and of the fp32 oracle at 720p
with the Wan2.1 channel widths, batch and input-dtype invariance, the bf16 VAE unchanged beside it, and the pipeline's decode.
Each comparison prints its errors as one JSON line."""
import json
import os

import pytest
import torch
import torch.nn.functional as F
from safetensors.torch import load_file

gpu = pytest.mark.gpu
RTOL, ATOL = 1e-3, 1e-4


def _L():
    import chronoedit_b200._lib as L

    return L


def _pair(x):
    """The split pair [..., 2, C] bf16 of fp32 x [..., C]."""
    hi = x.bfloat16()
    return torch.stack((hi, (x - hi.float()).bfloat16()), dim=-2).contiguous()


def _report(**kw):
    print(json.dumps(kw))


# ---------------------------------------------------------------------------------------------------------------- operator
def run_conv_fp32(Cin, Cout, T, H, W, k, stride=(1, 1, 1), hist=0, resid=False, split_time=False, planar=False, seed=0):
    """x channels-last [hist+T, H, W, Cin] fp32 with values bf16 cannot represent; reference = F.conv3d in fp64.

    Bound: with a = a_hi + a_lo + da, |da| <= 2^-17 |a| (and the same for w), the three products miss a_lo w_lo + da w + a dw,
    at most (2^-9 2^-9 + 2 * 2^-17) |a||w| < 2^-15.4 |a||w| per term.  The fp32 accumulation adds at most one part in 2^-23 of the
    running chunk sum per 16-wide k-step (48 steps per 768-long chunk) and 2^-24 per chunk add: below 2^-16.5 of sum |a||w| at the
    VAE's longest K.  So |y - ref| <= 2^-14 * sum |a||w| (+ the fp32 rounding of bias and residual)."""
    from chronoedit_b200.autoencoder import pack_parameter_fp32

    L = _L()
    g = torch.Generator(device="cpu").manual_seed(seed)
    kt, kh, kw = k
    st, sh, sw = stride
    ph, pw = (kh // 2, kw // 2) if sh == 1 else (0, 0)
    Tin = hist + T
    x = torch.randn(Tin, H, W, Cin, generator=g)
    w = torch.randn(Cout, Cin, kt, kh, kw, generator=g) / (Cin * kt * kh * kw) ** 0.5
    b = 0.1 * torch.randn(Cout, generator=g)
    assert not torch.equal(x, x.bfloat16().float()) and not torch.equal(w, w.bfloat16().float())
    xn = x.permute(3, 0, 1, 2)[None].double()
    pad = (0, 1, 0, 1) if sh == 2 else (pw, pw, ph, ph)
    ref = F.conv3d(F.pad(xn, pad), w.double(), b.double(), stride=(st, sh, sw))[0]          # [Cout, Tout, Hout, Wout]
    mag = F.conv3d(F.pad(xn.abs(), pad), w.double().abs(), None, stride=(st, sh, sw))[0]
    _, Tout, Hout, Wout = ref.shape
    c_store = Cout // 2 if split_time else Cout
    to_cl = lambda t: t.permute(1, 2, 3, 0)
    if planar:
        ref, mag = ref.clamp(-1, 1), mag
    else:
        ref, mag = to_cl(ref), to_cl(mag)
        if split_time:
            ref = torch.stack((ref[..., :c_store], ref[..., c_store:]), dim=1).reshape(2 * Tout, Hout, Wout, c_store)
            mag = torch.stack((mag[..., :c_store], mag[..., c_store:]), dim=1).reshape(2 * Tout, Hout, Wout, c_store)
    r = None
    if resid:
        r = torch.randn(ref.shape, generator=g)
        ref = ref + r.double()
        r = r.cuda()
    xp = _pair(x).cuda()
    wp = pack_parameter_fp32("layer.weight", w).cuda()
    bc = b.cuda()
    y = torch.full(ref.shape, float("nan"), device="cuda")
    y_pair = None if planar else torch.zeros(*ref.shape[:-1], 2, ref.shape[-1], dtype=torch.bfloat16, device="cuda")
    a = L.Conv3dArgsC()
    a.x, a.Tin, a.Hin, a.Win, a.Cin = L.ptr(xp), Tin, H, W, Cin
    a.w, a.bias, a.Cout, a.Cin_pad = L.ptr(wp), L.ptr(bc), Cout, (Cin + 63) // 64 * 64
    a.kt, a.kh, a.kw, a.st, a.sh, a.sw, a.ph, a.pw, a.t_base = kt, kh, kw, st, sh, sw, ph, pw, 0
    a.y, a.Tout, a.Hout, a.Wout = L.ptr(y), Tout, Hout, Wout
    a.resid, a.split_time = L.ptr(r), int(split_time)
    if planar:
        a.planar_out, a.clamp, a.planar_T, a.planar_t0 = 1, 1, Tout, 0
    L.check(L.lib().ce_conv3d_cl_ex_fp32(_L().ctypes.byref(a), L.ptr(y_pair), L.current_stream()))
    torch.cuda.synchronize()
    got = y.double().cpu()
    err = (got - ref).abs()
    bound = 2.0 ** -14 * mag + 2.0 ** -23 * (ref.abs() + 1)
    _report(op="conv_fp32", Cin=Cin, Cout=Cout, k=list(k), stride=list(stride), max_err=err.max().item(),
            max_rel_to_bound=(err / bound).max().item(), mean_err=err.mean().item())
    assert torch.isfinite(got).all()
    assert (err <= bound).all(), f"max err {err.max().item():.3g}, {(err / bound).max().item():.3g} of the bound"
    if y_pair is not None:   # the epilogue's pair is exactly the split of its fp32 output
        assert torch.equal(y_pair, _pair(y))


@gpu
@pytest.mark.parametrize("Cin,Cout", [(96, 96), (192, 384), (384, 192), (384, 384)])
def test_conv_fp32_causal_3x3x3(Cin, Cout):
    run_conv_fp32(Cin, Cout, T=2, H=19, W=37, k=(3, 3, 3), hist=2, seed=Cin + Cout)


@gpu
def test_conv_fp32_pointwise_residual_and_small_channels():
    run_conv_fp32(192, 384, T=3, H=16, W=24, k=(1, 1, 1), seed=1)                     # shortcut
    run_conv_fp32(96, 96, T=1, H=24, W=40, k=(3, 3, 3), hist=2, resid=True, seed=2)   # residual.6 + x
    run_conv_fp32(32, 32, T=3, H=12, W=20, k=(1, 1, 1), seed=3)                       # quant_conv (conv1)
    run_conv_fp32(16, 16, T=2, H=12, W=20, k=(1, 1, 1), seed=4)                       # post_quant_conv (conv2)
    run_conv_fp32(16, 384, T=1, H=9, W=13, k=(3, 3, 3), hist=2, seed=5)               # decoder.conv1
    run_conv_fp32(8, 96, T=4, H=16, W=24, k=(3, 3, 3), hist=2, seed=6)                # encoder.conv1 (3 channels padded to 8)


@gpu
def test_conv_fp32_resample_time_conv_and_head():
    run_conv_fp32(384, 192, T=2, H=20, W=28, k=(1, 3, 3), seed=7)                     # upsample's conv2d
    run_conv_fp32(96, 96, T=2, H=32, W=48, k=(1, 3, 3), stride=(1, 2, 2), seed=8)     # downsample: ZeroPad2d(0,1,0,1), stride 2
    run_conv_fp32(192, 192, T=1, H=31, W=45, k=(1, 3, 3), stride=(1, 2, 2), seed=9)   # odd sizes
    run_conv_fp32(384, 768, T=2, H=9, W=13, k=(3, 1, 1), hist=2, split_time=True, seed=10)   # upsample3d time_conv + interleave
    run_conv_fp32(192, 192, T=4, H=8, W=12, k=(3, 1, 1), stride=(2, 1, 1), hist=1, seed=11)  # downsample3d time_conv
    run_conv_fp32(96, 3, T=4, H=16, W=32, k=(3, 3, 3), hist=2, planar=True, seed=12)  # decoder head: planar, clamped


# ---------------------------------------------------------------------------------------------------------------- model
def _vae(cfg, sd, dtype=torch.float32, clamp=False):
    from chronoedit_b200.autoencoder import AutoencoderKLWan

    m = AutoencoderKLWan(base_dim=cfg.dim, z_dim=cfg.z_dim, dim_mult=tuple(cfg.dim_mult), num_res_blocks=cfg.num_res_blocks,
                         temperal_downsample=tuple(cfg.temperal_downsample), torch_dtype=dtype, clamp_output=clamp)
    m.load_state_dict(sd, strict=True)
    return m.cuda()


def _errors(got, ref):
    e = (got.double() - ref.double()).abs()
    return {"max_err": e.max().item(), "mean_err": e.mean().item(),
            "max_excess": (e - RTOL * ref.double().abs()).max().item()}


@gpu
@pytest.mark.parametrize("name", ["tiny_5f", "tiny_9f", "tiny_1f", "wan_5f_64"])
def test_vae_fp32_matches_reference(name, golden_dir):
    from oracle import cases

    case = cases.VAE_CASES[name]
    gold = load_file(os.path.join(golden_dir, f"vae_{name}.safetensors"))
    video, z = cases.vae_inputs(case)
    m = _vae(case.cfg, cases.vae_weights(case))
    assert m.dtype == torch.float32
    mu = m.encode(video.cuda()).latent_dist.mode()
    dec = m.decode(z.cuda(), return_dict=False)[0]
    assert mu.dtype == torch.float32 and dec.dtype == torch.float32
    for got, key in ((mu.cpu(), "mu"), (dec.cpu(), "dec")):
        ref32, ref16 = gold[f"{key}_fp32"], gold[f"{key}_bf16"].float()
        assert got.shape == ref32.shape and torch.isfinite(got).all()
        _report(case=name, out=key, **_errors(got, ref32), bf16_ref_max_err=(ref16 - ref32).abs().max().item())
        assert torch.allclose(got, ref32, rtol=RTOL, atol=ATOL), f"{key}: {_errors(got, ref32)}"


@gpu
def test_vae_fp32_720p_against_the_oracle():
    """Wan2.1 widths (96..384) at 720p with random fp32 weights: encode [1,3,5,720,1280] and decode [1,16,2,90,160] against the
    fp32 oracle on the GPU (TF32 off); the errors against fp64 and the bf16 mirror's error are printed for scale.  Then a
    29-frame decode (8 latent frames) at 240 x 416."""
    from oracle import vae_oracle as V

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = V.VAEConfig.wan21()
    sd = V.random_state_dict(cfg, seed=31)
    g = torch.Generator(device="cpu").manual_seed(32)
    cases = {"encode_5f_720p": (torch.rand(1, 3, 5, 720, 1280, generator=g) * 2 - 1).cuda(),
             "decode_5f_720p": torch.randn(1, 16, 2, 90, 160, generator=g).cuda(),
             "decode_29f_240x416": torch.randn(1, 16, 8, 30, 52, generator=g).cuda()}

    def call(m, what, x):
        return m.encode(x).latent_dist.mode() if what.startswith("encode") else m.decode(x, return_dict=False)[0]

    ours, mirror = {}, {}
    for dtype, res in ((torch.float32, ours), (torch.bfloat16, mirror)):   # one VAE at a time: the fp32 one needs 33 GB at 720p
        m = _vae(cfg, {k: v.to(dtype) for k, v in sd.items()}, dtype=dtype)
        for what, x in cases.items():
            res[what] = call(m, what, x).float()
        del m
        torch.cuda.empty_cache()
    for what, x in cases.items():
        ref = (lambda s, x: V.vae_encode(s, cfg, x)) if what.startswith("encode") else (lambda s, x: V.vae_decode(s, cfg, x, clamp=False))
        ref32 = ref({k: v.cuda() for k, v in sd.items()}, x)
        got = ours[what]
        rep = {"case": what, **_errors(got, ref32), "bf16_mirror_max_err": (mirror[what] - ref32).abs().max().item()}
        if what != "decode_29f_240x416":
            ref64 = ref({k: v.cuda().double() for k, v in sd.items()}, x.double())
            rep.update(ours_vs_fp64_max=(got.double() - ref64).abs().max().item(),
                       oracle_fp32_vs_fp64_max=(ref32.double() - ref64).abs().max().item())
            del ref64
        _report(**rep)
        assert torch.isfinite(got).all()
        assert torch.allclose(got, ref32, rtol=RTOL, atol=ATOL), rep
        del ref32
        torch.cuda.empty_cache()


@gpu
def test_vae_fp32_invariances():
    """A batch-2 call is two batch-1 calls bit for bit; a bf16 input gives the bits of its fp32 widening; the bf16 VAE gives the
    same bits and launch count before and after an fp32 VAE ran in the process."""
    from oracle import cases

    case = cases.VAE_CASES["tiny_5f"]
    sd = cases.vae_weights(case)
    video, z = cases.vae_inputs(case)
    video, z = video.cuda(), z.cuda()
    m16 = _vae(case.cfg, {k: v.bfloat16() for k, v in sd.items()}, dtype=torch.bfloat16)
    before = (m16.encode(video).latent_dist.mode().clone(), m16.launches(), m16.decode(z, return_dict=False)[0].clone(), m16.launches())

    m = _vae(case.cfg, sd)
    v2 = torch.cat([video, -0.5 * video.flip(3)])
    z2 = torch.cat([z, 0.5 * z.flip(4)])
    enc2 = m.encode(v2).latent_dist.mode()
    dec2 = m.decode(z2, return_dict=False)[0]
    for i in range(2):
        assert torch.equal(enc2[i:i + 1], m.encode(v2[i:i + 1]).latent_dist.mode()), f"encode sample {i}"
        assert torch.equal(dec2[i:i + 1], m.decode(z2[i:i + 1], return_dict=False)[0]), f"decode sample {i}"
    vb, zb = video.bfloat16(), z.bfloat16()
    enc_b = m.encode(vb).latent_dist.mode()
    assert enc_b.dtype == torch.float32 and torch.equal(enc_b, m.encode(vb.float()).latent_dist.mode())
    assert torch.equal(m.decode(zb, return_dict=False)[0], m.decode(zb.float(), return_dict=False)[0])

    after = (m16.encode(video).latent_dist.mode(), m16.launches(), m16.decode(z, return_dict=False)[0], m16.launches())
    assert torch.equal(before[0], after[0]) and torch.equal(before[2], after[2])
    assert before[1] == after[1] and before[3] == after[3]


@gpu
@pytest.mark.parametrize("name", ["edit_5f", "reason_full"])
def test_pipeline_with_the_fp32_vae(name):
    """The pipeline restated from ChronoEditPipeline.__call__ with the CUDA mirrors and the VAE in fp32: the conditioning video
    arrives in bf16 (prepare_latents) and is widened; every frame the VAE decodes is within rtol 1e-3 / atol 1e-4 of the fp32
    oracle VAE's decode of the same latents."""
    import chronoedit_b200 as ce
    from oracle import cases, pipeline_cases as PC
    from oracle.pipeline_oracle import OracleVAE

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda", 0)
    case = PC.PIPELINE_CASES[name]
    dsd, vsd = PC.weights()
    cfg = PC.DIT_CFG
    tr = ce.ChronoEditTransformer3DModel(
        patch_size=cfg.patch_size, num_attention_heads=cfg.num_attention_heads, attention_head_dim=cfg.attention_head_dim,
        in_channels=cfg.in_channels, out_channels=cfg.out_channels, text_dim=cfg.text_dim, freq_dim=cfg.freq_dim, ffn_dim=cfg.ffn_dim,
        num_layers=cfg.num_layers, eps=cfg.eps, image_dim=cfg.image_dim, added_kv_proj_dim=cfg.added_kv_proj_dim, cache_context=True)
    tr.load_state_dict(cases.to_bf16_state(dsd))
    vae = _vae(PC.VAE_CFG, vsd, clamp=True)
    calls = []
    decode = vae.decode

    def recording_decode(z, return_dict=True):
        out = decode(z, return_dict=return_dict)
        calls.append((z.clone(), (out[0] if not return_dict else out.sample).clone()))
        return out

    vae.decode = recording_decode
    video = PC.run_oracle_pipeline(case, torch.bfloat16, device=dev, transformer=tr.to(dev), vae=vae,
                                   scheduler=ce.FlowUniPCMultistepScheduler(shift=case.sched_shift))
    assert torch.isfinite(video.float()).all() and calls and vae.launches() > 0
    oracle = OracleVAE({k: v.to(dev) for k, v in vsd.items()}, PC.VAE_CFG, torch.float32)
    for z, ours in calls:
        assert z.dtype == torch.float32 and ours.dtype == torch.float32
        ref = oracle.decode(z, return_dict=False)[0]
        _report(case=name, latent_frames=z.shape[2], **_errors(ours, ref))
        assert torch.allclose(ours, ref, rtol=RTOL, atol=ATOL), _errors(ours, ref)
