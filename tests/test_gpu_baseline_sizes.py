"""Parity at the sizes BASELINE.json names (configs[1], configs[2]) -- not at reduced depth / width / resolution.

The CPU oracle cannot follow these sizes in seconds (one 14B forward = 222 TFLOP; fp32 weights = 65.6 GB), so here the
oracle's functional restatement (oracle/dit_oracle.py, oracle/vae_oracle.py -- plain torch ops on a state dict) is
evaluated on CUDA tensors on the test box: in fp32 with TF32 disabled (the "exact" answer) and in the reference's bf16
configuration (torch eager = cuBLAS / cuDNN / SDPA, i.e. the library path the unmodified reference itself executes on a
GPU).  The oracle stays the checker; the thing under test goes through the Python mirror -> C ABI -> sm_90a kernels.

Acceptance rule = tests/test_gpu_dit.py: the reference does not meet rtol=1e-3/atol=1e-4 against itself across precisions,
so OUR bf16 output must be as close to the fp32 answer as the REFERENCE's bf16 output is (mean-abs <= 1.25x, max-abs <= 2x);
the fp32 validation mode (tests/test_gpu_fp32_mode.py) is where the stated tolerance itself is asserted end to end.
For the DiT the rule is applied to the final sample AND to the output of every one of the 40 blocks; the per-layer error
curve is written to gpurun_out/dit_error_curve_14b.json.
"""
import json
import os

import pytest
import torch

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _exact_fp32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.set_float32_matmul_precision("highest")


def _init_dit_weights_(model, seed):
    """Random-init weights directly on the device (bench.py's recipe: Linear ~ N(0, 0.02), norms 1 + 0.1 N, tables N/sqrt(D))."""
    import math

    g = torch.Generator(device=model.device).manual_seed(seed)
    D = model.config.num_attention_heads * model.config.attention_head_dim
    for n, p in model.named_parameters():
        if n.endswith("scale_shift_table"):
            p.data.normal_(0, 1.0 / math.sqrt(D), generator=g)
        elif ".norm" in n and n.endswith("weight"):
            p.data.normal_(0, 0.1, generator=g).add_(1.0)
        elif ".norm" in n and n.endswith("bias"):
            p.data.normal_(0, 0.1, generator=g)
        else:
            p.data.normal_(0, 0.02, generator=g)


class _AsFloat32(dict):
    """The same bf16-representable weights, computed exactly: each tensor is widened to fp32 when the oracle reads it, so the 14B
    model is never held in fp32 as a whole (65.6 GB beside the 32.8 GB bf16 copy would not fit the H100's 80 GB)."""

    def __getitem__(self, key):
        return super().__getitem__(key).float()


def _dit_inputs(frames, seed, dev):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(1, 36, frames, 90, 160, generator=g)
    x[:, 16:20] = 0
    x[:, 16:20, 0] = 1     # mask channels of the condition (pipeline_chronoedit.py:447-453)
    text = torch.randn(1, 512, 4096, generator=g)
    text[:, 93:] = 0       # prompts are zero-padded past their length (pipeline_chronoedit.py:234-237)
    img = torch.randn(1, 257, 1280, generator=g)
    t = torch.tensor([757])
    return x.to(dev), t.to(dev), text.to(dev), img.to(dev)


def _run_dit_case(layers, frames, seed, curve_file=None):
    import chronoedit_b200 as ce
    from oracle import dit_oracle as O

    _exact_fp32()
    dev = torch.device("cuda", 0)
    cfg = O.DiTConfig(num_layers=layers)
    m = ce.ChronoEditTransformer3DModel(num_attention_heads=40, in_channels=36, out_channels=16, ffn_dim=13824, num_layers=layers,
                                        image_dim=1280, added_kv_proj_dim=5120, device=dev)
    _init_dit_weights_(m, seed)
    x, t, text, img = _dit_inputs(frames, seed + 1, dev)
    out = m(x, t, text, img, return_dict=False, capture_layers=tuple(range(layers)))[0].float()
    torch.cuda.synchronize()
    ours_layers = [m.last_captures[i].float() for i in range(layers)]
    # the reference's bf16 configuration: the mirror's own parameters (bf16, fp32 for _keep_in_fp32_modules), evaluated by torch
    sd16 = {k: v for k, v in m.state_dict().items()}
    with torch.no_grad():
        ref16, inter16 = O.dit_forward(sd16, cfg, x.bfloat16(), t, text.bfloat16(), img.bfloat16(), return_intermediates=True)
        ref16 = ref16.float()
        r16_layers = [inter16[f"block{i}"][0].float() for i in range(layers)]
        del inter16
        ref32, inter32 = O.dit_forward(_AsFloat32(sd16), cfg, x, t, text, img, return_intermediates=True)
    curve = []
    for i in range(layers):
        r32 = inter32[f"block{i}"][0]
        e_ref = (r16_layers[i] - r32).abs()
        e_our = (ours_layers[i] - r32).abs()
        curve.append({"layer": i, "mean_abs_ref32": r32.abs().mean().item(), "ours_mean": e_our.mean().item(), "ref_bf16_mean": e_ref.mean().item(),
                      "ours_max": e_our.max().item(), "ref_bf16_max": e_ref.max().item()})
    e_ref, e_our = (ref16 - ref32).abs(), (out - ref32).abs()
    summary = {"layers": layers, "tokens": frames * 45 * 80, "final": {"ours_mean": e_our.mean().item(), "ref_bf16_mean": e_ref.mean().item(),
                                                                        "ours_max": e_our.max().item(), "ref_bf16_max": e_ref.max().item(),
                                                                        "mean_abs_ref32": ref32.abs().mean().item()}, "per_layer": curve}
    if curve_file:
        os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
        with open(os.path.join(ROOT, "gpurun_out", curve_file), "w") as f:
            json.dump(summary, f, indent=1)
    print(json.dumps(summary["final"]))
    assert torch.isfinite(out).all()
    for c in curve:
        assert c["ours_mean"] <= 1.25 * c["ref_bf16_mean"] + 1e-7, f"block {c['layer']}: mean err {c['ours_mean']:.3g} vs reference bf16 {c['ref_bf16_mean']:.3g}"
    assert e_our.mean() <= 1.25 * e_ref.mean(), f"mean err {e_our.mean():.3g} vs reference bf16 {e_ref.mean():.3g}"
    assert e_our.max() <= 2.0 * e_ref.max(), f"max err {e_our.max():.3g} vs reference bf16 {e_ref.max():.3g}"


@gpu
def test_dit_14b_all_40_layers_at_720p():
    """BASELINE.json configs[1] exactly: ChronoEdit-14B (40 layers, dim 5120, ffn 13824), latent [1,36,2,90,160] = 7200 tokens."""
    _run_dit_case(layers=40, frames=2, seed=11, curve_file="dit_error_curve_14b.json")


@gpu
def test_dit_14b_width_temporal_reasoning_tokens():
    """BASELINE.json configs[2] geometry at full width: 8 latent frames = 28 800 tokens (225 key tiles per head), 2 blocks."""
    _run_dit_case(layers=2, frames=8, seed=13, curve_file="dit_error_curve_28800.json")


@gpu
def test_vae_720p_5_frames_matches_oracle():
    """VAE encode of [1,3,5,720,1280] and decode of [1,16,2,90,160] at Wan2.1 width -- the geometry bench.py times (90/8 = 11.25
    row tiles, TMA out-of-bounds fill, the multi-GB streaming workspace), against the oracle evaluated on the same device."""
    from chronoedit_b200.autoencoder import AutoencoderKLWan
    from oracle import vae_oracle as V

    _exact_fp32()
    dev = torch.device("cuda", 0)
    cfg = V.VAEConfig.wan21()
    sd32 = {k: v.to(dev) for k, v in V.random_state_dict(cfg, seed=5).items()}
    sd16 = {k: v.to(torch.bfloat16) for k, v in sd32.items()}
    sd32 = {k: v.float() for k, v in sd16.items()}    # the same bf16-representable weights, computed exactly
    g = torch.Generator(device="cpu").manual_seed(77)
    video = torch.zeros(1, 3, 5, 720, 1280)
    video[:, :, 0] = torch.rand(1, 3, 720, 1280, generator=g) * 2 - 1       # pipeline_chronoedit.py:421-425: image, then zero frames
    z = torch.randn(1, 16, 2, 90, 160, generator=g)
    video, z = video.to(dev), z.to(dev)
    m = AutoencoderKLWan(clamp_output=False)
    m.load_state_dict(sd16, strict=True)
    m = m.to(dev)
    mu = m.encode(video).latent_dist.mode().float()
    dec = m.decode(z, return_dict=False)[0].float()
    torch.cuda.synchronize()
    report = {}
    for got, key, fn, inp in ((mu, "encode", lambda sd, a: V.vae_encode(sd, cfg, a), video), (dec, "decode", lambda sd, a: V.vae_decode(sd, cfg, a, clamp=False), z)):
        ref32 = fn(sd32, inp)
        ref16 = fn(sd16, inp.bfloat16()).float()
        assert got.shape == ref32.shape, (got.shape, ref32.shape)
        assert torch.isfinite(got).all()
        e_ref, e_our = (ref16 - ref32).abs(), (got - ref32).abs()
        report[key] = {"ours_mean": e_our.mean().item(), "ref_bf16_mean": e_ref.mean().item(), "ours_max": e_our.max().item(),
                       "ref_bf16_max": e_ref.max().item(), "mean_abs_ref32": ref32.abs().mean().item()}
        del ref32, ref16
        torch.cuda.empty_cache()
    print(json.dumps(report))
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "vae_720p_parity.json"), "w") as f:
        json.dump(report, f, indent=1)
    for key, r in report.items():
        assert r["ours_mean"] <= 1.25 * r["ref_bf16_mean"], f"{key}: mean err {r['ours_mean']:.3g} vs reference's own bf16 error {r['ref_bf16_mean']:.3g}"
        assert r["ours_max"] <= 2.0 * r["ref_bf16_max"], f"{key}: max err {r['ours_max']:.3g} vs reference's own bf16 error {r['ref_bf16_max']:.3g}"


@gpu
def test_dit_context_cache_is_bit_identical():
    """cache_context=True (step-invariant text / image embedders and cross-attention K/V kept across steps) must not change a
    single bit, must survive alternating prompt / negative-prompt calls (two slots), and must notice in-place edits."""
    from oracle import cases

    import chronoedit_b200 as ce

    case = cases.DIT_CASES["tiny_b2"]
    cfg = case.cfg

    def build(cache):
        m = ce.ChronoEditTransformer3DModel(
            patch_size=cfg.patch_size, num_attention_heads=cfg.num_attention_heads, attention_head_dim=cfg.attention_head_dim,
            in_channels=cfg.in_channels, out_channels=cfg.out_channels, text_dim=cfg.text_dim, freq_dim=cfg.freq_dim,
            ffn_dim=cfg.ffn_dim, num_layers=cfg.num_layers, eps=cfg.eps, image_dim=cfg.image_dim,
            added_kv_proj_dim=cfg.added_kv_proj_dim, cache_context=cache)
        m.load_state_dict(cases.to_bf16_state(cases.dit_weights(case)))
        return m.cuda()

    x, t, text, img = (a.cuda() for a in cases.dit_inputs(case))
    text, img = text.bfloat16(), img.bfloat16()
    neg = torch.randn_like(text)
    plain, cached = build(False), build(True)
    for step in range(3):
        xs = x + 0.1 * step
        ts = t - 100 * step
        for ctx in (text, neg):
            a = plain(xs, ts, ctx, img, return_dict=False)[0]
            n_plain = plain.launches_per_forward()
            b = cached(xs, ts, ctx, img, return_dict=False)[0]
            assert torch.equal(a, b), f"step {step}: cached context changed the result"
            if step > 0:
                assert cached.launches_per_forward() < n_plain - 4 * cfg.num_layers + 1, "context was recomputed although it was cached"
    text.mul_(0.5)   # in-place edit bumps the version counter: the cache entry must not be reused
    a = plain(x, t, text, img, return_dict=False)[0]
    b = cached(x, t, text, img, return_dict=False)[0]
    assert torch.equal(a, b)
    assert cached.launches_per_forward() == plain.launches_per_forward()


@gpu
@pytest.mark.parametrize("cache", [False, True])
def test_dit_cuda_graph_replay_is_bit_identical(cache):
    """use_cuda_graph=True: the forward is captured on the second call of a configuration and replayed afterwards; every call must
    return exactly what the eager launch chain returns, with and without the context cache, across changing inputs."""
    from oracle import cases

    import chronoedit_b200 as ce

    case = cases.DIT_CASES["tiny_b2"]
    cfg = case.cfg

    def build(**kw):
        m = ce.ChronoEditTransformer3DModel(
            patch_size=cfg.patch_size, num_attention_heads=cfg.num_attention_heads, attention_head_dim=cfg.attention_head_dim,
            in_channels=cfg.in_channels, out_channels=cfg.out_channels, text_dim=cfg.text_dim, freq_dim=cfg.freq_dim,
            ffn_dim=cfg.ffn_dim, num_layers=cfg.num_layers, eps=cfg.eps, image_dim=cfg.image_dim,
            added_kv_proj_dim=cfg.added_kv_proj_dim, **kw)
        m.load_state_dict(cases.to_bf16_state(cases.dit_weights(case)))
        return m.cuda()

    x, t, text, img = (a.cuda() for a in cases.dit_inputs(case))
    text, img = text.bfloat16(), img.bfloat16()
    neg = torch.randn_like(text)
    eager, graphed = build(), build(use_cuda_graph=True, cache_context=cache)
    for step in range(5):
        xs, ts = x + 0.05 * step, t - 77 * step
        for ctx in (text, neg):
            a = eager(xs, ts, ctx, img, return_dict=False)[0]
            b = graphed(xs, ts, ctx, img, return_dict=False)[0]
            assert torch.equal(a, b), f"step {step}: graph replay differs from the eager forward"
    assert any(g.get("graph") is not None for g in graphed._graphs.values()), "no graph was ever captured"
