"""The sequence-parallel DiT forward on ONE GPU: `world` mirror instances with identical weights play the ranks, each driven from its
own host thread on its own stream, with ordinary device allocations as peer regions and the host barrier (ce_dit_sp_host_barrier)
between the phases of the exchange.  That runs every kernel, every peer-store address and every local-versus-global token count of
the sequence-parallel path (csrc/seqpar.cuh, the q | k scatter of the RMSNorm+RoPE kernel, the attention epilogue's row scatter, the
gate epilogue's rows per sample) at world 2 to 8 on a single device, and no kernel ever waits for another rank.

Asserted per case: every rank's sample is bit-identical to the single-GPU forward of the same weights and inputs (three steps with
the context cache on, prompt and negative prompt alternating, then the single-GPU forward again once sequence parallelism is off);
nothing is written outside the sub-buffers of the peer regions (a guard band after each region and the alignment gaps between its
q / k / v / attention / head-output buffers keep a byte pattern); the inputs are unchanged.  The refusals that come before any
launch are checked under the host barrier too, so a regression fails with a timeout message instead of reaching a device barrier.

tests/test_gpu_seqpar.py keeps what only several GPUs can show: the device flag barrier, CUDA IPC and NVLink peer stores."""
import time

import pytest
import torch

from tests.sp_one_gpu import BARRIER_MS, SHORT_MS, _clean_device, assert_pattern_kept, guarded_regions, run_ranks  # noqa: F401

gpu = pytest.mark.gpu


def sp_layout(B, L, D, No, world):
    """Python restatement of sp_layout (csrc/dit.cu): byte offsets of a rank's peer region for B samples of L tokens, width D and
    No = out_channels * 4 head outputs.  Sub-buffers start at multiples of 1024 bytes; the flags block (uint32 [8 * 32]) ends it."""
    al = lambda v: (v + 1023) & ~1023
    qkv = B * L * (D // world) * 2          # q, k, v: [B, L, D / world] bf16 each
    attn = B * (L // world) * D * 2         # [B * L / world, D] bf16
    yout = B * L * No * 2                   # [B * L, No] bf16
    g = al(qkv)
    lay = {"q": 0, "k": g, "v": 2 * g, "attn": 3 * g}
    lay["yout"] = lay["attn"] + al(attn)
    lay["flags"] = lay["yout"] + al(yout)
    lay["bytes"] = lay["flags"] + 1024
    lay["used"] = {"q": qkv, "k": qkv, "v": qkv, "attn": attn, "yout": yout}
    return lay


def sp_unwritten_ranges(lay):
    """[start, end) byte ranges of a region that the sequence-parallel forward never writes under the host barrier: the alignment gap
    after each sub-buffer and the flags block (only the device barrier uses it)."""
    out = []
    for name in ("q", "k", "v", "attn", "yout"):
        end = lay[name] + lay["used"][name]
        nxt = {"q": "k", "k": "v", "v": "attn", "attn": "yout", "yout": "flags"}[name]
        if end < lay[nxt]:
            out.append((name + " gap", end, lay[nxt]))
    out.append(("flags", lay["flags"], lay["bytes"]))
    return out


def _model(heads, layers, ffn, seed, dev):
    import chronoedit_b200 as ce

    D = heads * 128
    m = ce.ChronoEditTransformer3DModel(num_attention_heads=heads, in_channels=36, out_channels=16, ffn_dim=ffn, num_layers=layers,
                                        image_dim=1280, added_kv_proj_dim=D, device=dev, cache_context=True)
    g = torch.Generator(device=dev).manual_seed(seed)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if ".norm" in n and n.endswith("weight"):
                p.normal_(0, 0.1, generator=g).add_(1.0)
            elif p.dim() >= 2 and "scale_shift_table" not in n:
                p.normal_(0, p[0].numel() ** -0.5, generator=g)
            else:
                p.normal_(0, 0.05, generator=g)
    return m


def _mirrors(first, world):
    """`world` instances with the weights of `first` (which is rank 0)."""
    import chronoedit_b200 as ce

    c = first.config
    out = [first]
    for _ in range(world - 1):
        m = ce.ChronoEditTransformer3DModel(num_attention_heads=c.num_attention_heads, in_channels=c.in_channels, out_channels=c.out_channels,
                                            text_dim=c.text_dim, ffn_dim=c.ffn_dim, num_layers=c.num_layers, image_dim=c.image_dim,
                                            added_kv_proj_dim=c.added_kv_proj_dim, eps=c.eps, device=first.device, cache_context=True)
        m.load_state_dict(first.state_dict())
        out.append(m)
    return out


def _rank_diffs(out, ref, world):
    """Largest |out - ref| over the sample positions of each rank's tokens (rank r owns tokens [r L / world, (r + 1) L / world))."""
    _, _, T, H, W = ref.shape
    hp, wp = H // 2, W // 2
    f = torch.arange(T, device=ref.device).view(T, 1, 1)
    i = torch.arange(H, device=ref.device).view(1, H, 1) // 2
    j = torch.arange(W, device=ref.device).view(1, 1, W) // 2
    owner = (f * hp * wp + i * wp + j) // (T * hp * wp // world)
    d = (out.float() - ref.float()).abs().amax(dim=(0, 1))
    return ", ".join(f"rank {r} tokens: {float(d[owner == r].max()):.4g}" for r in range(world))


def _sequence_parallel_matches_single(models, steps, latent, world, oracle_check=None):
    from chronoedit_b200 import parallel

    m0 = models[0]
    B = steps[0][0].shape[0]
    T, H, W = latent
    inputs = [tuple(a.clone() for a in st) for st in steps]
    refs = [m0(*st, return_dict=False)[0].clone() for st in steps]
    torch.cuda.synchronize()
    for ref in refs:
        assert torch.isfinite(ref.float()).all() and ref.float().std() > 0
    if oracle_check is not None:
        oracle_check(refs[0])
    n = parallel.sp_region_bytes(m0, B, T, H, W, world)
    lay = sp_layout(B, T * (H // 2) * (W // 2), m0.config.num_attention_heads * 128, m0.config.out_channels * 4, world)
    assert lay["bytes"] == n
    regions = guarded_regions(n, world, m0.device)
    ptrs = [r.data_ptr() for r in regions]
    from chronoedit_b200 import _lib

    try:
        for r, m in enumerate(models):
            _lib.check(_lib.lib().ce_dit_sp_host_barrier(m._ensure_handle(), BARRIER_MS))
            parallel.configure_sequence_parallel(m, r, ptrs, n, {})
        bad = []
        for it, st in enumerate(steps):
            outs = run_ranks(lambda r: models[r](*st, return_dict=False)[0], world, timeout=600)
            torch.cuda.synchronize()
            for r, o in enumerate(outs):
                if not torch.equal(o, refs[it]):
                    bad.append(f"step {it}, rank {r}: max|diff| per token range: {_rank_diffs(o, refs[it], world)}")
        assert not bad, "sequence-parallel sample differs from the single-GPU forward:\n" + "\n".join(bad)
    finally:
        for m in models:
            parallel.disable_sequence_parallel(m)
    torch.cuda.synchronize()
    assert_pattern_kept(regions, n, sp_unwritten_ranges(lay))
    for m in models:   # every handle is back on the single-GPU forward
        assert torch.equal(m(*steps[0], return_dict=False)[0], refs[0])
    for st, before in zip(steps, inputs):
        assert all(torch.equal(a, b) for a, b in zip(st, before)), "the forward modified its inputs"


def _steps(B, latent, dev, seed):
    """Three denoising-step inputs: changing latents and timesteps, prompt and negative prompt alternating (the same tensor objects each
    time, so the context cache hits on the third step)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    T, H, W = latent
    prompt = torch.randn(B, 512, 4096, generator=g, device=dev).bfloat16()
    prompt[:, 100:] = 0
    negative = torch.randn(B, 512, 4096, generator=g, device=dev).bfloat16()
    negative[:, 20:] = 0
    img = torch.randn(B, 257, 1280, generator=g, device=dev).bfloat16()
    out = []
    for it in range(3):
        x = torch.randn(B, 36, T, H, W, generator=g, device=dev).bfloat16()
        t = torch.tensor([900 - 211 * it - 37 * b for b in range(B)], device=dev)
        out.append((x, t, prompt if it % 2 == 0 else negative, img))
    return out


# (name, heads, layers, ffn, latent (T, H, W), batch, worlds)
CASES = [
    ("small", 8, 2, 1024, (8, 24, 20), 1, (2, 4, 8)),      # 960 tokens: 120 rows per rank at world 8, every 128-row query tile spans two ranks
    ("odd", 4, 2, 1024, (2, 30, 42), 2, (2,)),             # 630 tokens: 315 local rows, the last row-pair CTA is half empty
    ("14b_width", 40, 1, 13824, (2, 32, 40), 2, (2, 4, 8)),  # 20 / 10 / 5 heads per rank, 80 rows per rank at world 8
    ("flagship_tokens", 40, 1, 13824, (8, 90, 160), 2, (2,)),  # 28 800 tokens: the geometry of scripts/bench_seqpar.py
]


@gpu
@pytest.mark.parametrize("name,heads,layers,ffn,latent,B,world",
                         [(c[0], c[1], c[2], c[3], c[4], c[5], w) for c in CASES for w in c[6]],
                         ids=[f"{c[0]}-w{w}" for c in CASES for w in c[6]])
def test_sequence_parallel_on_one_gpu_is_bit_identical(name, heads, layers, ffn, latent, B, world, _clean_device):
    dev = torch.device("cuda", torch.cuda.current_device())
    models = _mirrors(_model(heads, layers, ffn, seed=heads * 1000 + layers, dev=dev), world)
    _sequence_parallel_matches_single(models, _steps(B, latent, dev, seed=world + 17 * heads), latent, world)


@gpu
def test_sequence_parallel_on_one_gpu_golden_cfg0(golden_dir, _clean_device):
    """The 2048-token fixture (2 heads, 2 layers) at world 2: the first step is the fixture's own input, so the single-GPU forward the
    ranks must reproduce bit for bit also meets the oracle rule of test_gpu_dit.py against the reference's outputs."""
    import os

    from safetensors.torch import load_file

    from oracle import cases
    from tests.test_gpu_dit import _build

    case = cases.DIT_CASES["cfg0_64x64"]
    gold = load_file(os.path.join(golden_dir, "dit_cfg0_64x64.safetensors"))
    m = _build(case)
    m.cache_context = True
    models = _mirrors(m, 2)
    dev = m.device
    x, t, text, img = (v.to(dev) for v in cases.dit_inputs(case))
    x, text, img = x.bfloat16(), text.bfloat16(), img.bfloat16()
    more = _steps(1, (case.frames, case.height, case.width), dev, seed=5)
    steps = [(x, t, text, img), (more[1][0], more[1][1], more[1][2], img), (more[2][0], more[2][1], text, img)]

    def oracle_rule(out):
        out = out.float().cpu()
        ref32, ref16 = gold["out_fp32"], gold["out_bf16"].float()
        e_ref, e_our = (ref16 - ref32).abs(), (out - ref32).abs()
        assert e_our.mean() <= 1.25 * e_ref.mean(), f"mean err {e_our.mean():.3g} vs reference's own bf16 error {e_ref.mean():.3g}"
        assert e_our.max() <= 1.5 * e_ref.max(), f"max err {e_our.max():.3g} vs reference's own bf16 error {e_ref.max():.3g}"
        assert (out - ref16).abs().mean() <= 1.25 * e_ref.mean()

    _sequence_parallel_matches_single(models, steps, (case.frames, case.height, case.width), 2, oracle_check=oracle_rule)


# ---- refusals before the first launch: each its own message, never the host barrier's timeout
def _refusal(heads, world, latent, B=1, region_latent=None, prepare=None, **fwd):
    """Configure rank 0 of `world` (the other ranks never run) with the host barrier on and a region sized for `region_latent`, run one
    forward at `latent` and return the CEError it raised."""
    import chronoedit_b200 as ce
    from chronoedit_b200 import _lib, parallel

    dev = torch.device("cuda", torch.cuda.current_device())
    m = _model(heads, 1, 512, seed=7, dev=dev)
    if prepare:
        prepare(m)
    m.pack_weights()
    T, H, W = latent
    rT, rH, rW = region_latent or latent
    n = _lib.lib().ce_dit_sp_region_bytes(m._handle, B, rT, rH, rW, world)
    assert n > 0
    regions = [torch.zeros(n, dtype=torch.uint8, device=dev) for _ in range(world)]
    _lib.check(_lib.lib().ce_dit_sp_host_barrier(m._handle, SHORT_MS))
    parallel.configure_sequence_parallel(m, 0, [r.data_ptr() for r in regions], n, {})
    g = torch.Generator(device=dev).manual_seed(3)
    x = torch.randn(B, 36, T, H, W, generator=g, device=dev)
    text = torch.randn(B, 64, 4096, generator=g, device=dev)
    img = torch.randn(B, 257, 1280, generator=g, device=dev)
    try:
        with pytest.raises(ce.CEError) as e:
            m(x, torch.full((B,), 500, device=dev), text, img, **fwd)
    finally:
        parallel.disable_sequence_parallel(m)
    assert "host barrier" not in str(e.value)
    return str(e.value)


@gpu
def test_sequence_parallel_refuses_fp8_weights():
    assert "not built for FP8 weights" in _refusal(2, 2, (2, 32, 32), prepare=lambda m: m.enable_fp8())


@gpu
@pytest.mark.parametrize("how", [{"return_block0": True}, {"capture_layers": (0,)}], ids=["return_block0", "capture_layers"])
def test_sequence_parallel_refuses_block_capture(how):
    assert "no per-launch profiling / block capture" in _refusal(2, 2, (2, 32, 32), **how)


@gpu
def test_sequence_parallel_refuses_width_not_multiple_of_256():
    assert "the width must be a multiple of 256" in _refusal(3, 3, (2, 24, 32))   # D 384, 384 tokens


@gpu
def test_sequence_parallel_refuses_fewer_than_256_tokens():
    assert "at least 256 tokens" in _refusal(2, 2, (2, 16, 14))   # 112 tokens


@gpu
def test_sequence_parallel_refuses_tokens_not_divisible_by_world():
    # 270 tokens at world 4 (the region is sized for 256 tokens, the geometry the handle was configured for)
    assert "tokens must divide by the rank count" in _refusal(4, 4, (2, 18, 30), region_latent=(2, 16, 32))


@gpu
def test_host_barrier_times_out_with_the_rank_and_poisons_the_group():
    """Rank 0 alone reaches the first barrier: it fails after the timeout naming itself and the missing rank, and the group then fails
    at once."""
    import chronoedit_b200 as ce
    from chronoedit_b200 import _lib, parallel

    dev = torch.device("cuda", torch.cuda.current_device())
    m = _model(2, 1, 512, seed=7, dev=dev)
    n = parallel.sp_region_bytes(m, 1, 2, 32, 32, 2)
    regions = [torch.zeros(n, dtype=torch.uint8, device=dev) for _ in range(2)]
    _lib.check(_lib.lib().ce_dit_sp_host_barrier(m._handle, 500))
    parallel.configure_sequence_parallel(m, 0, [r.data_ptr() for r in regions], n, {})
    g = torch.Generator(device=dev).manual_seed(3)
    args = (torch.randn(1, 36, 2, 32, 32, generator=g, device=dev), torch.tensor([500], device=dev),
            torch.randn(1, 64, 4096, generator=g, device=dev), torch.randn(1, 257, 1280, generator=g, device=dev))
    try:
        t0 = time.perf_counter()
        with pytest.raises(ce.CEError, match=r"rank 0 timed out after 500 ms at barrier 1 waiting for rank\(s\) 1"):
            m(*args)
        assert time.perf_counter() - t0 < 30
        t0 = time.perf_counter()
        with pytest.raises(ce.CEError, match="the group failed earlier"):
            m(*args)
        assert time.perf_counter() - t0 < 5
    finally:
        parallel.disable_sequence_parallel(m)
    assert torch.isfinite(m(*args, return_dict=False)[0].float()).all()   # the single-GPU forward is unaffected
