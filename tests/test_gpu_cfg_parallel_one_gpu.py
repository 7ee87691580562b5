"""The batch split of the DiT forward (parallel.enable_cfg_parallel) on ONE GPU: `world` mirror instances with identical weights play the
ranks, each driven from its own host thread on its own stream, with ordinary device allocations as peer regions and the host barrier
(ce_dit_bp_host_barrier) at the exchange.  That runs the sample offsets, the exchange's peer stores and the alternating slot sets on a
single device, and no kernel ever waits for another rank.

Asserted per case: every rank returns the single-GPU forward of the full batch bit for bit, in the same mode (bf16, FP8 weights, FP8
attention), over three steps with the context cache on and prompt and negative prompt alternating, and again once the split is off;
nothing is written outside the parts of the regions the exchange owns (the flags block, each rank's own part of its slots, the slots'
alignment gaps and a guard band keep a byte pattern); the inputs are unchanged.  TeaCache decides on each rank's own samples, so its
reference is a single-GPU TeaCache run on that rank's half alone.  The grid (tokens over 2 ranks x batch over 2) runs on 4 handles.
The refusals are checked under a short host barrier, so a regression fails with a timeout message instead of a wrong answer.

tests/test_gpu_cfg_parallel.py keeps what only two GPUs can show: the device flag barrier, CUDA IPC and NVLink peer stores."""
import pytest
import torch

from tests.sp_one_gpu import BARRIER_MS, SHORT_MS, _clean_device, assert_pattern_kept, guarded_regions, run_ranks  # noqa: F401
from tests.test_cfg_parallel_cpu import bp_layout, bp_unwritten_ranges
from tests.test_gpu_seqpar_one_gpu import _mirrors, _model, _steps, sp_layout, sp_unwritten_ranges

gpu = pytest.mark.gpu


def _own_part_ranges(lay, B, world, r):
    """The part of each slot of rank r's region that only rank r's own samples would fill: the exchange never writes it."""
    part = lay["used"] // world
    return [(f"own part of slot {i}", a + r * part, a + (r + 1) * part) for i, a in enumerate(lay["slot"])]


def _configure(models, world, B, latent):
    """Host barrier on and the batch group configured for `models` (rank r = index); returns (regions, bytes, layout)."""
    from chronoedit_b200 import _lib, parallel

    T, H, W = latent
    m0 = models[0]
    n = parallel.cfg_region_bytes(m0, B, T, H, W, world)
    lay = bp_layout(B, m0.config.out_channels, T, H, W)
    assert n == lay["bytes"]
    regions = guarded_regions(n, world, m0.device)
    ptrs = [r.data_ptr() for r in regions]
    for r, m in enumerate(models):
        _lib.check(_lib.lib().ce_dit_bp_host_barrier(m._ensure_handle(), BARRIER_MS))
        parallel.configure_cfg_parallel(m, r, ptrs, n, {})
    return regions, n, lay


def _assert_regions_kept(regions, n, lay, B, world):
    for r, region in enumerate(regions):
        ranges = [(f"rank {r}: {what}", a, b) for what, a, b in bp_unwritten_ranges(lay) + _own_part_ranges(lay, B, world, r)]
        assert_pattern_kept([region], n, ranges)


def _split_matches_single(models, steps, latent, world):
    from chronoedit_b200 import parallel

    m0 = models[0]
    B = steps[0][0].shape[0]
    inputs = [tuple(a.clone() for a in st) for st in steps]
    refs = [m0(*st, return_dict=False)[0].clone() for st in steps]
    torch.cuda.synchronize()
    for ref in refs:
        assert torch.isfinite(ref.float()).all() and ref.float().std() > 0
    regions, n, lay = _configure(models, world, B, latent)
    try:
        bad = []
        for it, st in enumerate(steps):
            outs = run_ranks(lambda r: models[r](*st, return_dict=False)[0], world, timeout=600)
            torch.cuda.synchronize()
            for r, o in enumerate(outs):
                if not torch.equal(o, refs[it]):
                    d = (o.float() - refs[it].float()).abs().flatten(1).amax(dim=1)
                    bad.append(f"step {it}, rank {r}: max|diff| per sample {[round(float(v), 5) for v in d]}")
        assert not bad, "batch-split sample differs from the single-GPU forward:\n" + "\n".join(bad)
    finally:
        for m in models:
            parallel.disable_cfg_parallel(m)
    torch.cuda.synchronize()
    _assert_regions_kept(regions, n, lay, B, world)
    for m in models:   # every handle is back on the single-GPU forward
        assert torch.equal(m(*steps[0], return_dict=False)[0], refs[0])
    for st, before in zip(steps, inputs):
        assert all(torch.equal(a, b) for a, b in zip(st, before)), "the forward modified its inputs"


SMALL = (4, 2, 1024, (2, 30, 42))          # heads, layers, ffn, latent: 630 tokens, D = 512
WIDE = (40, 1, 13824, (2, 32, 40))         # the 14B model's width and FFN, 640 tokens


@gpu
@pytest.mark.parametrize("shape", [SMALL, WIDE], ids=["small", "14b_width"])
@pytest.mark.parametrize("B,world", [(2, 2), (4, 2), (4, 4)], ids=["B2-w2", "B4-w2", "B4-w4"])
def test_batch_split_on_one_gpu_is_bit_identical(shape, B, world, _clean_device):
    heads, layers, ffn, latent = shape
    dev = torch.device("cuda", torch.cuda.current_device())
    models = _mirrors(_model(heads, layers, ffn, seed=heads * 1000 + layers, dev=dev), world)
    _split_matches_single(models, _steps(B, latent, dev, seed=world + 17 * heads + B), latent, world)


@gpu
@pytest.mark.parametrize("mode", ["fp8", "fp8_attention", "fp8_both"])
def test_batch_split_with_fp8_is_bit_identical(mode, _clean_device):
    heads, layers, ffn = 4, 2, 1024
    latent = (2, 32, 32)
    dev = torch.device("cuda", torch.cuda.current_device())
    models = _mirrors(_model(heads, layers, ffn, seed=31, dev=dev), 2)
    for m in models:   # after loading: the mirrors copy the bf16 weights, then each quantizes them
        if mode in ("fp8", "fp8_both"):
            m.enable_fp8()
        if mode in ("fp8_attention", "fp8_both"):
            m.enable_fp8_attention()
    _split_matches_single(models, _steps(2, latent, dev, seed=5), latent, 2)


@gpu
@pytest.mark.parametrize("thresh", [0.3, 1e9])
def test_batch_split_with_teacache_equals_each_half_alone(thresh, _clean_device):
    """An 8-step CFG loop through step_cfg with TeaCache on under the split: every rank returns the same full batch, and sample r with
    rank r's records equals a single-GPU TeaCache run on half r alone (rel is summed over a call's own samples, so the full-batch
    TeaCache run decides on other sums and is not the reference)."""
    from chronoedit_b200 import parallel
    from chronoedit_b200.scheduler import FlowUniPCMultistepScheduler

    dev = torch.device("cuda", torch.cuda.current_device())
    T, H, W = latent = (2, 32, 32)
    models = _mirrors(_model(4, 2, 1024, seed=77, dev=dev), 2)
    g = torch.Generator(device=dev).manual_seed(9)
    lat = torch.randn(1, 16, T, H, W, generator=g, device=dev).bfloat16()
    cond = torch.randn(1, 20, T, H, W, generator=g, device=dev).bfloat16()
    text = torch.randn(2, 64, 4096, generator=g, device=dev).bfloat16()
    text[1, 20:] = 0
    img = torch.randn(1, 257, 1280, generator=g, device=dev).bfloat16().expand(2, -1, -1).contiguous()
    d_in = torch.cat([lat, cond], dim=1).contiguous()
    sched = FlowUniPCMultistepScheduler(num_train_timesteps=1000, shift=1, use_dynamic_shifting=False)
    sched.set_timesteps(8, device=dev, shift=5.0)
    for m in models:
        m.enable_teacache(thresh, num_inference_steps=8)
    regions, n, lay = _configure(models, 2, 2, latent)
    calls, outs_all = [], []
    try:
        for i in range(8):
            t = sched.timesteps[i]
            x, tt = d_in.expand(2, -1, -1, -1, -1).contiguous(), t.expand(2).contiguous()
            outs = run_ranks(lambda r: models[r](x, tt, text, img, return_dict=False)[0].clone(), 2, timeout=600)
            torch.cuda.synchronize()
            assert torch.equal(outs[0], outs[1]), f"step {i}: the ranks return different batches"
            calls.append((x.clone(), tt.clone()))
            outs_all.append(outs[0])
            lat = sched.step_cfg(outs[0][0:1], outs[0][1:2], 5.0, t, lat, model_input_out=d_in)
        records = [m.teacache_records for m in models]
    finally:
        for m in models:
            parallel.disable_cfg_parallel(m)
    torch.cuda.synchronize()
    _assert_regions_kept(regions, n, lay, 2, 2)
    print(f"  thresh {thresh}: computed per rank {[[e.computed for e in rec] for rec in records]}")
    if thresh > 1:
        assert any(not e.computed for rec in records for e in rec), "no call was skipped"
    alone = models[0]   # the split is off: a single-GPU TeaCache run on each half by itself
    for r in range(2):
        alone.reset_teacache()
        txt_r, img_r = text[r: r + 1].clone(), img[r: r + 1].clone()   # one conditioning: the same objects at every step
        for i, (x, tt) in enumerate(calls):
            ref = alone(x[r: r + 1], tt[r: r + 1], txt_r, img_r, return_dict=False)[0]
            assert torch.equal(outs_all[i][r: r + 1], ref), f"step {i}: sample {r} differs from half {r} alone"
        assert alone.teacache_records == records[r], f"rank {r}'s records differ from half {r} alone"
    for m in models:
        m.disable_teacache()


@gpu
def test_grid_tokens_by_batch_on_four_handles(_clean_device):
    """Tokens over 2 ranks inside each half of the CFG pair, the pair over 2 ranks: handle 2 i + j is batch rank i and token rank j.
    The token split is configured for the local batch (B / 2), the batch split for B."""
    from chronoedit_b200 import _lib, parallel

    heads, layers, ffn, latent = WIDE
    T, H, W = latent
    B = 2
    dev = torch.device("cuda", torch.cuda.current_device())
    models = _mirrors(_model(heads, layers, ffn, seed=4242, dev=dev), 4)
    steps = _steps(B, latent, dev, seed=11)
    refs = [models[0](*st, return_dict=False)[0].clone() for st in steps]
    L_tok = T * (H // 2) * (W // 2)
    n_sp = parallel.sp_region_bytes(models[0], B // 2, T, H, W, 2)
    n_bp = parallel.cfg_region_bytes(models[0], B, T, H, W, 2)
    sp_regions = [guarded_regions(n_sp, 2, dev) for _ in range(2)]   # [batch rank i] -> the regions of its token group
    bp_regions = [guarded_regions(n_bp, 2, dev) for _ in range(2)]   # [token rank j] -> the regions of its batch group
    try:
        for k, m in enumerate(models):
            i, j = divmod(k, 2)
            _lib.check(_lib.lib().ce_dit_sp_host_barrier(m._ensure_handle(), BARRIER_MS))
            _lib.check(_lib.lib().ce_dit_bp_host_barrier(m._handle, BARRIER_MS))
            parallel.configure_sequence_parallel(m, j, [r.data_ptr() for r in sp_regions[i]], n_sp, {})
            parallel.configure_cfg_parallel(m, i, [r.data_ptr() for r in bp_regions[j]], n_bp, {})
        for it, st in enumerate(steps):
            outs = run_ranks(lambda k: models[k](*st, return_dict=False)[0], 4, timeout=600)
            torch.cuda.synchronize()
            for k, o in enumerate(outs):
                assert torch.equal(o, refs[it]), f"step {it}, handle {k}: the grid differs from the single-GPU forward"
    finally:
        for m in models:
            parallel.disable_cfg_parallel(m)
            parallel.disable_sequence_parallel(m)
    torch.cuda.synchronize()
    lay_sp = sp_layout(B // 2, L_tok, heads * 128, 64, 2)
    for i in range(2):
        assert_pattern_kept(sp_regions[i], n_sp, sp_unwritten_ranges(lay_sp))
    for j in range(2):
        _assert_regions_kept(bp_regions[j], n_bp, bp_layout(B, 16, T, H, W), B, 2)
    for m in models:
        assert torch.equal(m(*steps[0], return_dict=False)[0], refs[0])


@gpu
def test_batch_split_forward_host(_clean_device):
    """One forward_host call (host inputs, staging on the device, host sample) per rank under the split."""
    from chronoedit_b200 import parallel

    heads, layers, ffn, latent = SMALL
    T, H, W = latent
    dev = torch.device("cuda", torch.cuda.current_device())
    models = _mirrors(_model(heads, layers, ffn, seed=3, dev=dev), 2)
    x, t, txt, img = (a.cpu() for a in _steps(2, latent, dev, seed=8)[0])
    t = t.float()
    ref = models[0].forward_host(x, t, txt, img).clone()
    regions, n, lay = _configure(models, 2, 2, latent)
    try:
        outs = run_ranks(lambda r: models[r].forward_host(x, t, txt, img).clone(), 2, timeout=600)
    finally:
        for m in models:
            parallel.disable_cfg_parallel(m)
    for r, o in enumerate(outs):
        assert torch.equal(o, ref), f"rank {r}: forward_host under the split differs from the single-GPU call"
    _assert_regions_kept(regions, n, lay, 2, 2)


# ---- refusals before the first launch: each its own message, never the host barrier's timeout
def _refusal(call, B=2, region_latent=(2, 32, 32), prepare=None):
    """Configure rank 0 of 2 (rank 1 never runs) with the host barrier on and a region sized for `region_latent`, then run `call(m,
    inputs(B, T, H, W))` and return the CEError it raised."""
    import chronoedit_b200 as ce
    from chronoedit_b200 import _lib, parallel

    dev = torch.device("cuda", torch.cuda.current_device())
    m = _model(2, 1, 512, seed=7, dev=dev)
    if prepare:
        prepare(m)
    m.pack_weights()
    n = parallel.cfg_region_bytes(m, 2, *region_latent, 2)
    regions = [torch.zeros(n, dtype=torch.uint8, device=dev) for _ in range(2)]
    _lib.check(_lib.lib().ce_dit_bp_host_barrier(m._handle, SHORT_MS))
    parallel.configure_cfg_parallel(m, 0, [r.data_ptr() for r in regions], n, {})
    g = torch.Generator(device=dev).manual_seed(3)

    def inputs(B, T=2, H=32, W=32):
        return (torch.randn(B, 36, T, H, W, generator=g, device=dev).bfloat16(), torch.full((B,), 500.0, device=dev),
                torch.randn(B, 64, 4096, generator=g, device=dev).bfloat16(), torch.randn(B, 257, 1280, generator=g, device=dev).bfloat16())

    try:
        with pytest.raises(ce.CEError) as e:
            call(m, inputs)
    finally:
        parallel.disable_cfg_parallel(m)
    assert "host barrier" not in str(e.value)
    torch.cuda.synchronize()
    assert all(int(r.count_nonzero()) == 0 for r in regions), "a refused call wrote into a peer region"
    return str(e.value)


@gpu
def test_batch_split_refuses_batch_one():
    msg = _refusal(lambda m, inp: m(*inp(1)))
    assert "the unchanged diffusers pipeline's batch-1 calls" in msg and "not split" in msg


@gpu
def test_batch_split_refuses_batch_one_with_teacache():
    msg = _refusal(lambda m, inp: m(*inp(1)), prepare=lambda m: m.enable_teacache(0.2, num_inference_steps=8))
    assert "the unchanged diffusers pipeline's batch-1 calls are not split" in msg


@gpu
def test_batch_split_refuses_a_sample_larger_than_the_slot():
    assert "needs a slot of" in _refusal(lambda m, inp: m(*inp(2, T=8)))   # region for 2 latent frames, call with 8


@gpu
@pytest.mark.parametrize("how", [{"return_block0": True}, {"capture_layers": (0,)}], ids=["return_block0", "capture_layers"])
def test_batch_split_refuses_block_capture(how):
    assert "no block capture / block0_out" in _refusal(lambda m, inp: m(*inp(2), **how))


@gpu
def test_batch_split_refuses_a_capturing_stream():
    def captured(m, inp):
        args = inp(2)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            m(*args)

    assert "the stream is capturing" in _refusal(captured)


@gpu
def test_batch_split_refuses_the_fp32_validation_forward():
    def fp32(m, inp):
        m.enable_fp32_validation({k: v.detach().float() for k, v in m.named_parameters()})
        x, t, txt, img = inp(2)
        m.forward_fp32(x.float(), t, txt.float(), img.float())

    assert "not built for the batch split" in _refusal(fp32)
