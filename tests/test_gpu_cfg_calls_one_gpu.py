"""The call-pair split (parallel.enable_cfg_parallel_calls) on ONE GPU: two mirror handles with identical weights play the two ranks,
each driven from its own host thread on its own stream, with ordinary device allocations of ce_dit_cp_region_bytes as peer regions
and the host barrier (ce_dit_cp_host_barrier) at the exchange.  That runs the pairing, the NaN fill, the exchange's peer stores and
the alternating slot sets on a single device, and no kernel ever waits for another rank.

Asserted per case: every rank's result equals the single-GPU run bit for bit -- the decoded video of the pipeline loop
(oracle/pipeline_oracle.run_pipeline, the restatement of the unchanged pipeline) for `edit_5f` and `reason_cut` (whose cut from 8 to 2
latent frames runs in a region sized for 8), and every combined noise prediction of a pipeline-order loop for the 14B width, FP8
weights + FP8 attention, TeaCache and the grid; nothing is written outside the parts of the regions the exchange owns (the flags
block, the slots' tails past the largest sample and a guard band keep a byte pattern).  With TeaCache, each rank's records equal the
single-GPU records of the conditioning it computes.  The grid (tokens over 2 handles x the pair over 2) runs on 4 handles with the
token split's host barrier.  Each refusal is checked under a short host barrier, so a regression fails with a timeout message instead
of a wrong answer.

tests/test_gpu_cfg_calls.py keeps what only two GPUs can show: the device flag barrier, CUDA IPC and NVLink peer stores."""
import dataclasses

import pytest
import torch

from tests.sp_one_gpu import BARRIER_MS, SHORT_MS, _clean_device, assert_pattern_kept, guarded_regions, run_ranks  # noqa: F401
from tests.test_cfg_parallel_cpu import bp_layout, bp_unwritten_ranges
from tests.test_gpu_seqpar_one_gpu import _mirrors, _model, sp_layout, sp_unwritten_ranges

gpu = pytest.mark.gpu


def _configure(models, latent, B=1, host_ms=BARRIER_MS):
    """Host barrier on and the call-pair group configured for `models` (rank r = index), regions sized for calls of batch B at
    `latent`; returns (regions, bytes, layout)."""
    from chronoedit_b200 import _lib, parallel

    T, H, W = latent
    m0 = models[0]
    n = parallel.cfg_calls_region_bytes(m0, B, T, H, W)
    lay = bp_layout(B, m0.config.out_channels, T, H, W)
    assert n == lay["bytes"]
    regions = guarded_regions(n, 2, m0.device)
    for r, m in enumerate(models):
        _lib.check(_lib.lib().ce_dit_cp_host_barrier(m._ensure_handle(), host_ms))
        parallel.configure_cfg_parallel_calls(m, r, [g.data_ptr() for g in regions], n, {})
    return regions, n, lay


def _disable(models):
    from chronoedit_b200 import parallel

    for m in models:
        parallel.disable_cfg_parallel_calls(m)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# the pipeline loop
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("name", ["edit_5f", "reason_cut"])
def test_pipeline_video_on_two_handles_equals_one_gpu(name, _clean_device):
    from oracle import pipeline_cases as PC
    from tests.test_gpu_pipeline import _mirrors as pipeline_mirrors

    dev = torch.device("cuda", torch.cuda.current_device())
    case = PC.PIPELINE_CASES[name]
    tr, vae, sch = pipeline_mirrors(case, dev)
    want = PC.run_oracle_pipeline(case, torch.bfloat16, device=dev, transformer=tr, vae=vae, scheduler=sch)
    torch.cuda.synchronize()
    assert torch.isfinite(want).all()
    ranks = [pipeline_mirrors(case, dev) for _ in range(2)]   # per rank: its own transformer, VAE and scheduler
    T = (case.num_frames - 1) // 4 + 1
    regions, n, lay = _configure([r[0] for r in ranks], (T, case.height // 8, case.width // 8))
    try:
        videos = run_ranks(lambda r: PC.run_oracle_pipeline(case, torch.bfloat16, device=dev, transformer=ranks[r][0], vae=ranks[r][1],
                                                            scheduler=ranks[r][2]), 2, timeout=600)
        torch.cuda.synchronize()
        assert all(m._cp_pair is None for m, _, _ in ranks)
    finally:
        _disable([r[0] for r in ranks])
    for r, v in enumerate(videos):
        assert torch.equal(v, want), f"rank {r}: max|diff| {float((v - want).abs().max())}"
    assert_pattern_kept(regions, n, bp_unwritten_ranges(lay))


# ---------------------------------------------------------------------------------------------------------------------
# a pipeline-order loop on a transformer alone: per step the prompt call, then the negative-prompt call with the same latents and
# timestep tensors, the guidance combine and an Euler step
# ---------------------------------------------------------------------------------------------------------------------
def _loop_inputs(latent, dev, seed, steps):
    T, H, W = latent
    g = torch.Generator(device=dev).manual_seed(seed)
    prompt = torch.randn(1, 512, 4096, generator=g, device=dev).bfloat16()
    prompt[:, 100:] = 0
    negative = torch.randn(1, 512, 4096, generator=g, device=dev).bfloat16()
    negative[:, 20:] = 0
    return dict(lat=torch.randn(1, 16, T, H, W, generator=g, device=dev).bfloat16(),
                cond=torch.randn(1, 20, T, H, W, generator=g, device=dev).bfloat16(), prompt=prompt, negative=negative,
                img=torch.randn(1, 257, 1280, generator=g, device=dev).bfloat16(),
                ts=[1000.0 * (1 - i / steps) ** 1.5 for i in range(steps)])


def _loop(model, inp):
    """The combined noise prediction of every step.  The encoder states are the same objects at every step (per thread: cloned once),
    as the pipeline passes them."""
    prompt, negative, img = inp["prompt"].clone(), inp["negative"].clone(), inp["img"].clone()
    lat, cond = inp["lat"].clone(), inp["cond"]
    outs = []
    for i, tv in enumerate(inp["ts"]):
        x = torch.cat([lat, cond], dim=1)
        t = torch.tensor([tv], device=lat.device)
        noise_pred = model(hidden_states=x, timestep=t, encoder_hidden_states=prompt, encoder_hidden_states_image=img, return_dict=False)[0]
        noise_uncond = model(hidden_states=x, timestep=t, encoder_hidden_states=negative, encoder_hidden_states_image=img,
                             return_dict=False)[0]
        noise = noise_uncond + 5.0 * (noise_pred - noise_uncond)
        outs.append(noise.clone())
        nxt = inp["ts"][i + 1] if i + 1 < len(inp["ts"]) else 0.0
        lat = (lat.float() + (nxt - tv) / 1000.0 * noise.float()).bfloat16()
    return outs


def _loop_matches_single(models, inp, latent, check_records=False):
    m0 = models[0]
    if check_records:
        for m in models:
            m.reset_teacache()
    want = _loop(m0, inp)
    torch.cuda.synchronize()
    single_records = m0.teacache_records if check_records else None
    for w in want:
        assert torch.isfinite(w.float()).all() and w.float().std() > 0
    regions, n, lay = _configure(models, latent)
    try:
        if check_records:
            for m in models:
                m.reset_teacache()
        outs = run_ranks(lambda r: _loop(models[r], inp), 2, timeout=900)
        torch.cuda.synchronize()
        records = [m.teacache_records for m in models] if check_records else None
    finally:
        _disable(models)
    bad = [f"step {i}, rank {r}: max|diff| {float((o[i].float() - want[i].float()).abs().max()):.4g}"
           for r, o in enumerate(outs) for i in range(len(want)) if not torch.equal(o[i], want[i])]
    assert not bad, "the call-pair split differs from one GPU:\n" + "\n".join(bad)
    assert_pattern_kept(regions, n, bp_unwritten_ranges(lay))
    return single_records, records


SMALL = (4, 2, 1024, (2, 30, 42))          # heads, layers, ffn, latent: 630 tokens, D = 512
WIDE = (40, 1, 13824, (2, 32, 40))         # the 14B model's width and FFN, 640 tokens


@gpu
@pytest.mark.parametrize("shape", [SMALL, WIDE], ids=["small", "14b_width"])
def test_pair_loop_on_two_handles_equals_one_gpu(shape, _clean_device):
    heads, layers, ffn, latent = shape
    dev = torch.device("cuda", torch.cuda.current_device())
    models = _mirrors(_model(heads, layers, ffn, seed=heads * 100 + layers, dev=dev), 2)
    _loop_matches_single(models, _loop_inputs(latent, dev, seed=heads, steps=3), latent)


@gpu
def test_pair_loop_with_fp8_weights_and_attention_equals_one_gpu(_clean_device):
    heads, layers, ffn, latent = SMALL
    dev = torch.device("cuda", torch.cuda.current_device())
    models = _mirrors(_model(heads, layers, ffn, seed=31, dev=dev), 2)
    for m in models:   # after loading: the mirrors copy the bf16 weights, then each quantizes them
        m.enable_fp8()
        m.enable_fp8_attention()
    _loop_matches_single(models, _loop_inputs(latent, dev, seed=5, steps=3), latent)


@gpu
@pytest.mark.parametrize("thresh", [1e9, float("-inf")], ids=["skips", "never_skips"])
def test_pair_loop_with_teacache_keeps_every_decision(thresh, _clean_device):
    """An 8-step loop with TeaCache (and FP8 weights) on: the videos are equal, and rank r's records are the single-GPU records of
    conditioning r (slot 0 the prompt, slot 1 the negative prompt; each rank numbers its one conditioning 0)."""
    heads, layers, ffn, latent = SMALL
    dev = torch.device("cuda", torch.cuda.current_device())
    models = _mirrors(_model(heads, layers, ffn, seed=77, dev=dev), 2)
    for m in models:
        m.enable_fp8()
        m.enable_teacache(thresh, num_inference_steps=8)
    single, records = _loop_matches_single(models, _loop_inputs(latent, dev, seed=9, steps=8), latent, check_records=True)
    assert len(single) == 16 and [len(r) for r in records] == [8, 8]
    skipped = sum(not e.computed for e in single)
    print(f"  thresh {thresh}: single-GPU computed {[e.computed for e in single]}")
    assert (skipped > 0) == (thresh > 1), f"{skipped} skipped calls at threshold {thresh}"
    for r in range(2):
        want = [dataclasses.replace(e, slot=0) for e in single if e.slot == r]
        assert list(records[r]) == want, f"rank {r}'s records differ from the single-GPU records of conditioning {r}"
    for m in models:
        m.disable_teacache()


@gpu
def test_grid_tokens_by_call_on_four_handles(_clean_device):
    """Tokens over 2 handles inside each call, the pair over 2: handle k = 2 i + j is token rank j of token group i (which computes
    role i) and rank i of pair group j.  The token split is configured for the call's own batch (1)."""
    from chronoedit_b200 import _lib, parallel

    heads, layers, ffn, latent = SMALL
    T, H, W = latent
    dev = torch.device("cuda", torch.cuda.current_device())
    models = _mirrors(_model(heads, layers, ffn, seed=4242, dev=dev), 4)
    inp = _loop_inputs(latent, dev, seed=11, steps=3)
    want = _loop(models[0], inp)
    n_sp = parallel.sp_region_bytes(models[0], 1, T, H, W, 2)
    n_cp = parallel.cfg_calls_region_bytes(models[0], 1, T, H, W)
    sp_regions = [guarded_regions(n_sp, 2, dev) for _ in range(2)]   # [token group i] -> its two regions
    cp_regions = [guarded_regions(n_cp, 2, dev) for _ in range(2)]   # [pair group j] -> its two regions
    try:
        for k, m in enumerate(models):
            i, j = divmod(k, 2)
            _lib.check(_lib.lib().ce_dit_sp_host_barrier(m._ensure_handle(), BARRIER_MS))
            _lib.check(_lib.lib().ce_dit_cp_host_barrier(m._handle, BARRIER_MS))
            parallel.configure_sequence_parallel(m, j, [r.data_ptr() for r in sp_regions[i]], n_sp, {})
            parallel.configure_cfg_parallel_calls(m, i, [r.data_ptr() for r in cp_regions[j]], n_cp, {})
        outs = run_ranks(lambda k: _loop(models[k], inp), 4, timeout=900)
        torch.cuda.synchronize()
    finally:
        for m in models:
            parallel.disable_cfg_parallel_calls(m)
            parallel.disable_sequence_parallel(m)
    torch.cuda.synchronize()
    for k, o in enumerate(outs):
        for s in range(len(want)):
            assert torch.equal(o[s], want[s]), f"step {s}, handle {k}: the grid differs from one GPU"
    lay_sp = sp_layout(1, T * (H // 2) * (W // 2), heads * 128, 64, 2)
    for i in range(2):
        assert_pattern_kept(sp_regions[i], n_sp, sp_unwritten_ranges(lay_sp))
    for j in range(2):
        assert_pattern_kept(cp_regions[j], n_cp, bp_unwritten_ranges(bp_layout(1, 16, T, H, W)))


@gpu
def test_a_pairing_mismatch_is_refused_and_the_next_pair_works(_clean_device):
    """Both ranks see a second call with other latents: both raise before any launch (no barrier is reached, the epoch stays), the
    pair is dropped, and the next correctly paired step equals one GPU."""
    from chronoedit_b200._lib import CEError

    heads, layers, ffn, latent = SMALL
    dev = torch.device("cuda", torch.cuda.current_device())
    models = _mirrors(_model(heads, layers, ffn, seed=12, dev=dev), 2)
    inp = _loop_inputs(latent, dev, seed=13, steps=1)
    want = _loop(models[0], inp)
    regions, n, lay = _configure(models, latent)

    def rank(r):
        m = models[r]
        x = torch.cat([inp["lat"], inp["cond"]], dim=1)
        t = torch.tensor([500.0], device=dev)
        m(x, t, inp["prompt"], inp["img"])
        try:
            m(x.clone(), t, inp["negative"], inp["img"])
        except CEError as e:
            msg = str(e)
        else:
            msg = None
        assert m._cp_pair is None
        return msg, _loop(m, inp)

    try:
        outs = run_ranks(rank, 2, timeout=600)
    finally:
        _disable(models)
    for r, (msg, got) in enumerate(outs):
        assert msg is not None and "does not pair with the previous one" in msg, f"rank {r}: {msg}"
        assert torch.equal(got[0], want[0]), f"rank {r}: the pair after the refused call differs from one GPU"
    assert_pattern_kept(regions, n, bp_unwritten_ranges(lay))


# ---- refusals before the first launch: each its own message, never the host barrier's timeout
def _refusal(call, region_latent=(2, 32, 32), prepare=None):
    """Configure rank 0 of 2 (rank 1 never runs) with the host barrier on and a region sized for `region_latent`, then run
    `call(m, inputs(T, H, W))` and return the CEError it raised."""
    import chronoedit_b200 as ce
    from chronoedit_b200 import _lib, parallel

    dev = torch.device("cuda", torch.cuda.current_device())
    m = _model(2, 1, 512, seed=7, dev=dev)
    if prepare:
        prepare(m)
    m.pack_weights()
    n = parallel.cfg_calls_region_bytes(m, 1, *region_latent)
    regions = [torch.zeros(n, dtype=torch.uint8, device=dev) for _ in range(2)]
    _lib.check(_lib.lib().ce_dit_cp_host_barrier(m._handle, SHORT_MS))
    parallel.configure_cfg_parallel_calls(m, 0, [r.data_ptr() for r in regions], n, {})
    g = torch.Generator(device=dev).manual_seed(3)

    def inputs(T=2, H=32, W=32):
        return (torch.randn(1, 36, T, H, W, generator=g, device=dev).bfloat16(), torch.full((1,), 500.0, device=dev),
                torch.randn(1, 64, 4096, generator=g, device=dev).bfloat16(), torch.randn(1, 257, 1280, generator=g, device=dev).bfloat16())

    try:
        with pytest.raises(ce.CEError) as e:
            call(m, inputs)
    finally:
        m._cp_pair = None   # a refused call may leave the first call of a pair open; nothing to warn about here
        parallel.disable_cfg_parallel_calls(m)
    assert "host barrier" not in str(e.value)
    torch.cuda.synchronize()
    assert all(int(r.count_nonzero()) == 0 for r in regions), "a refused call wrote into a peer region"
    return str(e.value)


@gpu
@pytest.mark.parametrize("how", [{"return_block0": True}, {"capture_layers": (0,)}], ids=["return_block0", "capture_layers"])
def test_call_pair_refuses_block_capture(how):
    assert "not available with the call-pair split" in _refusal(lambda m, inp: m(*inp(), **how))


@gpu
def test_call_pair_refuses_forward_host():
    def host(m, inp):
        x, t, txt, img = (a.cpu() for a in inp())
        m.forward_host(x, t, txt, img)

    assert "forward_host is not available with the call-pair split" in _refusal(host)


@gpu
def test_call_pair_refuses_the_fp32_validation_forward():
    def fp32(m, inp):
        m.enable_fp32_validation({k: v.detach().float() for k, v in m.named_parameters()})
        x, t, txt, img = inp()
        m.forward_fp32(x.float(), t, txt.float(), img.float())

    assert "forward_fp32 is not available with the call-pair split" in _refusal(fp32)


@gpu
def test_call_pair_refuses_a_capturing_stream():
    def captured(m, inp):
        args = inp()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            m(*args)

    assert "the stream is capturing" in _refusal(captured)


@gpu
def test_call_pair_refuses_a_sample_larger_than_the_slot():
    def larger(m, inp):   # region for 2 latent frames; the first call of the pair computes, the exchange of the second refuses
        args = inp(T=8)
        m(*args)
        m(args[0], args[1], torch.zeros_like(args[2]), args[3])

    assert "needs a slot of" in _refusal(larger)


@gpu
def test_call_pair_and_batch_split_are_exclusive():
    from chronoedit_b200 import parallel

    def with_bp(m, inp):
        parallel.configure_cfg_parallel(m, 0, [4096 * 256, 8192 * 256], 1 << 20, {})

    assert "the two CFG splits are exclusive" in _refusal(with_bp)
    m = _model(2, 1, 512, seed=7, dev=torch.device("cuda", torch.cuda.current_device()))
    n = parallel.cfg_region_bytes(m, 2, 2, 32, 32, 2)
    regions = [torch.zeros(n, dtype=torch.uint8, device=m.device) for _ in range(2)]
    parallel.configure_cfg_parallel(m, 0, [r.data_ptr() for r in regions], n, {})
    try:
        import chronoedit_b200 as ce

        with pytest.raises(ce.CEError, match="the two CFG splits are exclusive"):
            parallel.configure_cfg_parallel_calls(m, 0, [r.data_ptr() for r in regions], n, {})
        assert getattr(m, "_cp_state", None) is None
    finally:
        parallel.disable_cfg_parallel(m)
