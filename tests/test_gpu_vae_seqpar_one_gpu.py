"""The VAE split over ranks on ONE GPU: `world` AutoencoderKLWan instances with one state dict play the ranks, each driven from its own
host thread on its own stream, with ordinary device allocations (plus a guard band) as peer regions and the host barrier
(ce_vae_sp_host_barrier) between the exchanges.  That runs every kernel, every peer-store address and every band's row arithmetic of
the split at world 2 to 8 on a single device, and no kernel ever waits for another rank.

Asserted per case: every rank's encode moments and decode video are bit-identical to the single-GPU call, for several calls in a row
under one configuration; the guard band after each region and its barrier flags (only the device barrier writes them) keep their byte
pattern; the inputs are unchanged; after disabling the split each handle gives the single-GPU bits again.

tests/test_gpu_seqpar.py keeps what only several GPUs can show: the device flag barrier, CUDA IPC and NVLink peer stores."""
import os
import time

import pytest
import torch

from oracle.vae_oracle import VAEConfig
from tests.sp_one_gpu import BARRIER_MS, SHORT_MS, _clean_device, assert_pattern_kept, guarded_regions, run_ranks  # noqa: F401
from tests.test_vae_seqpar_cpu import vae_sp_layout

gpu = pytest.mark.gpu


def _vae(cfg, seed, dev, sd=None):
    from chronoedit_b200.autoencoder import AutoencoderKLWan

    m = AutoencoderKLWan(base_dim=cfg.dim, z_dim=cfg.z_dim, dim_mult=tuple(cfg.dim_mult), num_res_blocks=cfg.num_res_blocks,
                         temperal_downsample=tuple(cfg.temperal_downsample), clamp_output=False, device=dev)
    if sd is not None:
        m.load_state_dict(sd)
        return m
    g = torch.Generator(device=dev).manual_seed(seed)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith("gamma"):
                p.normal_(0, 0.1, generator=g).add_(1.0)
            elif n.endswith("bias"):
                p.normal_(0, 0.05, generator=g)
            else:
                p.normal_(0, p[0].numel() ** -0.5, generator=g)
    return m


def _mirrors(first, world):
    sd = first.state_dict()
    c = first.config
    cfg = VAEConfig(dim=c.base_dim, z_dim=c.z_dim, dim_mult=tuple(c.dim_mult), num_res_blocks=c.num_res_blocks,
                    temperal_downsample=tuple(c.temperal_downsample))
    return [first] + [_vae(cfg, 0, first.device, sd) for _ in range(world - 1)]


def _call(vae, call):
    """("enc", video, _) -> the moments (mean | logvar, unclamped) encode computes; ("dec", z, clamp) -> the decoded video."""
    kind, x, clamp = call
    if kind == "enc":
        B, _, T, H, W = x.shape
        out = torch.empty(B, 2 * vae.z_dim, 1 + (T - 1) // 4, H // 8, W // 8, dtype=torch.bfloat16, device=x.device)
        vae._native_encode(x, out)
        return out
    vae.clamp_output = clamp
    return vae.decode(x, return_dict=False)[0]


def _row_diffs(out, ref):
    d = (out.float() - ref.float()).abs()
    rows = d.amax(dim=tuple(i for i in range(d.dim()) if i != d.dim() - 2))
    bad = (rows > 0).nonzero().flatten().tolist()
    return f"max|diff| {float(d.max()):.4g}, differing rows {bad[:12]}{' ...' if len(bad) > 12 else ''} of {rows.numel()}"


def _split_matches_single(vaes, H, W, calls, world, refs=None):
    from chronoedit_b200 import _lib, parallel

    v0 = vaes[0]
    inputs = [c[1].clone() for c in calls]
    if refs is None:
        refs = [_call(v0, c).clone() for c in calls]
    torch.cuda.synchronize()
    for ref in refs:
        assert torch.isfinite(ref.float()).all() and ref.float().std() > 0
    n = parallel.vae_sp_region_bytes(v0, H, W, world)
    c = v0.config
    cfg = VAEConfig(dim=c.base_dim, z_dim=c.z_dim, dim_mult=tuple(c.dim_mult), num_res_blocks=c.num_res_blocks,
                    temperal_downsample=tuple(c.temperal_downsample))
    assert vae_sp_layout(cfg, H, W)["bytes"] == n
    regions = guarded_regions(n, world, v0.device)
    try:
        for r, v in enumerate(vaes):
            _lib.check(_lib.lib().ce_vae_sp_host_barrier(v._ensure_handle(), BARRIER_MS))
            parallel.configure_vae_sequence_parallel(v, r, [g.data_ptr() for g in regions], n, {})
        bad = []
        for i, call in enumerate(calls):
            outs = run_ranks(lambda r: _call(vaes[r], call), world, timeout=900)
            torch.cuda.synchronize()
            for r, o in enumerate(outs):
                if not torch.equal(o, refs[i]):
                    bad.append(f"call {i} ({call[0]}, {tuple(call[1].shape)}), rank {r}: {_row_diffs(o, refs[i])}")
        assert not bad, "the split VAE differs from the single-GPU call:\n" + "\n".join(bad)
    finally:
        for v in vaes:
            parallel.disable_vae_sequence_parallel(v)
            _lib.lib().ce_vae_sp_host_barrier(v._handle, 0)
    torch.cuda.synchronize()
    assert_pattern_kept(regions, n, [("barrier flags", 0, 1024)])
    for v in vaes:   # every handle is back on the single-GPU call
        assert torch.equal(_call(v, calls[0]), refs[0])
    for c, before in zip(calls, inputs):
        assert torch.equal(c[1], before), "the call modified its input"
    return refs


def _video(T, H, W, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return (torch.rand(1, 3, T, H, W, generator=g, device=dev) * 2 - 1).bfloat16()


def _latent(zc, T, h, w, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randn(1, zc, T, h, w, generator=g, device=dev).bfloat16()


def _calls(cfg, H, W, dev, seed, enc_frames=(5, 9), dec_frames=(2, 3)):
    """encode, decode (clamp off), decode at another frame count (clamp on), encode again"""
    h, w = H // 8, W // 8
    return [("enc", _video(enc_frames[0], H, W, dev, seed), False), ("dec", _latent(cfg.z_dim, dec_frames[0], h, w, dev, seed + 1), False),
            ("dec", 2.5 * _latent(cfg.z_dim, dec_frames[1], h, w, dev, seed + 2), True), ("enc", _video(enc_frames[1], H, W, dev, seed + 3), False)]


# (name, config, H, W, worlds): latent rows h = H / 8 split over the ranks
CASES = [
    ("tiny_h4", VAEConfig.tiny(32), 32, 48, (2, 3, 4)),       # world 3: bands of 1, 1, 2 rows; world 4: one latent row per rank
    ("tiny_h8", VAEConfig.tiny(32), 64, 40, (8,)),            # one latent row per rank at world 8
    ("tiny_h11", VAEConfig.tiny(32), 88, 56, (3, 8)),         # unequal bands of 3 / 4 rows, and of 1 / 2 rows
    ("wan_h8", VAEConfig.wan21(), 64, 64, (2, 4)),            # the Wan2.1 width at the golden geometry
    ("wan_h16", VAEConfig.wan21(), 128, 96, (2, 4)),          # several rows per rank
]


@gpu
@pytest.mark.parametrize("name,cfg,H,W,world", [(c[0], c[1], c[2], c[3], w) for c in CASES for w in c[4]],
                         ids=[f"{c[0]}-w{w}" for c in CASES for w in c[4]])
def test_split_vae_on_one_gpu_is_bit_identical(name, cfg, H, W, world, _clean_device):
    dev = torch.device("cuda", torch.cuda.current_device())
    vaes = _mirrors(_vae(cfg, seed=H * 7 + W, dev=dev), world)
    _split_matches_single(vaes, H, W, _calls(cfg, H, W, dev, seed=world + H), world)


@gpu
def test_split_vae_720p(_clean_device):
    """The edit's geometry at world 2: encode 5 frames, decode 2 latent frames (clamped, as the pipeline decodes)."""
    dev = torch.device("cuda", torch.cuda.current_device())
    cfg = VAEConfig.wan21()
    vaes = _mirrors(_vae(cfg, seed=720, dev=dev), 2)
    calls = [("enc", _video(5, 720, 1280, dev, 1), False), ("dec", _latent(16, 2, 90, 160, dev, 2), True)]
    _split_matches_single(vaes, 720, 1280, calls, 2)


@gpu
def test_split_vae_temporal_reasoning(_clean_device):
    """Temporal reasoning's shapes at a smaller size, under one configuration: encode 29 frames, decode 8 latent frames, then the
    first and last of them (pipeline_chronoedit.py:776-779)."""
    dev = torch.device("cuda", torch.cuda.current_device())
    cfg = VAEConfig.wan21()
    vaes = _mirrors(_vae(cfg, seed=29, dev=dev), 2)
    z = _latent(16, 8, 12, 16, dev, 3)
    calls = [("enc", _video(29, 96, 128, dev, 4), False), ("dec", z, True), ("dec", z[:, :, [0, -1]].contiguous(), True)]
    _split_matches_single(vaes, 96, 128, calls, 2)


@gpu
@pytest.mark.parametrize("name", ["tiny_5f", "wan_5f_64"])
def test_split_vae_golden(name, golden_dir, _clean_device):
    """The golden fixtures' inputs and weights at world 2: the single-GPU result the ranks reproduce bit for bit also meets the parity
    rule of test_gpu_vae.py against the reference's outputs."""
    from safetensors.torch import load_file

    from oracle import cases
    from tests.test_gpu_vae import _build_vae

    case = cases.VAE_CASES[name]
    gold = load_file(os.path.join(golden_dir, f"vae_{name}.safetensors"))
    m = _build_vae(case)
    video, z = cases.vae_inputs(case)
    video, z = video.cuda().bfloat16(), z.cuda().bfloat16()
    vaes = _mirrors(m, 2)
    calls = [("enc", video, False), ("dec", z, False)]
    refs = [_call(m, c).clone() for c in calls]
    zc = case.cfg.z_dim
    for got, key in ((refs[0][:, :zc], "mu"), (refs[1], "dec")):
        got = got.float().cpu()
        ref32, ref16 = gold[f"{key}_fp32"], gold[f"{key}_bf16"].float()
        e_ref, e_our = (ref16 - ref32).abs(), (got - ref32).abs()
        assert e_our.mean() <= 1.25 * e_ref.mean(), f"{key}: mean err {e_our.mean():.3g} vs reference's own bf16 error {e_ref.mean():.3g}"
        assert e_our.max() <= 2.0 * e_ref.max(), f"{key}: max err {e_our.max():.3g} vs reference's own bf16 error {e_ref.max():.3g}"
    _split_matches_single(vaes, case.height, case.width, calls, 2, refs=refs)


# ---- refusals before the first barrier: each its own message, never the host barrier's timeout
def _configured(world, H, W, ms=SHORT_MS):
    from chronoedit_b200 import _lib, parallel

    dev = torch.device("cuda", torch.cuda.current_device())
    v = _vae(VAEConfig.tiny(32), seed=5, dev=dev)
    v.pack_weights()
    n = parallel.vae_sp_region_bytes(v, H, W, world)
    regions = [torch.zeros(n, dtype=torch.uint8, device=dev) for _ in range(world)]
    _lib.check(_lib.lib().ce_vae_sp_host_barrier(v._ensure_handle(), ms))
    parallel.configure_vae_sequence_parallel(v, 0, [r.data_ptr() for r in regions], n, {})
    return v, regions


def _refusal(v, fn):
    import chronoedit_b200 as ce
    from chronoedit_b200 import _lib, parallel

    try:
        with pytest.raises(ce.CEError) as e:
            fn()
    finally:
        parallel.disable_vae_sequence_parallel(v)
        _lib.lib().ce_vae_sp_host_barrier(v._handle, 0)
    assert "host barrier" not in str(e.value)
    return str(e.value)


@gpu
def test_split_vae_refuses_fewer_rows_than_ranks():
    dev = torch.device("cuda", torch.cuda.current_device())
    v, _ = _configured(4, 64, 48)
    msg = _refusal(v, lambda: v.encode(_video(1, 24, 48, dev, 0)))
    assert "3 latent rows cannot be split over 4 ranks" in msg
    v, _ = _configured(4, 64, 48)
    assert "2 latent rows cannot be split over 4 ranks" in _refusal(v, lambda: v.decode(_latent(16, 1, 2, 6, dev, 0)))


@gpu
def test_split_vae_refuses_a_geometry_larger_than_the_region():
    dev = torch.device("cuda", torch.cuda.current_device())
    v, _ = _configured(2, 32, 48)
    assert "needs a peer region of" in _refusal(v, lambda: v.decode(_latent(16, 2, 8, 8, dev, 0)))


@gpu
def test_split_vae_refuses_stream_capture():
    from chronoedit_b200 import _lib

    dev = torch.device("cuda", torch.cuda.current_device())
    v, _ = _configured(2, 32, 48)
    z = _latent(16, 1, 4, 6, dev, 0)
    out = torch.empty(1, 3, 1, 32, 48, dtype=torch.bfloat16, device=dev)
    L = _lib.lib()
    n = L.ce_vae_workspace_bytes(v._handle, 1, 1, 4, 6)
    assert n > 0
    ws = torch.empty(n, dtype=torch.uint8, device=dev)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        rc = L.ce_vae_decode(v._handle, _lib.ptr(z[0]), _lib.ptr(out[0]), 1, 4, 6, 0, _lib.ptr(ws), n, _lib.current_stream())
        msg = L.ce_last_error().decode()
    assert rc != 0 and "the stream is capturing" in msg and "host barrier" not in msg, msg
    from chronoedit_b200 import parallel

    parallel.disable_vae_sequence_parallel(v)
    L.ce_vae_sp_host_barrier(v._handle, 0)


@gpu
def test_split_vae_lone_rank_times_out_and_poisons_the_group():
    """Rank 0 alone reaches the first barrier: it fails after the timeout naming itself and the missing rank, and the group then
    fails at once."""
    import chronoedit_b200 as ce
    from chronoedit_b200 import _lib, parallel

    dev = torch.device("cuda", torch.cuda.current_device())
    v, _ = _configured(2, 32, 48, ms=500)
    x = _video(1, 32, 48, dev, 0)
    try:
        t0 = time.perf_counter()
        with pytest.raises(ce.CEError, match=r"rank 0 timed out after 500 ms at barrier 1 waiting for rank\(s\) 1"):
            v.encode(x)
        assert time.perf_counter() - t0 < 30
        t0 = time.perf_counter()
        with pytest.raises(ce.CEError, match="the group failed earlier"):
            v.encode(x)
        assert time.perf_counter() - t0 < 5
    finally:
        parallel.disable_vae_sequence_parallel(v)
        _lib.lib().ce_vae_sp_host_barrier(v._handle, 0)
    assert torch.isfinite(v.encode(x).latent_dist.mean.float()).all()   # the single-GPU call is unaffected
