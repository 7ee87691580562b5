"""TeaCache on the GPU: the probe's sums, the recorded residual, the forward without blocks, and the pipeline with TeaCache on.

Acceptance:
  * the probe's two sums give rel values equal (as bf16) to torch's CUDA `(a - b).abs().mean() / b.abs().mean()` on the same
    timestep modulations, at every step of a 50-step shift-5 schedule, so the decisions are the same;
  * with the record on, the sample is bit-identical to the plain forward (bf16, FP8 weights, FP8 attention), and the residual is
    bf16(x_L - x_0) bit for bit (x_L: capture of the last block, x_0: the patch-embedding GEMM on its own);
  * the skipped forward meets tests/test_gpu_dit.py's rule against the oracle head on bf16(x_0 + residual), and is
    batch-invariant bit for bit;
  * tests/test_gpu_pipeline.py's cases with TeaCache on: the mirror's schedule is the rule on its own modulations, and the video
    meets the end-to-end rule against the oracle run under that schedule.
"""
import pytest
import torch

gpu = pytest.mark.gpu


def _model(cfg, sd, dev, **kw):
    import chronoedit_b200 as ce

    m = ce.ChronoEditTransformer3DModel(
        patch_size=cfg.patch_size, num_attention_heads=cfg.num_attention_heads, attention_head_dim=cfg.attention_head_dim,
        in_channels=cfg.in_channels, out_channels=cfg.out_channels, text_dim=cfg.text_dim, freq_dim=cfg.freq_dim, ffn_dim=cfg.ffn_dim,
        num_layers=cfg.num_layers, eps=cfg.eps, image_dim=cfg.image_dim, added_kv_proj_dim=cfg.added_kv_proj_dim, **kw)
    m.load_state_dict(sd)
    return m.to(dev)


@gpu
def test_probe_rel_equals_torch_on_the_same_modulations():
    from chronoedit_b200 import teacache as TCP
    from oracle import cases, dit_oracle as D, unipc_oracle as U

    dev = torch.device("cuda", 0)
    cfg = D.DiTConfig.tiny(num_layers=1, heads=40, ffn_dim=1024)   # D = 5120: the 14B model's modulation width
    sd = cases.to_bf16_state(D.random_state_dict(cfg, seed=3))
    b = "condition_embedder.time_proj.bias"
    sd[b] = (sd[b].float() * 20).bfloat16()   # rel ~ 0.01 (tests/golden/make_golden_teacache.py)
    m = _model(cfg, sd, dev)
    n = 2 * 6 * cfg.inner_dim
    _, ts = U.flow_sigmas(50, 5.0)
    bufs = [torch.empty(n, dtype=torch.bfloat16, device=dev) for _ in range(2)]
    mine, theirs = [], []
    for k, t in enumerate(ts):
        cur, prev = bufs[k % 2], bufs[(k + 1) % 2]
        sums = m._native_probe(t.float().expand(2).to(dev).contiguous(), prev if k else None, cur)
        if k:
            mine.append(TCP.rel_from_sums(sums[0], sums[1], n))
            a, p = cur.view(2, 6, -1), prev.view(2, 6, -1)
            theirs.append(((a - p).abs().mean() / p.abs().mean()).item())
    assert mine == theirs
    for thresh in (0.1, 0.2, 0.3):
        d = []
        for rels in (mine, theirs):
            pol = TCP.TeaCacheState(50, thresh)
            d.append([pol.decide(None)[1]] + [pol.decide(r)[1] for r in rels])
        assert d[0] == d[1]


def _tiny(dev, mode):
    from oracle import cases

    case = cases.DIT_CASES["tiny_t2"]
    sd32 = cases.dit_weights(case)
    m = _model(case.cfg, cases.to_bf16_state(sd32), dev)
    if mode in ("fp8", "fp8_attention"):
        m.enable_fp8()
    if mode == "fp8_attention":
        m.enable_fp8_attention()
    x, t, text, img = cases.dit_inputs(case)
    return m, case.cfg, sd32, (x.to(dev, torch.bfloat16), t.to(dev), text.to(dev, torch.bfloat16), img.to(dev, torch.bfloat16))


def _x0(m, x):
    """The patch-embedding GEMM on its own: im2row in torch (data movement), then ce_linear_bf16 with the bias epilogue."""
    from chronoedit_b200 import _lib

    B, C, T, H, W = x.shape
    patches = x.reshape(B, C, T, H // 2, 2, W // 2, 2).permute(0, 2, 3, 5, 1, 4, 6).reshape(-1, C * 4).contiguous()
    w = m.patch_embedding.weight.reshape(m.patch_embedding.weight.shape[0], -1).contiguous()
    out = torch.empty(patches.shape[0], w.shape[0], dtype=torch.bfloat16, device=x.device)
    _lib.check(_lib.lib().ce_linear_bf16(_lib.ptr(patches), C * 4, _lib.ptr(w), C * 4, _lib.ptr(m.patch_embedding.bias), _lib.ptr(out),
                                         w.shape[0], None, patches.shape[0], w.shape[0], C * 4, 0, None, 0, None, 0, 0,
                                         _lib.current_stream()))
    return out


@gpu
@pytest.mark.parametrize("mode", ["bf16", "fp8", "fp8_attention"])
def test_record_keeps_the_sample_and_stores_the_residual(mode):
    dev = torch.device("cuda", 0)
    m, cfg, _, (x, t, text, img) = _tiny(dev, mode)
    plain = m(x, t, text, img, capture_layers=(cfg.num_layers - 1,), return_dict=False)[0]
    xl = m.last_captures[cfg.num_layers - 1]
    resid = torch.empty(xl.numel(), dtype=torch.bfloat16, device=dev)
    out = torch.empty_like(plain)
    m._native_teacache_forward(x, t.float().contiguous(), text, img, out, text, img, resid, True)
    torch.cuda.synchronize()
    assert torch.equal(out, plain)
    assert torch.equal(resid.view_as(xl), (xl.float() - _x0(m, x).float()).bfloat16())


@gpu
def test_skipped_forward_against_the_oracle_head_and_batch_invariant():
    from oracle import cases, teacache_oracle as TC

    dev = torch.device("cuda", 0)
    m, cfg, sd32, (x, t, text, img) = _tiny(dev, "bf16")
    B = x.shape[0]
    g = torch.Generator().manual_seed(7)
    resid = (torch.randn(B, x.shape[2] * (x.shape[3] // 2) * (x.shape[4] // 2), cfg.inner_dim, generator=g) * 0.5).bfloat16().to(dev)
    tt = t.float().contiguous()
    out = torch.empty(B, cfg.out_channels, *x.shape[2:], dtype=torch.bfloat16, device=dev)
    m(x, t, text, img)   # packs the weights
    m._native_teacache_forward(x, tt, text, img, out, text, img, resid.flatten(), False)
    for b in range(B):   # batch invariance: one sample at a time, its own residual
        o1 = torch.empty_like(out[b:b + 1])
        m._native_teacache_forward(x[b:b + 1].contiguous(), tt[b:b + 1].contiguous(), text[b:b + 1].contiguous(),
                                   img[b:b + 1].contiguous(), o1, None, None, resid[b].flatten().contiguous(), False)
        torch.cuda.synchronize()
        assert torch.equal(o1, out[b:b + 1])
    xs = (_x0(m, x).view_as(resid).float() + resid.float()).bfloat16().cpu()   # bf16(x_0 + residual)
    sd16 = cases.to_bf16_state(sd32)
    ref16 = TC.head(sd16, cfg, xs, TC.time_embedding(sd16, cfg, t.cpu().float(), torch.bfloat16), x.shape[2:]).float()
    ref32 = TC.head(sd32, cfg, xs.float(), TC.time_embedding(sd32, cfg, t.cpu().float(), torch.float32), x.shape[2:])
    e_ref, e_our = (ref16 - ref32).abs(), (out.float().cpu() - ref32).abs()
    assert e_our.mean() <= 1.25 * e_ref.mean() and e_our.max() <= 2.0 * e_ref.max() + 1e-3


@gpu
def test_pack_weights_drops_the_states():
    """The lazy pack of the first call keeps the state it was made for; an explicit pack_weights() re-registers the weights, so the
    residuals computed from the old ones are dropped, as load_state_dict and fuse_lora drop them."""
    dev = torch.device("cuda", 0)
    m, _, _, (x, t, text, img) = _tiny(dev, "bf16")
    m.enable_teacache(1e9, num_inference_steps=4)
    m(x, t, text, img)
    m(x, t, text, img)
    assert [r.step for r in m.teacache_records] == [0, 1] and m._tc_states
    m.pack_weights()
    assert m._tc_states == []
    m(x, t, text, img)
    torch.cuda.synchronize()
    assert m.teacache_records[-1].step == 0 and m.teacache_records[-1].computed


@gpu
@pytest.mark.parametrize("name", ["edit_5f", "reason_cut"])
def test_pipeline_with_teacache(name):
    from chronoedit_b200 import teacache as TCP
    from oracle import cases, pipeline_cases as PC, teacache_oracle as TC
    from tests.test_gpu_pipeline import _mirrors

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda", 0)
    case = PC.PIPELINE_CASES[name]
    tr, vae, sch = _mirrors(case, dev)
    tr.enable_teacache(1e9, num_inference_steps=case.steps)   # every evaluated step skips unless forced
    seen = []
    probe = tr._native_probe

    def recording_probe(t, prev, cur):
        r = probe(t, prev, cur)
        seen.append(cur.clone())
        return r

    tr._native_probe = recording_probe
    ours = PC.run_oracle_pipeline(case, torch.bfloat16, device=dev, transformer=tr, vae=vae, scheduler=sch).float()
    recs = tr.teacache_records
    assert any(not r.computed for r in recs)
    # the rule on the mirror's own modulations, per conditioning slot, in torch on the device
    for slot in {r.slot for r in recs}:
        idx = [i for i, r in enumerate(recs) if r.slot == slot]
        mods = [seen[i].view(-1, 6, tr.config.num_attention_heads * tr.config.attention_head_dim) for i in idx]
        pol = TCP.TeaCacheState(case.steps, 1e9)
        for k, i in enumerate(idx):
            rel = TC.rel_l1(mods[k], mods[k - 1]) if pol.needs_rel() else None
            assert rel == recs[i].rel
            geom_change = k > 0 and name == "reason_cut" and pol.step == case.num_temporal_reasoning_steps
            assert pol.decide(rel, force_compute=geom_change)[1] == recs[i].computed
    computed = [r.computed for r in recs]
    dsd, _ = PC.weights()
    ref16 = PC.run_oracle_pipeline(case, torch.bfloat16, device=dev, transformer=TC.ScheduledTransformer(
        {k: v.to(dev) for k, v in cases.to_bf16_state(dsd).items()}, PC.DIT_CFG, torch.bfloat16, computed)).float()
    ref32 = PC.run_oracle_pipeline(case, torch.float32, device=dev, transformer=TC.ScheduledTransformer(
        {k: v.to(dev) for k, v in dsd.items()}, PC.DIT_CFG, torch.float32, computed)).float()
    e_ref, e_our = (ref16 - ref32).abs(), (ours - ref32).abs()
    print(name, computed, e_our.mean().item(), e_ref.mean().item(), e_our.max().item(), e_ref.max().item())
    assert e_our.mean() <= 1.25 * e_ref.mean() and e_our.max() <= 2.0 * e_ref.max() + 1e-3
