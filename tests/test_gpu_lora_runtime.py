"""Run-time LoRA on the GPU (DESIGN.md, "Run-time LoRA"): set_adapters / disable_lora / delete_adapters on bf16 and FP8 weights.

The rule is PEFT's unfused forward, base + sum_i bf16(bf16(bf16(x A_i^T) B_i^T) * scaling_i) (oracle/lora_oracle.py); the kernel
fuses the per-adapter roundings (one product over the stacked rank, B pre-scaled), so it is held to the DiT's oracle rule: mean and
max error against the fp32 oracle within 1.25x and 1.5x of the bf16 oracle's own.  Bit equalities: off means off, switching sets
gives each set's own bits, the context cache hits under one set, the batch split equals one GPU, and the epilogue addend equals
the kernel's own epilogue applied to bf16(bf16(acc + bias) + t)."""
import pytest
import torch

from tests.test_gpu_fp8 import _bf16_epilogue_of, _fp8_operands, _Fp8Linear, linear_fp8
from tests.test_gpu_row_stats import gemm_case, linear_ex, tile_width

gpu = pytest.mark.gpu


def _L():
    import chronoedit_b200._lib as L

    return L


def _p(t):
    return None if t is None else t.data_ptr()


# ---------------------------------------------------------------------------------------------------- the epilogue addend
def _linear_lora(A, W, out, term, *, fp8=None, bias=None, epi=0, resid=None, gate=None, rpb=1, stats=None, stats_mode=0):
    L = _L()
    M, K = A.shape
    N = W.shape[0]
    base = L.LinearArgsC(A=_p(A), lda=A.stride(0), W=_p(W), ldw=W.stride(0), M=M, N=N, K=K, out=_p(out), ldo=out.stride(0),
                         bias=_p(bias), epilogue=epi, resid=_p(resid), ldr=0 if resid is None else resid.stride(0), gate=_p(gate),
                         gate_stride=0 if gate is None else gate.shape[1], rows_per_batch=rpb, stats_out=_p(stats),
                         stats_ld=0 if stats is None else stats.shape[1], stats_mode=stats_mode)
    if fp8 is None:
        L.check(L.lib().ce_linear_lora_bf16(base, _p(term), term.stride(0), L.current_stream()))
    else:
        args = L.LinearFp8ArgsC(base=base, a_scale=_p(fp8[0]), w_scale=_p(fp8[1]))
        L.check(L.lib().ce_linear_lora_fp8(args, _p(term), term.stride(0), L.current_stream()))


@gpu
@pytest.mark.parametrize("dtype", ["bf16", "e4m3"])
@pytest.mark.parametrize("N", [512, 192, 64])   # tile widths 256, 128 (partial last tile), 64
def test_lora_epilogue_addend(N, dtype):
    """M = 1300 (the last M tile ragged), K = 320.  For epilogues 0-4 with row statistics, the LoRA kernel's output and statistics
    equal the plain kernel's epilogue applied to y = bf16(bf16(acc + bias) + t), bit for bit (t with a row stride wider than N)."""
    M, K, rpb = 1300, 320, 256
    tn = tile_width(N)
    tiles = (N + tn - 1) // tn
    A, W, bias, resid, gate = gemm_case("block_offset", M, N, K, rpb, seed=N)
    g = torch.Generator(device="cuda").manual_seed(N + 7)
    term = (torch.randn(M, N + 24, generator=g, device="cuda") * 0.5).bfloat16()
    y0 = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    if dtype == "bf16":
        linear_ex(A, W, y0, bias=bias)
        run = lambda out, **kw: _linear_lora(A, W, out, term, **kw)
    else:
        Aq, sa, Wq, sw = _fp8_operands(M, N, K, seed=N + 1)
        linear_fp8(Aq, sa, Wq, sw, y0, bias=bias)
        run = lambda out, **kw: _linear_lora(Aq, Wq, out, term, fp8=(sa, sw), **kw)
    y = (y0.float() + term[:, :N].float()).bfloat16().float()   # torch's bf16 add: the fp32 sum, rounded to nearest even
    for epi in range(5):
        mode = 1 if epi in (0, 3, 4) else 2
        kw = dict(epi=epi, resid=resid if epi in (3, 4) else None, gate=gate if epi == 3 else None, rpb=rpb, stats_mode=mode)
        out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
        st = torch.full((M, tiles, 2), float("nan"), device="cuda")
        run(out, bias=bias, stats=st, **kw)
        want, want_st = _bf16_epilogue_of(y, None, epi, kw["resid"], kw["gate"], rpb, mode, tn)
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int16), want.view(torch.int16)), f"{dtype} N={N} epi={epi}: output"
        assert torch.equal(st, want_st), f"{dtype} N={N} epi={epi}: statistics"


# ---------------------------------------------------------------------------------------------------- the DiT
def _model(cfg, sdb, fp8=False, fp8_attention=False, **kw):
    import chronoedit_b200 as ce

    m = ce.ChronoEditTransformer3DModel(
        patch_size=cfg.patch_size, num_attention_heads=cfg.num_attention_heads, attention_head_dim=cfg.attention_head_dim,
        in_channels=cfg.in_channels, out_channels=cfg.out_channels, text_dim=cfg.text_dim, freq_dim=cfg.freq_dim,
        ffn_dim=cfg.ffn_dim, num_layers=cfg.num_layers, eps=cfg.eps, image_dim=cfg.image_dim,
        added_kv_proj_dim=cfg.added_kv_proj_dim, rope_max_seq_len=cfg.rope_max_seq_len,
        rope_temporal_skip_len=cfg.rope_temporal_skip_len, **kw)
    m.load_state_dict(sdb)
    if fp8:
        m.enable_fp8()
    if fp8_attention:
        m.enable_fp8_attention()
    return m.cuda()


BLOCK_MODULES = ("attn1.to_q", "attn1.to_k", "attn1.to_v", "attn1.to_out.0", "attn2.to_q", "attn2.to_k", "attn2.to_v", "attn2.to_out.0",
                 "attn2.add_k_proj", "attn2.add_v_proj", "ffn.net.0.proj", "ffn.net.2")


def make_lora(sd, cfg, rank, seed, modules=BLOCK_MODULES, alpha=None, std=0.3):
    """A random adapter with diffusers keys on `modules` of every block: lora_A ~ N(0, 1/K), lora_B ~ N(0, std^2 / rank)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for i in range(cfg.num_layers):
        for mod in modules:
            w = sd[f"blocks.{i}.{mod}.weight"]
            N, K = w.shape
            out[f"transformer.blocks.{i}.{mod}.lora_A.weight"] = (torch.randn(rank, K, generator=g) / K ** 0.5).bfloat16()
            out[f"transformer.blocks.{i}.{mod}.lora_B.weight"] = (torch.randn(N, rank, generator=g) * std / rank ** 0.5).bfloat16()
            if alpha is not None:
                out[f"transformer.blocks.{i}.{mod}.alpha"] = torch.tensor(float(alpha))
    return out


def lora_rule_oracle(sd, cfg, entries, scale, *inputs, monkeypatch, fp8_weights=False, fp8_attention=False):
    """The oracle's forward with the adapters' terms (lora_oracle) on top of the bf16 rule, the FP8 GEMM rule (fp8_weights) and
    the FP8 attention rule (fp8_attention), in the dtype of `inputs`."""
    from oracle import dit_oracle as O
    from oracle import lora_oracle
    from chronoedit_b200.transformer import FP8_LINEARS, quantize_fp8_rows

    sd = dict(sd)
    inner = torch.nn.functional
    if fp8_weights:
        quantized = {}
        for i in range(cfg.num_layers):
            for name in FP8_LINEARS:
                k = f"blocks.{i}.{name}.weight"
                wq, sw = quantize_fp8_rows(sd[k])
                sd[k] = sd[k].clone()
                quantized[id(sd[k])] = (wq.to(sd[k].device), sw.to(sd[k].device))
        inner = _Fp8Linear(quantized)
    dev = inputs[0].device
    adapters = lora_oracle.adapters_of(entries, scale, device=dev)
    lf = lora_oracle._LoraF({id(sd[m + ".weight"]): lst for m, lst in adapters.items()}, inner)
    with monkeypatch.context() as mp:
        if fp8_attention:
            from tests.test_gpu_fp8_attention import _RuleF

            rule = _RuleF(lf)
            orig = O.attention

            def attention(sd_, p, cfg_, x, ctx, freqs):
                rule.self_attention = ctx is None
                try:
                    return orig(sd_, p, cfg_, x, ctx, freqs)
                finally:
                    rule.self_attention = False

            mp.setattr(O, "F", rule)
            mp.setattr(O, "attention", attention)
        else:
            mp.setattr(O, "F", lf)
        with torch.no_grad():
            return O.dit_forward(sd, cfg, *inputs)


def _check_rule(out, ref32, ref16, what):
    e_ref, e_our = (ref16 - ref32).abs(), (out - ref32).abs()
    assert out.shape == ref32.shape and torch.isfinite(out).all(), what
    assert e_our.mean() <= 1.25 * e_ref.mean(), f"{what}: mean err {e_our.mean():.3g} vs the bf16 oracle's {e_ref.mean():.3g}"
    assert e_our.max() <= 1.5 * e_ref.max(), f"{what}: max err {e_our.max():.3g} vs the bf16 oracle's {e_ref.max():.3g}"


def _tiny():
    from oracle import cases

    case = cases.DIT_CASES["tiny_t2"]
    sd32 = cases.dit_weights(case)
    return case.cfg, sd32, cases.to_bf16_state(sd32), cases.dit_inputs(case)


def _fwd(m, inputs, **kw):
    out = m(*[a.cuda() for a in inputs], return_dict=False, **kw)[0]
    torch.cuda.synchronize()
    return out.clone()


@gpu
@pytest.mark.parametrize("mode", ["bf16", "fp8", "fp8+fp8_attention"])
def test_lora_dit_matches_rule(mode, monkeypatch):
    """One adapter; two stacked adapters at different weights (with alpha); the same pair under attention_kwargs scale 0.6.
    Each against the oracle rule, in bf16, with FP8 weights and with FP8 weights + FP8 attention: one model serves all three
    sets and then no LoRA, with no reload and no fuse_lora."""
    cfg, sd32, sdb, (x, t, text, img) = _tiny()
    fp8, fp8_att = mode != "bf16", mode == "fp8+fp8_attention"
    m = _model(cfg, sdb, fp8=fp8, fp8_attention=fp8_att)
    base = _fwd(m, (x, t, text, img))
    la, lb = make_lora(sd32, cfg, 32, seed=1), make_lora(sd32, cfg, 16, seed=2, alpha=8)
    m.load_lora_adapter(la, adapter_name="distill")
    m.load_lora_adapter(lb, adapter_name="paint")
    assert torch.equal(_fwd(m, (x, t, text, img)), base), "loading alone changed the output"
    for names, weights, scale in [(["distill"], None, 1.0), (["distill", "paint"], [1.0, 0.7], 1.0), (["distill", "paint"], [1.0, 0.7], 0.6)]:
        m.set_adapters(names, weights)
        out = _fwd(m, (x, t, text, img), attention_kwargs={"scale": scale}).float().cpu()
        entries = [({"distill": la, "paint": lb}[n], w) for n, w in zip(names, weights or [1.0])]
        kw = dict(monkeypatch=monkeypatch, fp8_weights=fp8, fp8_attention=fp8_att)
        ref32 = lora_rule_oracle(sd32, cfg, entries, scale, x, t, text, img, **kw)
        ref16 = lora_rule_oracle(sdb, cfg, entries, scale, x.bfloat16(), t, text.bfloat16(), img.bfloat16(), **kw).float()
        _check_rule(out, ref32, ref16, f"{mode} {names} {weights} scale {scale}")
        assert (out - base.float().cpu()).abs().mean() > 4 * (ref16 - ref32).abs().mean(), "the adapters did not change the output"
    m.set_adapters([])
    assert torch.equal(_fwd(m, (x, t, text, img)), base), "an empty set is not the plain forward"


@gpu
def test_lora_dit_14b_width_two_layers_at_720p(monkeypatch):
    """Two blocks at the 14B width (D 5120, 40 heads, ffn 13 824) with 7200 tokens (720p, 2 latent frames), rank 32 and 64
    stacked at weights 1 and 0.5 under scale 0.8, against the oracle rule run on the GPU."""
    from oracle import cases, dit_oracle as O

    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    cfg = O.DiTConfig(num_layers=2)
    case = cases.DiTCase("w14b_2l", cfg, batch=1, frames=2, height=90, width=160, timestep=500, text_len=512)
    sd32 = {k: v.cuda() for k, v in cases.dit_weights(case).items()}
    sdb = cases.to_bf16_state(sd32)
    x, t, text, img = (a.cuda() for a in cases.dit_inputs(case))
    la, lb = make_lora(sd32, cfg, 32, seed=3), make_lora(sd32, cfg, 64, seed=4, alpha=32)
    m = _model(cfg, sdb)
    m.load_lora_adapter(la, adapter_name="a")
    m.load_lora_adapter(lb, adapter_name="b")
    m.set_adapters(["a", "b"], [1.0, 0.5])
    out = _fwd(m, (x, t, text, img), attention_kwargs={"scale": 0.8}).float()
    del m
    torch.cuda.empty_cache()
    entries = [(la, 1.0), (lb, 0.5)]
    ref32 = lora_rule_oracle(sd32, cfg, entries, 0.8, x, t, text, img, monkeypatch=monkeypatch)
    ref16 = lora_rule_oracle(sdb, cfg, entries, 0.8, x.bfloat16(), t, text.bfloat16(), img.bfloat16(), monkeypatch=monkeypatch).float()
    _check_rule(out, ref32, ref16, "14B width, 2 layers, 720p")


@gpu
def test_lora_off_means_off_and_switching():
    """No set: bit-identical to a model that never loaded an adapter, with the same launch count.  disable_lora() and
    delete_adapters give the pre-set output back bit for bit; enable_lora() gives the set's.  Alternating two sets across calls
    gives each set's own bits every time."""
    cfg, sd32, sdb, (x, t, text, img) = _tiny()
    plain = _model(cfg, sdb)
    ref = _fwd(plain, (x, t, text, img))
    n_plain = plain.launches_per_forward()
    m = _model(cfg, sdb)
    m.load_lora_adapter(make_lora(sd32, cfg, 8, seed=5), adapter_name="a")
    m.load_lora_adapter(make_lora(sd32, cfg, 24, seed=6), adapter_name="b")
    assert torch.equal(_fwd(m, (x, t, text, img)), ref) and m.launches_per_forward() == n_plain
    m.set_adapters("a")
    ya = _fwd(m, (x, t, text, img))
    assert not torch.equal(ya, ref) and m.launches_per_forward() > n_plain
    m.disable_lora()
    assert torch.equal(_fwd(m, (x, t, text, img)), ref) and m.launches_per_forward() == n_plain
    m.enable_lora()
    assert torch.equal(_fwd(m, (x, t, text, img)), ya)
    m.set_adapters(["a", "b"], [0.5, 1.5])
    yab = _fwd(m, (x, t, text, img))
    for _ in range(2):
        m.set_adapters("a")
        assert torch.equal(_fwd(m, (x, t, text, img)), ya)
        m.set_adapters(["a", "b"], [0.5, 1.5])
        assert torch.equal(_fwd(m, (x, t, text, img)), yab)
    m.delete_adapters(["a", "b"])
    assert m.active_adapters() == []
    assert torch.equal(_fwd(m, (x, t, text, img)), ref) and m.launches_per_forward() == n_plain


@gpu
def test_lora_switching_equals_fusing():
    """bf16 weights: one adapter at run time with weight s meets the oracle rule against the same model with fuse_lora(s)."""
    cfg, sd32, sdb, (x, t, text, img) = _tiny()
    from oracle import dit_oracle as O

    lora = make_lora(sd32, cfg, 16, seed=7, alpha=8)
    run = _model(cfg, sdb)
    run.load_lora_adapter(lora, adapter_name="s")
    run.set_adapters("s", 0.75)
    y_run = _fwd(run, (x, t, text, img)).float().cpu()
    fused = _model(cfg, sdb)
    fused.fuse_lora(lora, lora_scale=0.75)
    y_fused = _fwd(fused, (x, t, text, img)).float().cpu()
    sd_fused = {k: v.detach().float().cpu() for k, v in fused.state_dict().items()}
    ref32 = O.dit_forward(sd_fused, cfg, x, t, text, img)
    ref16 = O.dit_forward(cases_bf16(sd_fused), cfg, x.bfloat16(), t, text.bfloat16(), img.bfloat16()).float()
    _check_rule(y_run, ref32, ref16, "run-time adapter against the fused model's oracle")
    _check_rule(y_fused, ref32, ref16, "fused model against its oracle")


def cases_bf16(sd):
    from oracle import cases

    return cases.to_bf16_state(sd)


@gpu
def test_lora_context_projection_adapters_and_cache():
    """An adapter on attn2.to_k / to_v and add_k_proj / add_v_proj only, with the context cache on: a cache hit equals the uncached
    forward bit for bit under the same set, and a set change recomputes the cached K / V."""
    cfg, sd32, sdb, (x, t, text, img) = _tiny()
    ctx = make_lora(sd32, cfg, 16, seed=8, modules=("attn2.to_k", "attn2.to_v", "attn2.add_k_proj", "attn2.add_v_proj"), std=1.0)
    other = make_lora(sd32, cfg, 8, seed=9, modules=("attn2.to_k", "attn2.add_v_proj"), std=1.0)
    unc = _model(cfg, sdb)
    cac = _model(cfg, sdb, cache_context=True)
    for m in (unc, cac):
        m.load_lora_adapter(ctx, adapter_name="ctx")
        m.load_lora_adapter(other, adapter_name="other")
    txt, im = text.cuda(), img.cuda()
    plain = _fwd(unc, (x, t, txt, im))
    for names in (["ctx"], ["ctx", "other"], ["other"]):
        unc.set_adapters(names)
        cac.set_adapters(names)
        want = _fwd(unc, (x, t, txt, im))
        assert not torch.equal(want, plain), names
        first = _fwd(cac, (x, t, txt, im))    # fills the slot under this set
        hit = _fwd(cac, (x, t, txt, im))      # reads it
        assert torch.equal(first, want) and torch.equal(hit, want), f"{names}: cached forward differs from the uncached one"


@gpu
def test_lora_batch_split_equals_one_gpu():
    """Two handles under the host barrier (batch split, B = 2): every rank returns the single-GPU LoRA forward bit for bit."""
    from oracle import cases
    from tests.test_gpu_cfg_parallel_one_gpu import _split_matches_single

    case = cases.DIT_CASES["tiny_b2"]
    sd32 = cases.dit_weights(case)
    sdb = cases.to_bf16_state(sd32)
    x, t, text, img = (a.cuda() for a in cases.dit_inputs(case))
    lora = make_lora(sd32, case.cfg, 16, seed=10)
    models = []
    for _ in range(2):
        m = _model(case.cfg, sdb)
        m.load_lora_adapter(lora, adapter_name="a")
        m.set_adapters("a", 0.8)
        models.append(m)
    steps = [(x, t, text, img), (x * 0.5, t * 0.5, text, img)]
    _split_matches_single(models, steps, (case.frames, case.height, case.width), 2)


@gpu
def test_lora_set_change_drops_teacache_states():
    """TeaCache on: a set change drops the states, so the next call of a conditioning is its step 0 and computes."""
    cfg, sd32, sdb, (x, t, text, img) = _tiny()
    m = _model(cfg, sdb)
    m.load_lora_adapter(make_lora(sd32, cfg, 8, seed=11), adapter_name="a")
    m.enable_teacache(0.5, num_inference_steps=10)
    txt, im = text.cuda(), img.cuda()
    for k in range(3):
        _fwd(m, (x, t * (1 - 0.01 * k), txt, im))
    assert m.teacache_records[-1].step == 2
    m.set_adapters("a")
    assert m._tc_states == []
    _fwd(m, (x, t, txt, im))
    rec = m.teacache_records[-1]
    assert rec.step == 0 and rec.computed
