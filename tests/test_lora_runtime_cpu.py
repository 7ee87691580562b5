"""CPU tests (-m "not gpu") of run-time LoRA (set_adapters, DESIGN.md "Run-time LoRA"): the mirror's state machine with the oracle
standing in for the native forward (it reads the tables the handle was given), the packing of A_cat / B_cat, the scaling, the
refusals, the unchanged behaviours, and the oracle's restatement of the rule against PEFT-style layers on the reference's own
transformer when /root/reference is present."""
import warnings

import pytest
import torch

from oracle import cases, lora_oracle
from oracle import pipeline_cases as PC
from oracle import ref_loader

MODULES = ("attn1.to_q", "attn1.to_k", "attn1.to_v", "attn1.to_out.0", "attn2.to_q", "attn2.to_k", "attn2.to_v", "attn2.to_out.0",
           "attn2.add_k_proj", "attn2.add_v_proj", "ffn.net.0.proj", "ffn.net.2")


def _lora(m, rank, seed, modules=MODULES, alpha=None):
    g = torch.Generator().manual_seed(seed)
    shapes = {n: tuple(p.shape) for n, p in m.named_parameters()}
    shapes.update({n[: -len("_fp8")]: tuple(b.shape) for n, b in m.named_buffers() if n.endswith(".weight_fp8")})
    out = {}
    for i in range(len(m.blocks)):
        for mod in modules:
            N, K = shapes[f"blocks.{i}.{mod}.weight"]
            out[f"transformer.blocks.{i}.{mod}.lora_A.weight"] = (torch.randn(rank, K, generator=g) / K ** 0.5).bfloat16()
            out[f"transformer.blocks.{i}.{mod}.lora_B.weight"] = (torch.randn(N, rank, generator=g) * 0.3).bfloat16()
            if alpha is not None:
                out[f"transformer.blocks.{i}.{mod}.alpha"] = torch.tensor(float(alpha))
    return out


def _mirror():
    """The mirror on the CPU with the oracle behind _native_forward: the forward applies exactly the tables the handle holds."""
    import chronoedit_b200 as ce
    from chronoedit_b200.transformer import LORA_TARGETS

    cfg = PC.DIT_CFG
    m = ce.ChronoEditTransformer3DModel(
        patch_size=cfg.patch_size, num_attention_heads=cfg.num_attention_heads, attention_head_dim=cfg.attention_head_dim,
        in_channels=cfg.in_channels, out_channels=cfg.out_channels, text_dim=cfg.text_dim, freq_dim=cfg.freq_dim, ffn_dim=cfg.ffn_dim,
        num_layers=cfg.num_layers, eps=cfg.eps, image_dim=cfg.image_dim, added_kv_proj_dim=cfg.added_kv_proj_dim)
    m.load_state_dict(cases.to_bf16_state(PC.weights()[0]))
    m.native_calls = 0

    def native_forward(x, t, txt, img, out, b0, caps, txt_in, img_in):
        m.native_calls += 1
        adapters = {}
        for (layer, target), (a_cat, _, _, b_cat) in m._lora_tables.items():
            for sub, (tg, part, parts) in LORA_TARGETS.items():
                if tg == target:
                    n = b_cat.shape[0] // parts
                    adapters[f"blocks.{layer}.{sub}"] = [(a_cat, b_cat[part * n: (part + 1) * n], 1.0)]
        sd = {k: v.detach() for k, v in m.state_dict().items()}
        out.copy_(lora_oracle.dit_forward(sd, cfg, adapters, x, t, txt, img))

    m._native_forward = native_forward
    return m


def _inputs(seed=0):
    g = torch.Generator().manual_seed(seed)
    cfg = PC.DIT_CFG
    x = torch.randn(1, cfg.in_channels, 2, 8, 8, generator=g)
    txt = torch.randn(1, 16, cfg.text_dim, generator=g)
    img = torch.randn(1, 257, cfg.image_dim, generator=g)
    return x, torch.tensor([700.0]), txt, img


def _run(m, inp, **kw):
    return m(*inp, return_dict=False, **kw)[0].clone()


def test_state_machine_and_unchanged_behaviours():
    m, plain = _mirror(), _mirror()
    inp = _inputs()
    ref = _run(plain, inp)
    m.load_lora_adapter(_lora(m, 4, 1), adapter_name="a")
    m.load_lora_adapter(_lora(m, 8, 2, alpha=4), adapter_name="b")
    assert torch.equal(_run(m, inp), ref) and m._lora_key is None, "loading alone must leave the model as it is"
    assert m.active_adapters() == []
    m.set_adapters("a")
    assert m.active_adapters() == ["a"]
    ya = _run(m, inp)
    assert not torch.equal(ya, ref)
    m.disable_lora()
    assert m.active_adapters() == ["a"] and torch.equal(_run(m, inp), ref) and not m._lora_tables
    m.enable_lora()
    assert torch.equal(_run(m, inp), ya)
    m.set_adapters(["a", "b"], [0.5, 2.0])
    assert m.active_adapters() == ["a", "b"]
    yab = _run(m, inp)
    assert not torch.equal(yab, ya)
    m.set_adapters("a")
    assert torch.equal(_run(m, inp), ya)
    m.delete_adapters("a")
    assert m.active_adapters() == [] and torch.equal(_run(m, inp), ref)
    m.set_adapters(["b"], [2.0])
    m.delete_adapters(["b"])
    assert torch.equal(_run(m, inp), ref) and m._lora_key is None


def test_new_content_under_a_known_name_is_served():
    """Reloading an adapter name, while its set is active or after deleting it, serves the new factors, not the packed old ones."""
    inp = _inputs()
    old, new = None, None
    fresh = _mirror()
    new = _lora(fresh, 8, 7)
    fresh.load_lora_adapter(new, adapter_name="a")
    fresh.set_adapters("a")
    want = _run(fresh, inp)
    # (1) delete, load other content under the same name, set the same set again
    m = _mirror()
    old = _lora(m, 8, 3)
    m.load_lora_adapter(old, adapter_name="a")
    m.set_adapters("a")
    y_old = _run(m, inp)
    assert not torch.equal(y_old, want)
    m.delete_adapters("a")
    m.load_lora_adapter(new, adapter_name="a")
    m.set_adapters("a")
    assert torch.equal(_run(m, inp), want)
    # (2) overwrite the name while its set is active
    m = _mirror()
    m.load_lora_adapter(old, adapter_name="a")
    m.set_adapters("a")
    assert torch.equal(_run(m, inp), y_old)
    m._ctx_cache = [dict(buf=None)]
    m.load_lora_adapter(new, adapter_name="a")
    assert torch.equal(_run(m, inp), want)
    assert m._ctx_cache == [], "K / V cached under the old content must be dropped"
    # (3) unload everything, load the new content, set again
    m.unload_lora()
    m.load_lora_adapter(new, adapter_name="a")
    m.set_adapters("a")
    assert torch.equal(_run(m, inp), want)


def test_weights_none_means_one_and_forward_host_keeps_the_last_scale():
    m = _mirror()
    m.load_lora_adapter(_lora(m, 4, 1), adapter_name="a")
    m.load_lora_adapter(_lora(m, 4, 2), adapter_name="b")
    m.set_adapters(["a", "b"], [None, 0.5])
    assert [w for _, w in m._lora_set] == [1.0, 0.5]
    _run(m, _inputs(), attention_kwargs={"scale": 0.25})
    key = m._lora_key
    with pytest.raises(Exception):   # no CPU path: it fails after syncing the tables
        m.forward_host(*[t.bfloat16() if t.is_floating_point() and t.dim() > 1 else t for t in _inputs()])
    assert m._lora_key == key, "forward_host repacked the tables at another scale"


def test_the_packed_tables_restate_the_adapters():
    """A_cat stacks every adapter's lora_A in activation order (R padded to 8); B_cat holds each lora_B at its part's rows of the
    fused GEMM, scaled by weight * alpha / r * attention_kwargs["scale"]: B_cat A_cat = sum_i s_i B_i A_i per linear layer."""
    from chronoedit_b200.transformer import LORA_TARGETS

    m = _mirror()
    la = _lora(m, 4, 1, modules=("attn1.to_q", "attn1.to_v", "attn2.add_k_proj", "ffn.net.0.proj"))
    lb = _lora(m, 6, 2, modules=("attn1.to_v", "attn2.to_v", "ffn.net.0.proj"), alpha=3)
    m.load_lora_adapter(la, adapter_name="a")
    m.load_lora_adapter(lb, adapter_name="b")
    m.set_adapters(["a", "b"], [0.5, 1.5])
    for scale in (1.0, 0.25):
        with warnings.catch_warnings():
            warnings.simplefilter("error")   # the scale is used, not warned about, while a set is active
            _run(m, _inputs(), attention_kwargs={"scale": scale})
        want = lora_oracle.adapters_of([(la, 0.5), (lb, 1.5)], scale)
        seen = set()
        for (layer, target), (a_cat, b_raw, col_scale, b_cat) in m._lora_tables.items():
            assert a_cat.shape[0] % 8 == 0 and a_cat.dtype == b_cat.dtype == torch.bfloat16
            assert torch.equal(b_cat, (b_raw.float() * (col_scale * scale)).bfloat16())
            for sub, (tg, part, parts) in LORA_TARGETS.items():
                if tg != target:
                    continue
                n = b_cat.shape[0] // parts
                mod = f"blocks.{layer}.{sub}"
                got = b_raw[part * n: (part + 1) * n].float() * (col_scale * scale) @ a_cat.float()
                exp = sum((s * B.float() @ A.float() for A, B, s in want.get(mod, [])), torch.zeros_like(got))
                torch.testing.assert_close(got, exp, rtol=1e-6, atol=1e-6)
                seen.add(mod)
        assert {k for k in want} <= seen
    assert set(t for _, t in m._lora_tables) == {0, 3, 4, 6}   # fused QKV, context K | V, image K | V, ffn.0


def test_a_new_set_weight_or_scale_drops_cached_state():
    m = _mirror()
    m.load_lora_adapter(_lora(m, 4, 1), adapter_name="a")
    inp = _inputs()
    m.set_adapters("a")
    _run(m, inp)
    for change in (lambda: _run(m, inp, attention_kwargs={"scale": 0.5}), lambda: m.set_adapters("a", 0.3), m.disable_lora,
                   m.enable_lora, lambda: (m.load_lora_adapter(_lora(m, 4, 5), adapter_name="a"), _run(m, inp)),
                   lambda: m.set_adapters([])):
        m._ctx_cache, m._graphs, m._tc_states = [dict(buf=None)], {"k": 1}, [dict()]
        change()
        assert m._ctx_cache == [] and m._graphs == {} and m._tc_states == []
    _run(m, inp)   # the handle catches up with the empty set
    m._ctx_cache = [dict(buf=None)]
    _run(m, inp)   # no change: nothing is dropped, nothing repacked
    assert m._ctx_cache == [dict(buf=None)]


def test_refusals():
    from chronoedit_b200 import CEError

    m = _mirror()
    inp = _inputs()
    ref = _run(m, inp)
    m.load_lora_adapter(_lora(m, 4, 1), adapter_name="a")
    with pytest.raises(CEError, match="no loaded adapter"):
        m.set_adapters(["a", "nope"])
    assert m.active_adapters() == []
    g = torch.Generator().manual_seed(3)
    head = {"proj_out.lora_A.weight": torch.randn(4, m.proj_out.weight.shape[1], generator=g),
            "proj_out.lora_B.weight": torch.randn(m.proj_out.weight.shape[0], 4, generator=g)}
    m.load_lora_adapter(head, prefix=None, adapter_name="head")
    with pytest.raises(CEError, match="not a block linear layer.*fuse_lora"):
        m.set_adapters(["a", "head"])
    assert m.active_adapters() == [] and torch.equal(_run(m, inp), ref), "a refused set_adapters changed something"
    m.set_adapters("a")
    with pytest.raises(CEError, match="fuse_lora while adapters are active"):
        m.fuse_lora(lora_scale=1.0)
    m._fp32_keepalive = {"x": None}
    with pytest.raises(CEError, match="forward_fp32 is not built for run-time LoRA"):
        m.forward_fp32(*inp)
    m._sp_state = {"rank": 0, "world": 2}
    try:
        with pytest.raises(CEError, match="not built for sequence parallelism"):
            _run(m, inp)
        with pytest.raises(CEError, match="not built for sequence parallelism"):
            m.set_adapters("a")
    finally:
        m._sp_state = None
    m.disable_lora()
    assert m.fuse_lora(adapter_names=["a"], lora_scale=1.0) > 0   # switched off: fuse_lora merges as before


def test_scale_warns_only_without_an_active_adapter():
    m = _mirror()
    inp = _inputs()
    with pytest.warns(UserWarning, match="ineffective"):
        _run(m, inp, attention_kwargs={"scale": 0.5})
    m.load_lora_adapter(_lora(m, 4, 1), adapter_name="a")
    with pytest.warns(UserWarning, match="ineffective"):
        _run(m, inp, attention_kwargs={"scale": 0.5})
    m.set_adapters("a")
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        _run(m, inp, attention_kwargs={"scale": 0.5})


def test_load_and_set_after_enable_fp8():
    """FP8 weights keep no bf16 `weight`: the adapter's shapes are checked against `weight_fp8`, and the tables are the same."""
    m, m8 = _mirror(), _mirror()
    m8.enable_fp8()
    lora = _lora(m, 8, 4)
    for mm in (m, m8):
        mm.load_lora_adapter(lora, adapter_name="a")
        mm.set_adapters("a", 0.7)
        mm._lora_sync(1.0)
    assert m._lora_tables.keys() == m8._lora_tables.keys()
    for k, v in m._lora_tables.items():
        assert all(torch.equal(a, b) for a, b in zip(v, m8._lora_tables[k]))


@pytest.mark.skipif(not ref_loader.reference_available(), reason="/root/reference only exists in the build container")
def test_oracle_rule_matches_peft_style_layers_on_the_reference():
    """lora_oracle.dit_forward against the reference's transformer whose linear layers are wrapped PEFT-style
    (base(x) + lora_B(lora_A(x)) * scaling per adapter, in order), two stacked adapters, fp32 and bf16."""
    from tests.golden.make_golden import build_reference_dit

    case = cases.DIT_CASES["tiny_t2"]
    cfg = case.cfg
    sd32 = cases.dit_weights(case)
    x, t, text, img = cases.dit_inputs(case)
    ref = ref_loader.load_reference_dit()

    class PeftLinear(torch.nn.Module):
        def __init__(self, base, terms):
            super().__init__()
            self.base, self.terms = base, terms

        def forward(self, h):
            y = self.base(h)
            for A, B, s in self.terms:
                y = y + torch.nn.functional.linear(torch.nn.functional.linear(h, A.to(h.dtype)), B.to(h.dtype)) * s
            return y

    g = torch.Generator().manual_seed(5)
    entries = []
    for rank, w in ((4, 1.0), (8, 0.6)):
        sd = {}
        for i in range(cfg.num_layers):
            for mod in MODULES:
                N, K = sd32[f"blocks.{i}.{mod}.weight"].shape
                sd[f"blocks.{i}.{mod}.lora_A.weight"] = torch.randn(rank, K, generator=g) / K ** 0.5
                sd[f"blocks.{i}.{mod}.lora_B.weight"] = torch.randn(N, rank, generator=g) * 0.3
                sd[f"blocks.{i}.{mod}.alpha"] = torch.tensor(2.0 * rank)
        entries.append((sd, w))
    adapters = lora_oracle.adapters_of(entries, 0.8)
    for dtype in (torch.float32, torch.bfloat16):
        sd = sd32 if dtype == torch.float32 else cases.to_bf16_state(sd32)
        m = build_reference_dit(ref, cfg)
        m.load_state_dict(sd)
        if dtype == torch.bfloat16:
            from oracle import dit_oracle as O

            for n, p in m.named_parameters():
                if not any(k in n for k in O.KEEP_FP32):
                    p.data = p.data.bfloat16()
        for mod, terms in adapters.items():
            parent, _, leaf = mod.rpartition(".")
            holder = m.get_submodule(parent)
            setattr(holder, leaf, PeftLinear(getattr(holder, leaf), terms)) if not leaf.isdigit() else holder.__setitem__(
                int(leaf), PeftLinear(holder[int(leaf)], terms))
        ins = (x, t, text, img) if dtype == torch.float32 else (x.bfloat16(), t, text.bfloat16(), img.bfloat16())
        with torch.no_grad():
            y = m(*ins, return_dict=False)[0]
            o = lora_oracle.dit_forward(sd, cfg, adapters, *ins)
        torch.testing.assert_close(o.float(), y.float(), rtol=0, atol=1e-6 if dtype == torch.float32 else 0)
