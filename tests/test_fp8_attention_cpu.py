"""FP8 self-attention without a GPU: the torch statements of its two quantization rules, the key order of the stored V^T, the
switch's state on the Python mirror, and the device check of the new C exports."""
import pytest
import torch

from chronoedit_b200.transformer import fp8_attention_key_order, quantize_fp8_channels, quantize_fp8_heads, quantize_fp8_rows
from tests.test_fp8_cpu import _tiny


def test_heads_rule_exact_values():
    # two tokens x two heads: each head has its own scale; a head whose maximum is 448 keeps its values exactly
    x = torch.zeros(2, 256)
    x[0, :128] = torch.linspace(-448, 448, 128)
    x[0, 128:] = 1e-3
    x[0, 200] = -7.0
    x[1, 5] = 3.0
    q, s = quantize_fp8_heads(x)
    assert q.shape == (2, 256) and q.dtype == torch.float8_e4m3fn and s.shape == (2, 2)
    assert s[0, 0].item() == 1.0 and s[1, 1].item() == 1.0   # zero head: scale 1
    assert s[0, 1].item() == torch.tensor(7.0) / torch.tensor(448.0)
    assert s[1, 0].item() == torch.tensor(3.0) / torch.tensor(448.0)
    assert q[0, 200].float().item() == -448.0 and q[1, 5].float().item() == 448.0
    assert torch.equal(q[0, :128].float(), x[0, :128].to(torch.float8_e4m3fn).float())
    assert (q.view(torch.uint8)[1, 128:] == 0).all()
    # the same as quantize_fp8_rows on the [tokens * heads, 128] view, for any leading shape
    y = torch.randn(3, 5, 384).bfloat16()
    qa, sa = quantize_fp8_heads(y)
    qb, sb = quantize_fp8_rows(y.reshape(-1, 128))
    assert torch.equal(qa.view(torch.uint8).reshape(-1, 128), qb.view(torch.uint8)) and torch.equal(sa.reshape(-1), sb)


def test_channels_rule_exact_values():
    v = torch.zeros(2, 4, 3)   # [B, L, C]
    v[0, :, 0] = torch.tensor([1.0, -2.0, 0.5, 896.0])
    v[0, 2, 1] = -0.0
    v[1, :, 0] = torch.tensor([1.0, 1.0, 1.0, 1.0])   # the other sample: its own scale
    v[1, 1, 2] = 1e-3
    q, s = quantize_fp8_channels(v)
    assert q.shape == (2, 3, 4) and s.shape == (2, 3)
    assert s[0, 0].item() == 2.0 and s[0, 1].item() == 1.0 and s[0, 2].item() == 1.0
    assert s[1, 0].item() == torch.tensor(1.0) / torch.tensor(448.0)
    assert torch.equal(q[0, 0].float(), torch.tensor([0.5, -1.0, 0.25, 448.0]))
    assert q.view(torch.uint8)[0, 1, 2].item() == 0x80   # -0 keeps its sign
    assert (q[1, 0].float() == 448.0).all() and q[1, 2, 1].float().item() == 448.0
    # batch invariance: sample 1 alone gives the same
    q1, s1 = quantize_fp8_channels(v[1:])
    assert torch.equal(q1.view(torch.uint8), q.view(torch.uint8)[1:]) and torch.equal(s1, s[1:])


def test_key_order_is_a_permutation_matching_the_fragment():
    order = fp8_attention_key_order()
    assert sorted(order.tolist()) == list(range(32))
    # thread t of a warp holds the accumulator keys 8c + 2t + {0, 1}; fragment registers 0 and 2 want positions 4t .. 4t + 3 and
    # 16 + 4t .. 16 + 4t + 3, filled with the accumulator pairs c = 0, 1 and c = 2, 3
    for t in range(4):
        assert order[4 * t: 4 * t + 4].tolist() == [2 * t, 2 * t + 1, 8 + 2 * t, 9 + 2 * t]
        assert order[16 + 4 * t: 20 + 4 * t].tolist() == [16 + 2 * t, 17 + 2 * t, 24 + 2 * t, 25 + 2 * t]


def test_switch_state():
    m, sd = _tiny(num_layers=1)
    assert not m.fp8_attention_enabled
    before = {k: v.clone() for k, v in m.state_dict().items()}
    m._graphs = {"x": 1}
    m._workspaces = {"y": 2}
    m._ctx_cache = [{"buf": None}]
    m.enable_fp8_attention()
    assert m.fp8_attention_enabled
    assert m._graphs == {} and m._workspaces == {}, "toggling must drop captured graphs and workspaces"
    assert m._ctx_cache == [{"buf": None}], "the context cache stays valid: cross-attention is untouched"
    after = m.state_dict()
    assert before.keys() == after.keys() and all(torch.equal(before[k], after[k]) for k in before)
    m._graphs = {"x": 1}
    m.enable_fp8_attention(True)   # no change: nothing dropped
    assert m._graphs == {"x": 1}
    m = m.to(torch.device("cpu"))
    assert m.fp8_attention_enabled
    m.load_state_dict(sd)
    assert m.fp8_attention_enabled
    w = sd["blocks.0.attn2.to_k.weight"]
    lora = {"transformer.blocks.0.attn2.to_k.lora_A.weight": torch.zeros(4, w.shape[1]),
            "transformer.blocks.0.attn2.to_k.lora_B.weight": torch.zeros(w.shape[0], 4)}
    m.fuse_lora(lora, lora_scale=1.0)
    assert m.fp8_attention_enabled
    m.enable_fp8()
    assert m.fp8_attention_enabled and m.fp8_enabled
    m.enable_fp8_attention(False)
    assert not m.fp8_attention_enabled and m.fp8_enabled


def test_enable_fp8_does_not_switch_attention():
    m, _ = _tiny(num_layers=1)
    m.enable_fp8()
    assert m.fp8_enabled and not m.fp8_attention_enabled


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_fp8_attention_exports_fail_without_a_device():
    import chronoedit_b200._lib as L

    lib = L.lib()
    x = torch.zeros(4, 384, dtype=torch.bfloat16)
    q = torch.zeros(4, 256, dtype=torch.uint8)
    s = torch.ones(4, 2)
    vt = torch.zeros(1, 128, 32, dtype=torch.uint8)
    out = torch.zeros(4, 128, dtype=torch.bfloat16)
    assert lib.ce_quantize_heads_fp8(L.ptr(x), 384, 4, 2, L.ptr(q), 256, L.ptr(s), None) == -3
    assert b"no CPU fallback" in lib.ce_last_error()
    assert lib.ce_quantize_v_fp8(L.ptr(x[:, 256:]), 384, 1, 4, 1, L.ptr(vt), 32, L.ptr(s), None) == -3
    assert b"no CPU fallback" in lib.ce_last_error()
    assert lib.ce_attention_fp8(L.ptr(q), L.ptr(q[:, 128:]), 256, L.ptr(s), L.ptr(s[:, 1:]), 2, L.ptr(vt), 32, L.ptr(s), L.ptr(out), 128,
                                1, 1, 4, 0.088, None) == -3
    assert b"no CPU fallback" in lib.ce_last_error()
    # the switch itself is host state: it needs no device
    import ctypes

    from chronoedit_b200._lib import DiTConfigC

    cfg = DiTConfigC(2, 128, 16, 16, 64, 256, 256, 1, 0, 0, 1024, 8, 1e-6, 1, 2, 2)
    h = ctypes.c_void_p()
    L.check(lib.ce_dit_create(ctypes.byref(cfg), ctypes.byref(h)))
    try:
        off = lib.ce_dit_workspace_bytes(h, 1, 2, 16, 16, 8)
        L.check(lib.ce_dit_set_attention_fp8(h, 1))
        on = lib.ce_dit_workspace_bytes(h, 1, 2, 16, 16, 8)
        M, D, H, Lpad = 128, 256, 2, 128
        assert on - off >= M * 2 * D + M * 2 * H * 4 + D * Lpad + D * 4
        L.check(lib.ce_dit_set_attention_fp8(h, 0))
        assert lib.ce_dit_workspace_bytes(h, 1, 2, 16, 16, 8) == off
    finally:
        lib.ce_dit_destroy(h)
