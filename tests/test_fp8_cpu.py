"""FP8 mode without a GPU: the weight quantization rule, the mirror's buffers after enable_fp8(), the calls it forbids, and the
device check of the new C exports."""
import ctypes

import pytest
import torch

from chronoedit_b200.transformer import FP8_LINEARS, quantize_fp8_rows

E4M3_MAX = 448.0


def _tiny(num_layers=2):
    import chronoedit_b200 as ce
    from oracle import cases, dit_oracle as O

    cfg = O.DiTConfig.tiny(num_layers=num_layers)
    m = ce.ChronoEditTransformer3DModel(num_attention_heads=cfg.num_attention_heads, in_channels=cfg.in_channels,
                                        ffn_dim=cfg.ffn_dim, num_layers=cfg.num_layers, image_dim=cfg.image_dim,
                                        added_kv_proj_dim=cfg.added_kv_proj_dim, text_dim=cfg.text_dim)
    sd = cases.to_bf16_state(O.random_state_dict(cfg, seed=0))
    m.load_state_dict(sd)
    return m, sd


def _e4m3_values():
    """Every finite e4m3fn value (bit patterns 0x00-0x7e and their negatives) as fp32."""
    bits = torch.arange(256, dtype=torch.uint8)
    v = bits.view(torch.float8_e4m3fn).float()
    return v[torch.isfinite(v)]


def test_weight_rule_exact_values():
    # a row whose maximum is 448 has scale 1: every e4m3 value is kept exactly
    vals = _e4m3_values()
    row = torch.cat([vals, torch.tensor([448.0])]).reshape(1, -1)
    q, s = quantize_fp8_rows(row)
    assert s.item() == 1.0 and q.dtype == torch.float8_e4m3fn
    assert torch.equal(q.float(), row)


def test_weight_rule_scale_saturation_and_rounding():
    w = torch.tensor([[1000.0, -3.0, 0.5, 0.0],       # scale 1000/448: the maximum maps to exactly 448
                      [-2.0e-3, 1.0e-3, 0.0, 7.0e-4],
                      [1.0, 1.0625, 1.1875, -1.0625]])  # values between grid points of e4m3
    q, s = quantize_fp8_rows(w)
    ref_s = w.abs().amax(1) / 448
    assert torch.equal(s, ref_s)
    assert q[0, 0].float().item() == 448.0
    # the row maximum always lands on +-448 (no overflow to NaN, no saturation beyond the largest finite value)
    assert torch.equal(q.float().abs().amax(1), torch.full((3,), E4M3_MAX))
    for r in range(3):
        exact = (w[r] / s[r]).clamp(-448, 448)
        # round to nearest: the error is at most half a step of the e4m3 grid around each value
        vals = _e4m3_values()
        nearest = vals[(exact[:, None] - vals[None]).abs().argmin(1)]
        assert torch.equal((q[r].float() - exact).abs(), (nearest - exact).abs())


def test_weight_rule_zero_rows_and_negative_zero():
    w = torch.zeros(3, 32)
    w[1, 5] = -0.0
    w[2] = -0.0
    q, s = quantize_fp8_rows(w)
    assert torch.equal(s, torch.ones(3))
    assert torch.equal(q.view(torch.uint8)[0], torch.zeros(32, dtype=torch.uint8))
    assert q.view(torch.uint8)[1, 5].item() == 0x80   # -0.0 keeps its sign
    assert torch.equal(q.view(torch.uint8)[2], torch.full((32,), 0x80, dtype=torch.uint8))
    # bf16 input gives the same as its fp32 value
    x = torch.randn(5, 48).bfloat16()
    qa, sa = quantize_fp8_rows(x)
    qb, sb = quantize_fp8_rows(x.float())
    assert torch.equal(qa.view(torch.uint8), qb.view(torch.uint8)) and torch.equal(sa, sb)


def test_enable_fp8_buffers():
    m, sd = _tiny()
    assert not m.fp8_enabled
    m.enable_fp8()
    assert m.fp8_enabled
    params = dict(m.named_parameters())
    bufs = dict(m.named_buffers())
    D, F = 256, m.config.ffn_dim
    shapes = {"attn1.to_q": (D, D), "attn1.to_k": (D, D), "attn1.to_v": (D, D), "attn1.to_out.0": (D, D), "attn2.to_q": (D, D),
              "attn2.to_out.0": (D, D), "ffn.net.0.proj": (F, D), "ffn.net.2": (D, F)}
    assert set(shapes) == set(FP8_LINEARS)
    for i in range(m.config.num_layers):
        for name, (n, k) in shapes.items():
            p = f"blocks.{i}.{name}."
            assert p + "weight" not in params
            assert p + "bias" in params and params[p + "bias"].dtype == torch.bfloat16
            q, s = bufs[p + "weight_fp8"], bufs[p + "weight_scale"]
            assert q.dtype == torch.float8_e4m3fn and q.shape == (n, k)
            assert s.dtype == torch.float32 and s.shape == (n,)
            rq, rs = quantize_fp8_rows(sd[p + "weight"])
            assert torch.equal(q.view(torch.uint8), rq.view(torch.uint8)) and torch.equal(s, rs)
        # everything else keeps its bf16 / fp32 parameters
        for name in ("attn2.to_k", "attn2.to_v", "attn2.add_k_proj", "attn2.add_v_proj"):
            assert params[f"blocks.{i}.{name}.weight"].dtype == torch.bfloat16
    for name in ("patch_embedding.weight", "proj_out.weight", "condition_embedder.text_embedder.linear_1.weight"):
        assert params[name].dtype == torch.bfloat16
    assert len(bufs) == 2 * len(FP8_LINEARS) * m.config.num_layers
    m.enable_fp8()   # one-way: a second call changes nothing
    assert len(dict(m.named_buffers())) == len(bufs)
    m2 = m.to(torch.device("cpu"))
    assert m2.blocks[0].ffn.net[2].weight_fp8.dtype == torch.float8_e4m3fn


def test_fuse_lora_and_load_state_dict_raise_after_enable_fp8():
    import chronoedit_b200 as ce

    m, sd = _tiny(num_layers=1)
    m.enable_fp8()
    before = {k: v.clone() for k, v in m.state_dict().items()}
    w = sd["blocks.0.attn2.to_k.weight"]
    lora = {"transformer.blocks.0.attn2.to_k.lora_A.weight": torch.ones(4, w.shape[1]),
            "transformer.blocks.0.attn2.to_k.lora_B.weight": torch.ones(w.shape[0], 4)}
    with pytest.raises(ce.CEError, match="enable_fp8"):
        m.fuse_lora(lora, lora_scale=1.0)
    with pytest.raises(ce.CEError, match="enable_fp8"):
        m.load_state_dict(sd)
    after = m.state_dict()
    assert before.keys() == after.keys()
    assert all(torch.equal(before[k].view(torch.uint8) if before[k].dtype == torch.float8_e4m3fn else before[k],
                           after[k].view(torch.uint8) if after[k].dtype == torch.float8_e4m3fn else after[k]) for k in before)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_fp8_exports_fail_without_a_device():
    import chronoedit_b200._lib as L

    lib = L.lib()
    a = torch.zeros(16, 16, dtype=torch.uint8)
    sc = torch.ones(16)
    out = torch.zeros(16, 16, dtype=torch.bfloat16)
    base = L.LinearArgsC(A=a.data_ptr(), lda=16, W=a.data_ptr(), ldw=16, M=16, N=16, K=16, out=out.data_ptr(), ldo=16)
    args = L.LinearFp8ArgsC(base=base, a_scale=sc.data_ptr(), w_scale=sc.data_ptr())
    assert lib.ce_linear_fp8_ex(ctypes.byref(args), None) == -3 and b"no CPU fallback" in lib.ce_last_error()
    assert lib.ce_linear_fp8_ex(None, None) == -3 and b"no CPU fallback" in lib.ce_last_error()
    assert lib.ce_quantize_rows_fp8(L.ptr(out), 16, 16, 16, L.ptr(a), 16, L.ptr(sc), None) == -3
    assert b"no CPU fallback" in lib.ce_last_error()
