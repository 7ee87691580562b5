"""north_star's tolerance, asserted END TO END: "outputs match the reference ... within rtol=1e-3 / atol=1e-4".

In bf16 that band cannot be met by any implementation -- the reference misses it against itself across precisions (SURVEY.md
section 7, hard part 3) -- so the bf16 path is held to "as close to the fp32 answer as the reference's own bf16 run"
(tests/test_gpu_dit.py, tests/test_gpu_baseline_sizes.py).  Here the VALIDATION mode of the CUDA path (ce_dit_forward_fp32: fp32
I/O and residual stream, every matrix product on the wgmma GEMM with split-bf16 operands, csrc/dit_fp32.cu) is compared with
the golden outputs of the UNMODIFIED reference run in fp32 (tests/golden/dit_*.safetensors: `out_fp32`, `block0_fp32`), and every
element must satisfy |ours - ref| <= 1e-4 + 1e-3 |ref| -- torch.allclose(rtol=1e-3, atol=1e-4), no forgiven fraction -- on all
BASELINE configs[0] cases incl. the 64x64 latent (2048 tokens), the 8-frame RoPE branch, batch 2 and the ragged 3-head case."""
import json
import os

import pytest
import torch
from safetensors.torch import load_file

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@gpu
@pytest.mark.parametrize("name", ["tiny_t2", "tiny_t8", "tiny_b2", "tiny_ragged", "cfg0_64x64"])
def test_fp32_validation_mode_meets_the_stated_tolerance(name, golden_dir):
    import chronoedit_b200 as ce
    from oracle import cases

    case = cases.DIT_CASES[name]
    cfg = case.cfg
    gold = load_file(os.path.join(golden_dir, f"dit_{name}.safetensors"))
    sd32 = cases.dit_weights(case)
    x, t, text, img = cases.dit_inputs(case)
    m = ce.ChronoEditTransformer3DModel(
        patch_size=cfg.patch_size, num_attention_heads=cfg.num_attention_heads, attention_head_dim=cfg.attention_head_dim,
        in_channels=cfg.in_channels, out_channels=cfg.out_channels, text_dim=cfg.text_dim, freq_dim=cfg.freq_dim, ffn_dim=cfg.ffn_dim,
        num_layers=cfg.num_layers, eps=cfg.eps, image_dim=cfg.image_dim, added_kv_proj_dim=cfg.added_kv_proj_dim,
        rope_max_seq_len=cfg.rope_max_seq_len, rope_temporal_skip_len=cfg.rope_temporal_skip_len).cuda()
    m.enable_fp32_validation(sd32)
    out, b0 = m.forward_fp32(x.cuda(), t.cuda(), text.cuda(), img.cuda(), return_block0=True)
    torch.cuda.synchronize()
    out, b0 = out.cpu(), b0.cpu()
    ref = gold["out_fp32"]
    assert out.shape == ref.shape and torch.isfinite(out).all()
    err = (out - ref).abs()
    band = 1e-4 + 1e-3 * ref.abs()
    rep = {"case": name, "max_abs_err": err.max().item(), "mean_abs_err": err.mean().item(), "mean_abs_ref": ref.abs().mean().item(),
           "worst_err_over_band": (err / band).max().item(), "fraction_inside_band": (err <= band).float().mean().item()}
    if "block0_fp32" in gold:
        r0 = gold["block0_fp32"].reshape(b0.shape)
        e0 = (b0 - r0).abs()
        rep["block0_worst_err_over_band"] = (e0 / (1e-4 + 1e-3 * r0.abs())).max().item()
    print(json.dumps(rep))
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", f"fp32_mode_{name}.json"), "w") as f:
        json.dump(rep, f)
    assert torch.allclose(out, ref, rtol=1e-3, atol=1e-4), rep
    if "block0_fp32" in gold:
        assert torch.allclose(b0, gold["block0_fp32"].reshape(b0.shape), rtol=1e-3, atol=1e-4), rep
