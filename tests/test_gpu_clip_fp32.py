"""The fp32 CLIP image encoder against the class the reference CLI loads: `transformers.CLIPVisionModel` in fp32
(run_inference_diffusers.py:333-337, `torch_dtype=torch.float32`), with random fp32 weights that bf16 cannot represent, TF32 off.
The fp32 mode is held to the tolerance of the DiT's fp32 mode (rtol 1e-3 / atol 1e-4) on every hidden state it is asked for.  The
checkpoint path is the CLI's own call, `from_pretrained` on a sharded transformers directory, and each sample of a batch must come
out as it does alone."""
import copy
import json

import pytest
import torch

gpu = pytest.mark.gpu

SHAPES = {
    "clip_small": dict(hidden_size=256, intermediate_size=512, num_hidden_layers=3, num_attention_heads=4, image_size=56, patch_size=14,
                       hidden_act="quick_gelu"),
    # ViT-H/14 as the reference loads it: 1280 wide, 16 heads x 80, 32 layers, 224 px -> 257 tokens
    "clip_vit_h": dict(hidden_size=1280, intermediate_size=5120, num_hidden_layers=32, num_attention_heads=16, image_size=224, patch_size=14,
                       hidden_act="gelu"),
}
RTOL, ATOL = 1e-3, 1e-4
_CACHE = {}


def _reference(name):
    """(transformers model in fp32 on the GPU, its fp32 state dict on the host, pixel values [2, 3, S, S] fp32 on the host)"""
    if name not in _CACHE:
        from transformers import CLIPVisionConfig, CLIPVisionModel

        _CACHE.clear()
        kw = SHAPES[name]
        torch.manual_seed(7)
        ref = CLIPVisionModel(CLIPVisionConfig(attention_dropout=0.0, **kw)).eval()
        with torch.no_grad():
            for n, p in ref.named_parameters():   # O(1) activations, fp32 values that bf16 does not represent
                if "norm" in n and n.endswith("weight"):
                    p.normal_(1.0, 0.1)
                elif n.endswith("bias"):
                    p.normal_(0.0, 0.05)
                elif "embedding" in n:
                    p.normal_(0.0, 0.5)
                elif p.dim() == 2:
                    p.normal_(0.0, (1.0 / p.shape[1]) ** 0.5)
        sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
        assert not torch.equal(sd["vision_model.encoder.layers.0.mlp.fc1.weight"],
                               sd["vision_model.encoder.layers.0.mlp.fc1.weight"].bfloat16().float())
        px = torch.randn(2, 3, kw["image_size"], kw["image_size"])
        _CACHE[name] = (ref.cuda(), sd, px)
    return _CACHE[name]


def _mirror(name, sd, dtype):
    import chronoedit_b200 as ce

    m = ce.CLIPVisionModel(**SHAPES[name], torch_dtype=dtype)
    m.load_state_dict(sd)
    return m.cuda()


def _layer_counts(name):
    n = SHAPES[name]["num_hidden_layers"]
    return [0, 1, n - 1]


@gpu
@pytest.mark.parametrize("name", list(SHAPES))
def test_fp32_clip_matches_transformers_fp32(name):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    ref, sd, px = _reference(name)
    ours32, ours16 = _mirror(name, sd, torch.float32), _mirror(name, sd, None)
    assert ours32.dtype == torch.float32 and ours16.dtype == torch.bfloat16
    with torch.no_grad():
        r = ref(pixel_values=px.cuda(), output_hidden_states=True).hidden_states
        # fp64 as a yardstick for both fp32 results (reported, not asserted)
        r64 = copy.deepcopy(ref).double()(pixel_values=px.cuda().double(), output_hidden_states=True).hidden_states
    for k in _layer_counts(name):
        got = ours32(pixel_values=px.cuda(), output_hidden_states=True).hidden_states[k]
        assert got.dtype == torch.float32 and got.shape == r[k].shape
        b16 = ours16(pixel_values=px.cuda(), output_hidden_states=True).hidden_states[k].float()
        e32, e16 = (got - r[k]).abs(), (b16 - r[k]).abs()
        rep = {"case": name, "layers": k, "fp32_max": e32.max().item(), "fp32_mean": e32.mean().item(), "bf16_max": e16.max().item(),
               "bf16_mean": e16.mean().item(), "mean_abs_ref": r[k].abs().mean().item(), "fp32_launches": ours32.launches(),
               "fp32_vs_fp64_max": (got.double() - r64[k]).abs().max().item(), "ref_fp32_vs_fp64_max": (r[k].double() - r64[k]).abs().max().item()}
        print(json.dumps(rep))
        assert torch.isfinite(got).all()
        assert torch.allclose(got, r[k], rtol=RTOL, atol=ATOL), rep


@gpu
@pytest.mark.parametrize("name", list(SHAPES))
def test_from_pretrained_sharded_checkpoint_as_the_cli_loads_it(name, tmp_path):
    import chronoedit_b200 as ce

    ref, sd, px = _reference(name)
    d = tmp_path / "ckpt"
    ref.save_pretrained(str(d / "image_encoder"), max_shard_size="1MB" if name == "clip_small" else "300MB")
    assert (d / "image_encoder" / "model.safetensors.index.json").exists()
    n = SHAPES[name]["num_hidden_layers"]

    loaded = ce.CLIPVisionModel.from_pretrained(str(d), subfolder="image_encoder", torch_dtype=torch.float32).cuda()
    direct = _mirror(name, sd, torch.float32)
    a = loaded(pixel_values=px.cuda(), output_hidden_states=True).hidden_states[-2]
    b = direct(pixel_values=px.cuda(), output_hidden_states=True).hidden_states[-2]
    assert a.dtype == torch.float32 and torch.equal(a, b)
    assert loaded.launches() == direct.launches() > 0
    del loaded, direct

    loaded16 = ce.CLIPVisionModel.from_pretrained(str(d), subfolder="image_encoder", torch_dtype=torch.bfloat16).cuda()
    today = ce.CLIPVisionModel(**SHAPES[name])
    today.load_state_dict({k: v.to(torch.bfloat16) for k, v in sd.items()})
    today = today.cuda()
    a16 = loaded16(pixel_values=px.cuda(), output_hidden_states=True).hidden_states[n - 1]
    b16 = today(pixel_values=px.cuda(), output_hidden_states=True).hidden_states[n - 1]
    assert a16.dtype == torch.bfloat16 and torch.equal(a16.view(torch.int16), b16.view(torch.int16))
    assert loaded16.launches() == today.launches() > 0


@gpu
@pytest.mark.parametrize("name", list(SHAPES))
def test_fp32_clip_batch_invariance(name):
    _, sd, px = _reference(name)
    m = _mirror(name, sd, torch.float32)
    x = px.cuda()
    before = x.clone()
    both = m(pixel_values=x, output_hidden_states=True).hidden_states[-2]
    assert torch.equal(x, before)
    for b in range(2):
        one = m(pixel_values=x[b:b + 1].contiguous(), output_hidden_states=True).hidden_states[-2]
        assert torch.equal(one[0], both[b]), b
    assert torch.equal(x, before)
