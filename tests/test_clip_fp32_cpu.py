"""Host side of the fp32 CLIP image encoder and of the encoders' `from_pretrained`, without a GPU: the loader on transformers-format
directories (single file and sharded), the dtype rules of both mirrors, and the refusals of the fp32 C entry points, every one of
which comes before the first launch.  The arithmetic is compared on the GPU (tests/test_gpu_clip_fp32.py)."""
import ctypes
import json

import pytest
import torch

import chronoedit_b200 as ce
from chronoedit_b200 import _lib as L
from chronoedit_b200._lib import CEError

transformers = pytest.importorskip("transformers")
safetensors_torch = pytest.importorskip("safetensors.torch")

CLIP_KW = dict(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4, image_size=28, patch_size=14,
               hidden_act="quick_gelu")
UMT5_KW = dict(vocab_size=512, d_model=64, d_kv=16, d_ff=128, num_layers=2, num_heads=4)

CE_ERR_INVALID, CE_ERR_NO_DEVICE, CE_ERR_MISSING_WEIGHT, CE_ERR_WORKSPACE = -1, -3, -4, -5


def _hf_clip():
    torch.manual_seed(0)
    hf = transformers.CLIPVisionModel(transformers.CLIPVisionConfig(**CLIP_KW))
    with torch.no_grad():
        for p in hf.parameters():
            p.normal_(0.0, 1.0)   # fp32 values bf16 does not represent
    return hf


@pytest.fixture(params=["single", "sharded"])
def clip_dir(request, tmp_path):
    hf = _hf_clip()
    d = tmp_path / "image_encoder"
    hf.save_pretrained(str(d), max_shard_size="20KB" if request.param == "sharded" else "1GB")
    assert (d / "model.safetensors.index.json").exists() == (request.param == "sharded")
    return d, {k: v.detach().clone() for k, v in hf.state_dict().items() if not k.endswith("position_ids")}


def test_clip_from_pretrained_keeps_fp32_parameters(clip_dir):
    d, sd = clip_dir
    m = ce.CLIPVisionModel.from_pretrained(str(d.parent), subfolder=d.name, torch_dtype=torch.float32)
    assert m.dtype == torch.float32
    for k in ("hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads", "image_size", "patch_size", "hidden_act"):
        assert m.config[k] == CLIP_KW[k], k
    mine = m.state_dict()
    assert set(mine) == set(sd)
    for k, v in sd.items():
        assert mine[k].dtype == torch.float32 and torch.equal(mine[k], v), k


@pytest.mark.parametrize("dtype", [None, torch.bfloat16])
def test_clip_from_pretrained_bf16_is_todays_module(clip_dir, dtype):
    d, sd = clip_dir
    m = ce.CLIPVisionModel.from_pretrained(str(d), torch_dtype=dtype)
    today = ce.CLIPVisionModel(**CLIP_KW)
    today.load_state_dict({k: v.to(torch.bfloat16) for k, v in sd.items()})
    assert m.dtype == torch.bfloat16
    mine, theirs = m.state_dict(), today.state_dict()
    assert set(mine) == set(theirs)
    for k in mine:
        assert mine[k].dtype == torch.bfloat16 and torch.equal(mine[k].view(torch.int16), theirs[k].view(torch.int16)), k


def _synthetic_dir(tmp_path, sd, config):
    tmp_path.mkdir(parents=True, exist_ok=True)
    safetensors_torch.save_file({k: v.contiguous() for k, v in sd.items()}, str(tmp_path / "model.safetensors"))
    (tmp_path / "config.json").write_text(json.dumps(config))
    return str(tmp_path)


def test_clip_from_pretrained_refuses_unknown_and_missing_keys(tmp_path):
    sd = ce.CLIPVisionModel(**CLIP_KW, torch_dtype=torch.float32).state_dict()
    sd = {k: torch.randn(v.shape) for k, v in sd.items()}
    extra = _synthetic_dir(tmp_path / "extra", {**sd, "vision_model.encoder.layers.9.mlp.fc1.weight": torch.zeros(4)}, CLIP_KW)
    with pytest.raises(CEError, match="unexpected key in checkpoint: vision_model.encoder.layers.9.mlp.fc1.weight"):
        ce.CLIPVisionModel.from_pretrained(extra, torch_dtype=torch.float32)
    gone = "vision_model.encoder.layers.1.self_attn.k_proj.bias"
    short = _synthetic_dir(tmp_path / "short", {k: v for k, v in sd.items() if k != gone}, CLIP_KW)
    with pytest.raises(CEError, match=f"missing 1 parameters, first: {gone}"):
        ce.CLIPVisionModel.from_pretrained(short, torch_dtype=torch.float32)
    # the non-parameter position_ids buffer of older transformers checkpoints is not a key error
    old = _synthetic_dir(tmp_path / "old", {**sd, "vision_model.embeddings.position_ids": torch.arange(5).unsqueeze(0)}, CLIP_KW)
    assert ce.CLIPVisionModel.from_pretrained(old, torch_dtype=torch.float32).dtype == torch.float32


@pytest.mark.parametrize("dtype", [torch.float16, torch.float64, torch.int8])
def test_clip_refuses_other_dtypes(clip_dir, dtype):
    d, _ = clip_dir
    with pytest.raises(CEError, match="torch.bfloat16 or torch.float32"):
        ce.CLIPVisionModel(**CLIP_KW, torch_dtype=dtype)
    with pytest.raises(CEError, match="torch.bfloat16 or torch.float32"):
        ce.CLIPVisionModel.from_pretrained(str(d), torch_dtype=dtype)


def test_clip_fp32_has_no_cpu_path():
    m = ce.CLIPVisionModel(**CLIP_KW, torch_dtype=torch.float32)
    with pytest.raises(CEError, match="no CPU path"):
        m(pixel_values=torch.zeros(1, 3, 28, 28), output_hidden_states=True).hidden_states[-2]


@pytest.mark.parametrize("sharded", [False, True])
def test_umt5_from_pretrained_bf16_and_fp32_refused(tmp_path, sharded):
    torch.manual_seed(1)
    hf = transformers.UMT5EncoderModel(transformers.UMT5Config(**UMT5_KW, feed_forward_proj="gated-gelu", relative_attention_num_buckets=32,
                                                               relative_attention_max_distance=128))
    with torch.no_grad():
        for p in hf.parameters():
            p.normal_(0.0, 1.0)
    d = tmp_path / "text_encoder"
    hf.save_pretrained(str(d), max_shard_size="50KB" if sharded else "1GB")
    assert (d / "model.safetensors.index.json").exists() == sharded
    for dtype in (None, torch.bfloat16):
        m = ce.UMT5EncoderModel.from_pretrained(str(tmp_path), subfolder="text_encoder", torch_dtype=dtype)
        assert m.dtype == torch.bfloat16
        for k in UMT5_KW:
            assert m.config[k] == UMT5_KW[k], k
        today = ce.UMT5EncoderModel(**UMT5_KW)
        today.load_state_dict({k: v.to(torch.bfloat16) for k, v in hf.state_dict().items()})
        mine, theirs = m.state_dict(), today.state_dict()
        assert set(mine) == set(theirs)
        for k in mine:
            assert torch.equal(mine[k].view(torch.int16), theirs[k].view(torch.int16)), k
    for dtype in (torch.float32, torch.float16):
        with pytest.raises(CEError, match="bf16 only"):
            ce.UMT5EncoderModel.from_pretrained(str(d), torch_dtype=dtype)


# ------------------------------------------------------------------------------------------------------------------ C entry points
class _Aligned:
    """Aligned host addresses: the handle only keeps pointers, and nothing here dereferences them."""

    def __init__(self):
        self._buf = torch.zeros(1024, dtype=torch.uint8)
        self.base = (self._buf.data_ptr() + 255) & ~255
        self.ptr = ctypes.c_void_p(self.base)


BUF = _Aligned()
CLIP_C = dict(kind=1, d_model=256, d_kv=64, d_ff=512, num_layers=3, num_heads=4, eps=1e-5, image_size=56, patch_size=14, hidden_act=0)
UMT5_C = dict(kind=0, vocab_size=4096, d_model=512, d_kv=64, d_ff=1024, num_layers=3, num_heads=8, eps=1e-6)
no_device = pytest.mark.skipif(L.lib().ce_device_check() == 0, reason="a complete weight set would launch on fake host pointers")


def error():
    return (L.lib().ce_last_error() or b"").decode()


def clip_fp32_weights(c):
    """{transformers name: numel} of every fp32 parameter the fp32 entry reads"""
    D, F, ps = c["d_model"], c["d_ff"], c["patch_size"]
    vm = "vision_model."
    w = {vm + "embeddings.patch_embedding.weight": D * 3 * ps * ps, vm + "embeddings.class_embedding": D,
         vm + "embeddings.position_embedding.weight": (1 + (c["image_size"] // ps) ** 2) * D, vm + "pre_layrnorm.weight": D,
         vm + "pre_layrnorm.bias": D}
    for l in range(c["num_layers"]):
        p = f"{vm}encoder.layers.{l}."
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            w.update({p + f"self_attn.{n}.weight": D * D, p + f"self_attn.{n}.bias": D})
        for n in ("layer_norm1", "layer_norm2"):
            w.update({p + n + ".weight": D, p + n + ".bias": D})
        w.update({p + "mlp.fc1.weight": F * D, p + "mlp.fc1.bias": F, p + "mlp.fc2.weight": D * F, p + "mlp.fc2.bias": D})
    return w


class Handle:
    def __init__(self, c, fp32=None, bf16=None):
        self.lib, self.c = L.lib(), c
        self.h = ctypes.c_void_p()
        L.check(self.lib.ce_encoder_create(ctypes.byref(L.EncoderConfigC(**c)), ctypes.byref(self.h)))
        for name, numel in (fp32 or {}).items():
            L.check(self.lib.ce_encoder_set_weight_fp32(self.h, name.encode(), BUF.ptr, numel))
        for name, numel in (bf16 or {}).items():
            L.check(self.lib.ce_encoder_set_weight(self.h, name.encode(), BUF.ptr, numel))

    def ws_bytes(self, batch=2):
        return self.lib.ce_clip_vision_fp32_workspace_bytes(self.h, batch)

    def encode(self, px=BUF.ptr, out=BUF.ptr, batch=2, layers=None, ws=BUF.ptr, ws_bytes=None):
        layers = self.c["num_layers"] - 1 if layers is None else layers
        ws_bytes = 1 << 40 if ws_bytes is None else ws_bytes
        return self.lib.ce_clip_vision_encode_fp32(self.h, px, out, batch, layers, ws, ws_bytes, None)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.lib.ce_encoder_destroy(self.h)


def test_fp32_symbols_are_exported_and_refuse_null_handles():
    lib = L.lib()
    for name in ("ce_encoder_set_weight_fp32", "ce_clip_vision_fp32_workspace_bytes", "ce_clip_vision_encode_fp32"):
        assert hasattr(lib, name) and name in L.SIGNATURES
    assert lib.ce_encoder_set_weight_fp32(None, b"x", BUF.ptr, 4) == CE_ERR_INVALID and "null handle" in error()
    assert lib.ce_clip_vision_fp32_workspace_bytes(None, 1) == -1
    assert lib.ce_clip_vision_encode_fp32(None, BUF.ptr, BUF.ptr, 1, 0, BUF.ptr, 1 << 40, None) == CE_ERR_INVALID
    assert "null argument" in error()


def test_set_weight_fp32_refuses_null_and_misaligned_pointers():
    with Handle(CLIP_C) as e:
        assert e.lib.ce_encoder_set_weight_fp32(e.h, None, BUF.ptr, 4) == CE_ERR_INVALID and "null argument" in error()
        assert e.lib.ce_encoder_set_weight_fp32(e.h, b"x", None, 4) == CE_ERR_INVALID and "null argument" in error()
        assert e.lib.ce_encoder_set_weight_fp32(e.h, b"x", ctypes.c_void_p(BUF.base + 4), 4) == CE_ERR_INVALID
        assert "16-byte aligned" in error()


def test_fp32_workspace_query():
    with Handle(CLIP_C) as e:
        assert e.ws_bytes(0) == -1 and e.ws_bytes(-1) == -1
        sizes = [e.ws_bytes(b) for b in (1, 2, 3)]
        assert all(s > 0 and s % 256 == 0 for s in sizes) and sizes[0] < sizes[1] < sizes[2]
        # the fp32 residual stream alone: 7 [B*L, D] fp32 buffers and one [B*L, F]
        L_ = 1 + (56 // 14) ** 2
        assert sizes[1] > 4 * 2 * L_ * (7 * 256 + 512)
    with Handle(UMT5_C) as e:
        assert e.ws_bytes(1) == -1


def test_fp32_encode_refuses_bad_arguments_before_any_launch():
    w = clip_fp32_weights(CLIP_C)
    with Handle(CLIP_C, fp32=w) as e:
        for kw in (dict(px=None), dict(out=None), dict(ws=None)):
            assert e.encode(**kw) == CE_ERR_INVALID and "null argument" in error(), kw
        assert e.encode(batch=0) == CE_ERR_INVALID and "batch" in error()
        for layers in (-1, CLIP_C["num_layers"] + 1):
            assert e.encode(layers=layers) == CE_ERR_INVALID and "layers_to_run" in error()
        need = e.ws_bytes(2)
        assert e.encode(ws_bytes=need - 1) == CE_ERR_WORKSPACE and f"need {need}" in error()
        assert e.encode(ws=ctypes.c_void_p(BUF.base + 16)) == CE_ERR_INVALID and "256-byte aligned" in error()
    with Handle(UMT5_C, fp32={"shared.weight": 8}) as e:
        assert e.encode() == CE_ERR_INVALID and "not a CLIP vision encoder" in error()


def test_fp32_encode_refuses_a_handle_without_fp32_weights():
    # the same names registered as bf16 weights do not make an fp32 handle
    with Handle(CLIP_C, bf16=clip_fp32_weights(CLIP_C)) as e:
        assert e.encode() == CE_ERR_INVALID and "no fp32 weights" in error()


@pytest.mark.parametrize("case", ["missing", "short"])
def test_fp32_encode_names_each_missing_or_short_weight(case):
    w = clip_fp32_weights(CLIP_C)
    for name in w:
        ws = {k: v for k, v in w.items() if k != name} if case == "missing" else {**w, name: w[name] - 1}
        with Handle(CLIP_C, fp32=ws) as e:
            assert e.encode() == CE_ERR_MISSING_WEIGHT, name
            msg = error()
            assert msg == f"missing weight: {name}" or msg.startswith(f"weight {name} has "), (name, msg)


@no_device
def test_fp32_complete_weights_reach_the_device_check():
    with Handle(CLIP_C, fp32=clip_fp32_weights(CLIP_C)) as e:
        assert e.encode() == CE_ERR_NO_DEVICE and "no CPU fallback" in error()
