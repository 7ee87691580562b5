"""The DiT entries' input check without a GPU (-m "not gpu").

The C library takes pointers plus (B, T, H, W, Lt) and works out every extent from the config, so a tensor that is too small
would be read (or, for forward_host's `out`, written) past its end.  `forward`, `forward_host` and `forward_fp32` refuse such
inputs with a CEError that names the argument, before any copy or launch: `forward` never reaches its native seam, and
`forward_host` raises its input error rather than the missing device's.  The call shapes bench.py uses are still accepted.

With the C library stood in for, what reaches it: forward_host hands it one timestep per sample, a context-cache slot is not
left behind unfilled when anything fails between choosing it and the C call, and a new workspace geometry drops the captured
graphs that point at the old workspace.
"""
import contextlib

import pytest
import torch

import chronoedit_b200 as ce
from chronoedit_b200 import CEError

B, T, H, W, LT = 2, 2, 8, 8, 16


def _model(image_dim=1280):
    return ce.ChronoEditTransformer3DModel(num_attention_heads=2, in_channels=36, out_channels=16, ffn_dim=256, num_layers=1,
                                           text_dim=64, image_dim=image_dim, added_kv_proj_dim=image_dim and 256)


def _inputs(dtype=torch.bfloat16):
    return dict(x=torch.zeros(B, 36, T, H, W, dtype=dtype), t=torch.full((B,), 500.0), txt=torch.zeros(B, LT, 64, dtype=dtype),
                img=torch.zeros(B, 257, 1280, dtype=dtype), out=torch.zeros(B, 16, T, H, W, dtype=torch.bfloat16))


def _meta(a):
    """The same tensor's metadata on a device that is not the CPU."""
    return torch.empty(a.shape, dtype=a.dtype, device="meta")


# (argument the error names, change to the good inputs); every entry takes these
SHAPES = {
    "hidden_states_rank": ("hidden_states", lambda i: i.update(x=i["x"][0])),
    "hidden_states_channels": ("hidden_states", lambda i: i.update(x=i["x"][:, :16])),
    "timestep_count": ("timestep", lambda i: i.update(t=torch.full((3,), 500.0))),
    "timestep_empty": ("timestep", lambda i: i.update(t=torch.zeros(0))),
    "text_rank": ("encoder_hidden_states", lambda i: i.update(txt=i["txt"][0])),
    "text_batch": ("encoder_hidden_states", lambda i: i.update(txt=i["txt"][:1])),
    "text_dim": ("encoder_hidden_states", lambda i: i.update(txt=i["txt"][..., :32])),
    "image_missing": ("encoder_hidden_states_image", lambda i: i.update(img=None)),
    "image_rank": ("encoder_hidden_states_image", lambda i: i.update(img=i["img"][0])),
    "image_batch": ("encoder_hidden_states_image", lambda i: i.update(img=i["img"][:1])),
    "image_tokens": ("encoder_hidden_states_image", lambda i: i.update(img=i["img"][:, :256])),
    "image_dim": ("encoder_hidden_states_image", lambda i: i.update(img=i["img"][..., :1024])),
}
# forward_host only: its C call copies every input and the sample itself, from and to host memory
HOST = {
    "hidden_states_dtype": ("hidden_states", lambda i: i.update(x=i["x"].float())),
    "hidden_states_strided": ("hidden_states", lambda i: i.update(x=i["x"].transpose(3, 4))),
    "hidden_states_device": ("hidden_states", lambda i: i.update(x=_meta(i["x"]))),
    "timestep_device": ("timestep", lambda i: i.update(t=_meta(i["t"]))),
    "text_dtype": ("encoder_hidden_states", lambda i: i.update(txt=i["txt"].float())),
    "text_device": ("encoder_hidden_states", lambda i: i.update(txt=_meta(i["txt"]))),
    "image_dtype": ("encoder_hidden_states_image", lambda i: i.update(img=i["img"].float())),
    "image_strided": ("encoder_hidden_states_image", lambda i: i.update(img=i["img"].transpose(1, 2).contiguous().transpose(1, 2))),
    "image_device": ("encoder_hidden_states_image", lambda i: i.update(img=_meta(i["img"]))),
    "out_shape": ("out", lambda i: i.update(out=i["out"][:1])),
    "out_dtype": ("out", lambda i: i.update(out=i["out"].float())),
    "out_strided": ("out", lambda i: i.update(out=i["out"].transpose(3, 4))),
    "out_device": ("out", lambda i: i.update(out=_meta(i["out"]))),
}


def _bad(table, case, dtype=torch.bfloat16):
    name, change = table[case]
    inp = _inputs(dtype)
    change(inp)
    return name, inp


def _forward_recorder(m):
    calls = []
    m._native_forward = lambda *a: calls.append(a)
    return calls


@pytest.mark.parametrize("case", sorted(SHAPES))
def test_forward_refuses_before_the_native_forward(case):
    name, i = _bad(SHAPES, case)
    m = _model()
    calls = _forward_recorder(m)
    with pytest.raises(CEError, match=rf"\b{name}\b"):
        m(i["x"], i["t"], i["txt"], i["img"])
    assert calls == [], "the native forward was reached"


@pytest.mark.parametrize("case", sorted(SHAPES) + sorted(HOST))
def test_forward_host_refuses_before_the_device(case):
    name, i = _bad(HOST if case in HOST else SHAPES, case)
    with pytest.raises(CEError, match=rf"\b{name}\b"):
        _model().forward_host(i["x"], i["t"], i["txt"], i["img"], out=i["out"])


@pytest.mark.parametrize("case", sorted(SHAPES))
def test_forward_fp32_refuses_before_the_device(case):
    name, i = _bad(SHAPES, case, torch.float32)
    m = _model()
    m._fp32_keepalive = {"w": torch.zeros(1)}
    with pytest.raises(CEError, match=rf"\b{name}\b"):
        m.forward_fp32(i["x"], i["t"], i["txt"], i["img"])


def test_an_image_without_image_dim_is_refused():
    i = _inputs()
    m = _model(image_dim=None)
    calls = _forward_recorder(m)
    with pytest.raises(CEError, match=r"\bencoder_hidden_states_image\b"):
        m(i["x"], i["t"], i["txt"], i["img"])
    with pytest.raises(CEError, match=r"\bencoder_hidden_states_image\b"):
        m.forward_host(i["x"], i["t"], i["txt"], i["img"])
    assert calls == []


def test_the_call_shapes_of_bench_py_are_accepted():
    """bench.py's device step passes an expanded latent view and an expanded 0-dim timestep; its host step contiguous bf16 host
    tensors (pinned there), a CPU timestep expanded to the batch and its own `out`.  A 1-element timestep serves any batch."""
    i = _inputs()
    m = _model()
    calls = _forward_recorder(m)
    t = torch.tensor(999.0)
    m(i["x"][:1].expand(B, -1, -1, -1, -1), t.expand(B), i["txt"], i["img"])
    m(i["x"], torch.tensor([999.0]), i["txt"], i["img"])
    assert len(calls) == 2 and all(c[1].shape == (B,) for c in calls)
    for ts in (t.expand(B), torch.tensor(999).expand(B), torch.tensor([999.0])):
        with pytest.raises(CEError, match="must live on a CUDA"):   # past the input check: this host has no device
            m.forward_host(i["x"], ts, i["txt"], i["img"], out=i["out"], return_device_sample=True)
    m._fp32_keepalive = {"w": torch.zeros(1)}
    f = _inputs(torch.float32)
    with pytest.raises(CEError, match="unsupported geometry"):   # past the input check: no handle on this host
        m.forward_fp32(f["x"], t.expand(B), f["txt"], f["img"])


# ---------------------------------------------------------------------------------------------------------------------
# the C library stood in for: what the entries hand it
# ---------------------------------------------------------------------------------------------------------------------
class _StubLib:
    """Records every call; size queries return 1024 bytes, everything else 0, unless `ret` says otherwise."""

    def __init__(self):
        self.calls, self.ret = [], {"ce_last_error": b"stub failure"}

    def __getattr__(self, name):
        def call(*args):
            self.calls.append((name, args))
            return self.ret.get(name, 1024 if name.endswith("_bytes") else 0)
        return call

    def args(self, name):
        return [a for n, a in self.calls if n == name]


@pytest.fixture
def stub(monkeypatch):
    from chronoedit_b200 import _lib, transformer

    lib = _StubLib()
    monkeypatch.setattr(_lib, "lib", lambda: lib)
    monkeypatch.setattr(transformer, "ptr", lambda t: t)   # the stub sees the tensors themselves
    monkeypatch.setattr(transformer, "current_stream", lambda: None)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    return lib


def _stubbed_model(cache_context=False):
    m = ce.ChronoEditTransformer3DModel(num_attention_heads=2, in_channels=36, out_channels=16, ffn_dim=256, num_layers=1,
                                        text_dim=64, image_dim=1280, added_kv_proj_dim=256, cache_context=cache_context)
    m._packed = True   # stands in for the weights pack_weights would register on a device
    return m


@pytest.mark.parametrize("t", [torch.tensor([999.0]), torch.tensor(999.0), torch.tensor(999).expand(B)], ids=["one", "0-dim", "expanded"])
def test_forward_host_hands_the_c_call_one_timestep_per_sample(stub, t):
    i = _inputs()
    _stubbed_model().forward_host(i["x"], t, i["txt"], i["img"], out=i["out"])
    (args,) = stub.args("ce_dit_forward_host_ex")
    assert torch.equal(args[2], torch.full((B,), 999.0)) and args[2].is_contiguous()


def test_a_slot_is_not_left_unfilled_when_the_call_fails_before_the_launch(stub):
    """A failed set-up between choosing a new context-cache slot and the C call (the block-capture registration of forward, the
    staging allocation of forward_host) drops the slot, so the next call with the same prompt computes the context again."""
    i = _inputs()
    m = _stubbed_model(cache_context=True)
    stub.ret["ce_dit_set_capture"] = -1
    with pytest.raises(CEError, match="stub failure"):
        m(i["x"], i["t"], i["txt"], i["img"], capture_layers=(0,))
    assert m._ctx_cache == [] and stub.args("ce_dit_forward_ex") == []
    del stub.ret["ce_dit_set_capture"]
    m(i["x"], i["t"], i["txt"], i["img"])
    m(i["x"], i["t"], i["txt"], i["img"])
    assert [a[16] for a in stub.args("ce_dit_forward_ex")] == [0, 1]   # computed into the slot, then reused
    stub.ret["ce_dit_host_staging_bytes"] = -1   # the staging allocation fails
    other = torch.zeros(B, LT, 64, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError):
        m.forward_host(i["x"], i["t"], other, i["img"], out=i["out"])
    assert [e["txt"] is i["txt"] for e in m._ctx_cache] == [True], "the unfilled slot of the failed call was kept"
    assert stub.args("ce_dit_forward_host_ex") == []


def test_a_new_workspace_geometry_drops_the_captured_graphs(stub):
    """Captured graphs hold the workspace's address: when a new geometry replaces the workspace, they are dropped with it."""
    m = _stubbed_model()
    with m._pre_launch((B, 36, T, H, W), LT) as (ws, _, _):
        pass
    m._graphs = {"k": 1}
    with m._pre_launch((B, 36, T, H, W), LT) as (same, _, _):
        pass
    assert same is ws and m._graphs == {"k": 1}
    with m._pre_launch((B, 36, T, H + 2, W), LT):
        pass
    assert m._graphs == {}
