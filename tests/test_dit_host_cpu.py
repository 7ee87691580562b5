"""The DiT handle's host-side rules without a GPU: ce_dit_create, ce_dit_set_weight, ce_dit_weights_complete and the size
queries never touch the device, so they run here on fake 16-byte-aligned host pointers.

- which weights a configuration needs, with which dtype and element count, and the error that names the first one missing or
  wrong (including an FP8 handle with one block GEMM left in bf16);
- the workspace, context-cache and host-staging sizes, pinned to known values, and the staging layout (inputs, then the sample).
"""
import ctypes

import pytest
import torch

from chronoedit_b200 import _lib as L

BLOCK_GEMMS = ("attn1.to_qkv", "attn1.to_out.0", "attn2.to_q", "attn2.to_out.0", "ffn.net.0.proj", "ffn.net.2")
CE_ERR_MISSING_WEIGHT = -4

# (heads, ffn_dim, num_layers, image_dim); text_dim 4096, 36 -> 16 channels, freq_dim 256
CONFIGS = {
    "h2": (2, 1024, 2, 1280),
    "h3": (3, 640, 2, 1280),
    "h40": (40, 13824, 1, 1280),
    "h2_noimg": (2, 1024, 1, 0),
    "h3_noimg": (3, 640, 2, 0),
}
# (batch, frames, height, width, text_len) of the latent
GEOMETRIES = [(1, 2, 16, 24, 512), (2, 2, 90, 160, 512), (1, 8, 18, 26, 7)]


def _cfg(heads, ffn, layers, image_dim):
    return L.DiTConfigC(heads, 128, 36, 16, 4096, 256, ffn, layers, image_dim, heads * 128 if image_dim else 0, 1024, 8, 1e-6,
                        1, 2, 2)


def required(heads, ffn, layers, image_dim, fp8=False):
    """{name: (dtype, numel)} of every weight the forward reads: 0 bf16, 1 fp32, 2 e4m3 (include/chronoedit_b200.h)."""
    D, F, I, Kp, No = heads * 128, ffn, image_dim, 36 * 4, 16 * 4
    w = {}

    def linear(m, n, k, e4m3=False):
        w[m + ".weight"] = (2 if e4m3 else 0, n * k)
        if e4m3:
            w[m + ".weight_scale"] = (1, n)
        w[m + ".bias"] = (0, n)

    linear("patch_embedding", D, Kp)
    ce = "condition_embedder."
    w[ce + "time_embedder.linear_1.weight"] = (1, D * 256)
    w[ce + "time_embedder.linear_1.bias"] = (1, D)
    w[ce + "time_embedder.linear_2.weight"] = (1, D * D)
    w[ce + "time_embedder.linear_2.bias"] = (1, D)
    w[ce + "time_proj.weight"] = (0, 6 * D * D)
    w[ce + "time_proj.bias"] = (0, 6 * D)
    linear(ce + "text_embedder.linear_1", D, 4096)
    linear(ce + "text_embedder.linear_2", D, D)
    if I:
        w[ce + "image_embedder.norm1.weight"] = (1, I)
        w[ce + "image_embedder.norm1.bias"] = (1, I)
        linear(ce + "image_embedder.ff.net.0.proj", I, I)
        linear(ce + "image_embedder.ff.net.2", D, I)
        w[ce + "image_embedder.norm2.weight"] = (1, D)
        w[ce + "image_embedder.norm2.bias"] = (1, D)
    w["blocks.scale_shift_table"] = (1, layers * 6 * D)
    shapes = {"attn1.to_qkv": (3 * D, D), "attn1.to_out.0": (D, D), "attn2.to_q": (D, D), "attn2.to_out.0": (D, D),
              "ffn.net.0.proj": (F, D), "ffn.net.2": (D, F)}
    for i in range(layers):
        p = f"blocks.{i}."
        for m, (n, k) in shapes.items():
            linear(p + m, n, k, fp8)
        for m in ("attn1.norm_q", "attn1.norm_k", "attn2.norm_q", "attn2.norm_k"):
            w[p + m + ".weight"] = (0, D)
        w[p + "norm2.weight"] = (1, D)
        w[p + "norm2.bias"] = (1, D)
        linear(p + "attn2.to_kv", 2 * D, D)
        if I:
            linear(p + "attn2.add_kv_proj", 2 * D, D)
            w[p + "attn2.norm_added_k.weight"] = (0, D)
    w["scale_shift_table"] = (1, 2 * D)
    linear("proj_out", No, D)
    return w


class Handle:
    def __init__(self, config):
        self.lib = L.lib()
        self.cfg = _cfg(*config)
        self.h = ctypes.c_void_p()
        L.check(self.lib.ce_dit_create(ctypes.byref(self.cfg), ctypes.byref(self.h)))
        self._buf = torch.zeros(64, dtype=torch.uint8)   # the handle only keeps pointers: one aligned address serves all
        self.ptr = ctypes.c_void_p((self._buf.data_ptr() + 15) & ~15)

    def register(self, weights):
        for name, (dtype, numel) in weights.items():
            L.check(self.lib.ce_dit_set_weight(self.h, name.encode(), self.ptr, dtype, numel))
        return self

    def complete(self):
        rc = self.lib.ce_dit_weights_complete(self.h)
        return rc, (self.lib.ce_last_error() or b"").decode() if rc else ""

    def close(self):
        self.lib.ce_dit_destroy(self.h)


@pytest.fixture
def handle():
    made = []

    def make(config):
        made.append(Handle(config))
        return made[-1]

    yield make
    for h in made:
        h.close()


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_complete_weight_sets_are_accepted(handle, config, fp8):
    h = handle(CONFIGS[config]).register(required(*CONFIGS[config], fp8=fp8))
    assert h.complete() == (0, "")


@pytest.mark.parametrize("name", ["patch_embedding.weight", "condition_embedder.time_embedder.linear_1.bias",
                                  "condition_embedder.image_embedder.norm2.bias", "blocks.scale_shift_table",
                                  "blocks.1.attn2.add_kv_proj.bias", "blocks.1.attn2.norm_added_k.weight", "scale_shift_table",
                                  "proj_out.bias"])
def test_missing_weight_is_named(handle, name):
    w = required(*CONFIGS["h2"])
    del w[name]
    rc, msg = handle(CONFIGS["h2"]).register(w).complete()
    assert rc == CE_ERR_MISSING_WEIGHT and msg == f"missing weight: {name}"


@pytest.mark.parametrize("name", ["blocks.1.ffn.net.0.proj.weight_scale", "blocks.0.attn1.to_qkv.bias"])
def test_missing_fp8_weight_is_named(handle, name):
    w = required(*CONFIGS["h3"], fp8=True)
    del w[name]
    rc, msg = handle(CONFIGS["h3"]).register(w).complete()
    assert rc == CE_ERR_MISSING_WEIGHT and msg == f"missing weight: {name}"


@pytest.mark.parametrize("name,dtype", [("condition_embedder.time_embedder.linear_2.weight", 0), ("blocks.1.norm2.bias", 0),
                                        ("blocks.0.attn2.to_kv.weight", 1), ("proj_out.weight", 2)])
def test_wrong_dtype_is_named(handle, name, dtype):
    w = required(*CONFIGS["h2"])
    w[name] = (dtype, w[name][1])
    rc, msg = handle(CONFIGS["h2"]).register(w).complete()
    assert rc == CE_ERR_MISSING_WEIGHT and msg.startswith(f"weight {name} has dtype {dtype}, expected ")


@pytest.mark.parametrize("name", ["patch_embedding.weight", "condition_embedder.text_embedder.linear_1.weight",
                                  "blocks.1.attn2.to_out.0.weight", "blocks.0.ffn.net.2.bias", "blocks.scale_shift_table"])
def test_wrong_element_count_is_named(handle, name):
    w = required(*CONFIGS["h2"])
    dtype, numel = w[name]
    w[name] = (dtype, numel + 8)
    rc, msg = handle(CONFIGS["h2"]).register(w).complete()
    assert rc == CE_ERR_MISSING_WEIGHT and msg == f"weight {name} has {numel + 8} elements, expected {numel}"


@pytest.mark.parametrize("layer", [0, 1])
@pytest.mark.parametrize("gemm", BLOCK_GEMMS)
def test_fp8_handle_with_one_bf16_block_gemm_is_named(handle, gemm, layer):
    w = required(*CONFIGS["h3"], fp8=True)
    name = f"blocks.{layer}.{gemm}.weight"
    w[name] = (0, w[name][1])
    del w[f"blocks.{layer}.{gemm}.weight_scale"]
    rc, msg = handle(CONFIGS["h3"]).register(w).complete()
    assert rc == CE_ERR_MISSING_WEIGHT
    if (gemm, layer) == ("attn1.to_qkv", 0):   # layer 0's QKV weight sets the mode: the next e4m3 weight is the odd one out
        assert msg.startswith("weight blocks.0.attn1.to_out.0.weight has dtype 2, expected 0")
    else:
        assert msg.startswith(f"weight {name} has dtype 0, expected 2")
    assert msg.endswith("the six block GEMM weights of every layer are either all bf16 or all e4m3)")


# {config: [(workspace bf16, workspace fp8, context cache, staging, staging sample offset) per GEOMETRIES entry]}
SIZES = {
    "h2": [(3982336, 4179712, 1574912, 4932352, 4907776), (86117888, 100921088, 3149824, 15695104, 13851904),
           (7097088, 8059392, 540672, 1104896, 985088)],
    "h3": [(4934912, 5058560, 2362368, 4932352, 4907776), (99347968, 108621568, 4724736, 15695104, 13851904),
           (8133632, 8736512, 811008, 1104896, 985088)],
    "h40": [(50429952, 53084928, 15749120, 4932352, 4907776), (1366560768, 1565683968, 31498240, 15695104, 13851904),
            (96931328, 109874432, 5406720, 1104896, 985088)],
    "h2_noimg": [(2669056, 2866432, 524288, 4274688, 4250112), (83490816, 98294016, 1048576, 14379520, 12536320),
                 (5783808, 6746112, 7168, 447232, 327424)],
    "h3_noimg": [(3627776, 3751424, 1572864, 4274688, 4250112), (96733184, 106006784, 3145728, 14379520, 12536320),
                 (6826496, 7429376, 21504, 447232, 327424)],
}


def sizes(handle, config, geometry):
    out = []
    for fp8 in (False, True):
        h = handle(CONFIGS[config]).register(required(*CONFIGS[config], fp8=fp8))
        out.append(h.lib.ce_dit_workspace_bytes(h.h, *geometry))
    B, T, Hh, Ww, Lt = geometry
    out.append(h.lib.ce_dit_context_cache_bytes(h.h, B, Lt))
    out.append(h.lib.ce_dit_host_staging_bytes(h.h, *geometry))
    out.append(h.lib.ce_dit_host_staging_sample_offset(h.h, *geometry))
    return tuple(out)


@pytest.mark.parametrize("geo", range(len(GEOMETRIES)))
@pytest.mark.parametrize("config", list(CONFIGS))
def test_size_queries(handle, config, geo):
    geometry = GEOMETRIES[geo]
    got = sizes(handle, config, geometry)
    assert got == SIZES[config][geo]
    # the sample is the staging buffer's last slice: [B, 16, frames, height, width] bf16, rounded up to 256 bytes
    B, T, Hh, Ww, _ = geometry
    sample_bytes = (B * 16 * T * Hh * Ww * 2 + 255) // 256 * 256
    assert got[3] == got[4] + sample_bytes


def test_size_queries_reject_bad_geometry(handle):
    h = handle(CONFIGS["h2"]).register(required(*CONFIGS["h2"]))
    assert h.lib.ce_dit_workspace_bytes(h.h, 1, 3, 16, 24, 512) == -1    # frames must be 2 or rope_temporal_skip_len
    assert h.lib.ce_dit_workspace_bytes(h.h, 1, 2, 15, 24, 512) == -1    # odd latent height
    assert h.lib.ce_dit_workspace_bytes(h.h, 9, 2, 16, 24, 512) == -1    # batch 1..8
    assert h.lib.ce_dit_context_cache_bytes(h.h, 0, 512) == -1


def test_context_cache_slots_follow_any_prompt_order():
    """The context cache's two LRU slots (prompt and negative prompt) under any order of calls, not only strict alternation: a hit on
    the older slot must move it to the back without comparing the entries' tensors, and a third prompt evicts the least recently used
    slot and reuses its buffer."""
    import chronoedit_b200 as ce

    m = ce.ChronoEditTransformer3DModel(num_attention_heads=2, in_channels=36, ffn_dim=256, num_layers=1, image_dim=1280,
                                        added_kv_proj_dim=256, text_dim=64, cache_context=True)
    m._ensure_handle()
    prompt, negative, other = (torch.randn(1, 8, 64) for _ in range(3))
    img = torch.randn(1, 257, 1280)
    slot = lambda txt: m._context_slot(txt, img, txt, img)
    p_buf, reuse = slot(prompt)
    assert reuse == 0
    n_buf, reuse = slot(negative)
    assert reuse == 0 and n_buf is not p_buf
    for txt, buf in ((prompt, p_buf), (prompt, p_buf), (negative, n_buf), (negative, n_buf), (prompt, p_buf), (negative, n_buf)):
        got, reuse = slot(txt)
        assert reuse == 1 and got is buf
    assert [e["txt"] is negative for e in m._ctx_cache] == [False, True]
    got, reuse = slot(other)   # evicts the prompt, the least recently used
    assert reuse == 0 and got is p_buf
    assert slot(negative) == (n_buf, 1)
    prompt.add_(1)   # an in-place update invalidates the entry
    assert slot(other)[1] == 1 and slot(prompt)[1] == 0


def test_failed_forward_does_not_leave_a_half_filled_context_slot():
    """A forward that was to fill a context-cache slot and failed may have stopped before the K/V of later layers: its slot is dropped,
    so the next call with the same prompt computes the context again.  A failed call that only read the slot keeps it."""
    import chronoedit_b200 as ce

    m = ce.ChronoEditTransformer3DModel(num_attention_heads=2, in_channels=36, ffn_dim=256, num_layers=1, image_dim=1280,
                                        added_kv_proj_dim=256, text_dim=64, cache_context=True)
    m._ensure_handle()
    prompt, negative = torch.randn(1, 8, 64), torch.randn(1, 8, 64)
    img = torch.randn(1, 257, 1280)
    p_buf, _ = m._context_slot(prompt, img, prompt, img)
    m._check_forward(0, p_buf, 0)
    n_buf, reuse = m._context_slot(negative, img, negative, img)
    assert reuse == 0
    with pytest.raises(ce.CEError):
        m._check_forward(-1, n_buf, 0)
    assert [e["buf"] for e in m._ctx_cache] == [p_buf]
    assert m._context_slot(negative, img, negative, img)[1] == 0
    buf, reuse = m._context_slot(prompt, img, prompt, img)
    assert (buf, reuse) == (p_buf, 1)
    with pytest.raises(ce.CEError):
        m._check_forward(-1, buf, 1)
    assert m._context_slot(prompt, img, prompt, img) == (p_buf, 1)
