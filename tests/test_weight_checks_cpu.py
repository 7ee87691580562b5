"""The weight checks of the VAE, the UMT5 / CLIP encoders and the fp32 validation forward without a GPU.  Every one of them looks
its weights up by name and element count before anything is launched or the device is asked for, so a handle built on fake
16-byte-aligned host pointers reaches the point where a complete set fails with "no CPU fallback" (-3; checked only where no
usable device is present), and a missing or mis-sized weight fails with -4 (-1 from ce_vae_workspace_bytes) and its name.  The
workspace sizes are pinned as well.
"""
import ctypes

import pytest
import torch

from chronoedit_b200 import _lib as L

CE_ERR_NO_DEVICE = -3
CE_ERR_MISSING_WEIGHT = -4


class Fake:
    """One aligned host address: the handles only keep pointers, and nothing here dereferences them."""

    def __init__(self):
        self._buf = torch.zeros(64, dtype=torch.uint8)
        self.ptr = ctypes.c_void_p((self._buf.data_ptr() + 15) & ~15)


FAKE = Fake()

# A complete weight set passes every check, so on a machine with a usable device the forward would launch its kernels on the fake
# host pointers.  Those tests only run where the device check fails.
no_device = pytest.mark.skipif(L.lib().ce_device_check() == 0, reason="a complete weight set would launch on fake host pointers")


def error():
    return (L.lib().ce_last_error() or b"").decode()


def names(name):
    """The message names exactly this weight (as missing, or with its registered and expected element counts)."""
    msg = error()
    return msg == f"missing weight: {name}" or msg.startswith(f"weight {name} has ")


def one_short(weights):
    """(name, weights with that one weight one element short) for every weight."""
    for name in weights:
        yield name, {**weights, name: weights[name] - 1}


def one_missing(weights):
    for name in weights:
        yield name, {k: v for k, v in weights.items() if k != name}


# ---------------------------------------------------------------------------------------------------------------------- VAE
# (dim, z_dim, dim_mult, num_res_blocks, temporal_downsample)
VAE_CONFIGS = {"tiny": (32, 16, (1, 2, 4, 4), 2, (0, 1, 1)), "wan21": (96, 16, (1, 2, 4, 4), 2, (0, 1, 1))}
SMALL_CONVS = ("encoder.conv1", "conv1", "conv2", "decoder.conv1")


def vae_weights(dim, z, mult, nres, tdown):
    """{name: packed element count} of every VAE parameter (the layout include/chronoedit_b200.h documents)."""
    w = {}

    def conv(name, cout, cin, taps):
        k = taps * cin
        w[name + ".weight"] = cout * ((k + 7) // 8 * 8 if name in SMALL_CONVS else taps * ((cin + 63) // 64 * 64))
        w[name + ".bias"] = cout

    def res(name, cin, cout):
        w[name + ".residual.0.gamma"] = cin
        conv(name + ".residual.2", cout, cin, 27)
        w[name + ".residual.3.gamma"] = cout
        conv(name + ".residual.6", cout, cout, 27)
        if cin != cout:
            conv(name + ".shortcut", cout, cin, 1)

    def attn(name, c):
        w[name + ".norm.gamma"] = c
        w[name + ".to_qkv.weight"] = 3 * c * c
        w[name + ".to_qkv.bias"] = 3 * c
        w[name + ".proj.weight"] = c * c
        w[name + ".proj.bias"] = c

    top = dim * mult[3]
    conv("encoder.conv1", dim, 3, 27)
    dims = [dim] + [dim * m for m in mult]
    idx = 0
    for i in range(4):
        cin = dims[i]
        for _ in range(nres):
            res(f"encoder.downsamples.{idx}", cin, dims[i + 1])
            cin = dims[i + 1]
            idx += 1
        if i != 3:
            c = dims[i + 1]
            conv(f"encoder.downsamples.{idx}.resample.1", c, c, 9)
            if tdown[i]:
                conv(f"encoder.downsamples.{idx}.time_conv", c, c, 3)
            idx += 1
    res("encoder.middle.0", top, top)
    attn("encoder.middle.1", top)
    res("encoder.middle.2", top, top)
    w["encoder.head.0.gamma"] = top
    conv("encoder.head.2", 2 * z, top, 27)
    conv("conv1", 2 * z, 2 * z, 1)
    conv("conv2", z, z, 1)
    conv("decoder.conv1", top, z, 27)
    res("decoder.middle.0", top, top)
    attn("decoder.middle.1", top)
    res("decoder.middle.2", top, top)
    ddims = [top] + [dim * m for m in reversed(mult)]
    idx = 0
    for i in range(4):
        cin = ddims[i] // 2 if i >= 1 else ddims[i]
        for _ in range(nres + 1):
            res(f"decoder.upsamples.{idx}", cin, ddims[i + 1])
            cin = ddims[i + 1]
            idx += 1
        if i != 3:
            c = ddims[i + 1]
            conv(f"decoder.upsamples.{idx}.resample.1", c // 2, c, 9)
            if tdown[2 - i]:
                conv(f"decoder.upsamples.{idx}.time_conv", 2 * c, c, 3)
            idx += 1
    w["decoder.head.0.gamma"] = dim
    conv("decoder.head.2", 3, dim, 27)
    return w


class Vae:
    def __init__(self, config, weights):
        dim, z, mult, nres, tdown = VAE_CONFIGS[config]
        self.lib = L.lib()
        cfg = L.VAEConfigC(dim, z, (ctypes.c_int32 * 4)(*mult), nres, (ctypes.c_int32 * 3)(*tdown))
        self.h = ctypes.c_void_p()
        L.check(self.lib.ce_vae_create(ctypes.byref(cfg), ctypes.byref(self.h)))
        for name, numel in weights.items():
            L.check(self.lib.ce_vae_set_weight(self.h, name.encode(), FAKE.ptr, numel))

    def workspace(self, decode, frames, height, width):
        return self.lib.ce_vae_workspace_bytes(self.h, decode, frames, height, width)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.lib.ce_vae_destroy(self.h)


# (decode, frames, height, width): pixel geometry for encode, latent geometry for decode
VAE_GEOMETRIES = [(0, 1, 8, 8), (0, 5, 32, 48), (0, 9, 48, 32), (0, 1, 40, 24), (0, 5, 64, 64), (0, 5, 720, 1280),
                  (1, 1, 1, 1), (1, 2, 4, 6), (1, 3, 6, 4), (1, 1, 5, 3), (1, 2, 8, 8), (1, 2, 90, 160)]
VAE_SIZES = {
    "tiny": [221184, 8479488, 8481024, 3278592, 22626560, 6329549056, 353280, 12708864, 12708864, 5254912, 33904896, 8867174656],
    "wan21": [638976, 23261952, 23263488, 9492224, 62046464, 15199027456, 1055232, 38071296, 38071296, 15730944, 101538048,
              24084633856],
}


@pytest.mark.parametrize("config", list(VAE_CONFIGS))
def test_vae_workspace_sizes(config):
    with Vae(config, vae_weights(*VAE_CONFIGS[config])) as v:
        assert [v.workspace(*g) for g in VAE_GEOMETRIES] == VAE_SIZES[config]


@pytest.mark.parametrize("case", ["missing", "short"])
def test_vae_names_each_missing_or_short_weight(case):
    weights = vae_weights(*VAE_CONFIGS["tiny"])
    for name, w in (one_missing if case == "missing" else one_short)(weights):
        for decode in (0, 1):
            with Vae("tiny", w) as v:
                got = v.workspace(decode, 5, 32, 48) if not decode else v.workspace(decode, 2, 4, 6)
                if name.startswith(("decoder.", "conv2.") if decode else ("encoder.", "conv1.")):
                    assert got == -1, (name, decode)
                    assert names(name), (name, decode, error())
                else:   # a weight only the other direction reads
                    assert got > 0, (name, decode, error())



def test_vae_abi_checks_every_weight_before_a_launch():
    """ce_vae_encode / ce_vae_decode name a missing or short weight before they ask for the device or look at the arguments (the
    workspace here is not even 256-byte aligned)."""
    weights = vae_weights(*VAE_CONFIGS["tiny"])
    p = FAKE.ptr
    for name in ("encoder.conv1.weight", "decoder.middle.1.to_qkv.weight", "decoder.head.2.bias", "conv1.weight",
                 "encoder.downsamples.2.resample.1.weight", "decoder.upsamples.3.time_conv.weight"):
        decode = not name.startswith("encoder") and name != "conv1.weight"
        for w in ({**weights, name: weights[name] - 1}, {k: v for k, v in weights.items() if k != name}):
            with Vae("tiny", w) as v:
                rc = (v.lib.ce_vae_decode(v.h, p, p, 2, 4, 6, 0, p, 1 << 40, None) if decode else
                      v.lib.ce_vae_encode(v.h, p, p, 5, 32, 48, p, 1 << 40, None))
                assert rc == CE_ERR_MISSING_WEIGHT and names(name), (name, rc, error())


@no_device
def test_vae_abi_complete_set_reaches_the_device_check():
    p = FAKE.ptr
    with Vae("tiny", vae_weights(*VAE_CONFIGS["tiny"])) as v:
        assert v.lib.ce_vae_decode(v.h, p, p, 2, 4, 6, 0, p, 1 << 40, None) == CE_ERR_NO_DEVICE
        assert v.lib.ce_vae_encode(v.h, p, p, 5, 32, 48, p, 1 << 40, None) == CE_ERR_NO_DEVICE

# ------------------------------------------------------------------------------------------------------------------ encoders
UMT5 = dict(kind=0, vocab_size=4096, d_model=512, d_kv=64, d_ff=1024, num_layers=3, num_heads=8, eps=1e-6)
CLIP = dict(kind=1, d_model=256, d_kv=64, d_ff=512, num_layers=3, num_heads=4, eps=1e-5, image_size=56, patch_size=14, hidden_act=0)


def umt5_weights(c):
    D, I, F = c["d_model"], c["num_heads"] * c["d_kv"], c["d_ff"]
    w = {"shared.weight": c["vocab_size"] * D}
    for l in range(c["num_layers"]):
        p = f"encoder.block.{l}.layer."
        w.update({p + "0.layer_norm.weight": D, p + "0.SelfAttention.qk.weight": 2 * I * D, p + "0.SelfAttention.v.weight": I * D,
                  p + "0.SelfAttention.o.weight": D * I, p + "1.layer_norm.weight": D, p + "1.DenseReluDense.wi_0.weight": F * D,
                  p + "1.DenseReluDense.wi_1.weight": F * D, p + "1.DenseReluDense.wo.weight": D * F})
    w["encoder.final_layer_norm.weight"] = D
    return w


def clip_weights(c):
    D, I, F, ps = c["d_model"], c["num_heads"] * c["d_kv"], c["d_ff"], c["patch_size"]
    L_ = 1 + (c["image_size"] // ps) ** 2
    vm = "vision_model."
    w = {vm + "embeddings.patch_embedding.weight": D * ((3 * ps * ps + 7) // 8 * 8), vm + "embeddings.class_embedding": D,
         vm + "embeddings.position_embedding.weight": L_ * D, vm + "pre_layrnorm.weight_f32": D, vm + "pre_layrnorm.bias_f32": D}
    for l in range(c["num_layers"]):
        p = f"{vm}encoder.layers.{l}."
        w.update({p + "layer_norm1.weight_f32": D, p + "layer_norm1.bias_f32": D, p + "self_attn.qk_proj.weight": 2 * I * D,
                  p + "self_attn.qk_proj.bias": 2 * I, p + "self_attn.v_proj.weight": I * D, p + "self_attn.v_proj.bias": I,
                  p + "self_attn.out_proj.weight": D * I, p + "self_attn.out_proj.bias": D, p + "layer_norm2.weight_f32": D,
                  p + "layer_norm2.bias_f32": D, p + "mlp.fc1.weight": F * D, p + "mlp.fc1.bias": F, p + "mlp.fc2.weight": D * F,
                  p + "mlp.fc2.bias": D})
    return w


class Encoder:
    def __init__(self, c, weights):
        self.lib = L.lib()
        cfg = L.EncoderConfigC(**c)
        self.c = c
        self.h = ctypes.c_void_p()
        L.check(self.lib.ce_encoder_create(ctypes.byref(cfg), ctypes.byref(self.h)))
        for name, numel in weights.items():
            L.check(self.lib.ce_encoder_set_weight(self.h, name.encode(), FAKE.ptr, numel))

    def encode(self):
        p = FAKE.ptr
        if self.c["kind"] == 0:
            valid = (ctypes.c_int32 * 2)(512, 37)
            return self.lib.ce_umt5_encode(self.h, p, valid, p, 2, 512, p, p, 1 << 40, None)
        return self.lib.ce_clip_vision_encode(self.h, p, p, 2, self.c["num_layers"] - 1, p, 1 << 40, None)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.lib.ce_encoder_destroy(self.h)


ENCODERS = {"umt5": (UMT5, umt5_weights), "clip": (CLIP, clip_weights)}
# {encoder: [ce_encoder_workspace_bytes(batch, seq_len)] over ENCODER_GEOMETRIES}
ENCODER_GEOMETRIES = [(1, 8), (2, 17), (1, 257), (2, 512), (3, 200)]
ENCODER_SIZES = {
    "umt5": [85504, 487168, 5960704, 22544896, 7654912],
    "clip": [54528, 297728, 3414528, 13005568, 4839936],
}


@pytest.mark.parametrize("enc", list(ENCODERS))
def test_encoder_workspace_sizes(enc):
    c, weights = ENCODERS[enc]
    with Encoder(c, weights(c)) as e:
        assert [e.lib.ce_encoder_workspace_bytes(e.h, *g) for g in ENCODER_GEOMETRIES] == ENCODER_SIZES[enc]


@no_device
@pytest.mark.parametrize("enc", list(ENCODERS))
def test_encoder_complete_weights_reach_the_device_check(enc):
    c, weights = ENCODERS[enc]
    with Encoder(c, weights(c)) as e:
        assert e.encode() == CE_ERR_NO_DEVICE and "no CPU fallback" in error()


@pytest.mark.parametrize("case", ["missing", "short"])
@pytest.mark.parametrize("enc", list(ENCODERS))
def test_encoder_names_each_missing_or_short_weight(enc, case):
    c, weights = ENCODERS[enc]
    for name, w in (one_missing if case == "missing" else one_short)(weights(c)):
        with Encoder(c, w) as e:
            assert e.encode() == CE_ERR_MISSING_WEIGHT, name
            assert names(name), (name, error())


# ------------------------------------------------------------------------------------------------ fp32 validation forward
def dit_config(image_dim):
    return L.DiTConfigC(2, 128, 16, 16, 64, 256, 512, 2, image_dim, 256 if image_dim else 0, 1024, 8, 1e-6, 1, 2, 2)


def fp32_weights(image_dim, layers=2):
    D, F, I = 256, 512, image_dim
    w = {}

    def lin(m, n, k):
        w[m + ".weight"] = n * k
        w[m + ".bias"] = n

    ce = "condition_embedder."
    lin("patch_embedding", D, 16 * 4)
    lin(ce + "time_embedder.linear_1", D, 256)
    lin(ce + "time_embedder.linear_2", D, D)
    lin(ce + "time_proj", 6 * D, D)
    lin(ce + "text_embedder.linear_1", D, 64)
    lin(ce + "text_embedder.linear_2", D, D)
    if I:
        w[ce + "image_embedder.norm1.weight"] = w[ce + "image_embedder.norm1.bias"] = I
        lin(ce + "image_embedder.ff.net.0.proj", I, I)
        lin(ce + "image_embedder.ff.net.2", D, I)
        w[ce + "image_embedder.norm2.weight"] = w[ce + "image_embedder.norm2.bias"] = D
    for i in range(layers):
        p = f"blocks.{i}."
        w[p + "scale_shift_table"] = 6 * D
        for m in ("attn1.to_q", "attn1.to_k", "attn1.to_v", "attn1.to_out.0", "attn2.to_q", "attn2.to_k", "attn2.to_v", "attn2.to_out.0"):
            lin(p + m, D, D)
        for m in ("attn1.norm_q", "attn1.norm_k", "attn2.norm_q", "attn2.norm_k", "norm2"):
            w[p + m + ".weight"] = D
        w[p + "norm2.bias"] = D
        if I:
            lin(p + "attn2.add_k_proj", D, D)
            lin(p + "attn2.add_v_proj", D, D)
            w[p + "attn2.norm_added_k.weight"] = D
        lin(p + "ffn.net.0.proj", F, D)
        lin(p + "ffn.net.2", D, F)
    w["scale_shift_table"] = 2 * D
    lin("proj_out", 16 * 4, D)
    return w


def forward_fp32(image_dim, weights):
    lib = L.lib()
    cfg = dit_config(image_dim)
    h = ctypes.c_void_p()
    L.check(lib.ce_dit_create(ctypes.byref(cfg), ctypes.byref(h)))
    try:
        for name, numel in weights.items():
            L.check(lib.ce_dit_set_weight_fp32(h, name.encode(), FAKE.ptr, numel))
        p = FAKE.ptr
        return lib.ce_dit_forward_fp32(h, p, p, p, p if image_dim else None, p, 1, 2, 8, 8, 16, p, 1 << 40, None, None)
    finally:
        lib.ce_dit_destroy(h)


@no_device
@pytest.mark.parametrize("image_dim", [0, 128], ids=["no_image", "image"])
def test_fp32_complete_weights_reach_the_device_check(image_dim):
    assert forward_fp32(image_dim, fp32_weights(image_dim)) == CE_ERR_NO_DEVICE and "no CPU fallback" in error()


@pytest.mark.parametrize("case", ["missing", "short"])
@pytest.mark.parametrize("image_dim", [0, 128], ids=["no_image", "image"])
def test_fp32_names_each_missing_or_short_weight(image_dim, case):
    for name, w in (one_missing if case == "missing" else one_short)(fp32_weights(image_dim)):
        assert forward_fp32(image_dim, w) == CE_ERR_MISSING_WEIGHT, name
        assert names(name), (name, error())
