"""H100-native drop-in for diffusers `AutoencoderKLWan` as `ChronoEditPipeline` uses it.

What the unchanged pipeline touches (pipeline_chronoedit.py:119-129, 185-186, 427-445, 672, 765-781), plus the memory switches
scripts call on it (enable_tiling / disable_tiling / enable_slicing / disable_slicing):
    vae.encode(x).latent_dist.mode() / .sample(generator)      x  [B,3,T,H,W] in [-1,1]
    vae.decode(z, return_dict=False)[0]                         z  [B,16,Tl,h,w]
    vae.config.z_dim / .latents_mean / .latents_std, vae.temperal_downsample, vae.dtype
diffusers' class is un-vendored; the arithmetic follows the in-tree twin
/root/reference/chronoedit/_src/tokenizers/wan2pt1.py (WanVAE_, :467-581) with the diffusers deltas of SURVEY.md
section 8c: no latent mean/std inside encode/decode, decode clamps to [-1,1].  Parameter names are the twin's
(`encoder.downsamples.0.residual.2.weight`, ...); `diffusers_key_map()` gives the best-effort rename from a diffusers
checkpoint.  All arithmetic runs in libchronoedit_b200.so (wgmma implicit-GEMM convolutions etc.); no PyTorch fallback.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from . import _lib
from ._lib import CEError, VAEConfigC, check, current_stream, ptr

# latent statistics (values: wan2pt1.py:697-732); the pipeline reads them from vae.config
LATENTS_MEAN = [-0.7571, -0.7089, -0.9113, 0.1075, -0.1745, 0.9653, -0.1517, 1.5508,
                0.4134, -0.0715, 0.5517, -0.3632, -0.1922, -0.9497, 0.2503, -0.2921]
LATENTS_STD = [2.8184, 1.4541, 2.3275, 2.6558, 1.2196, 1.7708, 2.6052, 2.0743,
               3.2687, 2.1526, 2.8652, 1.5579, 1.6382, 1.1253, 2.8251, 1.9160]

# diffusers' tiled_decode returns the blended tiles without the [-1, 1] clamp its untiled decode applies ([diffusers-mem],
# DESIGN.md "Tiled VAE"); flip this to clamp the tiled output as well
TILED_DECODE_CLAMPS = False

# convolutions that run as im2row + GEMM (Cin < 64); every other convolution is the implicit-GEMM kernel
SMALL_CONVS = ("encoder.conv1", "decoder.conv1", "conv1", "conv2")


class _Config(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e


class DiagonalGaussianDistribution:
    """Posterior returned by encode(): same surface as diffusers' (mode / sample / mean / logvar)."""

    def __init__(self, moments: torch.Tensor):
        self.mean, self.logvar = moments.chunk(2, dim=1)
        self.logvar = self.logvar.clamp(-30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)

    def mode(self) -> torch.Tensor:
        return self.mean

    def sample(self, generator: Optional[torch.Generator] = None) -> torch.Tensor:
        noise = torch.randn(self.mean.shape, generator=generator, device=self.mean.device, dtype=self.mean.dtype)
        return self.mean + self.std * noise


@dataclass
class AutoencoderKLOutput:
    latent_dist: DiagonalGaussianDistribution


@dataclass
class DecoderOutput:
    sample: torch.Tensor


def _param_shapes(dim, z_dim, dim_mult, num_res_blocks, temporal_downsample) -> Dict[str, Tuple[int, ...]]:
    """Every parameter of WanVAE_ (wan2pt1.py:262-500), name -> shape."""
    s: Dict[str, Tuple[int, ...]] = {}

    def conv3(name, cout, cin, k):
        s[name + ".weight"] = (cout, cin) + tuple(k)
        s[name + ".bias"] = (cout,)

    def res(name, cin, cout):
        s[name + ".residual.0.gamma"] = (cin, 1, 1, 1)
        conv3(name + ".residual.2", cout, cin, (3, 3, 3))
        s[name + ".residual.3.gamma"] = (cout, 1, 1, 1)
        conv3(name + ".residual.6", cout, cout, (3, 3, 3))
        if cin != cout:
            conv3(name + ".shortcut", cout, cin, (1, 1, 1))

    def attn(name, c):
        s[name + ".norm.gamma"] = (c, 1, 1)
        s[name + ".to_qkv.weight"] = (3 * c, c, 1, 1)
        s[name + ".to_qkv.bias"] = (3 * c,)
        s[name + ".proj.weight"] = (c, c, 1, 1)
        s[name + ".proj.bias"] = (c,)

    def resample(name, c, mode):
        cout = c // 2 if mode.startswith("up") else c
        s[name + ".resample.1.weight"] = (cout, c, 3, 3)
        s[name + ".resample.1.bias"] = (cout,)
        if mode == "upsample3d":
            conv3(name + ".time_conv", 2 * c, c, (3, 1, 1))
        if mode == "downsample3d":
            conv3(name + ".time_conv", c, c, (3, 1, 1))

    top = dim * dim_mult[-1]
    conv3("encoder.conv1", dim, 3, (3, 3, 3))
    dims = [dim * u for u in (1,) + tuple(dim_mult)]
    idx = 0
    for i, (cin, cout) in enumerate(zip(dims[:-1], dims[1:])):
        for _ in range(num_res_blocks):
            res(f"encoder.downsamples.{idx}", cin, cout)
            idx += 1
            cin = cout
        if i != len(dim_mult) - 1:
            resample(f"encoder.downsamples.{idx}", cout, "downsample3d" if temporal_downsample[i] else "downsample2d")
            idx += 1
    res("encoder.middle.0", top, top)
    attn("encoder.middle.1", top)
    res("encoder.middle.2", top, top)
    s["encoder.head.0.gamma"] = (top, 1, 1, 1)
    conv3("encoder.head.2", 2 * z_dim, top, (3, 3, 3))
    conv3("conv1", 2 * z_dim, 2 * z_dim, (1, 1, 1))
    conv3("conv2", z_dim, z_dim, (1, 1, 1))
    conv3("decoder.conv1", top, z_dim, (3, 3, 3))
    res("decoder.middle.0", top, top)
    attn("decoder.middle.1", top)
    res("decoder.middle.2", top, top)
    ddims = [dim * u for u in (dim_mult[-1],) + tuple(dim_mult[::-1])]
    up = tuple(temporal_downsample[::-1])
    idx = 0
    for i, (cin, cout) in enumerate(zip(ddims[:-1], ddims[1:])):
        if i in (1, 2, 3):
            cin = cin // 2
        for _ in range(num_res_blocks + 1):
            res(f"decoder.upsamples.{idx}", cin, cout)
            idx += 1
            cin = cout
        if i != len(dim_mult) - 1:
            resample(f"decoder.upsamples.{idx}", cout, "upsample3d" if up[i] else "upsample2d")
            idx += 1
    s["decoder.head.0.gamma"] = (dim, 1, 1, 1)
    conv3("decoder.head.2", 3, dim, (3, 3, 3))
    return s


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def pack_parameter(name: str, w: torch.Tensor) -> torch.Tensor:
    """Reference layout -> the layout ce_vae_set_weight documents (include/chronoedit_b200.h)."""
    w = w.detach().to(torch.bfloat16)
    if name.endswith(".gamma") or name.endswith(".bias"):
        return w.reshape(-1).contiguous()
    base = name[: -len(".weight")]
    if base.endswith("to_qkv") or base.endswith(".proj"):
        return w.reshape(w.shape[0], w.shape[1]).contiguous()
    if w.dim() == 4:
        w = w[:, :, None]
    cout, cin, kt, kh, kw = w.shape
    w = w.permute(0, 2, 3, 4, 1).reshape(cout, kt * kh * kw, cin)
    if base in SMALL_CONVS:
        k = kt * kh * kw * cin
        out = torch.zeros(cout, _round_up(k, 8), dtype=torch.bfloat16, device=w.device)
        out[:, :k] = w.reshape(cout, k)
        return out
    out = torch.zeros(cout, kt * kh * kw, _round_up(cin, 64), dtype=torch.bfloat16, device=w.device)
    out[:, :, :cin] = w
    return out.reshape(cout, -1).contiguous()


def pack_parameter_fp32(name: str, w: torch.Tensor) -> torch.Tensor:
    """Reference layout -> the layout ce_vae_set_weight_fp32 documents: convolution weights (every one, the small ones included) as
    [Cout, taps, Cin_pad / 64, 3, 64] bf16 with W_hi | W_hi | W_lo per 64-channel block, the split the fp32 convolution multiplies
    with its input's hi / lo pair; everything else fp32 as it is."""
    w = w.detach().to(torch.float32)
    base = name[: -len(".weight")] if name.endswith(".weight") else None
    if base is None or base.endswith("to_qkv") or base.endswith(".proj"):
        return w.reshape(w.shape[0], -1).contiguous() if base else w.reshape(-1).contiguous()
    if w.dim() == 4:
        w = w[:, :, None]
    cout, cin, kt, kh, kw = w.shape
    cp = _round_up(cin, 64)
    full = torch.zeros(cout, kt * kh * kw, cp, dtype=torch.float32, device=w.device)
    full[:, :, :cin] = w.permute(0, 2, 3, 4, 1).reshape(cout, kt * kh * kw, cin)
    full = full.reshape(cout, kt * kh * kw, cp // 64, 64)
    hi = full.to(torch.bfloat16)
    lo = (full - hi.float()).to(torch.bfloat16)
    return torch.stack((hi, hi, lo), dim=3).reshape(cout, -1).contiguous()


class AutoencoderKLWan(nn.Module):
    """See module docstring.  Defaults = Wan2.1 VAE (wan2pt1.py:597-605)."""

    def __init__(self, base_dim: int = 96, z_dim: int = 16, dim_mult: Tuple[int, ...] = (1, 2, 4, 4), num_res_blocks: int = 2,
                 attn_scales: Tuple[float, ...] = (), temperal_downsample: Tuple[bool, ...] = (False, True, True),
                 dropout: float = 0.0, latents_mean: Optional[List[float]] = None, latents_std: Optional[List[float]] = None,
                 *, torch_dtype: torch.dtype = torch.bfloat16, device=None, clamp_output: bool = True):
        super().__init__()
        if torch_dtype not in (torch.bfloat16, torch.float32):
            raise CEError("chronoedit_b200 VAE computes in bf16 (run_inference_diffusers.py:341-345 loads it in bf16) or in fp32 "
                          f"(the reference pipeline's example loads it in fp32), not {torch_dtype}")
        if len(dim_mult) != 4 or len(temperal_downsample) != 3 or len(attn_scales) != 0:
            raise CEError("only the Wan2.1 layout (4 stages, no extra attention scales) is built")
        self.config = _Config(base_dim=base_dim, z_dim=z_dim, dim_mult=list(dim_mult), num_res_blocks=num_res_blocks,
                              attn_scales=list(attn_scales), temperal_downsample=list(temperal_downsample), dropout=dropout,
                              latents_mean=list(latents_mean or LATENTS_MEAN), latents_std=list(latents_std or LATENTS_STD))
        self.temperal_downsample = list(temperal_downsample)
        self._dtype = torch_dtype   # what encode / decode compute in, whatever .to() later does to the parameters
        self.z_dim = z_dim
        self.clamp_output = clamp_output
        self._shapes = _param_shapes(base_dim, z_dim, tuple(dim_mult), num_res_blocks, tuple(temperal_downsample))
        for name, shape in self._shapes.items():
            self._register(name, nn.Parameter(torch.empty(shape, dtype=torch_dtype, device=device), requires_grad=False))
        self._handle = None
        self._packed: Dict[str, torch.Tensor] = {}
        self._is_packed = False
        self._ws: Optional[torch.Tensor] = None
        self._sp_state: Optional[Dict] = None   # the split over ranks (parallel.enable_vae_sequence_parallel)
        # diffusers' memory switches (enable_tiling / enable_slicing), with its defaults; sizes in pixels
        self.use_slicing = False
        self.use_tiling = False
        self.tile_sample_min_height = 256
        self.tile_sample_min_width = 256
        self.tile_sample_stride_height = 192
        self.tile_sample_stride_width = 192

    def _register(self, dotted: str, p: nn.Parameter) -> None:
        mod = self
        parts = dotted.split(".")
        for part in parts[:-1]:
            if not hasattr(mod, part):
                mod.add_module(part, nn.Module())
            mod = getattr(mod, part)
        mod.register_parameter(parts[-1], p)

    @property
    def dtype(self) -> torch.dtype:
        """torch.bfloat16, or torch.float32 for a VAE built or loaded with torch_dtype=torch.float32 (fp32 encode / decode)."""
        return self._dtype

    @property
    def device(self) -> torch.device:
        return next(self.parameters()).device

    def _apply(self, fn, *a, **k):
        self._is_packed = False
        return super()._apply(fn, *a, **k)

    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                _lib.lib().ce_vae_destroy(self._handle)
        except Exception:
            pass

    def _ensure_handle(self):
        """The C handle (configuration only; pack_weights hands it the weights)."""
        if self._handle is None:
            c = self.config
            cfg = VAEConfigC(c.base_dim, c.z_dim, (_lib.c_int32 * 4)(*c.dim_mult), c.num_res_blocks,
                             (_lib.c_int32 * 3)(*[int(b) for b in c.temperal_downsample]))
            h = _lib.c_void_p()
            check(_lib.lib().ce_vae_create(_lib.ctypes.byref(cfg), _lib.ctypes.byref(h)))
            self._handle = h
        return self._handle

    @torch.no_grad()
    def pack_weights(self) -> None:
        L = _lib.lib()
        if self.device.type != "cuda":
            raise CEError("AutoencoderKLWan must live on a CUDA (sm_90) device; there is no CPU path")
        self._ensure_handle()
        packed = {}
        fp32 = self.dtype == torch.float32
        for name, p in self.named_parameters():
            t = (pack_parameter_fp32 if fp32 else pack_parameter)(name, p.data)
            packed[name] = t
            check((L.ce_vae_set_weight_fp32 if fp32 else L.ce_vae_set_weight)(self._handle, name.encode(), ptr(t), t.numel()))
        self._packed = packed
        self._is_packed = True

    def _workspace(self, nbytes: int) -> torch.Tensor:
        if self._ws is None or self._ws.numel() < nbytes or self._ws.device != self.device:
            self._ws = None
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        return self._ws

    # ------------------------------------------------------------------------------------------ memory switches
    def enable_tiling(self, tile_sample_min_height: Optional[int] = None, tile_sample_min_width: Optional[int] = None,
                      tile_sample_stride_height: Optional[int] = None, tile_sample_stride_width: Optional[int] = None) -> None:
        """Encode and decode frames larger than one tile tile by tile (diffusers' `enable_tiling`): the VAE's memory is then bounded by
        the tile size, whatever the frame size.  Sizes not given keep their current values.  Sizes and strides must be multiples of 8
        pixels with stride <= size (the C library refuses anything else at the first tiled call)."""
        self.use_tiling = True
        self.tile_sample_min_height = tile_sample_min_height or self.tile_sample_min_height
        self.tile_sample_min_width = tile_sample_min_width or self.tile_sample_min_width
        self.tile_sample_stride_height = tile_sample_stride_height or self.tile_sample_stride_height
        self.tile_sample_stride_width = tile_sample_stride_width or self.tile_sample_stride_width

    def disable_tiling(self) -> None:
        self.use_tiling = False

    def enable_slicing(self) -> None:
        """diffusers' `enable_slicing`: encode and decode a batch one sample at a time.  The samples of a batch already run one after
        another here, so this only records the switch."""
        self.use_slicing = True

    def disable_slicing(self) -> None:
        self.use_slicing = False

    def _tiles(self) -> Tuple[int, int, int, int]:
        return (self.tile_sample_min_height, self.tile_sample_min_width, self.tile_sample_stride_height, self.tile_sample_stride_width)

    def _tiled_encode(self, H: int, W: int) -> bool:   # diffusers' AutoencoderKLWan._encode
        return self.use_tiling and (W > self.tile_sample_min_width or H > self.tile_sample_min_height)

    def _tiled_decode(self, h: int, w: int) -> bool:   # diffusers' AutoencoderKLWan._decode, in latents
        return self.use_tiling and (w > self.tile_sample_min_width // 8 or h > self.tile_sample_min_height // 8)

    # ------------------------------------------------------------------------------------------ encode / decode
    # An fp32 VAE computes in fp32 and returns fp32.  It widens a bf16 x or z to fp32 (exact), so the unchanged pipeline's
    # prepare_latents, which casts the conditioning video to the transformer's bf16 before vae.encode, runs; diffusers' fp32 Conv3d
    # would reject that input instead.
    def _check_fp32_single_gpu(self) -> None:
        if self.dtype == torch.float32 and self._sp_state:
            raise CEError("the fp32 VAE does not run split over GPUs (parallel.enable_vae_sequence_parallel is built for bf16 only)")

    @torch.no_grad()
    def encode(self, x: torch.Tensor, return_dict: bool = True):
        """x [B,3,T,H,W] in [-1,1], T = 1+4k, H and W multiples of 8 -> posterior (mean|logvar [B,2z,1+k,H/8,W/8]), in the VAE's
        dtype.  With tiling on and a frame larger than one tile, tiled as diffusers' tiled_encode."""
        if x.dim() != 5 or x.shape[1] != 3:
            raise CEError("encode expects [B, 3, T, H, W]")
        B, _, T, H, W = x.shape
        if T < 1 or (T - 1) % 4 != 0 or H % 8 != 0 or W % 8 != 0:
            raise CEError("encode expects T = 1 + 4k frames and H, W multiples of 8")
        self._check_fp32_single_gpu()
        tiled = self._tiled_encode(H, W)
        if tiled:
            self._check_tiling_single_gpu()
        x = x.to(device=self.device, dtype=self.dtype).contiguous()
        out = torch.empty(B, 2 * self.z_dim, 1 + (T - 1) // 4, H // 8, W // 8, dtype=self.dtype, device=self.device)
        if tiled:
            self._native_tiled(x, out, decode=False)
        else:
            self._native_encode(x, out)
        post = DiagonalGaussianDistribution(out)
        if not return_dict:
            return (post,)
        return AutoencoderKLOutput(latent_dist=post)

    @torch.no_grad()
    def decode(self, z: torch.Tensor, return_dict: bool = True):
        """z [B,z_dim,Tl,h,w] -> video [B,3,1+4(Tl-1),8h,8w] (clamped to [-1,1] like diffusers), in the VAE's dtype.  With tiling
        on and a latent frame larger than one tile, tiled as diffusers' tiled_decode (not clamped)."""
        if z.dim() != 5 or z.shape[1] != self.z_dim:
            raise CEError(f"decode expects [B, {self.z_dim}, T, h, w]")
        B, _, Tl, h, w = z.shape
        self._check_fp32_single_gpu()
        tiled = self._tiled_decode(h, w)
        if tiled:
            self._check_tiling_single_gpu()
        z = z.to(device=self.device, dtype=self.dtype).contiguous()
        out = torch.empty(B, 3, 1 + 4 * (Tl - 1), 8 * h, 8 * w, dtype=self.dtype, device=self.device)
        if tiled:
            self._native_tiled(z, out, decode=True)
        else:
            self._native_decode(z, out)
        if not return_dict:
            return (out,)
        return DecoderOutput(sample=out)

    # the seams encode / decode reach the C ABI through (tests stand in for them), all one call of _native
    def _native_encode(self, x: torch.Tensor, out: torch.Tensor) -> None:
        self._native(x, out, decode=False, tiled=False)

    def _native_decode(self, z: torch.Tensor, out: torch.Tensor) -> None:
        self._native(z, out, decode=True, tiled=False)

    def _native_tiled(self, x: torch.Tensor, out: torch.Tensor, decode: bool) -> None:
        self._native(x, out, decode=decode, tiled=True)

    # (fp32, tiled) -> the workspace query and the encode / decode entry points
    _SYMBOLS = {
        (False, False): ("ce_vae_workspace_bytes", "ce_vae_encode", "ce_vae_decode"),
        (True, False): ("ce_vae_workspace_bytes_fp32", "ce_vae_encode_fp32", "ce_vae_decode_fp32"),
        (False, True): ("ce_vae_workspace_bytes_tiled", "ce_vae_encode_tiled", "ce_vae_decode_tiled"),
        (True, True): ("ce_vae_workspace_bytes_tiled_fp32", "ce_vae_encode_tiled_fp32", "ce_vae_decode_tiled_fp32"),
    }

    def _native(self, x: torch.Tensor, out: torch.Tensor, decode: bool, tiled: bool) -> None:
        """Encode (x = video) or decode (x = z), tiled or not.  Samples of a batch are independent streams (each has its own causal
        cache in the reference too), run back to back on the current stream.  The tiled decode does not clamp (TILED_DECODE_CLAMPS)."""
        if not self._is_packed:
            self.pack_weights()
        L = _lib.lib()
        query, enc, dec = (getattr(L, name) for name in self._SYMBOLS[(self.dtype == torch.float32, tiled)])
        B, _, T, H, W = x.shape
        tiles = self._tiles() if tiled else ()
        n = query(self._handle, int(decode), T, H, W, *tiles)
        if n < 0:
            check(-1)
        ws = self._workspace(n)
        clamp = (int(self.clamp_output and (TILED_DECODE_CLAMPS or not tiled)),) if decode else ()
        fn = dec if decode else enc
        with torch.cuda.device(self.device):
            for b in range(B):
                check(fn(self._handle, ptr(x[b]), ptr(out[b]), T, H, W, *tiles, *clamp, ptr(ws), ws.numel(), current_stream()))

    def _check_tiling_single_gpu(self) -> None:
        if self._sp_state:
            raise CEError("tiling is not built for the VAE split over GPUs (parallel.enable_vae_sequence_parallel); disable one of them")

    def launches(self) -> int:
        return int(_lib.lib().ce_vae_last_launch_count(self._handle)) if self._handle else 0

    # ------------------------------------------------------------------------------------------ checkpoint names / loading
    @classmethod
    def diffusers_key_map(cls, base_dim: int = 96, z_dim: int = 16, dim_mult=(1, 2, 4, 4), num_res_blocks: int = 2,
                          temperal_downsample=(False, True, True)) -> Dict[str, str]:
        """COMPLETE map  diffusers `AutoencoderKLWan` parameter name -> in-tree twin (`WanVAE_`) parameter name, generated from
        the architecture (one entry per parameter; `load_state_dict` / `from_pretrained` refuse anything unmapped or missing).

        diffusers 0.35.2 is not on this box, so the diffusers side is restated from its published module tree ([diffusers-mem],
        SURVEY.md section 8c): `encoder.conv_in`, flat `encoder.down_blocks.N` (WanResidualBlock: norm1 / conv1 / norm2 / conv2 /
        conv_shortcut; WanResample: resample.1 / time_conv), `{encoder,decoder}.mid_block.{resnets.0, attentions.0, resnets.1}`,
        `norm_out` / `conv_out`, `quant_conv` / `post_quant_conv`, and `decoder.up_blocks.I.{resnets.R, upsamplers.0}` --
        the same renames the Wan -> diffusers conversion applies to the original checkpoint whose names the twin keeps
        (wan2pt1.py:262-500)."""
        res = {"norm1.gamma": "residual.0.gamma", "conv1.weight": "residual.2.weight", "conv1.bias": "residual.2.bias",
               "norm2.gamma": "residual.3.gamma", "conv2.weight": "residual.6.weight", "conv2.bias": "residual.6.bias",
               "conv_shortcut.weight": "shortcut.weight", "conv_shortcut.bias": "shortcut.bias"}
        same = ("resample.1.weight", "resample.1.bias", "time_conv.weight", "time_conv.bias")
        attn = ("norm.gamma", "to_qkv.weight", "to_qkv.bias", "proj.weight", "proj.bias")
        twin = _param_shapes(base_dim, z_dim, tuple(dim_mult), num_res_blocks, tuple(temperal_downsample))
        m: Dict[str, str] = {}

        def put(dkey, tkey):
            if tkey in twin:
                m[dkey] = tkey

        for suf in ("weight", "bias"):
            put(f"quant_conv.{suf}", f"conv1.{suf}")
            put(f"post_quant_conv.{suf}", f"conv2.{suf}")
            for side in ("encoder", "decoder"):
                put(f"{side}.conv_in.{suf}", f"{side}.conv1.{suf}")
                put(f"{side}.conv_out.{suf}", f"{side}.head.2.{suf}")
        for side in ("encoder", "decoder"):
            put(f"{side}.norm_out.gamma", f"{side}.head.0.gamma")
            for dn, tn in (("mid_block.resnets.0", "middle.0"), ("mid_block.resnets.1", "middle.2")):
                for dk, tk in res.items():
                    put(f"{side}.{dn}.{dk}", f"{side}.{tn}.{tk}")
            for k in attn:
                put(f"{side}.mid_block.attentions.0.{k}", f"{side}.middle.1.{k}")
        n_stage = len(dim_mult)
        idx = 0   # encoder: both sides keep ONE flat list in the same order (res x num_res_blocks, then the resample)
        for i in range(n_stage):
            for _ in range(num_res_blocks):
                for dk, tk in res.items():
                    put(f"encoder.down_blocks.{idx}.{dk}", f"encoder.downsamples.{idx}.{tk}")
                idx += 1
            if i != n_stage - 1:
                for k in same:
                    put(f"encoder.down_blocks.{idx}.{k}", f"encoder.downsamples.{idx}.{k}")
                idx += 1
        idx = 0   # decoder: diffusers groups each stage into a WanUpBlock (resnets + upsamplers), the twin keeps a flat list
        for i in range(n_stage):
            for r in range(num_res_blocks + 1):
                for dk, tk in res.items():
                    put(f"decoder.up_blocks.{i}.resnets.{r}.{dk}", f"decoder.upsamples.{idx}.{tk}")
                idx += 1
            if i != n_stage - 1:
                for k in same:
                    put(f"decoder.up_blocks.{i}.upsamplers.0.{k}", f"decoder.upsamples.{idx}.{k}")
                idx += 1
        missing = sorted(set(twin) - set(m.values()))
        if missing or len(set(m.values())) != len(m):
            raise CEError(f"diffusers_key_map is not a bijection onto the twin's parameters (first missing: {missing[:1]})")
        return m

    def _map_from_config(self) -> Dict[str, str]:
        c = self.config
        return self.diffusers_key_map(c.base_dim, c.z_dim, tuple(c.dim_mult), c.num_res_blocks, tuple(c.temperal_downsample))

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        """Accepts the twin's names (`encoder.downsamples.0.residual.2.weight`, ...) or a diffusers `AutoencoderKLWan` state dict
        (`encoder.down_blocks.0.conv1.weight`, ...), recognised by `encoder.conv_in.weight`.  A diffusers dict must map
        completely: any unmapped or missing key is an error (strict or not), because a silently half-loaded VAE decodes garbage."""
        if "encoder.conv_in.weight" in state_dict or "decoder.conv_in.weight" in state_dict or "quant_conv.weight" in state_dict:
            kmap = self._map_from_config()
            unknown = sorted(k for k in state_dict if k not in kmap)
            absent = sorted(k for k in kmap if k not in state_dict)
            if unknown or absent:
                raise CEError(f"diffusers VAE state dict does not match the architecture: {len(unknown)} unmapped (first: {unknown[:1]}), "
                              f"{len(absent)} missing (first: {absent[:1]})")
            own = dict(self.named_parameters())
            converted = {}
            for k, v in state_dict.items():
                t = kmap[k]
                if tuple(v.shape) != tuple(own[t].shape):
                    if v.numel() != own[t].numel():
                        raise CEError(f"shape of '{k}' {tuple(v.shape)} does not match '{t}' {tuple(own[t].shape)}")
                    v = v.reshape(own[t].shape)
                converted[t] = v
            state_dict = converted
        self._is_packed = False
        return super().load_state_dict(state_dict, strict=strict, assign=assign)

    def diffusers_state_dict(self) -> Dict[str, torch.Tensor]:
        """The parameters under their diffusers names (inverse of the map above)."""
        own = dict(self.named_parameters())
        return {d: own[t].data for d, t in self._map_from_config().items()}

    @classmethod
    def from_config(cls, config: Dict, **kw) -> "AutoencoderKLWan":
        fields = ("base_dim", "z_dim", "dim_mult", "num_res_blocks", "attn_scales", "temperal_downsample", "dropout", "latents_mean",
                  "latents_std")
        args = {k: config[k] for k in fields if k in config}
        for k in ("dim_mult", "attn_scales", "temperal_downsample"):
            if k in args:
                args[k] = tuple(args[k])
        return cls(**args, **kw)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path: str, subfolder: Optional[str] = None, torch_dtype: torch.dtype = torch.bfloat16,
                        device=None, **unused) -> "AutoencoderKLWan":
        """`AutoencoderKLWan.from_pretrained(model_id, subfolder="vae", torch_dtype=torch.bfloat16)` (run_inference_diffusers.py:341-345)
        for a LOCAL diffusers checkpoint directory: config.json + diffusion_pytorch_model[.safetensors | sharded index].  Also accepts a
        directory / file holding the original `Wan2.1_VAE.pth`-style names (the twin's).  torch_dtype=torch.float32 keeps the
        checkpoint's fp32 values and builds the fp32 VAE."""
        import json
        import os

        from safetensors import safe_open

        root = os.path.join(pretrained_model_name_or_path, subfolder) if subfolder else pretrained_model_name_or_path
        cfg = {}
        cfg_path = os.path.join(root, "config.json")
        if os.path.exists(cfg_path):
            with open(cfg_path) as f:
                cfg = json.load(f)
        model = cls.from_config(cfg, torch_dtype=torch_dtype, device=device or "cpu")
        index = os.path.join(root, "diffusion_pytorch_model.safetensors.index.json")
        if os.path.exists(index):
            with open(index) as f:
                files = sorted(set(json.load(f)["weight_map"].values()))
        else:
            files = ["diffusion_pytorch_model.safetensors"]
        sd = {}
        for fn in files:
            with safe_open(os.path.join(root, fn), framework="pt", device="cpu") as sf:
                for k in sf.keys():
                    sd[k] = sf.get_tensor(k)
        model.load_state_dict({k: v.to(model.dtype) for k, v in sd.items()}, strict=True)
        return model
