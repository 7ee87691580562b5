"""Operator-level parity of the VAE's kernels, called one at a time through the C ABI: RMS_norm(+SiLU), the nearest 2x
upsample, im2row and the implicit-GEMM convolution with the options only the VAE's own launches use (planar clamped head,
sliding temporal window, small Cin, every BN tile choice, full 720p frames).

References are computed on the device from the same bf16 inputs, in fp64 or in fp32 with TF32 off.  Each test's docstring
derives its bound.  u = 2^-8 is the unit roundoff of bf16 (8 significant bits), so one rounding to bf16 moves a value by at
most u relative, and one bf16 ulp of v is between u|v| and 2u|v|.  Every output buffer is followed by a guard band, and
both the band and every element the kernel must write start as a NaN pattern: an element left unwritten stays NaN, a write
past the end changes the band.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

gpu = pytest.mark.gpu

U = 2.0 ** -8
GUARD = 4096                  # elements of guard band after every output
NAN_BITS = 0x7FA5             # a bf16 NaN, as the int16 bit pattern the guard band and unwritten outputs hold


def _L():
    import chronoedit_b200._lib as L

    return L


@pytest.fixture(autouse=True)
def _no_tf32():
    """fp32 references are true fp32: TF32 would round the operands to 10 bits, a bigger error than the kernels'."""
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def out_buf(n: int) -> torch.Tensor:
    """n bf16 elements plus the guard band, all NaN_BITS."""
    return torch.full((n + GUARD,), NAN_BITS, dtype=torch.int16, device="cuda").view(torch.bfloat16)


def check_guard(buf: torch.Tensor, n: int, what: str):
    assert bool((buf[n:].view(torch.int16) == NAN_BITS).all()), f"{what}: written past the end of the output"


def ordered(t: torch.Tensor) -> torch.Tensor:
    """bf16 bits as integers in the order of the values (+0 and -0 both 0): ulp distance = difference."""
    i = t.contiguous().view(torch.int16).int()
    return torch.where(i < 0, -(i & 0x7FFF), i)


def ulp_dist(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    return (ordered(a) - ordered(b)).abs()


def bf16_ulp(v: torch.Tensor) -> torch.Tensor:
    """One bf16 ulp at |v| (fp32 or fp64), 2^(e-8) for |v| in [2^(e-1), 2^e); the smallest normal's ulp below that."""
    _, e = torch.frexp(v.abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(v), e - 8)


def report(what: str, ratio: float):
    print(f"BOUND {what}: worst error / bound = {ratio:.3f}")


# ---------------------------------------------------------------------------------------------------------------- RMS + SiLU

def rms_input(pixels: int, C: int, seed: int):
    """Per-pixel magnitudes log-uniform in [1e-6, 1e4]; every 5th pixel (p % 5 == 3) exactly zero; every 5th (p % 5 == 1)
    with one channel 1000x the others."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    mag = 10.0 ** (torch.rand(pixels, 1, generator=g, device="cuda") * 10 - 6)
    x = torch.randn(pixels, C, generator=g, device="cuda") * mag
    p = torch.arange(pixels, device="cuda")
    dom = p[p % 5 == 1]
    x[dom, dom % C] *= 1000
    x[p % 5 == 3] = 0
    gamma = torch.randn(C, generator=g, device="cuda") * 0.5 + 1
    return x.bfloat16(), gamma.bfloat16(), p % 5 == 3


def run_rms(pixels: int, C: int, silu: int, seed: int = 0):
    """y = [silu](bf16(bf16(bf16(x / bf16(||x||)) * sqrt(C)) * gamma)).

    fp64 bound.  With a = x / ||x|| * sqrt(C) * gamma in fp64, the kernel's pre-SiLU value carries four bf16 roundings (the
    norm, the quotient, the two products), so its relative error is at most (1+u)^3 / (1-u) - 1 <= 4u + 8u^2, plus C 2^-24
    for the fp32 sum of C squares and the fp32 products rounded twice.  SiLU is 1.0998-Lipschitz, the exponential (__expf)
    adds 2^-20 |a|, and the output rounding u |y|.  Exact-zero pixels give exactly zero.

    Reference chain bound.  The oracle's own bf16 chain (vae_oracle._rms_norm, then F.silu; torch on the device) rounds at
    the same points.  Its norm and the kernel's are the same fp32 sum of squares in another order (relative difference below
    1e-6), so after rounding n is equal or a bf16 neighbour.  Hence every pixel must be bit-equal to the chain evaluated with
    bf16(||x||) or with one of its two neighbours, up to 1 ulp where SiLU's __expf and expf straddle a rounding boundary.
    Fewer than 0.1% of the elements may differ from the chain with the oracle's own n."""
    from oracle import vae_oracle

    L = _L()
    x, gamma, zero = rms_input(pixels, C, seed)
    n = pixels * C
    y = out_buf(n)
    L.check(L.lib().ce_rms_silu_cl_bf16(L.ptr(x), L.ptr(gamma), L.ptr(y), pixels, C, silu, L.current_stream()))
    y2 = out_buf(n)
    L.check(L.lib().ce_rms_silu_cl_bf16(L.ptr(x), L.ptr(gamma), L.ptr(y2), pixels, C, silu, L.current_stream()))
    torch.cuda.synchronize()
    what = f"rms_silu pixels={pixels} C={C} silu={silu}"
    check_guard(y, n, what)
    assert torch.equal(y.view(torch.int16), y2.view(torch.int16)), f"{what}: two launches differ"
    y = y[:n].view(pixels, C)
    assert bool(torch.isfinite(y).all()), f"{what}: non-finite output"
    assert bool((y[zero] == 0).all()), f"{what}: zero pixels must give exactly 0"

    xd = x.double()
    a = xd / xd.norm(dim=1, keepdim=True).clamp_min(1e-12) * math.sqrt(C) * gamma.double()
    rel = 4 * U + 8 * U * U + C * 2.0 ** -24
    if silu:
        y64 = F.silu(a)
        tol = (1.0998 * rel + 2.0 ** -20) * a.abs() * (1 + U) + U * y64.abs()
    else:
        y64 = a
        tol = rel * a.abs()
    err = (y.double() - y64).abs()
    ratio = (err / tol.clamp_min(1e-300)).max().item()
    report(what + " vs fp64", ratio)
    assert ratio <= 1.0, f"{what}: error {ratio:.3f}x the rounding chain's bound"

    def chain(nb):   # F.normalize's x / norm.clamp_min(eps), with the norm given
        pre = x / nb * (C ** 0.5) * gamma
        return F.silu(pre) if silu else pre

    nb = x.norm(dim=1, keepdim=True).clamp_min(1e-12)
    ref = chain(nb)
    oracle = vae_oracle._rms_norm(x, gamma)
    assert torch.equal(ref.view(torch.int16), (F.silu(oracle) if silu else oracle).view(torch.int16))
    bits = nb.view(torch.int16)
    d = ulp_dist(y, ref)
    best = torch.stack([d.amax(1)] + [ulp_dist(y, chain((bits + k).view(torch.bfloat16))).amax(1) for k in (-1, 1)]).amin(0)
    frac = (d > 0).float().mean().item()
    print(f"BOUND {what} vs bf16 oracle: {frac * 100:.4f}% differ (max {d.max().item()} ulp), "
          f"{(d.amax(1) > silu).float().mean().item() * 100:.4f}% of pixels need a neighbouring norm")
    assert int(best.max()) <= silu, f"{what}: {int((best > silu).sum())} pixels match the oracle chain with no norm of the three"
    assert frac < 1e-3, f"{what}: {frac * 100:.3f}% of elements differ from the oracle's bf16 chain"


@gpu
@pytest.mark.parametrize("silu", [0, 1])
@pytest.mark.parametrize("pixels", [1, 7, 4097])
@pytest.mark.parametrize("C", [16, 32, 96, 128, 136, 192, 384, 512])
def test_rms_silu(C, pixels, silu):
    """128 -> 136 is the switch from 16 to 32 lanes per pixel; 512 uses both 16-byte vectors of every lane."""
    run_rms(pixels, C, silu, seed=C * 10 + pixels + silu)


@gpu
@pytest.mark.parametrize("silu", [0, 1])
def test_rms_silu_full_frame(silu):
    """One 720 x 1280 frame at 96 channels: more pixel groups than threads, so the grid-stride loop wraps."""
    run_rms(720 * 1280, 96, silu, seed=11 + silu)


# ---------------------------------------------------------------------------------------------------------------- upsample

@gpu
@pytest.mark.parametrize("T,H,W,C", [(1, 7, 9, 8), (3, 5, 11, 96), (1, 3, 3, 384), (3, 9, 7, 384), (1, 90, 160, 384)])
def test_upsample2x(T, H, W, C):
    """A copy: bit-exact against repeat_interleave on both spatial dims."""
    L = _L()
    g = torch.Generator(device="cuda").manual_seed(T * H * W + C)
    x = torch.randn(T, H, W, C, generator=g, device="cuda").bfloat16()
    n = T * 4 * H * W * C
    y = out_buf(n)
    L.check(L.lib().ce_upsample2x_cl_bf16(L.ptr(x), L.ptr(y), T, H, W, C, L.current_stream()))
    torch.cuda.synchronize()
    check_guard(y, n, "upsample")
    ref = x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    assert torch.equal(y[:n].view(torch.int16), ref.reshape(-1).view(torch.int16))


# ---------------------------------------------------------------------------------------------------------------- im2row

def im2row_ref(xcl: torch.Tensor, Kpad, Tout, Hout, Wout, kt, kh, kw, ph, pw, t_base):
    """xcl: [Tin, Hin, Win, Cin] view of the input (any strides).  Built by indexing a zero-padded copy."""
    Tin, Hin, Win, Cin = xcl.shape
    pt = kt + abs(t_base) + Tout
    xp = torch.zeros(Tin + 2 * pt, Hin + 2 * ph + kh, Win + 2 * pw + kw, Cin, dtype=xcl.dtype, device=xcl.device)
    xp[pt:pt + Tin, ph:ph + Hin, pw:pw + Win] = xcl
    cols = []
    for dt in range(kt):
        for dh in range(kh):
            for dw in range(kw):
                t0 = pt + t_base + dt
                cols.append(xp[t0:t0 + Tout, dh:dh + Hout, dw:dw + Wout])
    K = kt * kh * kw * Cin
    A = torch.zeros(Tout * Hout * Wout, Kpad, dtype=xcl.dtype, device=xcl.device)
    A[:, :K] = torch.stack(cols, dim=3).reshape(-1, K)
    return A


def run_im2row(x, strides, shape, Kpad, Tout, k, pad, t_base):
    """x: any tensor; strides (sc, st, sh, sw) in elements and shape (Tin, Hin, Win, Cin) describe the input inside it."""
    L = _L()
    Tin, Hin, Win, Cin = shape
    kt, kh, kw = k
    ph, pw = pad
    Hout, Wout = Hin + 2 * ph - kh + 1, Win + 2 * pw - kw + 1
    sc, st, sh, sw = strides
    n = Tout * Hout * Wout * Kpad
    A = out_buf(n)
    L.check(L.lib().ce_im2row_bf16(L.ptr(x), sc, st, sh, sw, Tin, Hin, Win, Cin, L.ptr(A), Kpad, Tout, Hout, Wout, kt, kh, kw, ph, pw, t_base,
                                   L.current_stream()))
    torch.cuda.synchronize()
    what = f"im2row shape={shape} k={k} t_base={t_base} Kpad={Kpad}"
    check_guard(A, n, what)
    xcl = torch.as_strided(x, (Tin, Hin, Win, Cin), (st, sh, sw, sc))
    ref = im2row_ref(xcl, Kpad, Tout, Hout, Wout, kt, kh, kw, ph, pw, t_base)
    assert torch.equal(A[:n].view(torch.int16), ref.reshape(-1).view(torch.int16)), what
    return A[:n].view(-1, Kpad)


@gpu
@pytest.mark.parametrize("t_base,Tout", [(-2, 1), (-2, 4), (0, 4), (2, 4), (2, 8)])
def test_im2row_planar_video(t_base, Tout):
    """encoder.conv1: 3x3x3 from the planar video [3, T, H, W], K = 81 -> Kpad = 88 (zero tail); frames before 0 and from
    Tin on are causal / out-of-range zeros.  Bit-exact: the kernel only moves bits."""
    g = torch.Generator(device="cuda").manual_seed(t_base + 10 * Tout)
    T, H, W = 9, 19, 37
    v = torch.randn(3, T, H, W, generator=g, device="cuda").bfloat16()
    run_im2row(v, (T * H * W, H * W, W, 1), (T, H, W, 3), 88, Tout, (3, 3, 3), (1, 1), t_base)


@gpu
@pytest.mark.parametrize("Kpad", [432, 440])
def test_im2row_history_buffer(Kpad):
    """decoder.conv1: 3x3x3 over a channels-last [2 history + 1, h, w, 16] buffer; 440 adds a zero K tail."""
    g = torch.Generator(device="cuda").manual_seed(Kpad)
    x = torch.randn(3, 11, 13, 16, generator=g, device="cuda").bfloat16()
    run_im2row(x, (1, 11 * 13 * 16, 13 * 16, 16), (3, 11, 13, 16), Kpad, 1, (3, 3, 3), (1, 1), 0)


@gpu
def test_im2row_asymmetric_window():
    """kt, kh, kw and ph, pw all different, so that no index of the window can stand in for another."""
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(4, 10, 13, 8, generator=g, device="cuda").bfloat16()
    run_im2row(x, (1, 10 * 13 * 8, 13 * 8, 8), (4, 10, 13, 8), 2 * 3 * 5 * 8, 2, (2, 3, 5), (0, 2), 1)


@gpu
def test_im2row_pointwise_planar_z():
    """conv2: 1x1x1 on latent frame i of the planar z [16, Tl, h, w] (t_base = i)."""
    g = torch.Generator(device="cuda").manual_seed(5)
    Tl, h, w = 3, 9, 15
    z = torch.randn(16, Tl, h, w, generator=g, device="cuda").bfloat16()
    for i in range(Tl):
        run_im2row(z, (Tl * h * w, h * w, w, 1), (Tl, h, w, 16), 16, 1, (1, 1, 1), (0, 0), i)


@gpu
@pytest.mark.parametrize("f0,Tc", [(0, 1), (1, 4), (5, 4)])
def test_im2row_then_gemm_is_the_causal_conv(f0, Tc):
    """im2row + ce_linear_bf16 = F.conv3d of the causally padded video at output frames f0 .. f0+Tc-1.  The GEMM accumulates
    exactly representable products in fp32 as cuDNN does (TF32 off), so the two sums differ by fp32 rounding only: the bf16
    output is within one ulp of the fp32 reference, plus 2^-24 sqrt(K) sum |w x| where the sum cancels to near zero."""
    from chronoedit_b200.autoencoder import pack_parameter

    L = _L()
    g = torch.Generator(device="cuda").manual_seed(f0)
    T, H, W, Cout = 9, 19, 37, 96
    v = torch.randn(3, T, H, W, generator=g, device="cuda").bfloat16()
    w = (torch.randn(Cout, 3, 3, 3, 3, generator=g, device="cuda") / 9).bfloat16()
    b = (0.1 * torch.randn(Cout, generator=g, device="cuda")).bfloat16()
    A = run_im2row(v, (T * H * W, H * W, W, 1), (T, H, W, 3), 88, Tc, (3, 3, 3), (1, 1), f0 - 2)
    wp = pack_parameter("encoder.conv1.weight", w)
    M = Tc * H * W
    out = torch.empty(M, Cout, dtype=torch.bfloat16, device="cuda")
    L.check(L.lib().ce_linear_bf16(L.ptr(A), 88, L.ptr(wp), 88, L.ptr(b), L.ptr(out), Cout, None, M, Cout, 88, 0, None, 0, None, 0, 1,
                                   L.current_stream()))
    vp = F.pad(v[None].float(), (1, 1, 1, 1, 2, 0))
    ref = F.conv3d(vp, w.float(), b.float())[0, :, f0:f0 + Tc].permute(1, 2, 3, 0).reshape(M, Cout)
    absref = F.conv3d(vp.abs(), w.float().abs())[0, :, f0:f0 + Tc].permute(1, 2, 3, 0).reshape(M, Cout) + b.float().abs()
    tol = bf16_ulp(ref) + 2.0 ** -24 * math.sqrt(81) * absref
    ratio = ((out.float() - ref).abs() / tol).max().item()
    report(f"im2row+gemm f0={f0}", ratio)
    assert ratio <= 1.0


# ---------------------------------------------------------------------------------------------------------------- convolution

def run_conv(Cin, Cout, Tout, H, W, k, stride=(1, 1, 1), pad=(0, 0), Tin=None, t_base=0, split_time=0, planar=None, wscale=1.0,
             seed=0, gen_on_device=True):
    """One ce_conv3d_cl_ex_bf16 against F.conv3d in fp32 (TF32 off) on the same bf16 x, w, bias.

    Bound: the kernel and cuDNN both sum exactly representable bf16 products in fp32, in different orders, and the kernel
    rounds acc + bias to bf16 once, so |y - ref| <= one bf16 ulp of ref + 2^-24 sqrt(K) sum |w x| (the second term only
    matters where the sum cancels).  Clamping is 1-Lipschitz, so the clamped head has the same bound against clamp(ref).
    planar = (planar_T, planar_t0, clamp): y is a pre-filled planar video and only frames planar_t0 .. +Tout may change.
    Every case also checks the guard band behind y and that a second launch is bit-identical."""
    L = _L()
    g = torch.Generator(device="cuda").manual_seed(seed)
    kt, kh, kw = k
    st, sh, sw = stride
    ph, pw = pad
    Tin = Tin if Tin is not None else t_base + (Tout - 1) * st + kt
    x = torch.randn(Tin, H, W, Cin, generator=g, device="cuda").bfloat16()
    w = (wscale * torch.randn(Cout, Cin, kt, kh, kw, generator=g, device="cuda") / math.sqrt(Cin * kt * kh * kw)).bfloat16()
    b = (0.1 * torch.randn(Cout, generator=g, device="cuda")).bfloat16()
    Cin_pad = (Cin + 63) // 64 * 64
    wp = torch.zeros(Cout, kt * kh * kw, Cin_pad, dtype=torch.bfloat16, device="cuda")
    wp[:, :, :Cin] = w.permute(0, 2, 3, 4, 1).reshape(Cout, kt * kh * kw, Cin)

    xn = x.permute(3, 0, 1, 2)[None].float()[:, :, t_base:t_base + (Tout - 1) * st + kt]
    xp = F.pad(xn, (0, 1, 0, 1)) if sh == 2 else F.pad(xn, (pw, pw, ph, ph))   # stride 2: ZeroPad2d((0,1,0,1)) (wan2pt1.py:106-110)
    ref = F.conv3d(xp, w.float(), b.float(), stride=stride)[0]                   # [Cout, Tout, Hout, Wout]
    absref = F.conv3d(xp.abs(), w.float().abs(), b.float().abs(), stride=stride)[0]
    Hout, Wout = ref.shape[2], ref.shape[3]
    assert ref.shape[1] == Tout
    K = Cin * kt * kh * kw
    if planar is not None:
        planar_T, planar_t0, clamp = planar
        n = Cout * planar_T * Hout * Wout
        fill = torch.randn(n, generator=g, device="cuda").bfloat16() * 4
        if clamp:
            ref = ref.clamp(-1, 1)
    else:
        n = Cout * Tout * Hout * Wout
        if split_time:   # channels [0, C) -> even frames, [C, 2C) -> odd frames (wan2pt1.py:137-139)
            c = Cout // 2
            ref = torch.stack((ref[:c], ref[c:]), dim=2).reshape(c, 2 * Tout, Hout, Wout)
            absref = torch.stack((absref[:c], absref[c:]), dim=2).reshape(c, 2 * Tout, Hout, Wout)
    outs = []
    for _ in range(2):
        y = out_buf(n)
        if planar is not None:
            y[:n] = fill
        a = L.Conv3dArgsC(x=x.data_ptr(), Tin=Tin, Hin=H, Win=W, Cin=Cin, w=wp.data_ptr(), bias=b.data_ptr(), Cout=Cout, Cin_pad=Cin_pad,
                          kt=kt, kh=kh, kw=kw, st=st, sh=sh, sw=sw, ph=ph, pw=pw, t_base=t_base, y=y.data_ptr(), Tout=Tout, Hout=Hout,
                          Wout=Wout, split_time=split_time)
        if planar is not None:
            a.planar_out, a.planar_T, a.planar_t0, a.clamp = 1, planar_T, planar_t0, clamp
        L.check(L.lib().ce_conv3d_cl_ex_bf16(ctypes.byref(a), L.current_stream()))
        outs.append(y)
    torch.cuda.synchronize()
    what = f"conv Cin={Cin} Cout={Cout} k={k} stride={stride} {H}x{W} t_base={t_base} split={split_time} planar={planar}"
    y = outs[0]
    check_guard(y, n, what)
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16)), f"{what}: two launches differ"
    if planar is not None:
        yv = y[:n].view(Cout, planar_T, Hout, Wout)
        fv = fill.view(Cout, planar_T, Hout, Wout)
        keep = torch.ones(planar_T, dtype=torch.bool)
        keep[planar_t0:planar_t0 + Tout] = False
        assert torch.equal(yv[:, keep].view(torch.int16), fv[:, keep].view(torch.int16)), f"{what}: frames outside the chunk changed"
        got = yv[:, planar_t0:planar_t0 + Tout].float()
        if clamp:
            assert got.abs().max().item() <= 1.0, f"{what}: not clamped"
    else:
        got = y[:n].view(ref.shape[1], Hout, Wout, ref.shape[0]).permute(3, 0, 1, 2).float()
    assert bool(torch.isfinite(got).all()), f"{what}: non-finite or unwritten output"
    tol = bf16_ulp(ref) + 2.0 ** -24 * math.sqrt(K) * absref
    ratio = ((got - ref).abs() / tol).max().item()
    report(what, ratio)
    assert ratio <= 1.0, f"{what}: error {ratio:.3f}x the bound"
    return ref


@gpu
@pytest.mark.parametrize("clamp", [0, 1])
def test_conv_planar_head(clamp):
    """The decoder head: 96 -> 3, 3x3x3, stored planar at frames 3, 4 of a 7-frame video whose other frames must not change;
    the weights are scaled so that a good part of the outputs exceeds +-1."""
    ref = run_conv(96, 3, 2, 21, 35, (3, 3, 3), pad=(1, 1), Tin=4, planar=(7, 3, clamp), wscale=4.0, seed=20 + clamp)
    if not clamp:
        assert (ref.abs() > 1).float().mean().item() > 0.2, "the data must exceed +-1 for the clamp to be tested"


@gpu
def test_conv_planar_bounds_are_checked():
    """A planar store that would leave the video is refused before anything is launched."""
    L = _L()
    x = torch.zeros(3, 8, 16, 96, dtype=torch.bfloat16, device="cuda")
    w = torch.zeros(3, 27, 128, dtype=torch.bfloat16, device="cuda")
    y = torch.zeros(3, 4, 8, 16, dtype=torch.bfloat16, device="cuda")
    a = L.Conv3dArgsC(x=x.data_ptr(), Tin=3, Hin=8, Win=16, Cin=96, w=w.data_ptr(), Cout=3, Cin_pad=128, kt=3, kh=3, kw=3, st=1, sh=1, sw=1,
                      ph=1, pw=1, y=y.data_ptr(), Tout=1, Hout=8, Wout=16, planar_out=1, planar_T=4, planar_t0=4)
    assert L.lib().ce_conv3d_cl_ex_bf16(ctypes.byref(a), L.current_stream()) == -1
    assert b"planar output frames" in L.lib().ce_last_error()
    a.planar_t0 = 3
    L.check(L.lib().ce_conv3d_cl_ex_bf16(ctypes.byref(a), L.current_stream()))
    torch.cuda.synchronize()


@gpu
@pytest.mark.parametrize("t_base,Tout,st", [(3, 2, 1), (1, 2, 2)])
def test_conv_sliding_window(t_base, Tout, st):
    """t_base > 0 inside a longer buffer: output frame `to` reads input frames t_base + to*st .. + 2."""
    run_conv(96, 96, Tout, 19, 37, (3, 3, 3), stride=(st, 1, 1), pad=(1, 1), Tin=9, t_base=t_base, seed=30 + t_base)


@gpu
@pytest.mark.parametrize("Cin", [8, 16, 24, 72])
def test_conv_small_cin(Cin):
    """Most (8, 16, 24) or part (72 = 64 + 8) of a 64-channel block is the tensor map's out-of-bounds zero fill."""
    run_conv(Cin, 96, 2, 13, 21, (3, 3, 3), pad=(1, 1), Tin=4, seed=40 + Cin)


@gpu
@pytest.mark.parametrize("Cout", [3, 5, 8, 40, 200, 288])
def test_conv_cout_tiles(Cout):
    """Every BN choice: 32 (3, 5 and 8: 3 and 5 take the scalar channels-last store), 96 with a partial tile (40), 192 with a
    partial second tile (200), and three 96-wide tiles (288)."""
    run_conv(96, Cout, 1, 19, 37, (3, 3, 3), pad=(1, 1), Tin=3, seed=50 + Cout)


@gpu
def test_conv_full_720p_causal():
    """3x3x3 at 96 -> 96 on a 720 x 1280 frame with two history frames (the first decoder stage at 720p)."""
    run_conv(96, 96, 1, 720, 1280, (3, 3, 3), pad=(1, 1), Tin=3, seed=60)


@gpu
def test_conv_full_360p_causal():
    run_conv(192, 192, 1, 360, 640, (3, 3, 3), pad=(1, 1), Tin=3, seed=61)


@gpu
def test_conv_full_720p_downsample():
    """Stride-2 Resample 720 x 1280 -> 360 x 640: ZeroPad2d((0,1,0,1)) is the out-of-bounds fill on the right and bottom."""
    run_conv(96, 96, 1, 720, 1280, (1, 3, 3), stride=(1, 2, 2), seed=62)


@gpu
def test_conv_time_conv_split_90x160():
    """upsample3d's time_conv at 90 x 160: 384 -> 768 channels, split into two output frames."""
    run_conv(384, 768, 1, 90, 160, (3, 1, 1), Tin=3, split_time=1, seed=63)
