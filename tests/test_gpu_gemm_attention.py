"""Operator-level parity of gemm_attention, the GEMM-composed multi-head attention shared by the VAE mid-block and both
conditioning encoders, called through ce_gemm_attention_bf16 with each of its three score rules:
  scaled (VAE: H = 1, dk = C, up to 14 400 tokens), T5 (UMT5: relative-position bias table, key mask), CLIP (bf16 scores,
  L = 257, padding rows in the buffers).

Three checks per case, each with its bound derived in run_attention's docstring:
  - the projections q | k and V^T against fp32 GEMMs (TF32 off) of the same bf16 x and weights;
  - P against the rule's stated bf16 chain recomputed in torch from the kernel's own S (this is what sees a missing
    rounding point or a wrong mask);
  - the output against fp64 softmax attention over the kernel's own bf16 q, k, v.
u = 2^-8 is the unit roundoff of bf16 (8 significant bits).
"""
import ctypes
import math

import pytest
import torch

gpu = pytest.mark.gpu

U = 2.0 ** -8
SCALED, T5, CLIP = 0, 1, 2


def _L():
    import chronoedit_b200._lib as L

    return L


@pytest.fixture(autouse=True)
def _no_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = saved


def up8(v):
    return (v + 7) // 8 * 8


def bf16_ulp(v: torch.Tensor) -> torch.Tensor:
    _, e = torch.frexp(v.abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(v), e - 8)


def ordered(t: torch.Tensor) -> torch.Tensor:
    i = t.contiguous().view(torch.int16).int()
    return torch.where(i < 0, -(i & 0x7FFF), i)


def nan_bf16(*shape):
    return torch.full(shape, float("nan"), dtype=torch.bfloat16, device="cuda")


def run_attention(rule, H, dk, L, D, kpv=None, valid=None, pad_value=float("nan"), bias=True, seed=0):
    """One gemm_attention.  x has up8(L) rows; rows L.. hold pad_value, and qk, vT, S and P start as NaN.

    Projections: fp32 sums of exactly representable bf16 products, rounded once: within one bf16 ulp of the fp32 GEMM, plus
    2^-24 sqrt(D) sum |x w| where the sum cancels.

    P from the kernel's S.  The rule's chain -- score = s * scale (scaled), bf16(bf16(s) + bias) (T5), bf16(bf16(s) * scale)
    (CLIP); p = bf16(exp(score - max) * (1 / sum)) in fp32 over the keys that count, 0 elsewhere -- is recomputed in torch.
    Both sides round the same fp32 values, which differ only by the order of the sum (and __expf against expf in the scaled
    rule), so every element is within 1 ulp and fewer than 0.01% differ at all.  Masked keys are exactly 0.

    Output against fp64.  With the kernel's bf16 q, k, v and p64 = softmax of the rule's score in fp64, the kernel's row i
    differs from out64 = p64 v by at most f_i (p64 |v|) + u |out64|, where f_i = u (P's rounding) + 2 ds_i (a score error ds
    moves exp(score - max) / sum by up to 2 ds relatively) + kpv 2^-24 (fp32 P.V sum) + 2^-18 (fp32 exponentials), and ds_i
    bounds the error of row i's scores: dk 2^-24 max_j |q_i| . |k_j| for S in fp32, times the scale, plus u |s| + u |score|
    for the bf16 roundings of T5 and CLIP."""
    Lib = _L()
    g = torch.Generator(device="cuda").manual_seed(seed)
    I, L8 = H * dk, up8(L)
    kpv = kpv or L
    # unscaled rules: q, k of std dk^-1/4 so that scores are O(1); scaled: scale = dk^-1/2
    wstd = dk ** -0.25 if rule == T5 else 1.0
    scale = 1.0 if rule == T5 else 1.0 / math.sqrt(dk)
    x = torch.full((L8, D), pad_value, dtype=torch.bfloat16, device="cuda")
    x[:L] = torch.randn(L, D, generator=g, device="cuda").bfloat16()
    wqk = (wstd * torch.randn(2 * I, D, generator=g, device="cuda") / math.sqrt(D)).bfloat16()
    wv = (torch.randn(I, D, generator=g, device="cuda") / math.sqrt(D)).bfloat16()
    bqk = (0.1 * torch.randn(2 * I, generator=g, device="cuda")).bfloat16() if bias else None
    bv = (0.1 * torch.randn(I, generator=g, device="cuda")).bfloat16() if bias else None
    table = (2 * torch.randn(H, 2 * L - 1, generator=g, device="cuda")).bfloat16() if rule == T5 else None
    qk, vT, P, out = nan_bf16(L8, 2 * I), nan_bf16(I, L8), nan_bf16(H, L, L8), nan_bf16(L, I)
    S = torch.full((H, L, L8), float("nan"), dtype=torch.float32, device="cuda")
    a = Lib.GemmAttentionArgsC(x=x.data_ptr(), D=D, L=L, H=H, dk=dk, kpv=kpv, wqk=wqk.data_ptr(), bqk=Lib.ptr(bqk).value,
                               wv=wv.data_ptr(), bv=Lib.ptr(bv).value, rule=rule, scale=scale, bias=Lib.ptr(table).value,
                               bias_ld=2 * L - 1, valid=valid or 0, qk=qk.data_ptr(), vT=vT.data_ptr(), S=S.data_ptr(), P=P.data_ptr(),
                               out=out.data_ptr(), ldo=I)
    Lib.check(Lib.lib().ce_gemm_attention_bf16(ctypes.byref(a), Lib.current_stream()))
    torch.cuda.synchronize()
    what = f"gemm_attention rule={rule} H={H} dk={dk} L={L} kpv={kpv} valid={valid}"
    assert bool(torch.isfinite(out).all()), f"{what}: non-finite output"

    # projections
    xs = x[:L].float()
    for name, got, ref, absref in (
            ("qk", qk[:L].float(), xs @ wqk.float().t() + (bqk.float() if bias else 0),
             xs.abs() @ wqk.float().abs().t() + (bqk.float().abs() if bias else 0)),
            ("vT", vT[:, :L].float(), wv.float() @ xs.t() + (bv.float()[:, None] if bias else 0),
             wv.float().abs() @ xs.abs().t() + (bv.float().abs()[:, None] if bias else 0))):
        tol = bf16_ulp(ref) + 2.0 ** -24 * math.sqrt(D) * absref
        ratio = ((got - ref).abs() / tol).max().item()
        print(f"BOUND {what} {name}: worst error / bound = {ratio:.3f}")
        assert ratio <= 1.0, f"{what}: {name} projection {ratio:.3f}x its bound"

    # P from the kernel's own S, by the rule's chain
    s = S[:, :, :L]
    nk = L
    if rule == SCALED:
        m = s.amax(-1, keepdim=True)
        e = torch.exp((s - m) * scale)
    else:
        if rule == T5:
            i = torch.arange(L, device="cuda")
            rel = (i[None, :] - i[:, None]) + L - 1                     # key - query + L - 1
            sc = (s.bfloat16().float() + table.float()[:, rel]).bfloat16().float()
            nk = min(valid, L)
            sc = sc[:, :, :nk]
        else:
            sc = (s.bfloat16().float() * scale).bfloat16().float()
        e = torch.exp(sc - sc.amax(-1, keepdim=True))
    p_ref = torch.zeros(H, L, L8, dtype=torch.bfloat16, device="cuda")
    p_ref[:, :, :nk] = (e * (1.0 / e.sum(-1, keepdim=True))).bfloat16()
    assert bool((P[:, :, nk:] == 0).all()), f"{what}: masked or padding keys must get P = 0 exactly"
    d = (ordered(P) - ordered(p_ref)).abs()
    frac = (d > 0).float().mean().item()
    print(f"BOUND {what} P: {frac * 100:.4f}% differ from the rule's chain, max {d.max().item()} ulp")
    assert d.max().item() <= 1, f"{what}: P more than 1 ulp from the rule's bf16 chain"
    assert frac < 1e-4, f"{what}: {frac * 100:.3f}% of P differs from the rule's bf16 chain"

    # output against fp64 attention over the kernel's bf16 q, k, v
    q = qk[:L, :I].double().view(L, H, dk).transpose(0, 1)
    k = qk[:L, I:].double().view(L, H, dk).transpose(0, 1)
    v = vT[:, :L].double().view(H, dk, L).transpose(1, 2)
    s64 = q @ k.transpose(1, 2)
    ds = dk * 2.0 ** -24 * (q.abs() @ k.abs().transpose(1, 2)).amax(-1) * scale            # [H, L]
    if rule == T5:
        score = s64 + table.double()[:, rel]
        score[:, :, min(valid, L):] = float("-inf")
        ds = ds + U * (s64.abs() + score.abs()).nan_to_num(posinf=0).amax(-1)
    else:
        score = s64 * scale
        if rule == CLIP:
            ds = ds + 2 * U * score.abs().amax(-1)
    p64 = torch.softmax(score, -1)
    out64 = p64 @ v                                                                   # [H, L, dk]
    f = U + 2 * ds + kpv * 2.0 ** -24 + 2.0 ** -18
    tol = f[:, :, None] * (p64 @ v.abs()) + U * out64.abs()
    got = out.double().view(L, H, dk).transpose(0, 1)
    ratio = ((got - out64).abs() / tol).max().item()
    print(f"BOUND {what} out: worst error / bound = {ratio:.3f}")
    assert ratio <= 1.0, f"{what}: output {ratio:.3f}x its bound"
    return out, vT


@gpu
@pytest.mark.parametrize("dk", [96, 384])
@pytest.mark.parametrize("L", [64, 8100, 14400])
def test_scaled_vae(dk, L):
    """The VAE mid-block: one head as wide as the channels, kpv = L.  8100 = 90 x 90 tokens (a 720 x 720 edit) leaves
    L % 8 = 4: x's four padding rows are NaN, as is everything in qk, V^T, S and P before the call, and the output must still
    be finite and within its bound."""
    run_attention(SCALED, 1, dk, L, D=dk, seed=dk + L)


@gpu
@pytest.mark.parametrize("valid", [1, 37, 511, 512])
@pytest.mark.parametrize("H", [8, 64])
def test_t5(H, valid):
    """UMT5: dk = 64, L = 512, a random bias table [H, 2L - 1] (Toeplitz in query and key), keys >= valid masked.  With
    valid = 1 every query sees key 0 alone, so P = 1 there and the output is v_0 exactly."""
    out, vT = run_attention(T5, H, 64, 512, D=256, valid=valid, bias=False, seed=H + valid)
    if valid == 1:
        v0 = vT[:, 0].view(1, H * 64).expand(512, -1)
        assert torch.equal(out.view(torch.int16), v0.contiguous().view(torch.int16)), "valid = 1 must give v_0"


@gpu
def test_clip_padding_rows():
    """CLIP ViT-H: H = 16, dk = 80, L = 257 (L8 = 264) with kpv = L8 as the encoder runs it.  x's seven padding rows hold
    1e4: V^T gets large finite columns there, and only P's exact zeros keep them out of the output."""
    run_attention(CLIP, 16, 80, 257, D=256, kpv=264, pad_value=1e4, seed=3)


@gpu
def test_argument_checks():
    """T5 needs valid >= 1 and kpv may not exceed up8(L); both are refused before anything is launched."""
    Lib = _L()
    t = torch.zeros(4096, dtype=torch.bfloat16, device="cuda")
    s = torch.zeros(4096, dtype=torch.float32, device="cuda")
    p = t.data_ptr()
    a = Lib.GemmAttentionArgsC(x=p, D=8, L=8, H=1, dk=8, kpv=8, wqk=p, wv=p, rule=T5, scale=1.0, bias=p, bias_ld=15, valid=0, qk=p, vT=p,
                               S=s.data_ptr(), P=p, out=p, ldo=8)
    assert Lib.lib().ce_gemm_attention_bf16(ctypes.byref(a), Lib.current_stream()) == -1
    a.valid, a.kpv = 8, 16
    assert Lib.lib().ce_gemm_attention_bf16(ctypes.byref(a), Lib.current_stream()) == -1
    a.kpv, a.rule = 8, 3
    assert Lib.lib().ce_gemm_attention_bf16(ctypes.byref(a), Lib.current_stream()) == -1
