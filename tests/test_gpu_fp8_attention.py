"""The opt-in FP8 self-attention (DESIGN.md, "FP8 attention"): the two device quantizers against their torch statements, the
e4m3 attention kernel against fp64 softmax attention on the dequantized operands, and the DiT with the switch on against the
oracle with its self-attention replaced by the rule.

The rule, emulated in torch by `attention_rule` (fp32, online over 128-key tiles in key order):
    x = (q^ k^T) s_k,  m = running max of x s_q scale log2e,  P^ = e4m3(256 exp2(x s_q scale log2e - m)),
    l = l alpha + sum P^,  o = o alpha + P^ v^,  out = o s_v / l.

Operator tolerance.  Both the kernel and the emulation differ from fp64 attention on the dequantized operands mostly by the
quantization of P, which they apply at (almost) the same points, so the kernel is held to the error of the emulation rounded to
bf16 as the kernel stores it (mean <= 1.25x, max <= 2x, the repository's parity rule).  It must also meet an absolute bound.  P^_j = p_j (1 + d_j) + e_j with |d_j| <= 2^-4 + 2^-10
(3 mantissa bits, round to nearest; the exponentials the kernel takes by polynomial are within 8e-4) and |e_j| <= 2^-10 / 256 = 2^-18 (half the subnormal step of e4m3 at the factor 256).  The
running maximum's key has p = 1, so sum p >= 1, and the result is a weighted mean of v^ with weights perturbed by at most
eps = 2^-4 + 2^-10 + L 2^-18 + 2^-11 relative to their sum (the last term: the row sum, taken by the FP8 wgmma as P^ times
ones, 4 K32 instructions of about 14 bits); a weighted mean moves by at most 2 eps / (1 - eps) max_j |v^_j,c|.  The FP8 P V
accumulator (about 14 bits per K32 instruction, 4 per tile) adds 4 x 2^-13 of sum P^ |v^|, and the bf16 store 2^-9 |out|:
    |out - ref|_c <= (2 eps / (1 - eps) + 2^-11) max_j |v^_j,c| + 2^-8 |ref|.
"""
import math

import pytest
import torch

from chronoedit_b200.transformer import (FP8_LINEARS, fp8_attention_key_order, quantize_fp8_channels, quantize_fp8_heads,
                                         quantize_fp8_rows)
from tests.test_gpu_fp8 import BF16_MAX, _check_rule, _Fp8Linear, _rows

gpu = pytest.mark.gpu
LOG2E = 1.4426950408889634
SENTINEL = -12345


def _L():
    import chronoedit_b200._lib as L

    return L


def _p(t):
    return None if t is None else t.data_ptr()


def quantize_heads_dev(x, heads):
    """ce_quantize_heads_fp8 on bf16 x [rows, >= heads * 128] (any row stride) -> (q [rows, heads * 128] e4m3, s [rows, heads])."""
    L = _L()
    rows = x.shape[0]
    q = torch.empty(rows, heads * 128, dtype=torch.uint8, device="cuda")
    s = torch.empty(rows, heads, device="cuda")
    L.check(L.lib().ce_quantize_heads_fp8(_p(x), x.stride(0), rows, heads, _p(q), heads * 128, _p(s), L.current_stream()))
    return q.view(torch.float8_e4m3fn), s


def quantize_v_dev(v, B, Lk, H):
    """ce_quantize_v_fp8 on v [B * Lk, >= H * 128] -> (vt [B, H, 128, Lpad] e4m3 as stored, s [B, H * 128], Lpad)."""
    L = _L()
    Lpad = (Lk + 31) // 32 * 32
    vt = torch.full((B, H, 128, Lpad), 0x7F, dtype=torch.uint8, device="cuda")   # NaN bytes: every byte must be written
    s = torch.empty(B, H * 128, device="cuda")
    L.check(L.lib().ce_quantize_v_fp8(_p(v), v.stride(0), B, Lk, H, _p(vt), Lpad, _p(s), L.current_stream()))
    return vt.view(torch.float8_e4m3fn), s, Lpad


def keys_in_order(vt_stored, Lk):
    """Undo the key permutation within each 32-key group of the stored V^T and drop the pad keys."""
    order = fp8_attention_key_order().to(vt_stored.device)
    *lead, Lpad = vt_stored.shape
    g = vt_stored.view(torch.uint8).reshape(*lead, Lpad // 32, 32)
    out = torch.empty_like(g)
    out[..., order] = g
    return out.reshape(*lead, Lpad)[..., :Lk].view(torch.float8_e4m3fn)


def attention_fp8_dev(q8, k8, qs, ks, vt, vs, Lpad, B, H, Lk, out, ldqk):
    L = _L()
    L.check(L.lib().ce_attention_fp8(_p(q8), _p(k8), ldqk, _p(qs), _p(ks), qs.stride(0), _p(vt), Lpad, _p(vs), _p(out), out.stride(0),
                                     B, H, Lk, 1 / math.sqrt(128), L.current_stream()))


def attention_rule(qd, qs, kd, ks, vtd, vs, scale, tile=128):
    """The FP8 attention's rule in fp32 (module docstring).  qd, kd [G, L, 128] (e4m3 values), qs, ks [G, L], vtd [G, 128, L] (keys
    in order), vs [G, 128] -> [G, L, 128] fp32."""
    G, Lq, _ = qd.shape
    Lk = kd.shape[1]
    sl2 = torch.tensor(scale, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)
    rf = qs.float() * sl2.to(qs.device)
    m = torch.full((G, Lq), -math.inf, device=qd.device)
    l = torch.zeros(G, Lq, device=qd.device)
    o = torch.zeros(G, Lq, 128, device=qd.device)
    for j0 in range(0, Lk, tile):
        x = (qd.float() @ kd[:, j0:j0 + tile].float().transpose(1, 2)) * ks[:, None, j0:j0 + tile].float()
        m_new = torch.maximum(m, x.amax(-1) * rf)
        alpha = torch.exp2(m - m_new)
        ph = torch.exp2(x * rf[..., None] - m_new[..., None] + 8).to(torch.float8_e4m3fn).float()
        l = l * alpha + ph.sum(-1)
        o = o * alpha[..., None] + ph @ vtd[:, :, j0:j0 + tile].float().transpose(1, 2)
        m = m_new
    return o * vs.float()[:, None, :] / l[..., None]


# ---------------------------------------------------------------------------------------------------- quantizers
@gpu
@pytest.mark.parametrize("H", [1, 3, 40])
def test_quantize_heads_bit_identical_to_torch(H):
    """q | k read from the fused [M, 3D] buffer with ragged M; the difficult rows of test_gpu_fp8._rows in every head."""
    g = torch.Generator(device="cuda").manual_seed(H)
    D = H * 128
    M = 37
    x = torch.zeros(M, 3 * D, dtype=torch.bfloat16, device="cuda")
    for j in range(2 * H):   # every head of q | k gets the hard rows, in a different row order
        rows = _rows(128, g)
        x[:, j * 128:(j + 1) * 128] = rows[torch.randperm(M, generator=torch.Generator().manual_seed(j))]
    x[:, 2 * D:] = BF16_MAX   # v: must not be read
    q, s = quantize_heads_dev(x, 2 * H)
    rq, rs = quantize_fp8_heads(x[:, :2 * D])
    cq, cs = quantize_fp8_heads(x[:, :2 * D].cpu())
    vq, vs = quantize_fp8_rows(x[:, :2 * D].reshape(-1, 128))
    torch.cuda.synchronize()
    assert torch.equal(s, rs) and torch.equal(s.cpu(), cs) and torch.equal(s.reshape(-1), vs)
    assert torch.equal(q.view(torch.uint8), rq.view(torch.uint8)), f"{int((q.view(torch.uint8) != rq.view(torch.uint8)).sum())} bytes differ"
    assert torch.equal(q.view(torch.uint8).cpu(), cq.view(torch.uint8))
    assert torch.equal(q.view(torch.uint8).reshape(-1, 128), vq.view(torch.uint8))


@gpu
@pytest.mark.parametrize("B,Lk,H", [(1, 1, 1), (2, 100, 2), (1, 129, 3), (2, 2048, 40), (2, 7200, 4)])
def test_quantize_v_bit_identical_to_torch(B, Lk, H):
    g = torch.Generator(device="cuda").manual_seed(Lk + H)
    D = H * 128
    x = torch.randn(B * Lk, 3 * D, generator=g, device="cuda") * torch.logspace(-3, 3, 3 * D, device="cuda")
    x = x.bfloat16()
    v = x[:, 2 * D:]
    if Lk > 8:
        v[:, 5] = 0                  # a zero channel: scale 1
        v[:, 6] = -0.0
        v[:Lk, 7] = 2.0 ** -133      # subnormal channel in sample 0 only
        v[3, 9] = 1e4                # one outlier
        v[:, 10] = BF16_MAX
    vt, s, Lpad = quantize_v_dev(v, B, Lk, H)
    rq, rs = quantize_fp8_channels(v.reshape(B, Lk, D))
    cq, cs = quantize_fp8_channels(v.reshape(B, Lk, D).cpu())
    torch.cuda.synchronize()
    assert torch.equal(s, rs) and torch.equal(s.cpu(), cs)
    got = keys_in_order(vt, Lk).reshape(B, D, Lk)
    assert torch.equal(got.view(torch.uint8), rq.view(torch.uint8)), f"{int((got.view(torch.uint8) != rq.view(torch.uint8)).sum())} bytes differ"
    assert torch.equal(got.view(torch.uint8).cpu(), cq.view(torch.uint8))
    pad = vt.view(torch.uint8).reshape(B, H, 128, Lpad // 32, 32)
    order = fp8_attention_key_order().cuda()
    key = (torch.arange(Lpad // 32, device="cuda")[:, None] * 32 + order[None, :])
    assert (pad[..., key >= Lk] == 0).all(), "pad keys are not zero"
    # per-sample scales: sample 1's scales do not depend on sample 0
    if B == 2:
        _, s1, _ = quantize_v_dev(v[Lk:], 1, Lk, H)
        assert torch.equal(s1, s[1:])


# ---------------------------------------------------------------------------------------------------- attention operator
def _operands(B, H, Lk, seed):
    """Fused QKV [B * L, 3D] bf16: per-head magnitudes over 10^+-3, head 0 peaked (one dominant key), head 1 near-uniform."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    D = H * 128
    x = torch.randn(B, Lk, 3, H, 128, generator=g, device="cuda")
    e = torch.linspace(-3, 3, H, device="cuda") if H > 1 else torch.zeros(1, device="cuda")
    x[:, :, 0] *= (10.0 ** e)[:, None] * 0.3          # q
    x[:, :, 1] *= (10.0 ** -e)[:, None] * 0.3         # k: q.k stays of order 1 while each spans 10^+-3
    x[:, :, 2] *= (10.0 ** e.flip(0))[:, None]        # v
    if H > 2:
        base = torch.randn(128, generator=g, device="cuda")
        x[:, :, 0, 0] = base + 0.1 * x[:, :, 0, 0]
        x[:, Lk // 2, 1, 0] = base * 3                 # one key every query attends to
        x[:, :, 1, 1] *= 1e-3                          # scores near 0: p close to uniform
    return x.reshape(B * Lk, 3 * D).bfloat16()


def _reference64(qd, kd, vd, scale, chunk_bytes=2 ** 30):
    """fp64 softmax attention, [G, L, 128] each, chunked over queries."""
    G, Lq, _ = qd.shape
    out = torch.empty(G, Lq, 128, dtype=torch.float64, device=qd.device)
    step = max(1, chunk_bytes // (8 * kd.shape[1] * G))
    for i0 in range(0, Lq, step):
        s = (qd[:, i0:i0 + step].double() @ kd.double().transpose(1, 2)) * scale
        out[:, i0:i0 + step] = torch.softmax(s, -1) @ vd.double()
    return out


@gpu
@pytest.mark.parametrize("B,H,Lk", [(b, h, l) for l in (1, 100, 128, 129, 2048, 7200) for b, h in ((1, 1), (2, 40))] +
                         [(2, 1, 129), (1, 40, 2048), (1, 2, 28800)])
def test_attention_fp8_against_fp64(B, H, Lk):
    D = H * 128
    x = _operands(B, H, Lk, seed=B * 1000 + H * 10 + Lk)
    q8, s_qk = quantize_heads_dev(x, 2 * H)
    vt, vs, Lpad = quantize_v_dev(x[:, 2 * D:], B, Lk, H)
    ldo = D + 64
    buf = torch.full((B * Lk + 130, ldo), SENTINEL, dtype=torch.int16, device="cuda")
    out = buf[:B * Lk].view(torch.bfloat16)
    attention_fp8_dev(q8, q8[:, D:], s_qk, s_qk[:, H:], vt, vs, Lpad, B, H, Lk, out, 2 * D)
    torch.cuda.synchronize()
    assert (buf[B * Lk:] == SENTINEL).all(), "rows >= B * L written"
    assert (buf[:, D:] == SENTINEL).all(), "columns >= H * 128 written"
    got = out[:, :D].float().reshape(B, Lk, H, 128).permute(0, 2, 1, 3).reshape(B * H, Lk, 128)
    assert torch.isfinite(got).all()
    # operands per (sample, head)
    qd = q8[:, :D].float().reshape(B, Lk, H, 128).permute(0, 2, 1, 3).reshape(B * H, Lk, 128)
    kd = q8[:, D:].float().reshape(B, Lk, H, 128).permute(0, 2, 1, 3).reshape(B * H, Lk, 128)
    qs = s_qk[:, :H].reshape(B, Lk, H).permute(0, 2, 1).reshape(B * H, Lk)
    ks = s_qk[:, H:].reshape(B, Lk, H).permute(0, 2, 1).reshape(B * H, Lk)
    vtd = keys_in_order(vt, Lk).float().reshape(B * H, 128, Lk)
    vsd = vs.reshape(B * H, 128)
    scale = 1 / math.sqrt(128)
    emu = attention_rule(qd, qs, kd, ks, vtd, vsd, scale).bfloat16().float()   # the rule's result as the kernel stores it
    ref = _reference64(qd * qs[..., None], kd * ks[..., None], (vtd * vsd[..., None]).transpose(1, 2), scale)
    e_our, e_emu = (got.double() - ref).abs(), (emu.double() - ref).abs()
    vmax = (vtd.abs() * vsd[..., None]).amax(-1).double()       # [G, 128]
    eps = 2.0 ** -4 + 2.0 ** -10 + Lk * 2.0 ** -18 + 2.0 ** -11
    tol = (2 * eps / (1 - eps) + 2.0 ** -11) * vmax[:, None, :] + 2.0 ** -8 * ref.abs()
    ratio = (e_our / tol).max().item()
    print(f"B={B} H={H} L={Lk}: kernel mean {e_our.mean():.3g} max {e_our.max():.3g}; emulation mean {e_emu.mean():.3g} "
          f"max {e_emu.max():.3g}; worst err / bound {ratio:.3g}")
    assert ratio <= 1.0, f"beyond the absolute bound: worst err/bound {ratio:.3g}"
    assert e_our.mean() <= 1.25 * e_emu.mean() + 1e-30, f"mean err {e_our.mean():.3g} vs emulation {e_emu.mean():.3g}"
    assert e_our.max() <= 2.0 * e_emu.max() + 1e-30, f"max err {e_our.max():.3g} vs emulation {e_emu.max():.3g}"


# ---------------------------------------------------------------------------------------------------- end to end
class _RuleF:
    """Stands in for the oracle's F: the self-attention's scaled_dot_product_attention applies the FP8 attention rule; every other
    call (and F.linear, possibly the FP8 GEMM rule's) goes to `inner`."""

    def __init__(self, inner):
        self.inner = inner
        self.self_attention = False

    def __getattr__(self, name):
        return getattr(self.inner, name)

    def scaled_dot_product_attention(self, q, k, v):
        if not self.self_attention:
            return self.inner.scaled_dot_product_attention(q, k, v)
        B, H, Lk, hd = q.shape
        q8, qs = quantize_fp8_rows(q)
        k8, ks = quantize_fp8_rows(k)
        v8, vs = quantize_fp8_rows(v.transpose(-1, -2))   # per (sample, head, channel) = per (sample, channel)
        o = attention_rule(q8.float().reshape(B * H, Lk, hd), qs.reshape(B * H, Lk), k8.float().reshape(B * H, Lk, hd),
                           ks.reshape(B * H, Lk), v8.float().reshape(B * H, hd, Lk), vs.reshape(B * H, hd), 1 / math.sqrt(hd))
        return o.reshape(B, H, Lk, hd).to(q.dtype)


def rule_oracle(sd, cfg, *inputs, monkeypatch, fp8_weights):
    """The oracle's forward with its self-attention replaced by the FP8 attention rule and, with fp8_weights, the six block GEMMs
    by the FP8 GEMM rule (as test_gpu_fp8.fp8_oracle does), in the dtype of `inputs`."""
    from oracle import dit_oracle as O

    inner = torch.nn.functional
    if fp8_weights:
        sd = dict(sd)
        quantized = {}
        for i in range(cfg.num_layers):
            for name in FP8_LINEARS:
                k = f"blocks.{i}.{name}.weight"
                wq, sw = quantize_fp8_rows(sd[k])
                sd[k] = sd[k].clone()   # a tensor of its own, so that its id names this weight only
                quantized[id(sd[k])] = (wq.to(sd[k].device), sw.to(sd[k].device))
        inner = _Fp8Linear(quantized)
    rule = _RuleF(inner)
    orig = O.attention

    def attention(sd_, p, cfg_, x, ctx, freqs):
        rule.self_attention = ctx is None
        try:
            return orig(sd_, p, cfg_, x, ctx, freqs)
        finally:
            rule.self_attention = False

    with monkeypatch.context() as mp:
        mp.setattr(O, "F", rule)
        mp.setattr(O, "attention", attention)
        with torch.no_grad():
            return O.dit_forward(sd, cfg, *inputs)


def _model(cfg, sdb, fp8_weights, **kw):
    import chronoedit_b200 as ce

    m = ce.ChronoEditTransformer3DModel(
        patch_size=cfg.patch_size, num_attention_heads=cfg.num_attention_heads, attention_head_dim=cfg.attention_head_dim,
        in_channels=cfg.in_channels, out_channels=cfg.out_channels, text_dim=cfg.text_dim, freq_dim=cfg.freq_dim,
        ffn_dim=cfg.ffn_dim, num_layers=cfg.num_layers, eps=cfg.eps, image_dim=cfg.image_dim,
        added_kv_proj_dim=cfg.added_kv_proj_dim, rope_max_seq_len=cfg.rope_max_seq_len,
        rope_temporal_skip_len=cfg.rope_temporal_skip_len, **kw)
    m.load_state_dict(sdb)
    if fp8_weights:
        m.enable_fp8()
    m.enable_fp8_attention()
    return m.cuda()


@gpu
@pytest.mark.parametrize("fp8_weights", [False, True])
@pytest.mark.parametrize("name", ["tiny_t2", "tiny_b2", "tiny_ragged", "tiny_t8"])
def test_fp8_attention_dit_matches_rule(name, fp8_weights, monkeypatch):
    from oracle import cases

    case = cases.DIT_CASES[name]
    sd32 = cases.dit_weights(case)
    sdb = cases.to_bf16_state(sd32)
    x, t, text, img = cases.dit_inputs(case)
    m = _model(case.cfg, sdb, fp8_weights)
    out = m(x.cuda(), t.cuda(), text.cuda(), img.cuda(), return_dict=False)[0].float().cpu()
    ref32 = rule_oracle(sd32, case.cfg, x, t, text, img, monkeypatch=monkeypatch, fp8_weights=fp8_weights)
    ref16 = rule_oracle(sdb, case.cfg, x.bfloat16(), t, text.bfloat16(), img.bfloat16(), monkeypatch=monkeypatch,
                        fp8_weights=fp8_weights).float()
    _check_rule(out, ref32, ref16, f"{name} FP8 attention{' + FP8 GEMMs' if fp8_weights else ''}")


@gpu
def test_fp8_attention_dit_bit_equalities():
    """With the switch on: batch 2 against two batch-1 runs, CUDA graph against eager, context cache against none, forward_host
    against forward.  Switched off again, the output is the bits of a model that never enabled it."""
    from oracle import cases

    case = cases.DIT_CASES["tiny_b2"]
    sdb = cases.to_bf16_state(cases.dit_weights(case))
    x, t, text, img = (v.cuda() for v in cases.dit_inputs(case))
    plain = _model(case.cfg, sdb, False)
    plain.enable_fp8_attention(False)
    want_bf16 = plain(x, t, text, img, return_dict=False)[0]
    m = _model(case.cfg, sdb, False)
    assert m.fp8_attention_enabled
    both = m(x, t, text, img, return_dict=False)[0]
    assert not torch.equal(both, want_bf16), "the switch changed nothing"
    for b in range(2):
        one = m(x[b:b + 1], t[b:b + 1], text[b:b + 1], img[b:b + 1], return_dict=False)[0]
        assert torch.equal(both[b:b + 1], one), f"sample {b}: batched and single evaluation differ"
    host = m.forward_host(x.cpu().bfloat16().contiguous(), t.cpu(), text.cpu().bfloat16().contiguous(), img.cpu().bfloat16().contiguous())
    assert torch.equal(host, both.cpu()), "forward_host differs from forward"
    m.use_cuda_graph = True
    outs = [m(x, t, text, img, return_dict=False)[0] for _ in range(3)]   # eager, capture + replay, replay
    assert all(torch.equal(o, both) for o in outs), "CUDA-graph replay differs from eager"
    m.use_cuda_graph = False
    m.cache_context = True
    outs = [m(x, t, text, img, return_dict=False)[0] for _ in range(2)]   # fills the cache, reuses it
    assert all(torch.equal(o, both) for o in outs), "context cache differs from no cache"
    m.enable_fp8_attention(False)
    outs = [m(x, t, text, img, return_dict=False)[0] for _ in range(2)]   # the cache filled with the switch on stays valid
    assert all(torch.equal(o, want_bf16) for o in outs), "switched off again, the output differs from a model that never enabled it"
    m.enable_fp8_attention(True)
    assert torch.equal(m(x, t, text, img, return_dict=False)[0], both)


@gpu
def test_fp8_attention_temporal_frames_batch_invariant():
    """Tl = rope_temporal_skip_len (8 latent frames): batch 2 of the same sample equals batch 1, bit for bit."""
    from oracle import cases

    case = cases.DIT_CASES["tiny_t8"]
    sdb = cases.to_bf16_state(cases.dit_weights(case))
    x, t, text, img = (v.cuda() for v in cases.dit_inputs(case))
    assert x.shape[2] == case.cfg.rope_temporal_skip_len
    m = _model(case.cfg, sdb, False)
    one = m(x, t, text, img, return_dict=False)[0]
    two = m(x.expand(2, -1, -1, -1, -1).contiguous(), t.expand(2).contiguous(), text.expand(2, -1, -1).contiguous(),
            img.expand(2, -1, -1).contiguous(), return_dict=False)[0]
    assert torch.equal(two[0:1], one) and torch.equal(two[1:2], one)


@gpu
def test_fp8_attention_refuses_sequence_parallelism():
    import chronoedit_b200 as ce
    from oracle import cases

    case = cases.DIT_CASES["tiny_t2"]
    sdb = cases.to_bf16_state(cases.dit_weights(case))
    x, t, text, img = (v.cuda() for v in cases.dit_inputs(case))
    m = _model(case.cfg, sdb, False)
    m(x, t, text, img)
    L = _L()
    regions = [torch.empty(1 << 20, dtype=torch.uint8, device="cuda") for _ in range(2)]
    ptrs = (L.c_void_p * 2)(*[r.data_ptr() for r in regions])
    L.check(L.lib().ce_dit_sp_host_barrier(m._handle, 2000))   # a regression times out on the host, no kernel waits for rank 1
    L.check(L.lib().ce_dit_sp_configure(m._handle, 0, 2, ptrs, regions[0].numel()))
    try:
        with pytest.raises(ce.CEError, match="not built for FP8 attention"):
            m._native_forward(x.bfloat16().contiguous(), t.float(), text.bfloat16().contiguous(), img.bfloat16().contiguous(),
                              torch.empty_like(x, dtype=torch.bfloat16), None, {}, text, img)
    finally:
        L.check(L.lib().ce_dit_sp_configure(m._handle, 0, 1, None, 0))


@gpu
def test_fp8_attention_14b_width_two_layers_at_720p(monkeypatch):
    """Two blocks at the 14B width (D 5120, 40 heads, ffn 13 824) with 7200 tokens: bf16, FP8 GEMMs, FP8 GEMMs + FP8 attention
    against the unquantized fp32 oracle (printed), and the last against the rule oracle (FP8 GEMMs and attention)."""
    from oracle import cases, dit_oracle as O

    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    cfg = O.DiTConfig(num_layers=2)
    sd32 = {k: v.cuda() for k, v in O.random_state_dict(cfg, seed=3).items()}
    sdb = cases.to_bf16_state(sd32)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(1, 36, 2, 90, 160, generator=g).cuda()
    text = torch.randn(1, 512, 4096, generator=g)
    text[:, 77:] = 0
    text = text.cuda()
    img = torch.randn(1, 257, 1280, generator=g).cuda()
    t = torch.tensor([601]).cuda()
    import chronoedit_b200 as ce

    m = ce.ChronoEditTransformer3DModel(num_attention_heads=40, in_channels=36, out_channels=16, ffn_dim=13824, num_layers=2,
                                        image_dim=1280, added_kv_proj_dim=5120)
    m.load_state_dict(sdb)
    m = m.cuda()
    out_bf16 = m(x, t, text, img, return_dict=False)[0].float()
    m.enable_fp8()
    out_gemm = m(x, t, text, img, return_dict=False)[0].float()
    m.enable_fp8_attention()
    out = m(x, t, text, img, return_dict=False)[0].float()
    ref32 = rule_oracle(sd32, cfg, x, t, text, img, monkeypatch=monkeypatch, fp8_weights=True)
    ref16 = rule_oracle(sdb, cfg, x.bfloat16(), t, text.bfloat16(), img.bfloat16(), monkeypatch=monkeypatch, fp8_weights=True).float()
    _check_rule(out, ref32, ref16, "14B width, 2 layers, FP8 GEMMs + FP8 attention")
    with torch.no_grad():
        exact = O.dit_forward(sd32, cfg, x, t, text, img)
    errs = {k: (v - exact).abs() for k, v in (("bf16", out_bf16), ("fp8_gemm", out_gemm), ("fp8_gemm_attention", out))}
    print("against the unquantized fp32 oracle: " + "; ".join(f"{k} mean {e.mean():.3g} max {e.max():.3g}" for k, e in errs.items()) +
          f"; |exact| mean {exact.abs().mean():.3g}")
