"""The opt-in FP8 mode (DESIGN.md, "FP8 mode"): the device's row quantization against its torch statement, the e4m3 GEMM
against fp64 on the dequantized operands and against the bf16 GEMM's epilogue, and the FP8 DiT end to end against an FP8
emulation of the oracle.

GEMM tolerance.  The products of two e4m3 values are exact in fp32, so with fp32 accumulation over K terms
(u = 2^-24) and the two scale multiplies and the bias add of the epilogue, out_f32 = (sum_k qa qw) sa sw + bias satisfies
    |out_f32 - ref| <= s_a s_w (K + 2) u sum_k |qa qw| + u |ref|    (times 2 for second-order terms)
against the fp64 `ref` of the same formula.  Hopper's FP8 wgmma does not accumulate in full fp32 (its adder keeps about 14
bits, DESIGN.md "FP8 mode"), so every K is held to the same bound with u_acc = 2^-13 per K32 instruction in place of
(K + 2) u, and the block GEMMs' K (5120 and 13 824, where that question matters) also to the fp32 bound.

Epilogue.  "The existing epilogue applied to the kernel's own y" is computed by the bf16 GEMM itself: y (fp32, from the
FP8 GEMM's out_f32 without bias) is split exactly into three bf16 terms hi + mid + lo, and A = [hi | mid | lo] against
W = [I | I | I] makes the bf16 GEMM's accumulator equal y bit for bit; its epilogue with the same bias / residual / gate /
statistics then gives the bits the FP8 GEMM must store.

End to end.  The oracle's linears are swapped, for exactly the six block GEMMs, for the FP8 rule on its own operands (the
activation quantized per token with quantize_fp8_rows, the weight per output channel), in fp32 and in bf16.  The FP8 DiT
is held to the rule of test_gpu_dit.py with the bf16 emulation standing in for the reference's bf16 run.
"""
import math

import pytest
import torch

from chronoedit_b200.transformer import FP8_LINEARS, quantize_fp8_rows
from tests.test_gpu_row_stats import gemm_case, linear_ex, tile_width

gpu = pytest.mark.gpu
U = 2.0 ** -24
SENTINEL = -12345
BF16_MAX = torch.finfo(torch.bfloat16).max


def _L():
    import chronoedit_b200._lib as L

    return L


def _p(t):
    return None if t is None else t.data_ptr()


def quantize_dev(x):
    """ce_quantize_rows_fp8 on a bf16 [rows, K] CUDA tensor -> (q e4m3 [rows, K], s fp32 [rows])."""
    L = _L()
    rows, K = x.shape
    q = torch.empty(rows, K, dtype=torch.uint8, device="cuda")
    s = torch.empty(rows, device="cuda")
    L.check(L.lib().ce_quantize_rows_fp8(_p(x), x.stride(0), rows, K, _p(q), K, _p(s), L.current_stream()))
    return q.view(torch.float8_e4m3fn), s


def linear_fp8(Aq, sa, Wq, sw, out, *, out_f32=None, bias=None, epi=0, resid=None, gate=None, rpb=1, stats=None, stats_mode=0):
    L = _L()
    M, K = Aq.shape
    N = Wq.shape[0]
    base = L.LinearArgsC(A=_p(Aq), lda=Aq.stride(0), W=_p(Wq), ldw=Wq.stride(0), M=M, N=N, K=K, out=_p(out),
                         ldo=0 if out is None else out.stride(0), out_f32=_p(out_f32), ld_f32=0 if out_f32 is None else out_f32.stride(0),
                         bias=_p(bias), epilogue=epi, resid=_p(resid), ldr=0 if resid is None else resid.stride(0), gate=_p(gate),
                         gate_stride=0 if gate is None else gate.shape[1], rows_per_batch=rpb, stats_out=_p(stats),
                         stats_ld=0 if stats is None else stats.shape[1], stats_mode=stats_mode)
    args = L.LinearFp8ArgsC(base=base, a_scale=_p(sa), w_scale=_p(sw))
    L.check(L.lib().ce_linear_fp8_ex(args, L.current_stream()))


# ---------------------------------------------------------------------------------------------------- quantization
def _rows(K, g):
    """Ragged row count (not a multiple of anything) of every kind the rule has to handle."""
    n = 37
    x = torch.randn(n, K, generator=g, device="cuda") * torch.logspace(-3, 3, n, device="cuda")[:, None]
    x[1] = 0                                   # zero row: scale 1
    x[2] = -0.0                                # negative zeros keep their sign
    x[3] = 0.37                                # constant row
    x[4] = torch.randn(K, generator=g, device="cuda") * 1e-3
    x[4, K // 3] = 1e4                         # one outlier: everything else underflows towards the subnormals
    x[5] = BF16_MAX                            # +- the largest bf16
    x[5, ::2] = -BF16_MAX
    x[6] = 2.0 ** -133                         # bf16 subnormals
    x[7, K - 1] = -3e5                         # outlier in the last column
    return x.bfloat16()


@gpu
@pytest.mark.parametrize("K", [5120, 13824, 15360, 16])
def test_quantize_rows_bit_identical_to_torch(K):
    g = torch.Generator(device="cuda").manual_seed(K)
    x = _rows(K, g)
    q, s = quantize_dev(x)
    rq, rs = quantize_fp8_rows(x)
    cq, cs = quantize_fp8_rows(x.cpu())
    torch.cuda.synchronize()
    assert torch.equal(s, rs) and torch.equal(s.cpu(), cs)
    assert torch.equal(q.view(torch.uint8), rq.view(torch.uint8)), f"{int((q.view(torch.uint8) != rq.view(torch.uint8)).sum())} bytes differ"
    assert torch.equal(q.view(torch.uint8).cpu(), cq.view(torch.uint8))
    assert s[1].item() == 1.0 and (q.view(torch.uint8)[2] == 0x80).all()
    assert (q[5].float().abs() == 448).all()
    # a strided input (ldx > K) and a sub-range of rows give the same bits
    wide = torch.zeros(x.shape[0], K + 16, dtype=torch.bfloat16, device="cuda")
    wide[:, 8:8 + K] = x
    q2, s2 = quantize_dev(wide[3:, 8:8 + K])
    assert torch.equal(q2.view(torch.uint8), q.view(torch.uint8)[3:]) and torch.equal(s2, s[3:])


@gpu
def test_weight_quantization_cpu_equals_cuda():
    g = torch.Generator().manual_seed(11)
    w = (torch.randn(640, 384, generator=g) * torch.logspace(-4, 2, 640)[:, None]).bfloat16()
    w[3] = 0
    w[4, 7] = 1e30
    qc, sc = quantize_fp8_rows(w)
    qg, sg = quantize_fp8_rows(w.cuda())
    assert torch.equal(qc.view(torch.uint8), qg.view(torch.uint8).cpu()) and torch.equal(sc, sg.cpu())


# ---------------------------------------------------------------------------------------------------- GEMM
def _fp8_operands(M, N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    # per-row and per-column magnitudes that differ, so that a swapped or missing scale is visible
    A = (torch.randn(M, K, generator=g, device="cuda") * torch.logspace(-1, 1, M, device="cuda")[:, None]).bfloat16()
    W = (torch.randn(N, K, generator=g, device="cuda") / math.sqrt(K) * torch.logspace(1, -1, N, device="cuda")[:, None]).bfloat16()
    Aq, sa = quantize_dev(A)
    Wq, sw = quantize_fp8_rows(W)
    return Aq, sa, Wq, sw


def _ref_and_tol(Aq, sa, Wq, sw, bias, kblocks=None):
    qa, qw = Aq.double(), Wq.double()
    if kblocks is not None:   # planted defect: only the first `kblocks` k-blocks of 128
        qa, qw = qa[:, :128 * kblocks], qw[:, :128 * kblocks]
    acc = qa @ qw.t()
    absacc = qa.abs() @ qw.abs().t()
    y = acc * sa.double()[:, None] * sw.double()[None, :]
    ref = y + bias.double()[None, :]
    K = Aq.shape[1]
    tol = 2 * (sa.double()[:, None] * sw.double()[None, :] * (K + 2) * U * absacc + U * ref.abs())
    steps = (K + 31) // 32   # K32 instructions
    tol14 = 2 * (sa.double()[:, None] * sw.double()[None, :] * steps * 2.0 ** -13 * absacc + U * ref.abs())
    return ref, (tol, tol14), acc


def _err_ratio(got, ref, tol):
    return ((got.double() - ref).abs() / tol.clamp_min(1e-300)).max().item()


@gpu
@pytest.mark.parametrize("M,N,K", [(300, 512, 320), (1300, 192, 5120), (77, 64, 13824), (260, 5120, 13824), (129, 13824, 5120)])
def test_fp8_gemm_against_fp64(M, N, K):
    """Tile widths 256 / 128 / 64, ragged M and N, one or several waves, K with a partial last k-block (320 = 2.5 x 128)."""
    Aq, sa, Wq, sw = _fp8_operands(M, N, K, seed=M + N + K)
    bias = (torch.randn(N, device="cuda") * 0.1).bfloat16()
    f32 = torch.full((M, N), float("nan"), device="cuda")
    linear_fp8(Aq, sa, Wq, sw, None, out_f32=f32, bias=bias)
    torch.cuda.synchronize()
    ref, (tol32, tol), acc = _ref_and_tol(Aq, sa, Wq, sw, bias)
    assert torch.isfinite(f32).all()
    r32, r = _err_ratio(f32, ref, tol32), _err_ratio(f32, ref, tol)
    print(f"M={M} N={N} K={K}: worst err / fp32-accumulation bound {r32:.3g}, / 14-bit-accumulator bound {r:.3g}")
    assert r <= 1.0, f"out_f32 beyond the 14-bit-accumulator bound: worst err/bound {r:.3g}"
    if K >= 5120:
        assert r32 <= 1.0, f"out_f32 beyond the fp32-accumulation bound: worst err/bound {r32:.3g}"
    if K % 128:
        # the planted defects this bound must catch: swapped scales, the last partial k-block dropped, a scale ignored
        n = min(M, N)
        swapped = acc[:n, :n] * sw.double()[:n, None] * sa.double()[None, :n] + bias.double()[None, :n]
        assert _err_ratio(swapped, ref[:n, :n], tol[:n, :n]) > 1
        short, _, _ = _ref_and_tol(Aq, sa, Wq, sw, bias, kblocks=K // 128)
        assert _err_ratio(short, ref, tol) > 1
        assert _err_ratio(acc * sw.double()[None, :] + bias.double()[None, :], ref, tol) > 1
        assert _err_ratio(acc * sa.double()[:, None] + bias.double()[None, :], ref, tol) > 1


def _bf16_epilogue_of(y, bias, epi, resid, gate, rpb, stats_mode, tn, out_shape=None):
    """The bf16 GEMM's epilogue applied to an fp32 y [M, N] (module docstring): returns (out, stats)."""
    M, N = y.shape
    hi = y.bfloat16()
    mid = (y - hi.float()).bfloat16()
    lo = (y - hi.float() - mid.float()).bfloat16()
    assert torch.equal(hi.float() + mid.float() + lo.float(), y), "y does not split exactly into three bf16 terms"
    A = torch.cat([hi, mid, lo], dim=1).contiguous()
    eye = torch.eye(N, device="cuda", dtype=torch.bfloat16)
    W = torch.cat([eye, eye, eye], dim=1).contiguous()
    out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    st = torch.full((M, (N + tn - 1) // tn, 2), float("nan"), device="cuda") if stats_mode else None
    linear_ex(A, W, out, bias=bias, epi=epi, resid=resid, gate=gate, rpb=rpb, stats=st, stats_mode=stats_mode)
    return out, st


@gpu
@pytest.mark.parametrize("N", [512, 192, 64])   # tile widths 256, 128 (partial last tile), 64
def test_fp8_gemm_epilogues(N):
    """M = 1300 (11 M tiles, the last ragged), K = 320.  For epilogues 0-4 with statistics: the bf16 output and statistics equal
    the bf16 GEMM's epilogue applied to the FP8 GEMM's own y, and each 128-row slice equals the GEMM launched on that slice alone."""
    M, K, rpb = 1300, 320, 256
    tn = tile_width(N)
    tiles = (N + tn - 1) // tn
    _, _, bias, resid, gate = gemm_case("block_offset", M, N, K, rpb, seed=N)
    Aq, sa, Wq, sw = _fp8_operands(M, N, K, seed=N + 1)
    y = torch.empty(M, N, device="cuda")
    linear_fp8(Aq, sa, Wq, sw, None, out_f32=y)   # no bias: out_f32 = y + (-0.0) = y
    for epi in range(5):
        mode = 1 if epi in (0, 3, 4) else 2
        kw = dict(bias=bias, epi=epi, resid=resid if epi in (3, 4) else None, gate=gate if epi == 3 else None, rpb=rpb, stats_mode=mode)
        full = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
        st = torch.full((M, tiles, 2), float("nan"), device="cuda")
        linear_fp8(Aq, sa, Wq, sw, full, stats=st, **kw)
        want, want_st = _bf16_epilogue_of(y, bias, epi, kw["resid"], kw["gate"], rpb, mode, tn)
        torch.cuda.synchronize()
        assert torch.equal(full.view(torch.int16), want.view(torch.int16)), f"N={N} epi={epi}: output differs from the bf16 epilogue of y"
        assert torch.equal(st, want_st), f"N={N} epi={epi}: statistics differ from the bf16 epilogue of y"
        for r0 in range(0, M, 128):
            r1 = min(M, r0 + 128)
            out = torch.empty(r1 - r0, N, dtype=torch.bfloat16, device="cuda")
            sst = torch.full((r1 - r0, tiles, 2), float("nan"), device="cuda")
            linear_fp8(Aq[r0:r1], sa[r0:r1], Wq, sw, out, stats=sst, bias=bias, epi=epi,
                       resid=resid[r0:r1] if epi in (3, 4) else None, gate=gate[r0 // rpb:] if epi == 3 else None, rpb=rpb, stats_mode=mode)
            torch.cuda.synchronize()
            assert torch.equal(out.view(torch.int16), full[r0:r1].view(torch.int16)), f"N={N} epi={epi} rows {r0}:{r1}: output"
            assert torch.equal(sst, st[r0:r1]), f"N={N} epi={epi} rows {r0}:{r1}: statistics"


@gpu
def test_fp8_gemm_in_place_writes_nothing_outside():
    M, N, K, ld, rpb = 384, 320, 256, 400, 128
    tiles = 2
    _, _, bias, resid, gate = gemm_case("iid", M, N, K, rpb, seed=7)
    Aq, sa, Wq, sw = _fp8_operands(M, N, K, seed=8)
    for epi in (3, 4):
        buf = torch.full((M + 130, ld), SENTINEL, dtype=torch.int16, device="cuda").view(torch.bfloat16)
        buf[:M, :N] = resid
        st = torch.full((M + 130, tiles + 1, 2), float("nan"), device="cuda")
        out = buf[:M]
        linear_fp8(Aq, sa, Wq, sw, out, bias=bias, epi=epi, resid=out, gate=gate if epi == 3 else None, rpb=rpb, stats=st, stats_mode=1)
        sep = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
        linear_fp8(Aq, sa, Wq, sw, sep, bias=bias, epi=epi, resid=resid, gate=gate if epi == 3 else None, rpb=rpb)
        torch.cuda.synchronize()
        raw = buf.view(torch.int16)
        assert (raw[M:] == SENTINEL).all(), f"epi={epi}: rows >= M written"
        assert (raw[:, N:] == SENTINEL).all(), f"epi={epi}: columns >= N written"
        assert torch.equal(buf[:M, :N].view(torch.int16), sep.view(torch.int16)), f"epi={epi}: in place differs from out of place"
        assert torch.isnan(st[M:]).all() and torch.isnan(st[:, tiles:]).all(), f"epi={epi}: statistics written outside [M, tiles)"


# ---------------------------------------------------------------------------------------------------- end to end
class _Fp8Linear:
    """Stands in for torch.nn.functional inside the oracle: F.linear on one of the FP8 weights applies the FP8 rule."""

    def __init__(self, quantized):
        self.quantized = quantized   # id(placeholder weight) -> (Wq, s_w)

    def __getattr__(self, name):
        return getattr(torch.nn.functional, name)

    def linear(self, x, w, b=None):
        if id(w) not in self.quantized:
            return torch.nn.functional.linear(x, w, b)
        wq, sw = self.quantized[id(w)]
        qa, sa = quantize_fp8_rows(x)
        y = (qa.float() @ wq.float().t()) * sa.unsqueeze(-1) * sw
        if b is not None:
            y = y + b.float()
        return y.to(x.dtype)


def fp8_oracle(sd, cfg, *inputs, monkeypatch):
    """The oracle's forward with the FP8 rule on the six block GEMMs (module docstring), in the dtype of `inputs`."""
    from oracle import dit_oracle as O

    sd = dict(sd)
    quantized = {}
    for i in range(cfg.num_layers):
        for name in FP8_LINEARS:
            k = f"blocks.{i}.{name}.weight"
            wq, sw = quantize_fp8_rows(sd[k])
            sd[k] = sd[k].clone()   # a tensor of its own, so that its id names this weight only
            quantized[id(sd[k])] = (wq.to(sd[k].device), sw.to(sd[k].device))
    with monkeypatch.context() as mp:
        mp.setattr(O, "F", _Fp8Linear(quantized))
        with torch.no_grad():
            return O.dit_forward(sd, cfg, *inputs)


def _model(cfg, sdb, **kw):
    import chronoedit_b200 as ce

    m = ce.ChronoEditTransformer3DModel(
        patch_size=cfg.patch_size, num_attention_heads=cfg.num_attention_heads, attention_head_dim=cfg.attention_head_dim,
        in_channels=cfg.in_channels, out_channels=cfg.out_channels, text_dim=cfg.text_dim, freq_dim=cfg.freq_dim,
        ffn_dim=cfg.ffn_dim, num_layers=cfg.num_layers, eps=cfg.eps, image_dim=cfg.image_dim,
        added_kv_proj_dim=cfg.added_kv_proj_dim, rope_max_seq_len=cfg.rope_max_seq_len,
        rope_temporal_skip_len=cfg.rope_temporal_skip_len, **kw)
    m.load_state_dict(sdb)
    m.enable_fp8()
    return m.cuda()


def _check_rule(out, ref32, ref16, what):
    e_ref, e_our = (ref16 - ref32).abs(), (out - ref32).abs()
    assert out.shape == ref32.shape and torch.isfinite(out).all()
    print(f"{what}: FP8 DiT vs fp32 FP8 emulation mean {e_our.mean():.3g} max {e_our.max():.3g}; "
          f"bf16 FP8 emulation mean {e_ref.mean():.3g} max {e_ref.max():.3g}")
    assert e_our.mean() <= 1.25 * e_ref.mean(), f"{what}: mean err {e_our.mean():.3g} vs bf16 emulation {e_ref.mean():.3g}"
    assert e_our.max() <= 2.0 * e_ref.max(), f"{what}: max err {e_our.max():.3g} vs bf16 emulation {e_ref.max():.3g}"


@gpu
@pytest.mark.parametrize("name", ["tiny_t2", "tiny_b2", "tiny_ragged"])
def test_fp8_dit_matches_fp8_emulation(name, monkeypatch):
    from oracle import cases

    case = cases.DIT_CASES[name]
    sd32 = cases.dit_weights(case)
    sdb = cases.to_bf16_state(sd32)
    x, t, text, img = cases.dit_inputs(case)
    m = _model(case.cfg, sdb)
    out = m(x.cuda(), t.cuda(), text.cuda(), img.cuda(), return_dict=False)[0].float().cpu()
    ref32 = fp8_oracle(sd32, case.cfg, x, t, text, img, monkeypatch=monkeypatch)
    ref16 = fp8_oracle(sdb, case.cfg, x.bfloat16(), t, text.bfloat16(), img.bfloat16(), monkeypatch=monkeypatch).float()
    _check_rule(out, ref32, ref16, name)


@gpu
def test_fp8_dit_bit_equalities():
    """Batch 2 against two batch-1 runs, CUDA-graph replay against eager, context cache against none: all bit for bit."""
    from oracle import cases

    case = cases.DIT_CASES["tiny_b2"]
    sdb = cases.to_bf16_state(cases.dit_weights(case))
    x, t, text, img = (v.cuda() for v in cases.dit_inputs(case))
    m = _model(case.cfg, sdb)
    both = m(x, t, text, img, return_dict=False)[0]
    for b in range(2):
        one = m(x[b:b + 1], t[b:b + 1], text[b:b + 1], img[b:b + 1], return_dict=False)[0]
        assert torch.equal(both[b:b + 1], one), f"sample {b}: batched and single FP8 evaluation differ"
    m.use_cuda_graph = True
    outs = [m(x, t, text, img, return_dict=False)[0] for _ in range(3)]   # eager, capture + replay, replay
    assert all(torch.equal(o, both) for o in outs), "CUDA-graph replay differs from eager"
    m.use_cuda_graph = False
    m.cache_context = True
    outs = [m(x, t, text, img, return_dict=False)[0] for _ in range(2)]   # fills the cache, reuses it
    assert all(torch.equal(o, both) for o in outs), "context cache differs from no cache"
    assert m.fp8_enabled


@gpu
def test_fp8_dit_14b_width_two_layers_at_720p(monkeypatch):
    """Two blocks at the 14B width (D 5120, 40 heads, ffn 13 824) with 7200 tokens (720p, 2 latent frames), the oracle on
    the GPU.  Also prints the FP8 and the bf16 DiT's error against the unquantized fp32 oracle."""
    from oracle import cases, dit_oracle as O

    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)   # the fp32 oracle's patch-embedding conv in fp32
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
    out = m(x, t, text, img, return_dict=False)[0].float()
    ref32 = fp8_oracle(sd32, cfg, x, t, text, img, monkeypatch=monkeypatch)
    ref16 = fp8_oracle(sdb, cfg, x.bfloat16(), t, text.bfloat16(), img.bfloat16(), monkeypatch=monkeypatch).float()
    _check_rule(out, ref32, ref16, "14B width, 2 layers")
    with torch.no_grad():
        exact = O.dit_forward(sd32, cfg, x, t, text, img)
    e8, e16 = (out - exact).abs(), (out_bf16 - exact).abs()
    print(f"against the unquantized fp32 oracle: FP8 mean {e8.mean():.3g} max {e8.max():.3g}; "
          f"bf16 mean {e16.mean():.3g} max {e16.max():.3g}; |exact| mean {exact.abs().mean():.3g}")
