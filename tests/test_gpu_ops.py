"""Operator-level parity of the sm_90a kernels, called through the C ABI (ctypes), against a plain PyTorch fp32
restatement of the same op on the same seeded inputs (fp64 for LayerNorm).  Tolerance: north_star's rtol=1e-3 / atol=1e-4 wherever the
op can expose an fp32 result (GEMM accumulators); for bf16 outputs the check is "equal to the fp32 reference rounded
to bf16, up to 1 bf16 ulp at rounding ties" expressed as rtol=2^-7 on |y|, plus a mean-error bound that a systematic
error would break.
"""
import math

import pytest
import torch

gpu = pytest.mark.gpu


def _lib():
    import chronoedit_b200._lib as L

    return L


def _bf16_close(got: torch.Tensor, ref_f32: torch.Tensor, what: str, ulp: float = 1.0, mean_tol: float = 2.5e-3):
    got = got.float().cpu()
    ref = ref_f32.float().cpu()
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    err = (got - ref).abs()
    # `ulp` bf16 ulps of the element itself (spacing 2^-7 relative) plus a floor of the same size at the tensor's typical magnitude
    tol = ulp * (2.0 ** -7) * ref.abs() + ulp * (2.0 ** -8) * ref.abs().mean()
    bad = (err > tol).float().mean().item()
    rel_mean = (err.mean() / ref.abs().mean().clamp_min(1e-12)).item()
    assert bad < 1e-3, f"{what}: {bad * 100:.3f}% of elements beyond {ulp} bf16 ulp (max err {err.max().item():.4g})"
    assert rel_mean < mean_tol, f"{what}: mean relative error {rel_mean:.3g}"


ROW_KINDS = ("iid", "block_offset", "outlier", "constant", "tile_constant")


def structured_rows(kind: str, rows: int, D: int, g: torch.Generator, block: int = 256) -> torch.Tensor:
    """fp32 [rows, D] row data on g's device, shaped so that row statistics merged from per-block partials go visibly wrong:
      iid            N(0.5, 3^2)
      block_offset   N(0, 1) plus an offset ~ N(0, 2^2) per (row, block of `block` columns): the block means differ
      outlier        N(0, 1) with +-60 on the first column of a block (the pivot of a GEMM statistics tile) and -40 elsewhere
      constant       one value per row (LayerNorm must give exactly its shift)
      tile_constant  one value per (row, block): all of the variance is between blocks
    """
    dev = g.device
    nb = (D + block - 1) // block

    def per_block(v):
        return v.repeat_interleave(block, dim=1)[:, :D]

    if kind == "iid":
        return torch.randn(rows, D, generator=g, device=dev) * 3 + 0.5
    if kind == "block_offset":
        return torch.randn(rows, D, generator=g, device=dev) + per_block(torch.randn(rows, nb, generator=g, device=dev) * 2)
    if kind == "outlier":
        x = torch.randn(rows, D, generator=g, device=dev)
        k = nb // 2
        x[:, k * block] += 60 * torch.sign(torch.randn(rows, generator=g, device=dev))
        x[:, min(D - 1, k * block + block // 2 + 13)] -= 40
        return x
    if kind == "constant":
        return (torch.randn(rows, 1, generator=g, device=dev) * 3 + 0.5).expand(rows, D).contiguous()
    if kind == "tile_constant":
        return per_block(torch.randn(rows, nb, generator=g, device=dev) * 2 + 0.5)
    raise ValueError(kind)


def run_linear(M, N, K, epi, seed=0, rows_per_batch=None):
    L = _lib()
    lib = L.lib()
    g = torch.Generator(device="cpu").manual_seed(seed)
    A = (torch.randn(M, K, generator=g) * 0.5).bfloat16().cuda()
    W = (torch.randn(N, K, generator=g) / math.sqrt(K)).bfloat16().cuda()
    bias = (torch.randn(N, generator=g) * 0.1).bfloat16().cuda()
    resid = torch.randn(M, N, generator=g).bfloat16().cuda()
    rpb = rows_per_batch or M
    nb = (M + rpb - 1) // rpb
    gate = torch.randn(nb, N, generator=g).float().cuda()
    out = torch.zeros(M, N, dtype=torch.bfloat16, device="cuda")
    out32 = torch.zeros(M, N, dtype=torch.float32, device="cuda")
    L.check(lib.ce_linear_bf16(L.ptr(A), K, L.ptr(W), K, L.ptr(bias), L.ptr(out), N, L.ptr(out32), M, N, K, epi, L.ptr(resid), N,
                               L.ptr(gate), N, rpb, L.current_stream()))
    torch.cuda.synchronize()
    acc = A.float() @ W.float().t() + bias.float()
    # the stated tolerance on the fp32 accumulator
    torch.testing.assert_close(out32, acc, rtol=1e-3, atol=1e-4)
    y = acc.bfloat16().float()
    if epi == 1:
        ref = torch.nn.functional.gelu(y, approximate="tanh")
    elif epi == 2:
        ref = torch.nn.functional.gelu(y)
    elif epi == 3:
        gfull = gate.repeat_interleave(rpb, dim=0)[:M]
        ref = resid.float() + y * gfull
    elif epi == 4:
        ref = resid.float() + y
    else:
        ref = y
    _bf16_close(out, ref, f"linear M={M} N={N} K={K} epi={epi}")


@gpu
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (256, 512, 512), (300, 768, 1024), (7200, 256, 256), (77, 64, 144), (513, 128, 320),
                                   (1000, 1280, 1280)])
def test_linear_bias(M, N, K):
    run_linear(M, N, K, 0)


@gpu
@pytest.mark.parametrize("epi", [1, 2, 3, 4])
def test_linear_epilogues(epi):
    run_linear(391, 640, 384, epi, seed=epi, rows_per_batch=200)


@gpu
def test_linear_large_k_many_tiles():
    # more tiles than SMs, K deep enough to wrap the 4-stage ring many times
    run_linear(2304, 5120, 2048, 3, seed=7, rows_per_batch=1152)


@gpu
def test_linear_linearity():
    """Size-independent property at a 14B-shaped tile count: f(A1 + A2) == f(A1) + f(A2) on the fp32 accumulators."""
    L = _lib()
    lib = L.lib()
    M, N, K = 1024, 5120, 5120
    g = torch.Generator(device="cpu").manual_seed(3)
    A1 = (torch.randint(-4, 5, (M, K), generator=g).float() / 8).bfloat16().cuda()  # exactly representable sums
    A2 = (torch.randint(-4, 5, (M, K), generator=g).float() / 8).bfloat16().cuda()
    W = (torch.randint(-8, 9, (N, K), generator=g).float() / 16).bfloat16().cuda()
    outs = []
    for A in (A1, A2, (A1.float() + A2.float()).bfloat16()):
        o = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
        o32 = torch.empty(M, N, dtype=torch.float32, device="cuda")
        L.check(lib.ce_linear_bf16(L.ptr(A), K, L.ptr(W), K, None, L.ptr(o), N, L.ptr(o32), M, N, K, 0, None, 0, None, 0, 1, L.current_stream()))
        outs.append(o32)
    torch.cuda.synchronize()
    # all products/sums are exact in fp32 at these magnitudes -> bit-exact linearity
    assert torch.equal(outs[0] + outs[1], outs[2])
    assert torch.equal(outs[2], (A1.float() + A2.float()) @ W.float().t())


def run_attention(B, H, Lq, Lk, seed=0, accumulate=False, strided=True, key_ramp=0.0):
    L = _lib()
    lib = L.lib()
    hd = 128
    g = torch.Generator(device="cpu").manual_seed(seed)
    D = H * hd
    if strided and Lq == Lk:  # q|k|v packed like the QKV GEMM output
        qkv = torch.randn(B, Lq, 3 * D, generator=g).bfloat16().cuda()
        q, k, v = qkv[..., :D], qkv[..., D:2 * D], qkv[..., 2 * D:]
        ldq = ldk = ldv = 3 * D
    else:
        q = torch.randn(B, Lq, D, generator=g).bfloat16().cuda()
        kv = torch.randn(B, Lk, 2 * D, generator=g).bfloat16().cuda()
        k, v = kv[..., :D], kv[..., D:]
        ldq, ldk, ldv = D, 2 * D, 2 * D
    if key_ramp:  # keys grow along the sequence: the running row maximum keeps jumping by more than the lazy-rescale threshold
        ramp = (1.0 + key_ramp * torch.arange(Lk, dtype=torch.float32) / Lk).view(1, Lk, 1).cuda()
        k.copy_((k.float() * ramp).bfloat16())
    prev = torch.randn(B, Lq, D, generator=g).bfloat16().cuda()
    out = prev.clone() if accumulate else torch.zeros(B, Lq, D, dtype=torch.bfloat16, device="cuda")
    scale = 1.0 / math.sqrt(hd)
    L.check(lib.ce_attention_bf16(L.ptr(q), ldq, L.ptr(k), ldk, L.ptr(v), ldv, L.ptr(out), D, B, H, Lq, Lk, scale, int(accumulate),
                                  L.current_stream()))
    torch.cuda.synchronize()
    qf = q.float().reshape(B, Lq, H, hd).transpose(1, 2)
    kf = k.float().reshape(B, Lk, H, hd).transpose(1, 2)
    vf = v.float().reshape(B, Lk, H, hd).transpose(1, 2)
    p = torch.softmax(qf @ kf.transpose(-1, -2) * scale, dim=-1)
    ref = (p @ vf).transpose(1, 2).reshape(B, Lq, D)
    if accumulate:
        ref = ref.bfloat16().float() + prev.float()
    # P is rounded to bf16 before P@V (as flash kernels do): allow 2 bf16 ulp, keep the mean-error bound tight
    _bf16_close(out, ref, f"attention B={B} H={H} Lq={Lq} Lk={Lk} acc={accumulate}", ulp=2.0, mean_tol=4e-3)


@gpu
@pytest.mark.parametrize("B,H,Lq,Lk", [(1, 2, 128, 128), (1, 2, 256, 384), (2, 3, 234, 234), (1, 2, 2048, 2048), (1, 1, 130, 1),
                                       (1, 2, 100, 129)])
def test_attention_self(B, H, Lq, Lk):
    run_attention(B, H, Lq, Lk, seed=Lq + Lk)


@gpu
@pytest.mark.parametrize("Lq,ramp", [(1024, 6.0), (1500, 12.0), (640, -0.9)])
def test_attention_self_growing_and_shrinking_scores(Lq, ramp):
    """Exercises the rescale paths of the online softmax (incl. the redo after a failed speculation on the previous maximum):
    |k| grows (or shrinks) along the keys, so later key tiles raise the row maximum by far more than 2^8 again and again."""
    run_attention(1, 2, Lq, Lq, seed=Lq, key_ramp=ramp)


@gpu
@pytest.mark.parametrize("Lk,acc", [(512, False), (257, True), (257, False), (7, True)])
def test_attention_cross(Lk, acc):
    run_attention(2, 2, 300, Lk, seed=Lk, accumulate=acc, strided=False)


@gpu
def test_attention_rows_sum_property():
    """Full-size property (L = 7200, the 720p/2-frame token count): with V = 1 the output of softmax(QK^T)V is exactly
    the softmax row sum = 1, whatever Q and K are."""
    _rows_sum_property()


def _rows_sum_property():
    L = _lib()
    lib = L.lib()
    B, H, Lq, hd = 1, 2, 7200, 128
    D = H * hd
    g = torch.Generator(device="cpu").manual_seed(11)
    q = (torch.randn(B, Lq, D, generator=g) * 2).bfloat16().cuda()
    k = (torch.randn(B, Lq, D, generator=g) * 2).bfloat16().cuda()
    v = torch.ones(B, Lq, D, dtype=torch.bfloat16, device="cuda")
    out = torch.zeros(B, Lq, D, dtype=torch.bfloat16, device="cuda")
    L.check(lib.ce_attention_bf16(L.ptr(q), D, L.ptr(k), D, L.ptr(v), D, L.ptr(out), D, B, H, Lq, Lq, 1.0 / math.sqrt(hd), 0, L.current_stream()))
    torch.cuda.synchronize()
    torch.testing.assert_close(out.float(), torch.ones_like(out, dtype=torch.float32), rtol=0, atol=2 ** -7)


@gpu
@pytest.mark.parametrize("version", [0])
def test_attention_alternative_kernels(version):
    """The attention kernel selected by its explicit version number (the sm_90a build has one, version 0) against the same oracle
    comparisons and the full-size row-sum property -- the latter has thousands of running-maximum updates (scores scaled x2)."""
    L = _lib()
    L.check(L.lib().ce_debug_attention_kernel(version))
    try:
        for (B, H, Lq, Lk) in [(1, 2, 256, 384), (2, 3, 300, 300), (1, 2, 2048, 2048), (1, 1, 384, 257), (1, 2, 1000, 129 + 256)]:
            run_attention(B, H, Lq, Lk, seed=Lq + Lk + version)
        _rows_sum_property()
    finally:
        L.check(L.lib().ce_debug_attention_kernel(-1))


def layer_norm_f64(x: torch.Tensor, eps: float) -> torch.Tensor:
    """fp64 LayerNorm over the last dim of the stored x.  The mean is sum / D, which is exact for a constant row, so there
    x - mean is exactly 0 (torch's fp32 layer_norm is off by an ulp of the mean there, which rstd = 1/sqrt(eps) magnifies)."""
    xd = x.double()
    d = xd - xd.sum(-1, keepdim=True) / x.shape[-1]
    return d / torch.sqrt((d * d).mean(-1, keepdim=True) + eps)


def _with_kinds(iid_cases, structured_cases):
    """iid cases keep their plain ids; every structured case runs on each non-iid kind of structured_rows."""
    return ([pytest.param(*c, "iid", id="-".join(map(str, c))) for c in iid_cases] +
            [pytest.param(*c, k, id="-".join(map(str, c + (k,)))) for k in ROW_KINDS[1:] for c in structured_cases])


@gpu
@pytest.mark.parametrize("rows,D,mode,kind", _with_kinds(
    [(300, 256, "mod"), (77, 5120, "mod"), (64, 1280, "affine"), (33, 384, "plain"),
     (4739, 5120, "mod"), (4736, 3072, "affine"), (5003, 5120, "plain")],   # large row counts with ragged tails
    [(300, 384, "plain"), (64, 1280, "affine"), (4739, 5120, "mod")]))
def test_layernorm(rows, D, mode, kind):
    L = _lib()
    lib = L.lib()
    g = torch.Generator(device="cpu").manual_seed(rows)
    x = structured_rows(kind, rows, D, g).bfloat16().cuda()
    rpb = 100
    nb = (rows + rpb - 1) // rpb
    mod = torch.randn(nb, 6, D, generator=g).float().cuda()
    w = (1 + 0.1 * torch.randn(D, generator=g)).float().cuda()
    b = (0.1 * torch.randn(D, generator=g)).float().cuda()
    y = torch.zeros(rows, D, dtype=torch.bfloat16, device="cuda")
    eps = 1e-6
    if mode == "mod":
        scale, shift = mod[:, 1], mod[:, 0]
        L.check(lib.ce_layernorm_bf16(L.ptr(x), D, L.ptr(y), D, rows, D, eps, L.ptr(scale), L.ptr(shift), 6 * D, rpb, None, None, L.current_stream()))
        ln = layer_norm_f64(x, eps)
        ref = ln * (1 + scale.double().repeat_interleave(rpb, 0)[:rows]) + shift.double().repeat_interleave(rpb, 0)[:rows]
    elif mode == "affine":
        L.check(lib.ce_layernorm_bf16(L.ptr(x), D, L.ptr(y), D, rows, D, eps, None, None, 0, 0, L.ptr(w), L.ptr(b), L.current_stream()))
        ref = layer_norm_f64(x, eps) * w.double() + b.double()
    else:
        L.check(lib.ce_layernorm_bf16(L.ptr(x), D, L.ptr(y), D, rows, D, eps, None, None, 0, 0, None, None, L.current_stream()))
        ref = layer_norm_f64(x, eps)
    torch.cuda.synchronize()
    _bf16_close(y, ref, f"layernorm {mode} {kind} rows={rows} D={D}")
    if kind == "constant":   # x - mean is exactly 0: the output is exactly the shift / bias (or 0)
        assert torch.equal(y.float().cpu(), ref.bfloat16().float().cpu()), f"layernorm {mode} of constant rows is not exact"


@gpu
@pytest.mark.parametrize("rows,H,rope,kind", _with_kinds(
    [(234, 3, True), (126, 2, False), (600, 40, True), (4746, 40, True), (4740, 24, False)],   # last two: large, ragged
    [(600, 40, True), (126, 2, False)]))
def test_rmsnorm_rope(rows, H, rope, kind):
    from oracle import dit_oracle as O

    L = _lib()
    lib = L.lib()
    hd = 128
    D = H * hd
    g = torch.Generator(device="cpu").manual_seed(rows)
    ld = 3 * D
    buf = torch.randn(rows, ld, generator=g)
    if kind != "iid":
        buf[:, D:2 * D] = structured_rows(kind, rows, D, g)
    buf = buf.bfloat16().cuda()
    w = (1 + 0.1 * torch.randn(D, generator=g)).bfloat16().cuda()
    before = buf.clone()
    cfg = O.DiTConfig.tiny(heads=H)
    frames, hp, wp = 2, 3, rows // 6
    assert frames * hp * wp == rows
    cos = sin = None
    if rope:
        cos_h = torch.empty(rows, hd // 2, dtype=torch.float32)
        sin_h = torch.empty(rows, hd // 2, dtype=torch.float32)
        L.check(lib.ce_rope_table_host(hd, frames, hp, wp, 1024, 8, 10000.0, L.ptr(cos_h), L.ptr(sin_h)))
        # the table itself against the oracle's complex128 table (transformer_chronoedit.py:168-213)
        fr = O.rope_table(cfg, frames, hp * 2, wp * 2)[0, 0]
        torch.testing.assert_close(cos_h.double(), fr.real, rtol=0, atol=1e-7)
        torch.testing.assert_close(sin_h.double(), fr.imag, rtol=0, atol=1e-7)
        cos, sin = cos_h.cuda(), sin_h.cuda()
    L.check(lib.ce_rmsnorm_rope_bf16(L.ptr(buf[:, D:]), ld, rows, D, 1e-6, L.ptr(w), L.ptr(cos), L.ptr(sin), rows, hd, L.current_stream()))
    torch.cuda.synchronize()
    assert torch.equal(buf[:, :D], before[:, :D]) and torch.equal(buf[:, 2 * D:], before[:, 2 * D:]), "wrote outside its columns"
    x = before[:, D:2 * D].cpu()
    y = O._rms_norm_across_heads(x[None], w.cpu(), 1e-6)          # bf16 path of the oracle
    if rope:
        yh = y.unflatten(2, (H, hd)).transpose(1, 2)
        yh = O._apply_rope(yh, O.rope_table(cfg, frames, hp * 2, wp * 2))
        y = yh.transpose(1, 2).flatten(2, 3)
    _bf16_close(buf[:, D:2 * D], y[0].float(), f"rmsnorm_rope {kind} rows={rows} H={H} rope={rope}")


@gpu
@pytest.mark.parametrize("Lq,Lk,Lk2,version", [(300, 512, 257, -1), (7200, 512, 257, -1), (130, 7, 300, -1), (300, 7, 300, -1), (513, 640, 129, -1)])
def test_attention_dual_source(Lq, Lk, Lk2, version):
    """text + image cross-attention in one launch == sum of two separate bf16 SDPAs (transformer_chronoedit.py:84-104)."""
    L = _lib()
    lib = L.lib()
    L.check(lib.ce_debug_attention_kernel(version))
    try:
        _run_attention_dual(L, lib, Lq, Lk, Lk2)
    finally:
        L.check(lib.ce_debug_attention_kernel(-1))


def _run_attention_dual(L, lib, Lq, Lk, Lk2):
    B, H, hd = 2, 2, 128
    D = H * hd
    g = torch.Generator(device="cpu").manual_seed(Lq + Lk2)
    q = torch.randn(B, Lq, D, generator=g).bfloat16().cuda()
    kv = torch.randn(B, Lk, 2 * D, generator=g).bfloat16().cuda()
    kv2 = torch.randn(B, Lk2, 2 * D, generator=g).bfloat16().cuda()
    out = torch.zeros(B, Lq, D, dtype=torch.bfloat16, device="cuda")
    scale = 1.0 / math.sqrt(hd)
    L.check(lib.ce_attention_dual_bf16(L.ptr(q), D, L.ptr(kv), 2 * D, L.ptr(kv[..., D:]), 2 * D, L.ptr(kv2), 2 * D, L.ptr(kv2[..., D:]), 2 * D,
                                       L.ptr(out), D, B, H, Lq, Lk, Lk2, scale, L.current_stream()))
    torch.cuda.synchronize()

    def sdpa(k, v, n):
        qf = q.float().reshape(B, Lq, H, hd).transpose(1, 2)
        kf = k.float().reshape(B, n, H, hd).transpose(1, 2)
        vf = v.float().reshape(B, n, H, hd).transpose(1, 2)
        return (torch.softmax(qf @ kf.transpose(-1, -2) * scale, -1) @ vf).transpose(1, 2).reshape(B, Lq, D)

    ref = sdpa(kv[..., :D], kv[..., D:], Lk).bfloat16().float() + sdpa(kv2[..., :D], kv2[..., D:], Lk2).bfloat16().float()
    # a sum of two independently rounded bf16 tensors: one more rounding than a single SDPA -> 3 ulp
    _bf16_close(out, ref, f"dual attention Lq={Lq} Lk={Lk} Lk2={Lk2}", ulp=3.0, mean_tol=5e-3)
