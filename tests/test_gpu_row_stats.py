"""The DiT's fused row-statistics path, operator by operator, against fp64 statistics of the STORED bf16 tensors.

When D % 256 == 0 the GEMM that writes a row also writes, per (row, N tile), the statistics of the values it stored
(stats_mode 1: pivot-shifted (mean, M2); stats_mode 2: sum of squares), and the LayerNorm / RMSNorm that follows merges
those partials (Chan's pairwise update in a warp butterfly) instead of reducing over the row.  Every test runs on the
structured rows of test_gpu_ops.structured_rows (block offsets, outliers on a tile's pivot column, constant rows, rows
constant within each tile), because on iid rows every tile has the same mean and a merge that drops the between-tile
term, or weights a partial last tile as a full one, still passes.

Tolerances.  The GEMM partials are checked against bounds derived from fp32 arithmetic over the n <= 256 terms of a tile
(u = 2^-24), with d = y - y[pivot] the pivot-shifted values, A1 = sum |d|, A2 = sum d^2, S = |sum d|:
    mean   2u ((n + 2) A1 / n + |mean|)                 n-term sum, the division, the pivot add
    M2     2u ((n + 3) A2 + (2n + 3) S A1 / n)          sum of squares minus (sum d)^2 / n, each with its own roundings
    sum y^2   2u (n + 1) sum y^2
(the factor 2 covers second-order terms).  The normalised bf16 outputs use the rule of test_gpu_ops.py: within 1 bf16
ulp of the fp64 reference for all but 0.1% of the elements and a mean relative error < 2.5e-3; constant rows must give
exactly bf16(shift).
"""
import math
import os

import pytest
import torch

from tests.test_gpu_ops import ROW_KINDS, _bf16_close, layer_norm_f64, structured_rows

gpu = pytest.mark.gpu
U = 2.0 ** -24   # fp32 unit roundoff
EPS = 1e-6


def _lib():
    import chronoedit_b200._lib as L

    return L


def _p(t):
    return None if t is None else t.data_ptr()


def tile_width(N):
    """N tile width of the GEMM (gemm_tile_n): the granularity of its statistics."""
    return 256 if N >= 256 else (128 if N >= 128 else 64)


def linear_ex(A, W, out, *, bias=None, epi=0, resid=None, gate=None, rpb=1, stats=None, stats_mode=0, group_m=0):
    L = _lib()
    M, K = A.shape
    N = W.shape[0]
    a = L.LinearArgsC(A=_p(A), lda=K, W=_p(W), ldw=K, M=M, N=N, K=K, out=_p(out), ldo=out.shape[1], bias=_p(bias), epilogue=epi,
                      resid=_p(resid), ldr=0 if resid is None else resid.shape[1], gate=_p(gate),
                      gate_stride=0 if gate is None else gate.shape[1], rows_per_batch=rpb, stats_out=_p(stats),
                      stats_ld=0 if stats is None else stats.shape[1], stats_mode=stats_mode, group_m=group_m)
    L.check(L.lib().ce_linear_ex_bf16(a, L.current_stream()))


def gemm_case(kind, M, N, K, rpb, seed):
    """Operands of one Linear whose output rows have the structure `kind` (see structured_rows), on the GPU.
    Without a residual the structure comes from the bias (the same for every row); with one, from the residual rows.
    For the constant kinds W = 0, so the output is exactly bias / residual / gate combined per row or per tile."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    tn = tile_width(N)
    nbat = (M + rpb - 1) // rpb
    A = (torch.randn(M, K, generator=g, device="cuda") * 0.5).bfloat16()
    const = kind in ("constant", "tile_constant")
    W = torch.zeros(N, K, device="cuda") if const else torch.randn(N, K, generator=g, device="cuda") / math.sqrt(K)
    bias = structured_rows(kind, 1, N, g, block=tn)[0] * (1.0 if const else 0.1)
    if kind == "outlier":   # structured_rows' outliers at full size on the bias too
        bias = bias * 10
    resid = structured_rows(kind, M, N, g, block=tn)
    if kind == "constant":
        gate = torch.randn(nbat, 1, generator=g, device="cuda").expand(nbat, N)
    elif kind == "tile_constant":
        gate = torch.randn(nbat, (N + tn - 1) // tn, generator=g, device="cuda").repeat_interleave(tn, dim=1)[:, :N]
    else:
        gate = torch.randn(nbat, N, generator=g, device="cuda")
    return A, W.bfloat16(), bias.bfloat16(), resid.bfloat16(), gate.float().contiguous()


def ref_output(A, W, bias, resid, gate, epi, rpb):
    """fp32 restatement of the epilogue on the bf16-rounded Linear output (as test_gpu_ops.run_linear)."""
    y = (A.float() @ W.float().t() + bias.float()).bfloat16().float()
    if epi == 3:
        return resid.float() + y * gate.repeat_interleave(rpb, dim=0)[:A.shape[0]]
    if epi == 4:
        return resid.float() + y
    return y


def ref_partials(z, tn):
    """fp64 per-tile statistics of the stored z [M, N] and their fp32 error bounds (module docstring).  All [M, tiles]."""
    z = z.double()
    M, N = z.shape
    r = {k: [] for k in ("mean", "m2", "ss", "tol_mean", "tol_m2", "tol_ss")}
    for t in range((N + tn - 1) // tn):
        c = z[:, t * tn:min(N, (t + 1) * tn)]
        n = c.shape[1]
        mean = c.mean(1)
        d = c - c[:, :1]
        a1, a2, s = d.abs().sum(1), (d * d).sum(1), d.sum(1).abs()
        ss = (c * c).sum(1)
        r["mean"].append(mean)
        r["m2"].append(((c - mean[:, None]) ** 2).sum(1))
        r["ss"].append(ss)
        r["tol_mean"].append(2 * U * ((n + 2) * a1 / n + mean.abs()))
        r["tol_m2"].append(2 * U * ((n + 3) * a2 + (2 * n + 3) * s * a1 / n))
        r["tol_ss"].append(2 * U * (n + 1) * ss)
    return {k: torch.stack(v, 1) for k, v in r.items()}


def _within(got, ref, tol, what):
    err = (got.double() - ref).abs()
    bad = err > tol
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.numel()} beyond the fp32 bound; worst err/bound "
                           f"{(err / tol.clamp_min(1e-300)).max().item():.3g} (err {err.max().item():.3g})")


def run_gemm_stats(kind, M, N, K, epi, rpb, seed, pad_rows=37, pad_tiles=3):
    """One Linear without statistics and with stats_mode 1 and 2; returns (out, {mode: stats [M, tiles, 2]}) after checking
    that `out` does not depend on the statistics and that nothing outside [M, tiles) of the stats buffer is written."""
    A, W, bias, resid, gate = gemm_case(kind, M, N, K, rpb, seed)
    tiles = (N + tile_width(N) - 1) // tile_width(N)
    kw = dict(bias=bias, epi=epi, resid=resid if epi in (3, 4) else None, gate=gate if epi == 3 else None, rpb=rpb)
    plain = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    linear_ex(A, W, plain, **kw)
    res = {}
    for mode in (1, 2):
        out = torch.empty_like(plain)
        st = torch.full((M + pad_rows, tiles + pad_tiles, 2), float("nan"), device="cuda")
        linear_ex(A, W, out, stats=st, stats_mode=mode, **kw)
        torch.cuda.synchronize()
        assert torch.equal(out, plain), f"{kind} N={N} epi={epi}: stats_mode {mode} changed the stored output"
        assert torch.isnan(st[M:]).all(), f"stats_mode {mode} wrote rows >= M"
        assert torch.isnan(st[:M, tiles:]).all(), f"stats_mode {mode} wrote entries past the last tile"
        res[mode] = st[:M, :tiles]
    return plain, res, (A, W, bias, resid, gate)


# ---------------------------------------------------------------------------------------------------- a. GEMM partials
@gpu
@pytest.mark.parametrize("epi", [0, 3, 4])
@pytest.mark.parametrize("M,N", [(300, 64), (300, 192), (300, 640), (300, 5120), (300, 3 * 5120), (300, 8192),
                                 (4739, 5120), (4739, 3 * 5120), (4739, 8192)])
def test_gemm_stats_partials(M, N, epi):
    """stats_mode 1 (mean, M2) and 2 (sum y^2) of every (row, tile) against fp64 statistics of the stored bf16 output, at each
    tile width (64, 128 with a partial last tile, 256 with a 128-wide last tile, 20 / 60 / 32 tiles), ragged M and a ragged
    rows_per_batch.  The stored output itself is checked against the fp32 epilogue, so partials taken before the residual /
    gate, or counting columns that were not stored, fail here.  Bounds: module docstring."""
    K, rpb = 200, 97 if M == 300 else 1200
    for i, kind in enumerate(ROW_KINDS):
        out, st, ops = run_gemm_stats(kind, M, N, K, epi, rpb, seed=1000 * epi + N + M + i)
        what = f"{kind} M={M} N={N} epi={epi}"
        _bf16_close(out, ref_output(*ops, epi, rpb), what)
        ref = ref_partials(out, tile_width(N))
        _within(st[1][..., 0], ref["mean"], ref["tol_mean"], what + " tile mean")
        _within(st[1][..., 1], ref["m2"], ref["tol_m2"], what + " tile M2")
        _within(st[2][..., 0], ref["ss"], ref["tol_ss"], what + " tile sum of squares")
        assert (st[2][..., 1] == 0).all(), what + ": stats_mode 2 second component"
        if kind == "constant":
            assert (st[1][..., 1] == 0).all() and torch.equal(st[1][..., 0].double(), ref["mean"]), what + ": constant rows are exact"


@gpu
def test_gemm_stats_group_m_invariant():
    """Tile rasterisation must not change any result: group_m in {1, 3, 16, 64} at 38 x 20 tiles (more than the SMs, and 38 is
    not a multiple of 3, 16 or 64, so the last group is partial) gives bit-identical outputs and statistics."""
    M, N, K, rpb = 4739, 5120, 200, 1200
    A, W, bias, resid, gate = gemm_case("block_offset", M, N, K, rpb, seed=5)
    tiles = N // 256
    first = None
    for gm in (1, 3, 16, 64):
        got = []
        for mode in (1, 2):
            out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
            st = torch.full((M, tiles, 2), float("nan"), device="cuda")
            linear_ex(A, W, out, bias=bias, epi=3, resid=resid, gate=gate, rpb=rpb, stats=st, stats_mode=mode, group_m=gm)
            got += [out, st]
        torch.cuda.synchronize()
        if first is None:
            first = got
            assert not any(torch.isnan(t).any() for t in got[1::2]), "a (row, tile) statistic was not written"
        else:
            for a, b in zip(first, got):
                assert torch.equal(a, b), f"group_m={gm} differs from group_m=1"


# ---------------------------------------------------------------------------------------------------- b. stats LayerNorm
def _mod_tables(g, nbat, D):
    mod = torch.randn(nbat, 6, D, generator=g, device="cuda")
    mod1p = mod.clone()
    mod1p[:, 1] += 1   # the (1 + scale) table the DiT keeps
    w = 1 + 0.1 * torch.randn(D, generator=g, device="cuda")
    b = 0.1 * torch.randn(D, generator=g, device="cuda")
    return mod, mod1p, w, b


def _ln_ref(x, mode, mod, w, b, rpb):
    """fp64 LayerNorm of the stored bf16 x, then the modulation / affine in fp64."""
    ln = layer_norm_f64(x, EPS)
    if mode.startswith("mod"):
        rows = x.shape[0]
        scale = mod[:, 1].double().repeat_interleave(rpb, 0)[:rows]
        shift = mod[:, 0].double().repeat_interleave(rpb, 0)[:rows]
        return ln * (1 + scale) + shift
    if mode == "affine":
        return ln * w.double() + b.double()
    return ln


def _ln_args(mode, mod, mod1p, w, b, D):
    """(scale, shift, mod_stride, weight, bias, scale_is_1p) of the C call."""
    L = _lib()
    if mode == "mod0":
        return L.ptr(mod[:, 1]), L.ptr(mod[:, 0]), 6 * D, None, None, 0
    if mode == "mod1":
        return L.ptr(mod1p[:, 1]), L.ptr(mod1p[:, 0]), 6 * D, None, None, 1
    if mode == "affine":
        return None, None, 0, L.ptr(w), L.ptr(b), 0
    return None, None, 0, None, None, 0


def _check_ln(y, ref, what, kind):
    _bf16_close(y, ref, what)
    if kind == "constant":
        assert torch.equal(y.float(), ref.bfloat16().float()), what + ": constant rows must give exactly bf16(shift)"


LN_CASES = [(300, D, m) for D in (256, 640, 5120, 8192) for m in ("mod0", "mod1", "affine", "plain")] + \
           [(4739, 5120, "mod1"), (4739, 8192, "plain")]


@gpu
@pytest.mark.parametrize("rows,D,mode", LN_CASES)
def test_layernorm_stats_after_gemm(rows, D, mode):
    """GEMM (stats_mode 1, residual epilogue, as the DiT's out-projections) -> ce_layernorm_stats_bf16, against fp64 LayerNorm of
    the stored x, and against the row-reducing ce_layernorm_bf16 on the same x (2 ulp: both are within 1 ulp of the reference).
    Catches a merge without Chan's between-tile term (block offsets, tile-constant rows), a partial last tile weighted as a full
    one (D = 640), and an ignored scale_is_1p (mod0 vs mod1).  rows_per_batch does not divide the row count.  In mode mod1 the
    call is also made with stats = NULL (the kernel reduces over the row): with the (1 + scale) table added in fp32 by torch it must
    give ce_layernorm_bf16's bits for the plain scale."""
    L = _lib()
    lib = L.lib()
    rpb = 97 if rows == 300 else 1200
    tn = tile_width(D)
    tiles = (D + tn - 1) // tn
    for i, kind in enumerate(ROW_KINDS):
        A, W, bias, resid, gate = gemm_case(kind, rows, D, 136, rpb, seed=D + rows + i)
        x = torch.empty(rows, D, dtype=torch.bfloat16, device="cuda")
        st = torch.full((rows, tiles + 1, 2), float("nan"), device="cuda")
        linear_ex(A, W, x, bias=bias, epi=4, resid=resid, stats=st, stats_mode=1)
        g = torch.Generator(device="cuda").manual_seed(i)
        mod, mod1p, w, b = _mod_tables(g, (rows + rpb - 1) // rpb, D)
        scale, shift, ms, wp, bp, is1p = _ln_args(mode, mod, mod1p, w, b, D)
        y = torch.empty_like(x)
        L.check(lib.ce_layernorm_stats_bf16(L.ptr(x), D, L.ptr(y), D, rows, D, EPS, scale, shift, ms, rpb, wp, bp, is1p, L.ptr(st),
                                            tiles + 1, tiles, tn, L.current_stream()))
        y_row = torch.empty_like(x)
        s0, h0, ms0, _, _, _ = _ln_args("mod0" if mode.startswith("mod") else mode, mod, mod1p, w, b, D)
        L.check(lib.ce_layernorm_bf16(L.ptr(x), D, L.ptr(y_row), D, rows, D, EPS, s0, h0, ms0, rpb, wp, bp, L.current_stream()))
        if mode == "mod1":
            y_null = torch.empty_like(x)
            L.check(lib.ce_layernorm_stats_bf16(L.ptr(x), D, L.ptr(y_null), D, rows, D, EPS, scale, shift, ms, rpb, wp, bp, is1p, None, 0, 0,
                                                0, L.current_stream()))
        torch.cuda.synchronize()
        what = f"layernorm(stats) {mode} {kind} rows={rows} D={D}"
        _check_ln(y, _ln_ref(x, mode, mod, w, b, rpb), what, kind)
        _bf16_close(y, y_row.float(), what + " vs ce_layernorm_bf16", ulp=2.0)
        if mode == "mod1":
            assert torch.equal(y_null, y_row), what + ": stats = NULL with (1 + scale) differs from ce_layernorm_bf16 with scale"


@gpu
@pytest.mark.parametrize("D,tile_n", [(768, 256), (640, 64), (5120, 176), (8192, 256), (5120, 5120)])
def test_layernorm_stats_hand_built_partials(D, tile_n):
    """The merge on its own: exact (fp64, rounded to fp32) tile partials built on the host, 1 to 32 tiles, including a 16-column
    last tile (5120 = 29 x 176 + 16) whose count must not be taken as tile_n."""
    L = _lib()
    lib = L.lib()
    rows, rpb = 301, 100
    tiles = (D + tile_n - 1) // tile_n
    for i, kind in enumerate(ROW_KINDS):
        g = torch.Generator(device="cuda").manual_seed(D + tile_n + i)
        x = structured_rows(kind, rows, D, g).bfloat16()
        xd = x.double()
        st = torch.full((rows, tiles + 2, 2), float("nan"), device="cuda")
        for t in range(tiles):
            c = xd[:, t * tile_n:min(D, (t + 1) * tile_n)]
            m = c.mean(1)
            st[:, t, 0] = m.float()
            st[:, t, 1] = ((c - m[:, None]) ** 2).sum(1).float()
        mod, mod1p, w, b = _mod_tables(g, (rows + rpb - 1) // rpb, D)
        for mode in ("mod1", "plain"):
            scale, shift, ms, wp, bp, is1p = _ln_args(mode, mod, mod1p, w, b, D)
            y = torch.empty_like(x)
            L.check(lib.ce_layernorm_stats_bf16(L.ptr(x), D, L.ptr(y), D, rows, D, EPS, scale, shift, ms, rpb, wp, bp, is1p, L.ptr(st),
                                                tiles + 2, tiles, tile_n, L.current_stream()))
            torch.cuda.synchronize()
            _check_ln(y, _ln_ref(x, mode, mod, w, b, rpb), f"layernorm(hand-built stats) {mode} {kind} D={D} tile_n={tile_n}", kind)


# ---------------------------------------------------------------------------------------------------- c. stats RMSNorm + RoPE
def _rope(L, H, frames, hp, wp):
    hd = 128
    n = frames * hp * wp
    cos = torch.empty(n, hd // 2)
    sin = torch.empty(n, hd // 2)
    L.check(L.lib().ce_rope_table_host(hd, frames, hp, wp, 1024, 8, 10000.0, L.ptr(cos), L.ptr(sin)))
    return cos.cuda(), sin.cuda()


def _rms_ref(x, w, H, freqs=None, B=1):
    """The oracle's bf16 RMSNorm across heads (and RoPE) of the stored x [B * L, D]."""
    from oracle import dit_oracle as O

    y = O._rms_norm_across_heads(x.cpu().reshape(B, -1, x.shape[1]), w.cpu(), EPS)
    if freqs is not None:
        yh = O._apply_rope(y.unflatten(2, (H, 128)).transpose(1, 2), freqs)
        y = yh.transpose(1, 2).flatten(2, 3)
    return y.reshape(x.shape).float()


@gpu
@pytest.mark.parametrize("H", [2, 4, 40])   # D = 256, 512, 5120: 1, 2 and 20 tiles per matrix
def test_rmsnorm_rope_stats_qkv(H):
    """The self-attention q | k path: a [M, 3D] QKV buffer written by the GEMM with stats_mode 2, then nmat = 2 with different q and
    k weights (and k twice the scale of q, so reading q's partials for k fails), RoPE from ce_rope_table_host, B = 2 so the token
    is row % L.  v must stay bit-untouched.  Rule of test_rmsnorm_rope (1 bf16 ulp of the oracle).  The same call with stats = NULL
    (the kernel reduces over each row) must give the bits of two ce_rmsnorm_rope_bf16 launches, on q and on k, and leave v alone."""
    from oracle import dit_oracle as O

    L = _lib()
    D = H * 128
    frames, hp, wp = 2, 3, 25
    Lt = frames * hp * wp
    M = 2 * Lt
    tiles = D // 256
    cos, sin = _rope(L, H, frames, hp, wp)
    freqs = O.rope_table(O.DiTConfig.tiny(heads=H), frames, 2 * hp, 2 * wp)
    for i, kind in enumerate(ROW_KINDS):
        A, W, bias, _, _ = gemm_case(kind, M, 3 * D, 136, M, seed=H + i)
        W[D:2 * D] *= 2
        bias[D:2 * D] *= 2
        qkv = torch.empty(M, 3 * D, dtype=torch.bfloat16, device="cuda")
        st = torch.full((M, 3 * tiles + 1, 2), float("nan"), device="cuda")
        linear_ex(A, W, qkv, bias=bias, stats=st, stats_mode=2)
        g = torch.Generator(device="cuda").manual_seed(100 + i)
        wq = (1 + 0.1 * torch.randn(D, generator=g, device="cuda")).bfloat16()
        wk = (1 - 0.2 * torch.randn(D, generator=g, device="cuda")).bfloat16()
        before = qkv.clone()
        L.check(L.lib().ce_rmsnorm_rope_stats_bf16(L.ptr(qkv), 3 * D, M, D, EPS, L.ptr(wq), L.ptr(wk), 2, L.ptr(cos), L.ptr(sin), Lt, 128,
                                                   L.ptr(st), 3 * tiles + 1, tiles, L.current_stream()))
        in_kernel, two = before.clone(), before.clone()
        L.check(L.lib().ce_rmsnorm_rope_stats_bf16(L.ptr(in_kernel), 3 * D, M, D, EPS, L.ptr(wq), L.ptr(wk), 2, L.ptr(cos), L.ptr(sin), Lt,
                                                   128, None, 0, 0, L.current_stream()))
        for m, wm in ((0, wq), (1, wk)):
            L.check(L.lib().ce_rmsnorm_rope_bf16(L.ptr(two[:, m * D:]), 3 * D, M, D, EPS, L.ptr(wm), L.ptr(cos), L.ptr(sin), Lt, 128,
                                                 L.current_stream()))
        torch.cuda.synchronize()
        what = f"rmsnorm_rope(stats) {kind} H={H}"
        assert torch.equal(qkv[:, 2 * D:], before[:, 2 * D:]), what + ": v columns were written"
        assert torch.equal(in_kernel, two), what + ": stats = NULL differs from two ce_rmsnorm_rope_bf16 launches"
        _bf16_close(qkv[:, :D], _rms_ref(before[:, :D], wq, H, freqs, B=2), what + " q")
        _bf16_close(qkv[:, D:2 * D], _rms_ref(before[:, D:2 * D], wk, H, freqs, B=2), what + " k")


@gpu
@pytest.mark.parametrize("H", [2, 4, 40])
def test_rmsnorm_stats_cross_attention_q(H):
    """nmat = 1 without RoPE (the cross-attention q): GEMM [M, D] with stats_mode 2 -> ce_rmsnorm_rope_stats_bf16, M ragged."""
    L = _lib()
    D = H * 128
    M = 301
    tiles = D // 256
    for i, kind in enumerate(ROW_KINDS):
        A, W, bias, _, _ = gemm_case(kind, M, D, 136, M, seed=7 * H + i)
        q = torch.empty(M, D, dtype=torch.bfloat16, device="cuda")
        st = torch.full((M, tiles, 2), float("nan"), device="cuda")
        linear_ex(A, W, q, bias=bias, stats=st, stats_mode=2)
        w = (1 + 0.1 * torch.randn(D, generator=torch.Generator(device="cuda").manual_seed(i), device="cuda")).bfloat16()
        before = q.clone()
        L.check(L.lib().ce_rmsnorm_rope_stats_bf16(L.ptr(q), D, M, D, EPS, L.ptr(w), None, 1, None, None, 0, 128, L.ptr(st), tiles, tiles,
                                                   L.current_stream()))
        torch.cuda.synchronize()
        _bf16_close(q, _rms_ref(before, w, H), f"rmsnorm(stats) nmat=1 {kind} H={H}")


# ---------------------------------------------------------------------------------------------------- d. DiT, three stats tiles
def _dit_case():
    """heads 6 (D = 768: three 256-column tiles), 2 layers, 2 frames of a 16 x 24 latent (192 tokens); the patch embedding bias
    has a different offset per 256-column block, so the residual stream's tile means differ."""
    from oracle import cases, dit_oracle as O

    cfg = O.DiTConfig.tiny(heads=6)
    sd32 = O.random_state_dict(cfg, seed=21)
    sd32["patch_embedding.bias"] = sd32["patch_embedding.bias"] + torch.tensor([-1.5, 0.75, 2.0]).repeat_interleave(256)
    g = torch.Generator().manual_seed(22)
    x = torch.randn(1, 36, 2, 16, 24, generator=g)
    text = torch.randn(1, 512, cfg.text_dim, generator=g)
    text[:, 77:] = 0
    img = torch.randn(1, 257, cfg.image_dim, generator=g)
    t = torch.tensor([601])
    return cfg, sd32, cases.to_bf16_state(sd32), (x, t, text, img)


def _dit_run_cuda():
    """The CUDA forward of _dit_case -> (out, block0) as fp32 CPU tensors."""
    import chronoedit_b200 as ce

    cfg, _, sdb, (x, t, text, img) = _dit_case()
    m = ce.ChronoEditTransformer3DModel(
        patch_size=cfg.patch_size, num_attention_heads=cfg.num_attention_heads, attention_head_dim=cfg.attention_head_dim,
        in_channels=cfg.in_channels, out_channels=cfg.out_channels, text_dim=cfg.text_dim, freq_dim=cfg.freq_dim,
        ffn_dim=cfg.ffn_dim, num_layers=cfg.num_layers, eps=cfg.eps, image_dim=cfg.image_dim,
        added_kv_proj_dim=cfg.added_kv_proj_dim, rope_max_seq_len=cfg.rope_max_seq_len,
        rope_temporal_skip_len=cfg.rope_temporal_skip_len)
    m.load_state_dict(sdb)
    m = m.cuda()
    out = m(x.cuda(), t.cuda(), text.cuda(), img.cuda(), return_dict=False, return_block0=True)[0]
    torch.cuda.synchronize()
    return out.float().cpu(), m.last_block0.float().cpu().reshape(1, -1, cfg.inner_dim)


@gpu
def test_dit_three_stats_tiles():
    """The end-to-end stats path with a cross-tile merge (D = 768) on a tile-structured residual stream: block 0 and the output
    against the CPU oracle under the rule of test_dit_forward_matches_reference (as close to the fp32 oracle as the oracle's own
    bf16 run)."""
    from oracle import dit_oracle as O

    out, b0 = _dit_run_cuda()
    cfg, sd32, sdb, (x, t, text, img) = _dit_case()
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    with torch.no_grad():
        ref32, i32 = O.dit_forward(sd32, cfg, x, t, text, img, return_intermediates=True)
        ref16, i16 = O.dit_forward(sdb, cfg, x.bfloat16(), t, text.bfloat16(), img.bfloat16(), return_intermediates=True)
    ref16, b16, b32 = ref16.float(), i16["block0"].float(), i32["block0"].float()
    assert torch.isfinite(out).all() and out.shape == ref32.shape
    eb_ref = (b16 - b32).abs()
    assert (b0 - b32).abs().mean() <= 1.25 * eb_ref.mean() + 1e-6, f"block0 mean err {(b0 - b32).abs().mean():.3g} vs {eb_ref.mean():.3g}"
    e_ref, e_our = (ref16 - ref32).abs(), (out - ref32).abs()
    assert e_our.mean() <= 1.25 * e_ref.mean(), f"mean err {e_our.mean():.3g} vs reference's own bf16 error {e_ref.mean():.3g}"
    assert e_our.max() <= 1.5 * e_ref.max(), f"max err {e_our.max():.3g} vs reference's own bf16 error {e_ref.max():.3g}"
    assert (out - ref16).abs().mean() <= 1.25 * e_ref.mean()
