"""The GEMM's epilogue hand-over: the consumers write each tile, rounded to bf16, into a shared-memory staging buffer and go on to
the next tile's main loop while warps 1-3 of the producer warpgroup apply GELU / residual / gate, store and compute the row
statistics.  A CTA that overwrote its staging tile before the epilogue warps had drained it, or a role that lost step with the
other across tiles, would store another tile's values.  So every case runs many tiles per CTA at a small K (>= 30 tiles per SM,
one or two k-blocks each), where the epilogue is most of the time.

Operands are small integers: each row of A has a single 1, W, bias, residual and gate are in {-2, ..., 2} and the FP8 scales are
1 or 2.  Every value and every statistics sum is then exact in fp32 in any order, so every non-GELU output and both
statistics modes are compared bit for bit with a float64 restatement of the documented epilogue.  GELU is compared with the same
kernel's EPI_BIAS output passed through the documented formula.
"""
import pytest
import torch

from tests.test_gpu_fp8 import linear_fp8
from tests.test_gpu_row_stats import linear_ex, tile_width

gpu = pytest.mark.gpu
KIND_K = {"bf16": 64, "fp8": 128}   # one k-block of either kernel


def _operands(M, N, K, rpb, fp8, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    kidx = torch.randint(0, K, (M,), generator=g, device="cuda")
    A = torch.zeros(M, K, device="cuda")
    A[torch.arange(M, device="cuda"), kidx] = 1.0
    W = torch.randint(-1, 2, (N, K), generator=g, device="cuda").float()
    acc = W[:, kidx].t().double()                                              # A @ W^T, exactly
    op = {"bias": torch.randint(-1, 2, (N,), generator=g, device="cuda").bfloat16(),
          "resid": torch.randint(-2, 3, (M, N), generator=g, device="cuda").bfloat16(),
          "gate": torch.randint(-1, 2, ((M + rpb - 1) // rpb, N), generator=g, device="cuda").float()}
    if fp8:
        sa = 2.0 ** torch.randint(0, 2, (M,), generator=g, device="cuda").float()
        sw = 2.0 ** torch.randint(0, 2, (N,), generator=g, device="cuda").float()
        op.update(A=A.to(torch.float8_e4m3fn), W=W.to(torch.float8_e4m3fn), sa=sa, sw=sw)
        acc = acc * sa.double()[:, None] * sw.double()[None, :]
    else:
        op.update(A=A.bfloat16(), W=W.bfloat16())
    op["y"] = (acc + op["bias"].double()).bfloat16()                            # nn.Linear's bf16 output
    return op


def _run(op, fp8, out, epi, rpb, stats, mode, resid):
    kw = dict(bias=op["bias"], epi=epi, resid=resid if epi in (3, 4) else None, gate=op["gate"] if epi == 3 else None, rpb=rpb,
              stats=stats if mode else None, stats_mode=mode)
    if fp8:
        linear_fp8(op["A"], op["sa"], op["W"], op["sw"], out, **kw)
    else:
        linear_ex(op["A"], op["W"], out, **kw)


def _ref_stats(z, tn, mode):
    """Per (row, N tile): mode 1 (pivot + s / n, ss - s * s / n) about the tile's first column, mode 2 (sum z^2, 0)."""
    z = z.double()
    M, N = z.shape
    parts = []
    for t in range((N + tn - 1) // tn):
        c = z[:, t * tn:min(N, (t + 1) * tn)]
        if mode == 1:
            d = c - c[:, :1]
            s, ss, n = d.sum(1), (d * d).sum(1), c.shape[1]
            parts.append(torch.stack([c[:, 0] + s / n, (ss - s * s / n).clamp_min(0)], 1))
        else:
            parts.append(torch.stack([(c * c).sum(1), torch.zeros_like(c[:, 0])], 1))
    return torch.stack(parts, 1).float()


# (M, N): ragged M; N with a partial last tile of a power-of-two width (the statistics divide by it exactly); >= 30 tiles per SM
SHAPES = {256: (128 * 124 + 37, 256 * 31 + 64), 128: (128 * 1990 + 37, 160), 64: (128 * 1990 + 37, 96)}


@gpu
@pytest.mark.parametrize("kind", ["bf16", "fp8"])
@pytest.mark.parametrize("bn", [256, 128, 64])
def test_gemm_overlap_many_tiles(bn, kind):
    fp8 = kind == "fp8"
    M, N = SHAPES[bn]
    assert tile_width(N) == bn
    K, rpb, tn = KIND_K[kind], 1000, bn
    tiles = (N + tn - 1) // tn
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert ((M + 127) // 128) * tiles >= 30 * sms
    op = _operands(M, N, K, rpb, fp8, seed=bn + fp8)
    y = op["y"]
    gate_rows = op["gate"].repeat_interleave(rpb, dim=0)[:M].double()
    ref = {0: y, 3: (op["resid"].double() + y.double() * gate_rows).bfloat16(), 4: (op["resid"].double() + y.double()).bfloat16()}
    base = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    _run(op, fp8, base, 0, rpb, None, 0, None)
    for epi in range(5):
        for mode in (0, 1, 2):
            what = f"{kind} BN={bn} epi={epi} stats_mode={mode}"
            st = torch.full((M, tiles, 2), float("nan"), device="cuda")
            if epi in (3, 4):   # in place, as the DiT's residual GEMMs
                out = op["resid"].clone()
                _run(op, fp8, out, epi, rpb, st, mode, out)
            else:
                out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
                _run(op, fp8, out, epi, rpb, st, mode, None)
            torch.cuda.synchronize()
            if epi in (1, 2):
                want = torch.nn.functional.gelu(base.float(), approximate="tanh" if epi == 1 else "none").bfloat16()
                diff = (out.view(torch.int16).int() - want.view(torch.int16).int()).abs()
                assert diff.max().item() <= 1, f"{what}: GELU output more than 1 bf16 ulp from GELU of the EPI_BIAS output"
                want_st = _ref_stats(out, tn, mode) if mode else None
                if mode:
                    torch.testing.assert_close(st, want_st, rtol=1e-5, atol=1e-5, msg=what + ": statistics")
                continue
            assert torch.equal(out.view(torch.int16), ref[epi].view(torch.int16)), f"{what}: output"
            if epi == 0:
                assert torch.equal(out.view(torch.int16), base.view(torch.int16)), f"{what}: output depends on the statistics"
            if mode:
                assert torch.equal(st, _ref_stats(out, tn, mode)), f"{what}: statistics"
            else:
                assert torch.isnan(st).all(), f"{what}: statistics written without stats_mode"
