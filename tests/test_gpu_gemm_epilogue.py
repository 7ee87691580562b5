"""The GEMM epilogue in passes: bias / rounding / GELU for the whole tile into packed registers, then per row chunks of eight
column groups whose residual and gate loads are issued before the chunk's stores.  out and resid alias in the DiT's residual
GEMMs (in place), so the tests check in-place against out-of-place bit for bit, that nothing outside [M, N) or the statistics
tiles is written, and that a tile's result depends only on its own rows: the same GEMM launched on one 128-row slice of A gives
the same bits, outputs and statistics, whichever CTA computes the tile and wherever it sits in the tile walk.
"""
import pytest
import torch

from tests.test_gpu_ops import _bf16_close
from tests.test_gpu_row_stats import gemm_case, linear_ex, ref_output, tile_width

gpu = pytest.mark.gpu
SENTINEL = -12345   # int16 bit pattern of a finite negative bf16


def _stats_mode(epi):
    return 1 if epi in (0, 3, 4) else 2


@gpu
@pytest.mark.parametrize("N", [512, 192, 64])   # tile widths 256, 128 (partial last tile), 64
def test_gemm_epilogue_slices_bit_exact(N):
    """M = 1300: 11 M tiles (odd, the last one ragged).  For epilogues 0-4 with statistics, each 128-row slice of the full
    GEMM equals the GEMM launched on that slice alone, bit for bit, outputs and statistics."""
    M, K, rpb = 1300, 320, 256   # rows_per_batch a multiple of 128: a slice never straddles two gate rows
    tn = tile_width(N)
    tiles = (N + tn - 1) // tn
    A, W, bias, resid, gate = gemm_case("block_offset", M, N, K, rpb, seed=N)
    for epi in range(5):
        mode = _stats_mode(epi)
        kw = dict(bias=bias, epi=epi, stats_mode=mode)
        full = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
        st = torch.full((M, tiles, 2), float("nan"), device="cuda")
        linear_ex(A, W, full, resid=resid if epi in (3, 4) else None, gate=gate if epi == 3 else None, rpb=rpb, stats=st, **kw)
        ref = ref_output(A, W, bias, resid, gate, epi, rpb)
        if epi in (1, 2):
            ref = torch.nn.functional.gelu(ref, approximate="tanh" if epi == 1 else "none")
        _bf16_close(full, ref, f"N={N} epi={epi}")
        for r0 in range(0, M, 128):
            r1 = min(M, r0 + 128)
            out = torch.empty(r1 - r0, N, dtype=torch.bfloat16, device="cuda")
            sst = torch.full((r1 - r0, tiles, 2), float("nan"), device="cuda")
            linear_ex(A[r0:r1], W, out, resid=resid[r0:r1] if epi in (3, 4) else None,
                      gate=gate[r0 // rpb:] if epi == 3 else None, rpb=rpb, stats=sst, **kw)
            torch.cuda.synchronize()
            assert torch.equal(out.view(torch.int16), full[r0:r1].view(torch.int16)), f"N={N} epi={epi} rows {r0}:{r1}: output"
            assert torch.equal(sst, st[r0:r1]), f"N={N} epi={epi} rows {r0}:{r1}: statistics"


@gpu
def test_gemm_epilogue_in_place_writes_nothing_outside():
    """M = 384, N = 320 (a 64-column last tile), in place as the DiT's residual GEMMs, with ldo > N in an allocation that
    extends past row M: the result equals the out-of-place one bit for bit, and rows >= M, columns >= N and statistics
    outside [M, tiles) stay untouched."""
    M, N, K, ld, rpb = 384, 320, 256, 400, 128
    tiles = 2
    A, W, bias, resid, gate = gemm_case("iid", M, N, K, rpb, seed=7)
    for epi in (3, 4):
        buf = torch.full((M + 130, ld), SENTINEL, dtype=torch.int16, device="cuda").view(torch.bfloat16)
        buf[:M, :N] = resid
        st = torch.full((M + 130, tiles + 1, 2), float("nan"), device="cuda")
        out = buf[:M + 130]
        linear_ex(A, W, out[:M], bias=bias, epi=epi, resid=out[:M], gate=gate if epi == 3 else None, rpb=rpb, stats=st,
                  stats_mode=1)
        sep = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
        linear_ex(A, W, sep, bias=bias, epi=epi, resid=resid, gate=gate if epi == 3 else None, rpb=rpb)
        torch.cuda.synchronize()
        raw = buf.view(torch.int16)
        assert (raw[M:] == SENTINEL).all(), f"epi={epi}: rows >= M written"
        assert (raw[:, N:] == SENTINEL).all(), f"epi={epi}: columns >= N written"
        assert torch.equal(buf[:M, :N].view(torch.int16), sep.view(torch.int16)), f"epi={epi}: in place differs from out of place"
        assert torch.isnan(st[M:]).all() and torch.isnan(st[:, tiles:]).all(), f"epi={epi}: statistics written outside [M, tiles)"
        assert not torch.isnan(st[:M, :tiles]).any(), f"epi={epi}: a statistic was not written"


@gpu
@pytest.mark.parametrize("M,N", [(77, 64), (256, 512), (4739, 5120)])
def test_gemm_epilogue_grid_shapes(M, N):
    """Fewer tiles than SMs (one ragged tile; 2 x 2 tiles) and many more (38 x 20 tiles, several waves with a partial last
    one), against the fp32 epilogue."""
    K, rpb = 192, 97
    A, W, bias, resid, gate = gemm_case("iid", M, N, K, rpb, seed=M + N)
    for epi in (0, 3):
        out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
        linear_ex(A, W, out, bias=bias, epi=epi, resid=resid if epi == 3 else None, gate=gate if epi == 3 else None, rpb=rpb)
        torch.cuda.synchronize()
        _bf16_close(out, ref_output(A, W, bias, resid, gate, epi, rpb), f"M={M} N={N} epi={epi}")
