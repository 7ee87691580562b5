"""The bf16 attention's two schedules against each other: the pipelined one (version 0, the default: S of key tile j and P V of
tile j-1 issued together, the softmax of tile j under that P V, warpgroups in ping-pong) must give the serial one's output
(version 1: S, softmax, P V per tile) bit for bit, since both apply the same operations in the same order to every value.
The output buffer has a column gap (ldo > H * 128) and a guard band after its last row, both filled with a sentinel that
neither schedule may touch."""
import math

import pytest
import torch

gpu = pytest.mark.gpu

SENTINEL = -12345   # int16 bit pattern of the guard cells (a bf16 NaN would compare unequal to itself)
GUARD_ROWS = 3
GAP = 64            # extra columns per row beyond H * 128


def _lib():
    import chronoedit_b200._lib as L

    return L


def _out_buffer(B, Lq, D, prev=None):
    """[B * Lq + GUARD_ROWS, D + GAP] bf16, all sentinel; the first D columns of the first B * Lq rows hold `prev` if given."""
    buf = torch.full((B * Lq + GUARD_ROWS, D + GAP), SENTINEL, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    if prev is not None:
        buf[:B * Lq, :D] = prev.reshape(B * Lq, D)
    return buf


def _check_pair(outs, B, Lq, D, what):
    o0, o1 = (o.view(torch.int16) for o in outs)
    guard = torch.full_like(o0[B * Lq:], SENTINEL)
    for v, o in ((0, o0), (1, o1)):
        assert torch.equal(o[B * Lq:], guard), f"{what}: version {v} wrote into the guard rows"
        assert bool((o[:B * Lq, D:] == SENTINEL).all()), f"{what}: version {v} wrote into the column gap"
        assert torch.isfinite(o[:B * Lq, :D].view(torch.bfloat16).float()).all(), f"{what}: version {v} non-finite output"
    diff = (o0 != o1).sum().item()
    assert diff == 0, f"{what}: pipelined and serial schedules differ in {diff} of {o0.numel()} values"


def _both_versions(launch):
    """Runs launch(version) under version 1 and then 0 and restores the default."""
    L = _lib()
    lib = L.lib()
    try:
        for v in (1, 0):
            L.check(lib.ce_debug_attention_kernel(v))
            launch(v)
        torch.cuda.synchronize()
    finally:
        L.check(lib.ce_debug_attention_kernel(-1))


def _run_single(B, H, Lq, Lk, seed, accumulate=False, key_ramp=0.0, fused=True):
    L = _lib()
    lib = L.lib()
    hd = 128
    D = H * hd
    g = torch.Generator(device="cpu").manual_seed(seed)
    if fused:   # q | k | v packed per row, as the DiT's self-attention reads them
        assert Lq == Lk
        qkv = torch.randn(B, Lq, 3 * D, generator=g).bfloat16().cuda()
        q, k, v = qkv[..., :D], qkv[..., D:2 * D], qkv[..., 2 * D:]
        ldq = ldk = ldv = 3 * D
    else:
        q = torch.randn(B, Lq, D, generator=g).bfloat16().cuda()
        kv = torch.randn(B, Lk, 2 * D, generator=g).bfloat16().cuda()
        k, v = kv[..., :D], kv[..., D:]
        ldq, ldk, ldv = D, 2 * D, 2 * D
    if key_ramp:   # the inputs of test_attention_self_growing_and_shrinking_scores: the running maximum keeps moving
        ramp = (1.0 + key_ramp * torch.arange(Lk, dtype=torch.float32) / Lk).view(1, Lk, 1).cuda()
        k.copy_((k.float() * ramp).bfloat16())
    prev = torch.randn(B, Lq, D, generator=g).bfloat16().cuda() if accumulate else None
    outs = [_out_buffer(B, Lq, D, prev) for _ in range(2)]

    def launch(version):
        out = outs[version]
        L.check(lib.ce_attention_bf16(L.ptr(q), ldq, L.ptr(k), ldk, L.ptr(v), ldv, L.ptr(out), D + GAP, B, H, Lq, Lk, 1.0 / math.sqrt(hd),
                                      int(accumulate), L.current_stream()))

    _both_versions(launch)
    _check_pair(outs, B, Lq, D, f"attention B={B} H={H} Lq={Lq} Lk={Lk} acc={accumulate} ramp={key_ramp}")


@gpu
@pytest.mark.parametrize("L_", [1, 7, 127, 128, 129, 255, 256, 257, 2048])
def test_self_attention_schedules_equal(L_):
    _run_single(1, 2, L_, L_, seed=L_)


@gpu
def test_self_attention_schedules_equal_full_size():
    """The benchmark's self-attention: batch 2 (CFG), 40 heads, 7200 tokens."""
    _run_single(2, 40, 7200, 7200, seed=7200)


@gpu
def test_self_attention_schedules_equal_long():
    """28 800 tokens (temporal reasoning): 225 key tiles per query tile."""
    _run_single(1, 40, 28800, 28800, seed=28800)


@gpu
@pytest.mark.parametrize("Lq,ramp", [(1024, 6.0), (1500, 12.0), (640, -0.9)])
def test_schedules_equal_growing_and_shrinking_scores(Lq, ramp):
    _run_single(1, 2, Lq, Lq, seed=Lq, key_ramp=ramp)


@gpu
@pytest.mark.parametrize("Lq,Lk", [(300, 257), (300, 7), (7200, 512), (1000, 1000)])
def test_accumulate_schedules_equal(Lq, Lk):
    _run_single(2, 2, Lq, Lk, seed=Lq + Lk, accumulate=True, fused=False)


@gpu
@pytest.mark.parametrize("Lq", [300, 7200])
@pytest.mark.parametrize("Lk,Lk2", [(512, 257), (7, 300), (640, 129)])
def test_dual_source_schedules_equal(Lq, Lk, Lk2):
    L = _lib()
    lib = L.lib()
    B, H, hd = 2, 2, 128
    D = H * hd
    g = torch.Generator(device="cpu").manual_seed(Lq + Lk + Lk2)
    q = torch.randn(B, Lq, D, generator=g).bfloat16().cuda()
    kv = torch.randn(B, Lk, 2 * D, generator=g).bfloat16().cuda()
    kv2 = torch.randn(B, Lk2, 2 * D, generator=g).bfloat16().cuda()
    outs = [_out_buffer(B, Lq, D) for _ in range(2)]

    def launch(version):
        out = outs[version]
        L.check(lib.ce_attention_dual_bf16(L.ptr(q), D, L.ptr(kv), 2 * D, L.ptr(kv[..., D:]), 2 * D, L.ptr(kv2), 2 * D, L.ptr(kv2[..., D:]),
                                           2 * D, L.ptr(out), D + GAP, B, H, Lq, Lk, Lk2, 1.0 / math.sqrt(hd), L.current_stream()))

    _both_versions(launch)
    _check_pair(outs, B, Lq, D, f"dual attention Lq={Lq} Lk={Lk} Lk2={Lk2}")


def test_schedule_selection_abi():
    """Versions -1, 0 and 1 are accepted, every other one refused; no device needed."""
    import os

    L = _lib()
    if not os.path.exists(L.LIB_PATH):
        from chronoedit_b200 import build

        build.build()
    lib = L.lib()
    try:
        for v in (1, 0, -1):
            assert lib.ce_debug_attention_kernel(v) == 0
        for v in (2, 7, -2):
            assert lib.ce_debug_attention_kernel(v) == -1
    finally:
        lib.ce_debug_attention_kernel(-1)
