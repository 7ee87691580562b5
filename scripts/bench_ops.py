#!/usr/bin/env python
"""Operator micro-benchmarks at the 14B / 720p shapes (CUDA events, warm-up, L2-busting operand rotation).
    python scripts/bench_ops.py [attn] [attn8] [attnab] [gemm [cublas]] [gemmk] [rows] [conv]
`attnab` times the bf16 attention's pipelined schedule (version 0) against its serial one (version 1, ce_debug_attention_kernel)
in alternating rounds, and prints the median of each, the speed-up and the phase cycles of ce_debug_attention_timing.
`attn8` times the self-attention in bf16 and as the FP8 attention runs it: the q | k and v quantizers and the e4m3 kernel.
`gemm` times each block GEMM in bf16 and, in the fp8_* fields, as the FP8 mode runs it (quantization and e4m3 GEMM).
`gemmk` times the bf16 o-proj GEMM over K and fits the time per wave of tiles to a + b K: `a` is the per-tile cost that does not
scale with K (epilogue, hand-overs), `b` the main loop, printed as the TFLOP/s of all SMs while it runs.
Prints one JSON line per op; used to iterate on a kernel without running the whole 40-layer step."""
import json
import math
import sys
import time

import torch

sys.path.insert(0, ".")
import chronoedit_b200._lib as L  # noqa: E402

lib = L.lib()


def timeit(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def bench_attn(B=2, H=40, Lq=7200, Lk=7200, nbuf=3):
    D = H * 128
    bufs = [torch.randn(B, Lq, 3 * D, device="cuda", dtype=torch.bfloat16) for _ in range(nbuf)] if Lq == Lk else None
    out = torch.empty(B, Lq, D, device="cuda", dtype=torch.bfloat16)
    i = [0]
    if bufs is None:
        q = torch.randn(B, Lq, D, device="cuda", dtype=torch.bfloat16)
        kv = torch.randn(B, Lk, 2 * D, device="cuda", dtype=torch.bfloat16)

    def fn():
        if bufs is not None:
            x = bufs[i[0] % nbuf]
            i[0] += 1
            L.check(lib.ce_attention_bf16(L.ptr(x), 3 * D, L.ptr(x[..., D:]), 3 * D, L.ptr(x[..., 2 * D:]), 3 * D, L.ptr(out), D, B, H, Lq, Lk,
                                          1 / math.sqrt(128), 0, L.current_stream()))
        else:
            L.check(lib.ce_attention_bf16(L.ptr(q), D, L.ptr(kv), 2 * D, L.ptr(kv[..., D:]), 2 * D, L.ptr(out), D, B, H, Lq, Lk,
                                          1 / math.sqrt(128), 0, L.current_stream()))

    ms = timeit(fn)
    fl = 4.0 * B * H * Lq * Lk * 128
    print(json.dumps({"op": "attention", "B": B, "H": H, "Lq": Lq, "Lk": Lk, "ms": round(ms, 4), "tflops": round(fl / ms / 1e9, 1)}), flush=True)


def bench_attn8(B=2, H=40, Lk=7200, nbuf=2):
    """Self-attention at [B, Lk, H x 128]: the bf16 kernel, then the FP8 path's three parts on the same fused QKV buffers."""
    D = H * 128
    bufs = [torch.randn(B, Lk, 3 * D, device="cuda", dtype=torch.bfloat16) for _ in range(nbuf)]
    out = torch.empty(B, Lk, D, device="cuda", dtype=torch.bfloat16)
    Lpad = (Lk + 31) // 32 * 32
    qk8 = torch.empty(B * Lk, 2 * D, device="cuda", dtype=torch.uint8)
    qks = torch.empty(B * Lk, 2 * H, device="cuda")
    vt8 = torch.empty(B, D, Lpad, device="cuda", dtype=torch.uint8)
    vs = torch.empty(B, D, device="cuda")
    i = [0]
    s = L.current_stream()

    def nxt():
        x = bufs[i[0] % nbuf]
        i[0] += 1
        return x

    def bf16():
        x = nxt()
        L.check(lib.ce_attention_bf16(L.ptr(x), 3 * D, L.ptr(x[..., D:]), 3 * D, L.ptr(x[..., 2 * D:]), 3 * D, L.ptr(out), D, B, H, Lk, Lk,
                                      1 / math.sqrt(128), 0, s))

    def quant_qk():
        L.check(lib.ce_quantize_heads_fp8(L.ptr(nxt()), 3 * D, B * Lk, 2 * H, L.ptr(qk8), 2 * D, L.ptr(qks), s))

    def quant_v():
        L.check(lib.ce_quantize_v_fp8(L.ptr(nxt()[..., 2 * D:]), 3 * D, B, Lk, H, L.ptr(vt8), Lpad, L.ptr(vs), s))

    def fp8():
        L.check(lib.ce_attention_fp8(L.ptr(qk8), L.ptr(qk8[:, D:]), 2 * D, L.ptr(qks), L.ptr(qks[:, H:]), 2 * H, L.ptr(vt8), Lpad, L.ptr(vs),
                                     L.ptr(out), D, B, H, Lk, 1 / math.sqrt(128), s))

    quant_qk()
    quant_v()
    fl = 4.0 * B * H * Lk * Lk * 128
    res = {}
    for name, fn in (("bf16", bf16), ("fp8", fp8), ("quant_qk", quant_qk), ("quant_v", quant_v), ("bf16_again", bf16), ("fp8_again", fp8)):
        res[name] = timeit(fn)
    qk_bytes, v_bytes = B * Lk * 2 * D * 3 + B * Lk * 2 * H * 4, B * Lk * D * 2 * 2 + B * D * Lpad + B * D * 4
    print(json.dumps({"op": "attention_fp8", "B": B, "H": H, "Lk": Lk,
                      "bf16_ms": [round(res["bf16"], 3), round(res["bf16_again"], 3)],
                      "fp8_ms": [round(res["fp8"], 3), round(res["fp8_again"], 3)],
                      "bf16_tflops": round(fl / min(res["bf16"], res["bf16_again"]) / 1e9, 1),
                      "fp8_tflops": round(fl / min(res["fp8"], res["fp8_again"]) / 1e9, 1),
                      "quant_qk_ms": round(res["quant_qk"], 3), "quant_qk_GBps": round(qk_bytes / res["quant_qk"] / 1e6, 1),
                      "quant_v_ms": round(res["quant_v"], 3), "quant_v_GBps": round(v_bytes / res["quant_v"] / 1e6, 1),
                      "fp8_total_ms": round(min(res["fp8"], res["fp8_again"]) + res["quant_qk"] + res["quant_v"], 3)}), flush=True)


def bench_attn_libs(B=2, H=40, L=7200, Lk=None):
    """The library bar for the self-attention (SURVEY K6): what the unmodified reference executes on a cc-10.0 GPU --
    torch SDPA with the cuDNN fused-attention backend (chronoedit/_src/modules/attention.py:129-138 picks it on Blackwell), torch's
    built-in flash backend, and the flash-attn 2.8 package -- on the same shapes, same timing loop."""
    from torch.nn.attention import SDPBackend, sdpa_kernel

    Lk = Lk or L
    q = torch.randn(B, H, L, 128, device="cuda", dtype=torch.bfloat16)
    k = torch.randn(B, H, Lk, 128, device="cuda", dtype=torch.bfloat16)
    v = torch.randn(B, H, Lk, 128, device="cuda", dtype=torch.bfloat16)
    fl = 4.0 * B * H * L * Lk * 128
    for name, backend in (("sdpa_cudnn", SDPBackend.CUDNN_ATTENTION), ("sdpa_flash", SDPBackend.FLASH_ATTENTION),
                          ("sdpa_efficient", SDPBackend.EFFICIENT_ATTENTION)):
        try:
            with sdpa_kernel(backend):
                ms = timeit(lambda: torch.nn.functional.scaled_dot_product_attention(q, k, v), iters=5, warmup=2)
            print(json.dumps({"op": name, "B": B, "H": H, "Lq": L, "Lk": Lk, "ms": round(ms, 4), "tflops": round(fl / ms / 1e9, 1)}), flush=True)
        except Exception as e:  # noqa: BLE001
            print(json.dumps({"op": name, "Lq": L, "error": str(e)[:160]}), flush=True)
    try:
        from flash_attn import flash_attn_func

        qf, kf, vf = (t.transpose(1, 2).contiguous() for t in (q, k, v))
        ms = timeit(lambda: flash_attn_func(qf, kf, vf), iters=5, warmup=2)
        print(json.dumps({"op": "flash_attn_2.8_pkg", "B": B, "H": H, "Lq": L, "Lk": Lk, "ms": round(ms, 4), "tflops": round(fl / ms / 1e9, 1)}), flush=True)
    except Exception as e:  # noqa: BLE001
        print(json.dumps({"op": "flash_attn_2.8_pkg", "error": str(e)[:160]}), flush=True)


def bench_attn_dual(B=2, H=40, Lq=7200, Lk=512, Lk2=257):
    """The cross-attention launch of the DiT block: text keys + image keys in one kernel."""
    D = H * 128
    q = torch.randn(B, Lq, D, device="cuda", dtype=torch.bfloat16)
    kv = torch.randn(B, Lk, 2 * D, device="cuda", dtype=torch.bfloat16)
    kv2 = torch.randn(B, Lk2, 2 * D, device="cuda", dtype=torch.bfloat16)
    out = torch.empty(B, Lq, D, device="cuda", dtype=torch.bfloat16)

    def fn():
        L.check(lib.ce_attention_dual_bf16(L.ptr(q), D, L.ptr(kv), 2 * D, L.ptr(kv[..., D:]), 2 * D, L.ptr(kv2), 2 * D, L.ptr(kv2[..., D:]), 2 * D,
                                           L.ptr(out), D, B, H, Lq, Lk, Lk2, 1 / math.sqrt(128), L.current_stream()))

    ms = timeit(fn)
    fl = 4.0 * B * H * Lq * (Lk + Lk2) * 128
    print(json.dumps({"op": "attention_dual", "B": B, "H": H, "Lq": Lq, "Lk": Lk, "Lk2": Lk2, "ms": round(ms, 4), "tflops": round(fl / ms / 1e9, 1)}), flush=True)


def bench_attn_ab(B=2, H=40, Lq=7200, Lk=7200, Lk2=0, rounds=12, iters=5):
    """Version 0 (pipelined) against version 1 (serial) of the bf16 attention on the same buffers: one timing of each per
    round, alternated, median over the rounds.  Then one launch of each with the phase-timing hook on."""
    import statistics

    D = H * 128
    self_attn = Lq == Lk and Lk2 == 0
    nbuf = 2
    if self_attn:
        bufs = [torch.randn(B, Lq, 3 * D, device="cuda", dtype=torch.bfloat16) for _ in range(nbuf)]
    else:
        q = torch.randn(B, Lq, D, device="cuda", dtype=torch.bfloat16)
        kv = torch.randn(B, Lk, 2 * D, device="cuda", dtype=torch.bfloat16)
        kv2 = torch.randn(B, max(Lk2, 1), 2 * D, device="cuda", dtype=torch.bfloat16)
    out = torch.empty(B, Lq, D, device="cuda", dtype=torch.bfloat16)
    i = [0]
    s = L.current_stream()

    def fn():
        if self_attn:
            x = bufs[i[0] % nbuf]
            i[0] += 1
            L.check(lib.ce_attention_bf16(L.ptr(x), 3 * D, L.ptr(x[..., D:]), 3 * D, L.ptr(x[..., 2 * D:]), 3 * D, L.ptr(out), D, B, H, Lq, Lk,
                                          1 / math.sqrt(128), 0, s))
        elif Lk2:
            L.check(lib.ce_attention_dual_bf16(L.ptr(q), D, L.ptr(kv), 2 * D, L.ptr(kv[..., D:]), 2 * D, L.ptr(kv2), 2 * D, L.ptr(kv2[..., D:]),
                                               2 * D, L.ptr(out), D, B, H, Lq, Lk, Lk2, 1 / math.sqrt(128), s))
        else:
            L.check(lib.ce_attention_bf16(L.ptr(q), D, L.ptr(kv), 2 * D, L.ptr(kv[..., D:]), 2 * D, L.ptr(out), D, B, H, Lq, Lk,
                                          1 / math.sqrt(128), 0, s))

    ms = {0: [], 1: []}
    try:
        for v in (1, 0):   # warm-up of both
            L.check(lib.ce_debug_attention_kernel(v))
            timeit(fn, iters=2, warmup=2)
        for _ in range(rounds):
            for v in (1, 0):
                L.check(lib.ce_debug_attention_kernel(v))
                ms[v].append(timeit(fn, iters=iters, warmup=1))
        phases = {}
        buf = torch.zeros(16, dtype=torch.int64, device="cuda")
        L.check(lib.ce_debug_attention_timing(L.ptr(buf)))
        for v in (1, 0):
            L.check(lib.ce_debug_attention_kernel(v))
            buf.zero_()
            fn()
            torch.cuda.synchronize()
            phases[v] = buf[:4].tolist()
    finally:
        L.check(lib.ce_debug_attention_timing(None))
        L.check(lib.ce_debug_attention_kernel(-1))
    fl = 4.0 * B * H * Lq * (Lk + Lk2) * 128
    m0, m1 = statistics.median(ms[0]), statistics.median(ms[1])
    print(json.dumps({"op": "attention_ab", "B": B, "H": H, "Lq": Lq, "Lk": Lk, "Lk2": Lk2, "rounds": rounds,
                      "pipelined_ms": round(m0, 4), "serial_ms": round(m1, 4), "speedup": round(m1 / m0, 4),
                      "pipelined_range_ms": [round(min(ms[0]), 4), round(max(ms[0]), 4)],
                      "serial_range_ms": [round(min(ms[1]), 4), round(max(ms[1]), 4)],
                      "pipelined_tflops": round(fl / m0 / 1e9, 1), "serial_tflops": round(fl / m1 / 1e9, 1),
                      "phase_cycles_pipelined": phases[0], "phase_cycles_serial": phases[1]}), flush=True)


# The six block GEMMs of the DiT at the 14B / 720p step (dit.cu), as dit.cu calls them: in-place residual (out == resid == x),
# a batch-2 gate read from the modulation table (row stride 6 D), statistics for the LayerNorm / RMSNorm that follows.
#   name, N, K, epilogue, stats_mode
DIT_GEMMS = [("qkv", 15360, 5120, 0, 2), ("o_proj", 5120, 5120, 3, 1), ("cross_q", 5120, 5120, 0, 2),
             ("cross_out", 5120, 5120, 4, 1), ("ffn_up", 13824, 5120, 1, 0), ("ffn_down", 5120, 13824, 3, 1),
             # EPI_BIAS without statistics at the o-proj / FFN-down shapes: the difference to those rows is the epilogue's cost
             ("o_proj_bias_only", 5120, 5120, 0, 0), ("ffn_down_bias_only", 5120, 13824, 0, 0),
             # FFN up without GELU: the difference to the ffn_up row is GELU's cost
             ("ffn_up_bias_only", 13824, 5120, 0, 0),
             # the qkv shape at K = 64: one k-block per tile, so the time is nearly all epilogue
             ("qkv_k64", 15360, 64, 0, 2)]


def bench_gemm(name, N, K, epi, stats_mode, M=14400, rows_per_batch=7200, nbuf=3, cublas=True, fp8=True):
    A = [torch.randn(M, K, device="cuda", dtype=torch.bfloat16) for _ in range(nbuf)]
    W = [torch.randn(N, K, device="cuda", dtype=torch.bfloat16) * 0.02 for _ in range(nbuf)]
    bias = (torch.randn(N, device="cuda") * 0.02).bfloat16()
    x = torch.randn(M, N, device="cuda", dtype=torch.bfloat16)   # output, and residual in place for epilogues 3 / 4
    mod = torch.randn(M // rows_per_batch, 6, N, device="cuda") * 0.1
    tn = 256 if N >= 256 else (128 if N >= 128 else 64)
    stats = torch.empty(M, (N + tn - 1) // tn, 2, device="cuda")
    resid_epi = epi in (3, 4)
    i = [0]

    def fn():
        a, w = A[i[0] % nbuf], W[i[0] % nbuf]
        i[0] += 1
        args = L.LinearArgsC(A=a.data_ptr(), lda=K, W=w.data_ptr(), ldw=K, M=M, N=N, K=K, out=x.data_ptr(), ldo=N, bias=bias.data_ptr(),
                             epilogue=epi, resid=x.data_ptr() if resid_epi else None, ldr=N if resid_epi else 0,
                             gate=mod[:, 2].data_ptr() if epi == 3 else None, gate_stride=6 * N if epi == 3 else 0,
                             rows_per_batch=rows_per_batch, stats_out=stats.data_ptr() if stats_mode else None,
                             stats_ld=stats.shape[1] if stats_mode else 0, stats_mode=stats_mode)
        L.check(lib.ce_linear_ex_bf16(args, L.current_stream()))

    ms = timeit(fn)
    row = {"op": "gemm", "name": name, "M": M, "N": N, "K": K, "epi": epi, "stats_mode": stats_mode, "ms": round(ms, 4),
           "tflops": round(2.0 * M * N * K / ms / 1e9, 1)}
    if not fp8:
        print(json.dumps(row), flush=True)
        return ms
    # FP8 column: the same GEMM as the FP8 mode runs it (ce_linear_fp8_ex on e4m3 operands), and the row quantization of A
    # that precedes it in dit.cu (ce_quantize_rows_fp8, one launch per GEMM)
    from chronoedit_b200.transformer import quantize_fp8_rows

    Aq = [torch.empty(M, K, device="cuda", dtype=torch.uint8) for _ in range(nbuf)]
    sa = [torch.empty(M, device="cuda") for _ in range(nbuf)]
    Wq, sw = zip(*[quantize_fp8_rows(w) for w in W])

    def quant():
        j = i[0] % nbuf
        i[0] += 1
        L.check(lib.ce_quantize_rows_fp8(L.ptr(A[j]), K, M, K, L.ptr(Aq[j]), K, L.ptr(sa[j]), L.current_stream()))

    def fn8():
        j = i[0] % nbuf
        i[0] += 1
        base = L.LinearArgsC(A=Aq[j].data_ptr(), lda=K, W=Wq[j].data_ptr(), ldw=K, M=M, N=N, K=K, out=x.data_ptr(), ldo=N,
                             bias=bias.data_ptr(), epilogue=epi, resid=x.data_ptr() if resid_epi else None, ldr=N if resid_epi else 0,
                             gate=mod[:, 2].data_ptr() if epi == 3 else None, gate_stride=6 * N if epi == 3 else 0,
                             rows_per_batch=rows_per_batch, stats_out=stats.data_ptr() if stats_mode else None,
                             stats_ld=stats.shape[1] if stats_mode else 0, stats_mode=stats_mode)
        args = L.LinearFp8ArgsC(base=base, a_scale=sa[j].data_ptr(), w_scale=sw[j].data_ptr())
        L.check(lib.ce_linear_fp8_ex(args, L.current_stream()))

    msq = timeit(quant)
    ms8 = timeit(fn8)
    row.update(fp8_ms=round(ms8, 4), fp8_tflops=round(2.0 * M * N * K / ms8 / 1e9, 1), fp8_quant_ms=round(msq, 4),
               fp8_quant_GBps=round(3.0 * M * K / msq / 1e6, 1))
    print(json.dumps(row), flush=True)
    if cublas:   # library bar: cuBLAS through torch on the same shapes
        ms2 = timeit(lambda: torch.matmul(A[0], W[0].t()))
        print(json.dumps({"op": "cublas_gemm", "M": M, "N": N, "K": K, "ms": round(ms2, 4), "tflops": round(2.0 * M * N * K / ms2 / 1e9, 1)}), flush=True)


def bench_gemm_k(Ks=(1280, 2560, 5120, 10240, 13824), M=14400, N=5120):
    """The o-proj GEMM (gate * residual + statistics) at several K: least-squares fit of ms per wave = a + b K."""
    import numpy as np

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = ((M + 127) // 128) * ((N + 255) // 256)
    waves = (tiles + sms - 1) // sms
    per_wave = [bench_gemm(f"o_proj_k{K}", N, K, 3, 1, M=M, cublas=False, fp8=False) / waves for K in Ks]
    b, a = np.polyfit(np.array(Ks, dtype=float), np.array(per_wave), 1)
    print(json.dumps({"op": "gemmk_fit", "M": M, "N": N, "tiles": tiles, "waves": waves, "sms": sms,
                      "a_us_per_tile": round(a * 1e3, 2), "b_ns_per_k": round(b * 1e6, 3),
                      "main_loop_tflops": round(sms * 2.0 * 128 * 256 / (b * 1e-3) / 1e12, 1)}), flush=True)


def bench_rows(M=14400, D=5120):
    x = torch.randn(M, D, device="cuda", dtype=torch.bfloat16)
    y = torch.empty_like(x)
    mod = torch.randn(2, 6, D, device="cuda")
    ms = timeit(lambda: L.check(lib.ce_layernorm_bf16(L.ptr(x), D, L.ptr(y), D, M, D, 1e-6, L.ptr(mod[:, 1]), L.ptr(mod[:, 0]), 6 * D, M // 2, None,
                                                      None, L.current_stream())))
    print(json.dumps({"op": "layernorm_mod", "M": M, "D": D, "ms": round(ms, 4), "GBps": round(4.0 * M * D / ms / 1e6, 1)}), flush=True)
    w = torch.ones(D, device="cuda", dtype=torch.bfloat16)
    cos = torch.randn(M // 2, 64, device="cuda")
    ms = timeit(lambda: L.check(lib.ce_rmsnorm_rope_bf16(L.ptr(x), D, M, D, 1e-6, L.ptr(w), L.ptr(cos), L.ptr(cos), M // 2, 128, L.current_stream())))
    print(json.dumps({"op": "rmsnorm_rope", "M": M, "D": D, "ms": round(ms, 4), "GBps": round(4.0 * M * D / ms / 1e6, 1)}), flush=True)
    # the same two operators with their row statistics from the epilogue of the GEMM that wrote the rows, as the DiT runs them at
    # D % 256 == 0: the (1 + scale) modulation, and q | k of the fused QKV output in one launch.  Outputs of the GEMM have rms ~ 1, so
    # the in-place RMSNorm, which keeps the GEMM's statistics over its repeats, stays in range.
    def gemm_with_stats(N, mode, K=256):
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        st = torch.empty(M, N // 256, 2, device="cuda")
        a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
        wt = (torch.randn(N, K, device="cuda") / math.sqrt(K)).bfloat16()
        args = L.LinearArgsC(A=a.data_ptr(), lda=K, W=wt.data_ptr(), ldw=K, M=M, N=N, K=K, out=out.data_ptr(), ldo=N,
                             stats_out=st.data_ptr(), stats_ld=N // 256, stats_mode=mode)
        L.check(lib.ce_linear_ex_bf16(args, L.current_stream()))
        return out, st

    x, st = gemm_with_stats(D, 1)
    mod1p = mod.clone()
    mod1p[:, 1] += 1
    ms = timeit(lambda: L.check(lib.ce_layernorm_stats_bf16(L.ptr(x), D, L.ptr(y), D, M, D, 1e-6, L.ptr(mod1p[:, 1]), L.ptr(mod1p[:, 0]), 6 * D,
                                                            M // 2, None, None, 1, L.ptr(st), D // 256, D // 256, 256, L.current_stream())))
    print(json.dumps({"op": "layernorm_mod_stats", "M": M, "D": D, "ms": round(ms, 4), "GBps": round(4.0 * M * D / ms / 1e6, 1)}), flush=True)
    qkv, st = gemm_with_stats(3 * D, 2)
    ang = torch.rand(M // 2, 64, device="cuda") * (2 * math.pi)   # a true rotation: the repeats keep the norm
    cos, sin = ang.cos(), ang.sin()
    ms = timeit(lambda: L.check(lib.ce_rmsnorm_rope_stats_bf16(L.ptr(qkv), 3 * D, M, D, 1e-6, L.ptr(w), L.ptr(w), 2, L.ptr(cos), L.ptr(sin), M // 2,
                                                               128, L.ptr(st), 3 * D // 256, D // 256, L.current_stream())))
    print(json.dumps({"op": "rmsnorm_rope_qk_stats", "M": M, "D": D, "ms": round(ms, 4), "GBps": round(8.0 * M * D / ms / 1e6, 1)}), flush=True)


def bench_conv(Cin=96, Cout=96, T=4, H=720, W=1280):
    from chronoedit_b200.autoencoder import pack_parameter

    x = torch.randn(T + 2, H, W, Cin, device="cuda", dtype=torch.bfloat16)
    w = pack_parameter("l.weight", torch.randn(Cout, Cin, 3, 3, 3, device="cuda") * 0.02)
    b = torch.zeros(Cout, device="cuda", dtype=torch.bfloat16)
    y = torch.empty(T, H, W, Cout, device="cuda", dtype=torch.bfloat16)
    ms = timeit(lambda: L.check(lib.ce_conv3d_cl_bf16(L.ptr(x), T + 2, H, W, Cin, L.ptr(w), L.ptr(b), Cout, 3, 3, 3, 1, 1, 1, 1, 1, 0, L.ptr(y), T, H, W,
                                                      None, 0, L.current_stream())), iters=5, warmup=2)
    fl = 2.0 * 27 * Cin * Cout * T * H * W
    print(json.dumps({"op": "conv3x3x3", "Cin": Cin, "Cout": Cout, "T": T, "H": H, "W": W, "ms": round(ms, 3), "tflops": round(fl / ms / 1e9, 1)}), flush=True)
    xt = x.permute(3, 0, 1, 2)[None].contiguous(memory_format=torch.channels_last_3d)
    wt = torch.randn(Cout, Cin, 3, 3, 3, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last_3d)
    try:
        ms2 = timeit(lambda: torch.nn.functional.conv3d(xt, wt, padding=(0, 1, 1)), iters=3, warmup=1)
        print(json.dumps({"op": "cudnn_conv3d", "ms": round(ms2, 3), "tflops": round(fl / ms2 / 1e9, 1)}), flush=True)
    except Exception as e:  # noqa: BLE001
        print(json.dumps({"op": "cudnn_conv3d", "error": str(e)[:200]}), flush=True)


if __name__ == "__main__":
    what = sys.argv[1:] or ["attn", "gemm", "rows"]
    if "attn" in what:
        bench_attn()
        bench_attn(B=1)
        bench_attn(Lk=512)
        bench_attn(Lk=257)
        bench_attn_dual()
    if "attn8" in what:
        bench_attn8()
        bench_attn8(B=2, Lk=28800)
    if "attnab" in what:
        bench_attn_ab()
        bench_attn_ab(B=1, Lq=28800, Lk=28800, rounds=10, iters=2)
        bench_attn_ab(Lk=512, Lk2=257)
    if "attnself" in what:
        bench_attn()
        bench_attn(B=1, Lq=28800, Lk=28800, nbuf=2)
    if "attncross" in what:
        bench_attn(Lk=512)
        bench_attn(Lk=257)
        bench_attn_dual()
    if "attnlib" in what:
        bench_attn()
        bench_attn_libs()
        bench_attn(B=1, Lq=28800, Lk=28800, nbuf=2)
        bench_attn_libs(B=1, L=28800)
        bench_attn(Lk=512)
        bench_attn_libs(L=7200, Lk=512)
    if "gemm" in what:
        for case in DIT_GEMMS:
            bench_gemm(*case, cublas="cublas" in what)
    if "gemmk" in what:
        bench_gemm_k()
    if "rows" in what:
        bench_rows()
    if "conv" in what:
        bench_conv(96, 96, 4, 720, 1280)
        bench_conv(192, 192, 4, 360, 640)
        bench_conv(384, 384, 2, 180, 320)
