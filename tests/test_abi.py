"""Host-side checks that need no GPU: the C-ABI library loads, exports every symbol the header declares, fails loudly
without a device, and its host-only entry points agree with the oracle."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _built():
    import chronoedit_b200._lib as L

    if not os.path.exists(L.LIB_PATH):
        from chronoedit_b200 import build

        build.build()
    return L


def test_library_exports_every_header_symbol():
    L = _built()
    hdr = open(os.path.join(ROOT, "include", "chronoedit_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(ce_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"ce_dit_config"}
    assert len(declared) >= 15
    so = ctypes.CDLL(L.LIB_PATH)
    for name in sorted(declared):
        assert hasattr(so, name), f"{name} declared in include/chronoedit_b200.h but not exported"
    assert declared == set(L.SIGNATURES), "ctypes binding and header disagree: " + str(declared ^ set(L.SIGNATURES))
    assert L.lib().ce_abi_version() == 1


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    L = _built()
    lib = L.lib()
    assert lib.ce_device_check() != 0
    assert b"no CPU fallback" in lib.ce_last_error()
    import chronoedit_b200 as ce

    m = ce.ChronoEditTransformer3DModel(num_attention_heads=2, in_channels=36, ffn_dim=256, num_layers=1, image_dim=1280,
                                        added_kv_proj_dim=256, text_dim=64)
    with pytest.raises(ce.CEError, match="no CPU path"):
        m(torch.zeros(1, 36, 2, 4, 4), torch.tensor([1]), torch.zeros(1, 8, 64), torch.zeros(1, 257, 1280))
    a = torch.zeros(8, 8, dtype=torch.bfloat16)
    rc = lib.ce_linear_bf16(L.ptr(a), 8, L.ptr(a), 8, None, L.ptr(a), 8, None, 8, 8, 8, 0, None, 0, None, 0, 1, None)
    assert rc != 0
    # the fused-statistics operators: the device check comes first, whatever the arguments
    st = torch.zeros(8, 2)
    la = L.LinearArgsC(A=a.data_ptr(), lda=8, W=a.data_ptr(), ldw=8, M=8, N=8, K=8, out=a.data_ptr(), ldo=8, stats_out=st.data_ptr(),
                       stats_ld=1, stats_mode=1)
    assert lib.ce_linear_ex_bf16(ctypes.byref(la), None) == -3 and b"no CPU fallback" in lib.ce_last_error()
    assert lib.ce_linear_ex_bf16(None, None) == -3 and b"no CPU fallback" in lib.ce_last_error()
    assert lib.ce_layernorm_stats_bf16(L.ptr(a), 8, L.ptr(a), 8, 8, 8, 1e-6, None, None, 0, 0, None, None, 0, L.ptr(st), 1, 1, 8,
                                       None) == -3 and b"no CPU fallback" in lib.ce_last_error()
    assert lib.ce_rmsnorm_rope_stats_bf16(L.ptr(a), 8, 8, 8, 1e-6, L.ptr(a), None, 1, None, None, 0, 8, L.ptr(st), 1, 1,
                                          None) == -3 and b"no CPU fallback" in lib.ce_last_error()
    # the VAE and encoder operators: the device check comes first, valid arguments or not
    assert lib.ce_rms_silu_cl_bf16(L.ptr(a), L.ptr(a), L.ptr(a), 8, 8, 1, None) == -3 and b"no CPU fallback" in lib.ce_last_error()
    assert lib.ce_upsample2x_cl_bf16(L.ptr(a), L.ptr(a), 1, 1, 1, 8, None) == -3 and b"no CPU fallback" in lib.ce_last_error()
    assert lib.ce_im2row_bf16(L.ptr(a), 1, 1, 1, 1, 1, 1, 1, 1, L.ptr(a), 8, 1, 1, 1, 1, 1, 1, 0, 0, 0,
                              None) == -3 and b"no CPU fallback" in lib.ce_last_error()
    ca = L.Conv3dArgsC(x=a.data_ptr(), Tin=1, Hin=1, Win=1, Cin=8, w=a.data_ptr(), Cout=8, Cin_pad=64, kt=1, kh=1, kw=1, st=1, sh=1, sw=1,
                       y=a.data_ptr(), Tout=1, Hout=1, Wout=1, planar_out=1, clamp=1, planar_T=1)
    assert lib.ce_conv3d_cl_ex_bf16(ctypes.byref(ca), None) == -3 and b"no CPU fallback" in lib.ce_last_error()
    assert lib.ce_conv3d_cl_ex_bf16(None, None) == -3 and b"no CPU fallback" in lib.ce_last_error()
    ga = L.GemmAttentionArgsC(x=a.data_ptr(), D=8, L=8, H=1, dk=8, kpv=8, wqk=a.data_ptr(), wv=a.data_ptr(), rule=1, scale=1.0,
                              bias=a.data_ptr(), bias_ld=15, valid=0, qk=a.data_ptr(), vT=a.data_ptr(), S=st.data_ptr(), P=a.data_ptr(),
                              out=a.data_ptr(), ldo=8)
    assert lib.ce_gemm_attention_bf16(ctypes.byref(ga), None) == -3 and b"no CPU fallback" in lib.ce_last_error()
    assert lib.ce_gemm_attention_bf16(None, None) == -3 and b"no CPU fallback" in lib.ce_last_error()
    # the sampler entry point: argument validation first, then the device check -- never a CPU evaluation
    args = L.UniPCStepArgsC()
    x = torch.zeros(64)
    args.sample_dtype, args.model_dtype, args.n, args.p_order = 0, 0, 64, 1
    args.cond = args.sample = args.x0_out = args.prev_sample_out = x.data_ptr()
    assert lib.ce_unipc_step(ctypes.byref(args), None) == -3 and b"no CPU fallback" in lib.ce_last_error()
    args.p_order = 3
    assert lib.ce_unipc_step(ctypes.byref(args), None) == -1
    assert lib.ce_debug_attention_kernel(7) == -1 and lib.ce_debug_attention_kernel(-1) == 0


def test_rope_table_host_matches_oracle():
    from oracle import dit_oracle as O

    L = _built()
    cfg = O.DiTConfig.tiny()
    for frames, hp, wp in [(2, 5, 7), (8, 3, 4)]:
        n = frames * hp * wp
        cos = torch.empty(n, 64, dtype=torch.float32)
        sin = torch.empty(n, 64, dtype=torch.float32)
        L.check(L.lib().ce_rope_table_host(128, frames, hp, wp, 1024, 8, 10000.0, L.ptr(cos), L.ptr(sin)))
        fr = O.rope_table(cfg, frames, 2 * hp, 2 * wp)[0, 0]
        torch.testing.assert_close(cos.double(), fr.real, rtol=0, atol=1e-7)
        torch.testing.assert_close(sin.double(), fr.imag, rtol=0, atol=1e-7)
    cos = torch.empty(5 * 4, 64)
    assert L.lib().ce_rope_table_host(128, 5, 2, 2, 1024, 8, 10000.0, L.ptr(cos), L.ptr(cos)) != 0
    assert b"num_frames must be 2 or" in L.lib().ce_last_error()


def test_mirror_parameter_names_match_reference_state_dict():
    """The Python mirror must accept a reference state_dict unchanged (names and shapes)."""
    import chronoedit_b200 as ce
    from oracle import dit_oracle as O

    cfg = O.DiTConfig.tiny()
    m = ce.ChronoEditTransformer3DModel(num_attention_heads=2, in_channels=36, ffn_dim=cfg.ffn_dim, num_layers=2, image_dim=1280,
                                        added_kv_proj_dim=256)
    mine = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert mine == O.param_shapes(cfg)
    assert m.config.patch_size[1] == 2 and m.dtype == torch.bfloat16
    for k, v in m.state_dict().items():
        want = torch.float32 if any(s in k for s in O.KEEP_FP32) else torch.bfloat16
        assert v.dtype == want, k
