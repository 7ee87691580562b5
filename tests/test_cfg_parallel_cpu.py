"""The batch split of the DiT forward (parallel.enable_cfg_parallel, ce_dit_bp_*) without a GPU: the region layout, the host-only
refusals, and the Python state it keeps apart from the token split's.  The data path runs in tests/test_gpu_cfg_parallel_one_gpu.py
(one GPU, host barrier) and tests/test_gpu_cfg_parallel.py (two GPUs)."""
import contextlib
import ctypes

import pytest
import torch
import torch.distributed as dist

from chronoedit_b200 import parallel


def bp_layout(B, out_channels, T, H, W):
    """Python restatement of the batch split's peer region (csrc/dit.cu): the flags block (uint32 [8 * 32]) first, then two slots of
    the call's full sample [B, out_channels, T, H, W] bf16, each rounded up to 1024 bytes."""
    used = B * out_channels * T * H * W * 2
    slot = (used + 1023) & ~1023
    return {"flags": 0, "slot": [1024, 1024 + slot], "used": used, "slot_bytes": slot, "bytes": 1024 + 2 * slot}


def bp_unwritten_ranges(lay, used=None):
    """[start, end) byte ranges of a region that a split call writing `used` sample bytes (default: the layout's) never writes under the
    host barrier: the flags block (only the device barrier uses it) and each slot's tail."""
    used = lay["used"] if used is None else used
    out = [("flags", 0, 1024)]
    for i, a in enumerate(lay["slot"]):
        if used < lay["slot_bytes"]:
            out.append((f"slot {i} gap", a + used, a + lay["slot_bytes"]))
    return out


def _handle(heads=2, out_channels=16):
    import chronoedit_b200 as ce

    m = ce.ChronoEditTransformer3DModel(num_attention_heads=heads, in_channels=36, out_channels=out_channels, ffn_dim=256, num_layers=1,
                                        image_dim=1280, added_kv_proj_dim=heads * 128, text_dim=64)
    return m, m._ensure_handle()


def test_bp_region_bytes_matches_the_layout_restatement():
    from chronoedit_b200 import _lib

    L = _lib.lib()
    gaps = 0
    for oc in (16, 12):
        m, h = _handle(out_channels=oc)
        for world in range(2, 9):
            for B in (world, 2 * world):
                if B > 8:
                    continue
                for T, H, W in ((2, 16, 16), (8, 90, 160), (2, 30, 42), (1, 2, 2)):
                    lay = bp_layout(B, oc, T, H, W)
                    assert L.ce_dit_bp_region_bytes(h, B, T, H, W, world) == lay["bytes"], (oc, world, B, T, H, W)
                    assert lay["slot"][1] % 1024 == 0 and lay["bytes"] - lay["slot"][1] == lay["slot_bytes"] >= lay["used"]
                    gaps += len(bp_unwritten_ranges(lay)) - 1
    assert gaps > 0, "no case exercised the alignment gap after a slot"


def test_bp_region_bytes_refusals():
    from chronoedit_b200 import _lib

    L = _lib.lib()
    m, h = _handle(heads=3)
    assert L.ce_dit_bp_region_bytes(h, 2, 2, 16, 16, 2) > 0
    assert L.ce_dit_bp_region_bytes(h, 6, 2, 16, 16, 3) > 0        # no head-count rule: the samples are split, not the heads
    assert L.ce_dit_bp_region_bytes(None, 2, 2, 16, 16, 2) == -1
    assert L.ce_dit_bp_region_bytes(h, 2, 2, 16, 16, 1) == -1     # world 1 is no split
    assert L.ce_dit_bp_region_bytes(h, 2, 2, 16, 16, 9) == -1     # at most 8 ranks
    assert L.ce_dit_bp_region_bytes(h, 0, 2, 16, 16, 2) == -1     # batch
    assert L.ce_dit_bp_region_bytes(h, 10, 2, 16, 16, 2) == -1    # batch at most 8, as the forward
    assert L.ce_dit_bp_region_bytes(h, 1, 2, 16, 16, 2) == -1     # the diffusers pipeline's batch-1 calls are not split
    assert L.ce_dit_bp_region_bytes(h, 6, 2, 16, 16, 4) == -1     # 6 % 4
    assert L.ce_dit_bp_region_bytes(h, 2, 0, 16, 16, 2) == -1     # geometry
    assert L.ce_dit_bp_region_bytes(h, 2, 2, 16, -2, 2) == -1


def test_bp_configure_refusals():
    """The batch group's configure refuses what the token group's does, except the head count; world 1 switches it off."""
    from chronoedit_b200 import _lib

    L = _lib.lib()
    m, h = _handle(heads=3)
    table = (ctypes.c_void_p * 8)(*[4096 * (w + 1) for w in range(8)])   # configure never dereferences the addresses

    def refused(*args, msg):
        assert L.ce_dit_bp_configure(*args) == -1
        assert msg in L.ce_last_error().decode()

    refused(None, 0, 2, table, 64, msg="null handle")
    refused(h, 0, 9, table, 64, msg="ce_dit_bp_configure: arguments")
    refused(h, 0, 0, table, 64, msg="ce_dit_bp_configure: arguments")
    refused(h, -1, 2, table, 64, msg="ce_dit_bp_configure: arguments")
    refused(h, 2, 2, table, 64, msg="ce_dit_bp_configure: arguments")
    refused(h, 0, 2, None, 64, msg="ce_dit_bp_configure: arguments")
    refused(h, 0, 2, table, 0, msg="ce_dit_bp_configure: arguments")
    refused(h, 0, 2, (ctypes.c_void_p * 2)(4096, None), 64, msg="null region pointer")
    refused(h, 0, 2, (ctypes.c_void_p * 2)(4096, 8192 + 16), 64, msg="256-byte aligned")
    assert L.ce_dit_bp_configure(h, 1, 2, table, 64) == 0           # 3 heads over 2 ranks: fine for the batch split
    assert L.ce_dit_sp_configure(h, 0, 2, table, 64) == -1          # but not for the token split
    assert L.ce_dit_bp_configure(h, 0, 1, None, 0) == 0             # world 1 switches it off


def test_bp_host_barrier_arguments():
    from chronoedit_b200 import _lib

    L = _lib.lib()
    m, h = _handle()
    assert L.ce_dit_bp_host_barrier(None, 1000) == -1 and b"ce_dit_bp_host_barrier: arguments" in L.ce_last_error()
    assert L.ce_dit_bp_host_barrier(h, -1) == -1 and b"ce_dit_bp_host_barrier: arguments" in L.ce_last_error()
    assert L.ce_dit_bp_host_barrier(h, 60000) == 0
    assert L.ce_dit_bp_host_barrier(h, 0) == 0


def test_enable_cfg_parallel_needs_a_process_group():
    from chronoedit_b200._lib import CEError

    assert not dist.is_initialized()
    with pytest.raises(CEError, match="enable_cfg_parallel needs an initialised torch.distributed process group"):
        parallel.enable_cfg_parallel(object(), 2, 2, 16, 16)
    parallel.disable_cfg_parallel(object())   # a model that never enabled it: no-op
    m, _ = _handle()
    with pytest.raises(CEError, match=r"batch \(1\) must divide by the world size \(2"):
        parallel.cfg_region_bytes(m, 1, 2, 16, 16, 2)


@pytest.fixture
def host_only_configure(monkeypatch):
    """configure_cfg_parallel on a CPU model: the device context and synchronise of the peer-region helpers become no-ops."""
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "synchronize", lambda device=None: None)


def test_batch_group_is_kept_apart_from_the_token_group(host_only_configure):
    """Configuring the batch group sets model._bp_state only: every refusal the token split's _sp_state drives stays as it was, and
    enable_teacache (refused under the token split) still works.  Disable switches the C handle back and drops the per-sample caches."""
    from chronoedit_b200 import _lib
    from chronoedit_b200._lib import CEError

    m, h = _handle()
    m._ctx_cache = ["stale"]
    parallel.configure_cfg_parallel(m, 1, [4096, 8192], 1 << 20, {})
    assert m._bp_state == {"rank": 1, "world": 2, "bytes": 1 << 20}
    assert getattr(m, "_sp_state", None) is None
    assert m._ctx_cache == []                                       # K/V of the old share of samples
    assert m._local_samples(2) == (1, 1) and m._local_samples(4) == (2, 2) and m._local_samples(1) == (0, 1)
    m.enable_teacache(0.2, num_inference_steps=8)
    assert m.teacache_enabled
    m.disable_teacache()
    parallel.disable_cfg_parallel(m)
    assert m._bp_state is None and m._local_samples(2) == (0, 2)
    assert _lib.lib().ce_dit_bp_region_bytes(h, 2, 2, 16, 16, 2) > 0
    m._sp_state = {"world": 2}
    with pytest.raises(CEError, match="sequence parallelism"):
        m.enable_teacache(0.2, num_inference_steps=8)


def test_teacache_under_the_batch_split_sizes_by_the_local_samples(host_only_configure):
    """With TeaCache on, rank 1 of 2 probes its own timestep only, and its modulation and residual hold one sample of a batch-2 call.
    The two native seams are stood in for; the call still reaches the forward with the full batch (the C side splits it)."""
    m, _ = _handle()
    parallel.configure_cfg_parallel(m, 1, [4096, 8192], 1 << 20, {})
    m.enable_teacache(1e9, num_inference_steps=4)
    seen = []

    def probe(t, prev, cur):
        seen.append(("probe", t.tolist(), cur.numel(), None if prev is None else prev.numel()))
        return None if prev is None else (1.0, 100.0)

    def fwd(x, t, txt, img, out, txt_in, img_in, resid, record):
        seen.append(("forward", x.shape[0], t.numel(), out.shape[0], resid.numel(), record))

    m._native_probe, m._native_teacache_forward = probe, fwd
    D = 2 * 128
    x = torch.zeros(2, 36, 2, 8, 8)
    txt = torch.zeros(2, 16, 64)
    img = torch.zeros(2, 257, 1280)
    for tv in (900, 700):
        m(x, torch.tensor([tv, tv - 50]), txt, img)
    L = 2 * 4 * 4
    assert seen == [("probe", [850.0], 6 * D, None), ("forward", 2, 2, 2, L * D, True),
                    ("probe", [650.0], 6 * D, 6 * D), ("forward", 2, 2, 2, L * D, False)]
    with pytest.raises(Exception, match="unchanged diffusers pipeline's batch-1 calls are not split"):
        m(x[:1], torch.tensor([500]), txt[:1], img[:1])
    assert len(seen) == 4                                           # refused before the probe
    parallel.disable_cfg_parallel(m)
