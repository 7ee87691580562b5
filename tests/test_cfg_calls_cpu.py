"""The call-pair split (parallel.enable_cfg_parallel_calls) without a GPU, driven by the pipeline's own call order.

Two "ranks" run in two threads, each with its own pipeline loop and its own mirror instances.  The mirrors' native seams are stood in
for by the oracle exactly as in tests/test_pipeline_cpu.py, and the exchange seam (`_native_cp_exchange`, ce_dit_cp_exchange) by a
Python stand-in: a threading.Barrier and a copy, with the two slot sets alternating by the barrier's parity as on the device.  Driven
by the UNMODIFIED reference pipeline file where it exists, and everywhere by its restatement in oracle/pipeline_oracle.py (pinned bit
for bit against that file by tests/test_pipeline_cpu.py).

Asserted: both ranks return the video of the single-instance run bit for bit, each rank runs exactly one native forward per step (the
prompt calls on rank 0, the negative-prompt calls on rank 1), and a guidance-free run raises the pairing check's CEError on both ranks
instead of returning a video.  The device path runs in tests/test_gpu_cfg_calls_one_gpu.py."""
import contextlib
import ctypes
import threading

import pytest
import torch
import torch.distributed as dist

from chronoedit_b200 import parallel
from oracle import pipeline_cases as PC, ref_loader
from tests.test_pipeline_cpu import _mirror_scheduler, _mirror_transformer, _mirror_vae

needs_ref = pytest.mark.skipif(not ref_loader.reference_available(), reason="the reference pipeline file is not on this machine")
TIMEOUT_S = 300


@pytest.fixture
def host_only_configure(monkeypatch):
    """configure_cfg_parallel_calls on a CPU model: the device context and synchronise of the peer-region helpers become no-ops."""
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "synchronize", lambda device=None: None)


def _counted_mirror(dsd):
    """The transformer mirror with the oracle behind its native forward, counting the native forwards."""
    m = _mirror_transformer(dsd)
    inner = m._native_forward
    m.native_calls = 0

    def native_forward(*args):
        m.native_calls += 1
        inner(*args)

    m._native_forward = native_forward
    return m


def _exchange_stand_in(models):
    """ce_dit_cp_exchange for `models` [rank 0, rank 1]: own into the peer's slot of set (epoch & 1), one barrier, the peer's sample
    out of the own slot of that set."""
    barrier = threading.Barrier(2, timeout=TIMEOUT_S)
    slots = [[None, None], [None, None]]   # [set][rank]: what rank wrote for its peer
    epoch = [0, 0]

    for r, m in enumerate(models):
        def native(own, other, r=r):
            p = epoch[r] & 1
            slots[p][r] = own.clone()
            barrier.wait()
            epoch[r] += 1
            other.copy_(slots[p][1 - r])

        m._native_cp_exchange = native


def _run(driver, case):
    """Both ranks through `driver(case, transformer, vae, scheduler)` at once; returns (videos, errors, models)."""
    dsd, vsd = PC.weights()
    models = [_counted_mirror(dsd) for _ in range(2)]
    for r, m in enumerate(models):
        m._ensure_handle()
        parallel.configure_cfg_parallel_calls(m, r, [4096, 8192], 1 << 20, {})
    _exchange_stand_in(models)
    videos, errors = [None, None], [None, None]

    def work(r):
        try:
            videos[r] = driver(case, models[r], _mirror_vae(vsd), _mirror_scheduler(case.sched_shift))
        except BaseException as e:   # noqa: BLE001 -- examined by the test
            errors[r] = e

    threads = [threading.Thread(target=work, args=(r,), daemon=True) for r in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(TIMEOUT_S)
    assert not any(t.is_alive() for t in threads), "a rank is still running"
    return videos, errors, models


def _unmodified(case, tr, vae, sch):
    return PC.run_reference_pipeline(case, torch.bfloat16, transformer=tr, vae=vae, scheduler=sch)


def _restated(case, tr, vae, sch):
    return PC.run_oracle_pipeline(case, torch.bfloat16, transformer=tr, vae=vae, scheduler=sch)


DRIVERS = [pytest.param(_unmodified, marks=needs_ref, id="unmodified_pipeline"), pytest.param(_restated, id="restated_pipeline")]


@pytest.mark.parametrize("driver", DRIVERS)
@pytest.mark.parametrize("name", ["edit_5f", "reason_cut", "reason_full"])
def test_pipeline_calls_split_over_two_ranks_equal_one_instance(name, driver, host_only_configure):
    if driver is _unmodified:
        ref_loader.load_reference_pipeline()   # loaded once, before the threads
    case = PC.PIPELINE_CASES[name]
    dsd, vsd = PC.weights()
    single = _counted_mirror(dsd)
    want = driver(case, single, _mirror_vae(vsd), _mirror_scheduler(case.sched_shift))
    assert single.native_calls == 2 * case.steps
    videos, errors, models = _run(driver, case)
    try:
        for r, e in enumerate(errors):
            assert e is None, f"rank {r} failed: {e!r}"
        for r, v in enumerate(videos):
            assert v.shape == want.shape
            assert torch.equal(v, want), f"rank {r}: max|diff| {float((v.float() - want.float()).abs().max())}"
        assert [m.native_calls for m in models] == [case.steps, case.steps], "each rank computes one call per step"
        assert all(m._cp_pair is None for m in models), "a pair is still open after the last step"
    finally:
        for m in models:
            parallel.disable_cfg_parallel_calls(m)


@pytest.mark.parametrize("driver", DRIVERS)
def test_guidance_free_pipeline_is_refused_by_the_pairing_check(driver, host_only_configure):
    """guidance_scale <= 1: one call per step, so the second call of the first "pair" is the next step's prompt call with new
    latents.  Both ranks raise there, before any launch, and neither returns a video."""
    from chronoedit_b200._lib import CEError

    if driver is _unmodified:
        ref_loader.load_reference_pipeline()
    case = PC.PIPELINE_CASES["edit_nocfg"]
    videos, errors, models = _run(driver, case)
    try:
        for r in range(2):
            assert videos[r] is None, f"rank {r} returned a video"
            assert isinstance(errors[r], CEError), f"rank {r}: {errors[r]!r}"
            assert "does not pair with the previous one" in str(errors[r]) and "guidance_scale > 1" in str(errors[r])
        assert [m.native_calls for m in models] == [1, 0], "only rank 0 computes the first step's call"
        assert all(m._cp_pair is None for m in models), "the refused call left the pair open"
    finally:
        for m in models:
            parallel.disable_cfg_parallel_calls(m)


# ---------------------------------------------------------------------------------------------------------------------
# the C ABI's host-only parts and the Python state
# ---------------------------------------------------------------------------------------------------------------------
def _handle(out_channels=16):
    import chronoedit_b200 as ce

    m = ce.ChronoEditTransformer3DModel(num_attention_heads=2, in_channels=36, out_channels=out_channels, ffn_dim=256, num_layers=1,
                                        image_dim=1280, added_kv_proj_dim=256, text_dim=64)
    return m, m._ensure_handle()


def test_cp_region_bytes_is_the_batch_split_layout_for_one_call():
    from chronoedit_b200 import _lib
    from tests.test_cfg_parallel_cpu import bp_layout

    L = _lib.lib()
    for oc in (16, 12):
        m, h = _handle(out_channels=oc)
        for B in (1, 2, 8):
            for T, H, W in ((2, 16, 16), (8, 90, 160), (2, 30, 42), (1, 2, 2)):
                assert L.ce_dit_cp_region_bytes(h, B, T, H, W) == bp_layout(B, oc, T, H, W)["bytes"], (oc, B, T, H, W)
    m, h = _handle()
    assert L.ce_dit_cp_region_bytes(None, 1, 2, 16, 16) == -1
    assert L.ce_dit_cp_region_bytes(h, 0, 2, 16, 16) == -1
    assert L.ce_dit_cp_region_bytes(h, 9, 2, 16, 16) == -1
    assert L.ce_dit_cp_region_bytes(h, 1, 0, 16, 16) == -1
    assert L.ce_dit_cp_region_bytes(h, 1, 2, -16, 16) == -1
    assert parallel.cfg_calls_region_bytes(m, 1, 8, 90, 160) == bp_layout(1, 16, 8, 90, 160)["bytes"]


def test_cp_configure_refusals():
    """The call-pair group refuses what the batch group does, a world other than 1 or 2, and the batch group beside it (and the
    batch group refuses it); the token group composes with it."""
    from chronoedit_b200 import _lib

    L = _lib.lib()
    m, h = _handle()
    table = (ctypes.c_void_p * 8)(*[4096 * (w + 1) for w in range(8)])   # configure never dereferences the addresses

    def refused(entry, *args, msg):
        assert getattr(L, entry)(*args) == -1
        assert msg in L.ce_last_error().decode()

    refused("ce_dit_cp_configure", None, 0, 2, table, 64, msg="null handle")
    refused("ce_dit_cp_configure", h, 0, 0, table, 64, msg="ce_dit_cp_configure: arguments")
    refused("ce_dit_cp_configure", h, 2, 2, table, 64, msg="ce_dit_cp_configure: arguments")
    refused("ce_dit_cp_configure", h, 0, 2, None, 64, msg="ce_dit_cp_configure: arguments")
    refused("ce_dit_cp_configure", h, 0, 2, table, 0, msg="ce_dit_cp_configure: arguments")
    refused("ce_dit_cp_configure", h, 0, 2, (ctypes.c_void_p * 2)(4096, None), 64, msg="null region pointer")
    refused("ce_dit_cp_configure", h, 0, 2, (ctypes.c_void_p * 2)(4096, 8192 + 16), 64, msg="256-byte aligned")
    for world in (3, 4, 8):
        refused("ce_dit_cp_configure", h, 0, world, table, 64, msg="a CFG pair has two calls")
    assert L.ce_dit_bp_configure(h, 0, 2, table, 64) == 0
    refused("ce_dit_cp_configure", h, 0, 2, table, 64, msg="the two CFG splits are exclusive")
    assert L.ce_dit_bp_configure(h, 0, 1, None, 0) == 0
    assert L.ce_dit_cp_configure(h, 1, 2, table, 64) == 0
    refused("ce_dit_bp_configure", h, 0, 2, table, 64, msg="the two CFG splits are exclusive")
    assert L.ce_dit_sp_configure(h, 0, 2, table, 64) == 0             # the token split composes with it
    assert L.ce_dit_sp_configure(h, 0, 1, None, 0) == 0
    assert L.ce_dit_bp_configure(h, 0, 1, None, 0) == 0               # switching the other group off is always accepted
    assert L.ce_dit_cp_configure(h, 0, 1, None, 0) == 0
    assert L.ce_dit_bp_configure(h, 0, 2, table, 64) == 0
    assert L.ce_dit_bp_configure(h, 0, 1, None, 0) == 0


def test_cp_exchange_and_host_barrier_arguments():
    from chronoedit_b200 import _lib

    L = _lib.lib()
    m, h = _handle()
    buf = ctypes.c_void_p(4096)
    assert L.ce_dit_cp_exchange(None, buf, buf, 1, 2, 16, 16, None) == -1 and b"null argument" in L.ce_last_error()
    assert L.ce_dit_cp_exchange(h, buf, buf, 1, 2, 16, 16, None) == -1 and b"not configured" in L.ce_last_error()
    assert L.ce_dit_cp_host_barrier(None, 1000) == -1 and b"ce_dit_cp_host_barrier: arguments" in L.ce_last_error()
    assert L.ce_dit_cp_host_barrier(h, -1) == -1 and b"ce_dit_cp_host_barrier: arguments" in L.ce_last_error()
    assert L.ce_dit_cp_host_barrier(h, 60000) == 0
    assert L.ce_dit_cp_host_barrier(h, 0) == 0


def test_enable_cfg_parallel_calls_needs_a_process_group():
    from chronoedit_b200._lib import CEError

    assert not dist.is_initialized()
    with pytest.raises(CEError, match="enable_cfg_parallel_calls needs an initialised torch.distributed process group"):
        parallel.enable_cfg_parallel_calls(object(), 1, 2, 16, 16)
    parallel.disable_cfg_parallel_calls(object())   # a model that never enabled it: no-op


def test_call_pair_state_and_refusals(host_only_configure):
    """The Python side of the mode on a CPU model: the state is kept apart from the other groups, every refusal comes before the first
    seam is reached, a refused second call drops the pair, and disabling with an open pair warns."""
    from chronoedit_b200._lib import CEError

    m, h = _handle()
    seen = []
    m._native_forward = lambda x, t, txt, img, out, *a: (seen.append("forward"), out.fill_(1.0))
    m._native_cp_exchange = lambda own, other: (seen.append("exchange"), other.copy_(own))
    m._ctx_cache = ["stale"]
    parallel.configure_cfg_parallel_calls(m, 1, [4096, 8192], 1 << 20, {})
    assert m._cp_state == {"rank": 1, "world": 2, "bytes": 1 << 20} and m._cp_pair is None
    assert getattr(m, "_bp_state", None) is None and getattr(m, "_sp_state", None) is None
    assert m._ctx_cache == []
    with pytest.raises(CEError, match="the two CFG splits are exclusive"):
        parallel.configure_cfg_parallel(m, 0, [4096, 8192], 1 << 20, {})
    x, t = torch.zeros(1, 36, 2, 8, 8), torch.tensor([900.0])
    txt, neg, img = torch.zeros(1, 16, 64), torch.ones(1, 16, 64), torch.zeros(1, 257, 1280)
    for kw in ({"return_block0": True}, {"capture_layers": (0,)}):
        with pytest.raises(CEError, match="not available with the call-pair split"):
            m(x, t, txt, img, **kw)
    with pytest.raises(CEError, match="forward_host is not available with the call-pair split"):
        m.forward_host(x.bfloat16(), t, txt.bfloat16(), img.bfloat16())
    with pytest.raises(CEError, match="forward_fp32 is not available with the call-pair split"):
        m._fp32_keepalive = {"w": torch.zeros(1)}
        m.forward_fp32(x, t, txt, img)
    assert seen == []
    # rank 1: the prompt call is not computed (NaN, no seam), the negative-prompt call is, then the exchange fills the first sample
    out0 = m(x, t, txt, img, return_dict=False)[0]
    assert seen == [] and m._cp_pair is not None
    assert (out0.view(torch.int16) == -1).all() and torch.isnan(out0.float()).all()
    out1 = m(x, t, neg, img, return_dict=False)[0]
    assert seen == ["forward", "exchange"] and m._cp_pair is None
    assert (out0 == 1).all() and (out1 == 1).all()
    # a second call with other latents, an in-place change, another timestep or another image: refused, the pair dropped
    for change in ("x", "x_inplace", "t", "img"):
        seen.clear()
        m(x, t, txt, img)
        x2, t2, img2 = x, t, img
        if change == "x":
            x2 = x.clone()
        elif change == "x_inplace":
            x.add_(0)
        elif change == "t":
            t2 = t.clone()
        else:
            img2 = img.clone()
        with pytest.raises(CEError, match="does not pair with the previous one"):
            m(x2, t2, neg, img2)
        assert seen == [] and m._cp_pair is None
    m(x, t, txt, img)
    with pytest.warns(UserWarning, match="still open"):
        parallel.disable_cfg_parallel_calls(m)
    assert m._cp_state is None and m._cp_pair is None
