"""world_size-2 gloo test (CPU) of the N>1 path: edit sharding and the one-time weight broadcast."""
import os
import socket
import types

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from chronoedit_b200 import parallel


def test_shard_edits_covers_every_edit_once():
    for n in (0, 1, 7, 8, 13):
        for world in (1, 2, 4, 8):
            seen = sorted(i for r in range(world) for i in parallel.shard_edits(n, r, world))
            assert seen == list(range(n))
            sizes = [len(parallel.shard_edits(n, r, world)) for r in range(world)]
            assert max(sizes) - min(sizes) <= 1
    with pytest.raises(ValueError):
        parallel.shard_edits(4, 2, 2)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import chronoedit_b200 as ce

        torch.manual_seed(100 + rank)  # different garbage on every rank before the broadcast
        m = ce.ChronoEditTransformer3DModel(num_attention_heads=2, in_channels=36, ffn_dim=256, num_layers=2, image_dim=1280,
                                            added_kv_proj_dim=256, text_dim=64)
        for p in m.parameters():
            p.data.copy_(torch.randn(p.shape).to(p.dtype))
        nbytes = parallel.broadcast_module_weights(m, src=0)
        expect = sum(p.numel() * p.element_size() for p in m.parameters())
        fingerprint = float(sum(p.data.double().sum() for p in m.parameters()))
        edits = parallel.shard_edits(5, rank, world)
        gathered = parallel.gather_objects([rank, fingerprint, edits, nbytes, expect])
        if rank == 0:
            q.put(gathered)
    finally:
        dist.destroy_process_group()


def test_weight_broadcast_and_sharding_gloo_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = q.get(timeout=180)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    (r0, f0, e0, n0, x0), (r1, f1, e1, n1, x1) = res
    assert (r0, r1) == (0, 1)
    assert f0 == f1, "weights differ across ranks after the broadcast"
    assert sorted(e0 + e1) == [0, 1, 2, 3, 4] and e0 == [0, 2, 4] and e1 == [1, 3]
    assert n0 == x0 and n1 == x1, "broadcast byte count must equal the parameter bytes"


def test_sequence_parallel_host_checks():
    """enable_sequence_parallel fails loudly (never silently falls back to a single-GPU forward) without a process group, and the
    region-size query rejects a missing handle; the data path itself needs NVLink peers (tests/test_gpu_seqpar.py, 2 GPUs)."""
    from chronoedit_b200 import _lib
    from chronoedit_b200._lib import CEError

    assert not dist.is_initialized()
    with pytest.raises(CEError, match="process group"):
        parallel.enable_sequence_parallel(object(), 1, 2, 4, 4)
    assert _lib.lib().ce_dit_sp_region_bytes(None, 1, 2, 4, 4, 2) == -1
    parallel.disable_sequence_parallel(object())   # a model that never enabled it: no-op


def _sp_handle(heads):
    """A C handle of a 1-layer model with `heads` heads (no device needed: the sequence-parallel set-up calls are host-only)."""
    import chronoedit_b200 as ce

    m = ce.ChronoEditTransformer3DModel(num_attention_heads=heads, in_channels=36, ffn_dim=256, num_layers=1, image_dim=1280,
                                        added_kv_proj_dim=heads * 128, text_dim=64)
    return m, m._ensure_handle()


def test_sp_region_bytes_matches_the_layout_restatement():
    """ce_dit_sp_region_bytes against the Python sp_layout the one-GPU test derives its guard ranges from, for world 2 to 8, with
    sub-buffer sizes that are and are not multiples of the 1024-byte alignment."""
    from chronoedit_b200 import _lib
    from tests.test_gpu_seqpar_one_gpu import sp_layout, sp_unwritten_ranges

    L = _lib.lib()
    padded = 0
    for world in range(2, 9):
        heads = world * (1 if world > 4 else 2)
        m, h = _sp_handle(heads)
        D = heads * 128
        for B, (T, H, W) in ((1, (2, 16, 16)), (2, (2, 24, 20)), (1, (8, 18, 10)), (3, (2, 30, 42)), (2, (8, 90, 160))):
            tokens = T * (H // 2) * (W // 2)
            if tokens % world:
                assert L.ce_dit_sp_region_bytes(h, B, T, H, W, world) == -1
                continue
            lay = sp_layout(B, tokens, D, 64, world)
            assert L.ce_dit_sp_region_bytes(h, B, T, H, W, world) == lay["bytes"], (world, B, T, H, W)
            offs = [lay[k] for k in ("q", "k", "v", "attn", "yout", "flags")]
            assert all(o % 1024 == 0 for o in offs) and offs == sorted(offs)
            assert lay["bytes"] - lay["flags"] == 1024 == 8 * 32 * 4   # the flags block: uint32 [8 * 32]
            for name, nxt in (("q", "k"), ("k", "v"), ("v", "attn"), ("attn", "yout"), ("yout", "flags")):
                assert 0 <= lay[nxt] - (lay[name] + lay["used"][name]) < 1024
            gaps = sp_unwritten_ranges(lay)
            assert gaps[-1] == ("flags", lay["flags"], lay["bytes"])
            padded += len(gaps) - 1
        del m
    assert padded > 0, "no case exercised the alignment padding"


def test_sp_region_bytes_refusals():
    from chronoedit_b200 import _lib

    L = _lib.lib()
    m, h = _sp_handle(4)
    assert L.ce_dit_sp_region_bytes(h, 1, 2, 32, 32, 2) > 0
    assert L.ce_dit_sp_region_bytes(h, 1, 2, 32, 32, 1) == -1     # world 1 is not sequence parallel
    assert L.ce_dit_sp_region_bytes(h, 1, 2, 32, 32, 9) == -1     # at most 8 ranks
    assert L.ce_dit_sp_region_bytes(h, 0, 2, 32, 32, 2) == -1     # batch
    assert L.ce_dit_sp_region_bytes(h, 1, 2, 18, 30, 4) == -1     # 270 tokens % 4
    m3, h3 = _sp_handle(3)
    assert L.ce_dit_sp_region_bytes(h3, 1, 2, 32, 32, 2) == -1    # 3 heads % 2
    assert L.ce_dit_sp_region_bytes(h3, 1, 2, 24, 32, 3) > 0


def test_sp_configure_refusals_with_aligned_regions():
    """The DiT's configure refuses what the VAE's does (world outside 1..8, rank, table, size, null or not 256-byte aligned region)
    and a head count the world does not divide; it accepts 256-byte aligned regions and world 1 switches it off."""
    import ctypes

    from chronoedit_b200 import _lib

    L = _lib.lib()
    m, h = _sp_handle(4)
    table = (ctypes.c_void_p * 8)(*[4096 * (w + 1) for w in range(8)])   # configure never dereferences the addresses

    def refused(*args, msg):
        assert L.ce_dit_sp_configure(*args) == -1
        assert msg in L.ce_last_error().decode()

    refused(None, 0, 2, table, 64, msg="null handle")
    refused(h, 0, 9, table, 64, msg="arguments")
    refused(h, 0, 0, table, 64, msg="arguments")
    refused(h, -1, 2, table, 64, msg="arguments")
    refused(h, 2, 2, table, 64, msg="arguments")
    refused(h, 0, 2, None, 64, msg="arguments")
    refused(h, 0, 2, table, 0, msg="arguments")
    refused(h, 0, 8, table, 64, msg="head count must be divisible")
    holes = (ctypes.c_void_p * 2)(4096, None)
    refused(h, 0, 2, holes, 64, msg="null region pointer")
    misaligned = (ctypes.c_void_p * 2)(4096, 8192 + 16)
    refused(h, 0, 2, misaligned, 64, msg="256-byte aligned")
    assert L.ce_dit_sp_configure(h, 1, 4, table, 64) == 0
    assert L.ce_dit_sp_configure(h, 0, 1, None, 0) == 0            # world 1 switches it off


@pytest.mark.parametrize("disable,entry", [("disable_sequence_parallel", "ce_dit_sp_configure"),
                                           ("disable_vae_sequence_parallel", "ce_vae_sp_configure")])
def test_disable_barriers_on_the_group_of_the_regions(monkeypatch, disable, entry):
    """Before the own region is freed, disable waits for the ranks of the group the regions were opened with, not the default group."""
    from chronoedit_b200 import _lib

    calls = []

    class Lib:
        def __getattr__(self, name):
            return lambda *a: calls.append((name,) + a) or 0

    monkeypatch.setattr(_lib, "lib", lambda: Lib())
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "barrier", lambda group=None: calls.append(("barrier", group)))
    monkeypatch.setattr(torch.cuda, "synchronize", lambda device=None: None)
    group = object()
    obj = types.SimpleNamespace(device="cuda:0", _handle="handle", _sp_state={"own": "own", "opened": ["peer"], "group": group})
    getattr(parallel, disable)(obj)
    assert calls == [(entry, "handle", 0, 1, None, 0), ("ce_ipc_close", "peer"), ("barrier", group), ("ce_ipc_free", "own")]
    assert obj._sp_state is None


def test_sp_host_barrier_arguments():
    from chronoedit_b200 import _lib

    L = _lib.lib()
    m, h = _sp_handle(2)
    assert L.ce_dit_sp_host_barrier(None, 1000) == -1 and b"ce_dit_sp_host_barrier: arguments" in L.ce_last_error()
    assert L.ce_dit_sp_host_barrier(h, -1) == -1 and b"ce_dit_sp_host_barrier: arguments" in L.ce_last_error()
    assert L.ce_dit_sp_host_barrier(h, 60000) == 0
    assert L.ce_dit_sp_host_barrier(h, 0) == 0                     # back to the device barrier
