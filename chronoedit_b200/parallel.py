"""Data-parallel plumbing for a batch of independent edits (SURVEY.md section 8e).

The hot path shards naturally on the edit (batch) dimension: no operator of the DiT or the VAE mixes samples, so edit i
simply runs on rank i % world.  The ONLY collective is the one-time replication of the weights from rank 0 (the
reference's closest analogue is `sync_model_states`, chronoedit/_ext/imaginaire/utils/distributed.py:351-443); there is
no per-step collective.  Works with the NCCL backend (GPU tensors, NVLink/NVSwitch) and with gloo (CPU tensors; used by
the CPU tests at world_size 2).
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Sequence

import torch
import torch.distributed as dist


def shard_edits(n_edits: int, rank: int, world: int) -> List[int]:
    """Indices of the edits rank `rank` processes: round-robin, every edit exactly once, |shards| differ by <= 1."""
    if not (0 <= rank < world):
        raise ValueError(f"rank {rank} outside world {world}")
    return list(range(rank, n_edits, world))


def broadcast_tensors(tensors: Iterable[torch.Tensor], src: int = 0, bucket_bytes: int = 256 << 20) -> int:
    """Replicate `tensors` (same shapes/dtypes on every rank) from rank `src`, coalescing small tensors into flat
    buckets of at most `bucket_bytes` so that launch latency, not link count, is what is amortised (NVSwitch gives every
    GPU full bandwidth to every peer).  Returns the number of bytes broadcast."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size() == 1:
        return 0
    total = 0
    by_dtype: Dict[torch.dtype, List[torch.Tensor]] = {}
    for t in tensors:
        by_dtype.setdefault(t.dtype, []).append(t)
    for dtype, ts in by_dtype.items():
        bucket: List[torch.Tensor] = []
        size = 0

        def flush():
            nonlocal bucket, size, total
            if not bucket:
                return
            if len(bucket) == 1 and bucket[0].is_contiguous():
                dist.broadcast(bucket[0], src=src)
            else:
                flat = torch.cat([b.reshape(-1) for b in bucket])
                dist.broadcast(flat, src=src)
                off = 0
                for b in bucket:
                    n = b.numel()
                    b.copy_(flat[off: off + n].view_as(b))
                    off += n
            total += size
            bucket, size = [], 0

        for t in ts:
            nbytes = t.numel() * t.element_size()
            if nbytes >= bucket_bytes:
                flush()
                if t.is_contiguous():
                    dist.broadcast(t, src=src)
                else:
                    c = t.contiguous()
                    dist.broadcast(c, src=src)
                    t.copy_(c)
                total += nbytes
                continue
            if size + nbytes > bucket_bytes:
                flush()
            bucket.append(t)
            size += nbytes
        flush()
    return total


def broadcast_module_weights(module: torch.nn.Module, src: int = 0) -> int:
    """Broadcast every parameter / buffer of a module.  For a packed ChronoEditTransformer3DModel the fused buffers are
    broadcast instead of the per-parameter views (same storage, fewer and larger messages)."""
    keep = getattr(module, "_pack_keepalive", None)
    if keep and getattr(module, "_packed", False):
        return broadcast_tensors(keep.values(), src=src)
    return broadcast_tensors([p.data for p in module.parameters()] + [b for b in module.buffers()], src=src)


def gather_objects(local: Sequence, dst: int = 0):
    """Gather small per-rank python results (timings, checksums) on rank `dst`."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return [list(local)]
    out = [None] * dist.get_world_size() if dist.get_rank() == dst else None
    dist.gather_object(list(local), out, dst=dst)
    return out


# ----------------------------------------------------------------------------------------------------------------------
# The peer group of a split model: one region per rank, opened by every other rank through CUDA IPC (csrc/seqpar.cuh)
# ----------------------------------------------------------------------------------------------------------------------
def _open_peer_regions(n: int, group) -> tuple:
    """Allocates this rank's peer region of `n` bytes (ce_ipc_alloc), all-gathers the 64-byte CUDA IPC handles over `group` (plumbing
    only) and opens the other ranks' regions.  Returns the pointer table (one address per rank, as seen from this process) and the
    state _release_peer_regions frees."""
    import ctypes

    from . import _lib
    from ._lib import check

    L = _lib.lib()
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    own = ctypes.c_void_p()
    check(L.ce_ipc_alloc(n, ctypes.byref(own)))
    hbuf = (ctypes.c_uint8 * 64)()
    check(L.ce_ipc_get_handle(own, hbuf))
    handles = [None] * world
    dist.all_gather_object(handles, bytes(hbuf), group=group)
    ptrs, opened = [], []
    for w in range(world):
        if w == rank:
            ptrs.append(own.value)
            continue
        p = ctypes.c_void_p()
        hb = (ctypes.c_uint8 * 64).from_buffer_copy(handles[w])
        check(L.ce_ipc_open(hb, ctypes.byref(p)))
        ptrs.append(p.value)
        opened.append(p)
    return ptrs, {"own": own, "opened": opened, "group": group}


def _configure_peer_regions(obj, entry: str, rank: int, region_ptrs: Sequence[int], region_bytes: int, state: Dict,
                            attr: str = "_sp_state") -> None:
    """Hands the pointer table to the C configure `entry` of obj's handle and keeps `state` as obj.<attr> (the token split's
    "_sp_state", the batch split's "_bp_state" or the call pair's "_cp_state"), with "rank", "world" and "bytes" added."""
    import ctypes

    from . import _lib
    from ._lib import check

    world = len(region_ptrs)
    table = (ctypes.c_void_p * world)(*region_ptrs)
    with torch.cuda.device(obj.device):
        check(getattr(_lib.lib(), entry)(obj._ensure_handle(), rank, world, table, region_bytes))
        torch.cuda.synchronize(obj.device)
    setattr(obj, attr, dict(state, rank=rank, world=world, bytes=region_bytes))


def _release_peer_regions(obj, entry: str, attr: str = "_sp_state") -> bool:
    """Switches obj's handle back to one GPU (C configure `entry`, world 1), closes the opened peer mappings of the state obj.<attr>
    and frees the own region once no rank of the state's group still maps it.  Returns False when obj had no such split on."""
    from . import _lib

    st = getattr(obj, attr, None)
    if not st:
        return False
    L = _lib.lib()
    torch.cuda.synchronize(obj.device)
    getattr(L, entry)(obj._handle, 0, 1, None, 0)
    for p in st.get("opened", ()):
        L.ce_ipc_close(p)
    if st.get("own") is not None:
        if dist.is_initialized():
            dist.barrier(group=st.get("group"))
        L.ce_ipc_free(st["own"])
    setattr(obj, attr, None)
    return True


def _enable_split(obj, who: str, group, disable, region_bytes, configure) -> int:
    """What every enable_* does: refuse without a process group, `disable(obj)` and stop at world 1; otherwise size the region
    with `region_bytes(world)`, open the peer regions, hand them to `configure` (a configure_* function) and wait for every rank.
    Returns the region size in bytes."""
    from ._lib import CEError

    if not dist.is_initialized():
        raise CEError(f"{who} needs an initialised torch.distributed process group (one process per GPU)")
    disable(obj)
    world = dist.get_world_size(group)
    if world == 1:
        return 0
    n = region_bytes(world)
    with torch.cuda.device(obj.device):
        ptrs, state = _open_peer_regions(n, group)
        configure(obj, dist.get_rank(group), ptrs, n, state)
    dist.barrier(group=group)   # every region exists, is zeroed and is mapped everywhere before the first flag is written
    return int(n)


# ----------------------------------------------------------------------------------------------------------------------
# Sequence parallelism for single-edit latency (SURVEY.md section 8(f) row 2)
# ----------------------------------------------------------------------------------------------------------------------
def enable_sequence_parallel(model, batch: int, frames: int, height: int, width: int, group=None) -> int:
    """Split the tokens of ONE edit over the ranks of `group` (one process per GPU of a node; reference: the Ulysses path of
    chronoedit_diffsynth/wan_video_new_chronoedit.py:330-355 and the TE ring of chronoedit/_src/networks/wan2pt1.py:352-353).

    Allocates this rank's peer region (ce_ipc_alloc), exchanges the 64-byte CUDA IPC handles through torch.distributed (plumbing
    only), opens the peers' regions and hands the pointer table to the C handle (ce_dit_sp_configure).  From then on
    `model(hidden_states, timestep, encoder_hidden_states, encoder_hidden_states_image)` -- called with the SAME full inputs on every
    rank -- computes 1/world of the tokens per rank, exchanges q/k/v and the attention output by peer stores over NVLink inside the
    kernels (no collective call on the data path), and returns the same full sample on every rank, bit-identical to the single-GPU
    forward.  Geometry-specific: call again for another latent shape.  Returns the region size in bytes."""
    return _enable_split(model, "enable_sequence_parallel", group, disable_sequence_parallel,
                         lambda world: sp_region_bytes(model, batch, frames, height, width, world), configure_sequence_parallel)


def sp_region_bytes(model, batch: int, frames: int, height: int, width: int, world: int) -> int:
    """Bytes of the peer region every rank needs for this geometry (ce_dit_sp_region_bytes); packs the weights first."""
    from . import _lib
    from ._lib import CEError

    model._ensure_packed()
    n = _lib.lib().ce_dit_sp_region_bytes(model._handle, batch, frames, height, width, world)
    if n < 0:
        raise CEError(f"sequence parallel: tokens and heads must be divisible by the world size {world} (2 to 8)")
    return int(n)


def configure_sequence_parallel(model, rank: int, region_ptrs: Sequence[int], region_bytes: int, state: Dict) -> None:
    """Hand rank `rank`'s table of peer-region addresses (one per rank, as seen from this process) to the model's C handle
    (ce_dit_sp_configure) and switch the model into sequence-parallel mode.  `state` is kept as `model._sp_state` (with "world" and
    "bytes" added) and holds whatever disable_sequence_parallel releases: the own region under "own" (freed with ce_ipc_free, after a
    barrier on the process group under "group") and the opened peer mappings under "opened" (closed with ce_ipc_close)."""
    model._ensure_packed()
    _configure_peer_regions(model, "ce_dit_sp_configure", rank, region_ptrs, region_bytes, state)
    model._invalidate("layout")


def disable_sequence_parallel(model) -> None:
    """Back to the single-GPU forward; releases what enable_sequence_parallel allocated and opened."""
    _release_peer_regions(model, "ce_dit_sp_configure")


# ----------------------------------------------------------------------------------------------------------------------
# The batch of a DiT forward split over the ranks of a node: the CFG pair of one edit on two GPUs (include/chronoedit_b200.h, ce_dit_bp_*)
# ----------------------------------------------------------------------------------------------------------------------
def enable_cfg_parallel(model, batch: int, frames: int, height: int, width: int, group=None) -> int:
    """Split the batch of every forward over the ranks of `group` (one process per GPU of a node): rank r computes samples
    [r B / world, (r + 1) B / world) of a call's batch B with the unchanged forward, and one exchange of the finished samples by peer
    stores over NVLink gives every rank the full batch, bit-identical to the single-GPU forward.  For the CFG pair (prompt and negative
    prompt as one batch-2 call, as `scheduler.step_cfg` and bench.py run it) that puts each half of the pair on its own GPU.
    Called with the SAME full inputs on every rank.  FP8 weights (`enable_fp8`), FP8 attention (`enable_fp8_attention`) and TeaCache
    (`enable_teacache`, one state per conditioning, decided on the rank's own samples) work unchanged with it on.  A call whose batch
    the ranks do not divide is refused: the unchanged diffusers pipeline's two batch-1 calls per step are not split.  CUDA graphs are
    not replayed while it is on.

    `batch` x (frames, height, width) sizes the region: any later call whose full sample is no larger is accepted (a region for 8
    latent frames also serves the cut to 2).  Returns the region size in bytes.

    On 4 or 8 GPUs it composes with the token split as a grid: the batch over 2 ranks, the tokens of each half over W / 2 ranks.
    With dist.new_group, token groups {0 .. W/2 - 1} and {W/2 .. W - 1}, pair groups {r, r + W/2}; every rank calls:

        parallel.enable_sequence_parallel(model, B // 2, T, H, W, group=token_group)   # the token split sees the local batch
        parallel.enable_cfg_parallel(model, B, T, H, W, group=pair_group)
    """
    from ._lib import CEError

    if dist.is_initialized() and model._cp_state:   # before any region is allocated; ce_dit_bp_configure refuses it too
        raise CEError("enable_cfg_parallel: the call-pair split (enable_cfg_parallel_calls) is on: the two CFG splits are exclusive, "
                      "disable it first")
    return _enable_split(model, "enable_cfg_parallel", group, disable_cfg_parallel,
                         lambda world: cfg_region_bytes(model, batch, frames, height, width, world), configure_cfg_parallel)


def cfg_region_bytes(model, batch: int, frames: int, height: int, width: int, world: int) -> int:
    """Bytes of the peer region every rank of the batch split needs for this geometry (ce_dit_bp_region_bytes)."""
    from . import _lib
    from ._lib import CEError

    n = _lib.lib().ce_dit_bp_region_bytes(model._ensure_handle(), batch, frames, height, width, world)
    if n < 0:
        raise CEError(f"batch split: the batch ({batch}) must divide by the world size ({world}, 2 to 8) and the geometry must be valid")
    return int(n)


def configure_cfg_parallel(model, rank: int, region_ptrs: Sequence[int], region_bytes: int, state: Dict) -> None:
    """Hand rank `rank`'s table of peer-region addresses (one per rank, as seen from this process) to the model's C handle
    (ce_dit_bp_configure) and switch the model's batch split on.  `state` is kept as `model._bp_state` (with "rank", "world" and
    "bytes" added) and holds what disable_cfg_parallel releases, as for configure_sequence_parallel.  The token split's state
    (`model._sp_state`) is not touched."""
    _configure_peer_regions(model, "ce_dit_bp_configure", rank, region_ptrs, region_bytes, state, "_bp_state")
    model._invalidate("results")   # the context cache's K/V and the TeaCache states hold the old share of samples


def disable_cfg_parallel(model) -> None:
    """Back to computing every sample of a call on this GPU; releases what enable_cfg_parallel allocated and opened."""
    if _release_peer_regions(model, "ce_dit_bp_configure", "_bp_state"):
        model._invalidate("results")


# ----------------------------------------------------------------------------------------------------------------------
# The two calls of the unchanged pipeline's CFG pair on two ranks (include/chronoedit_b200.h, ce_dit_cp_*)
# ----------------------------------------------------------------------------------------------------------------------
def enable_cfg_parallel_calls(model, batch: int, frames: int, height: int, width: int, group=None) -> int:
    """Compute the two calls of each CFG step of the unchanged diffusers pipeline on two ranks (one process per GPU): the pipeline
    calls the transformer once with `prompt_embeds` and once with `negative_prompt_embeds`, with the same latents and timestep.  From
    then on the model takes its calls in pairs: rank 0 of `group` computes the first call (the prompt), rank 1 the second (the negative
    prompt), each with the ordinary single-GPU forward, and at the second call one exchange by peer stores over NVLink gives each rank
    the other's sample.  Every rank runs the same pipeline with the SAME inputs and gets both samples, bit-identical to one GPU.

    Rank 1 returns a sample filled with NaN from the first call of a pair; the exchange of the second call overwrites it in place,
    stream-ordered before the pipeline's guidance combine reads it.  So the mode needs classifier-free guidance
    (`guidance_scale > 1`, the pipeline's `do_classifier_free_guidance`): the second call of a pair must pass the same
    `hidden_states` and `timestep` objects (unchanged in place) and the same `encoder_hidden_states_image` as the first, or it raises
    CEError on every rank before any launch.  A guidance-free run therefore raises at its second step.

    FP8 weights (`enable_fp8`), FP8 attention (`enable_fp8_attention`), TeaCache and the context cache work unchanged: a rank keeps
    the state of the one conditioning it computes, so every TeaCache decision equals the single-GPU run's.  Refused while on:
    `return_block0`, `capture_layers`, `forward_host`, `forward_fp32`, a capturing stream and `enable_cfg_parallel`.  CUDA graphs are
    not replayed.

    `batch` x (frames, height, width) sizes the region for one call: any later call whose sample is no larger is accepted (a region for
    8 latent frames also serves temporal reasoning's cut to 2).  Returns the region size in bytes.

    On 4 or 8 GPUs it composes with the token split as a grid: each call's tokens over W / 2 ranks, the pair over 2.  With
    dist.new_group, token groups {0 .. W/2 - 1} and {W/2 .. W - 1}, pair groups {j, j + W/2}; every rank calls:

        parallel.enable_sequence_parallel(model, B, T, H, W, group=token_group)   # the call's own batch (1 in the pipeline)
        parallel.enable_cfg_parallel_calls(model, B, T, H, W, group=pair_group)

    and every rank of token group 0 computes the prompt calls, every rank of token group 1 the negative-prompt calls.
    """
    from ._lib import CEError

    if dist.is_initialized() and model._bp_state:   # before any region is allocated; ce_dit_cp_configure refuses it too
        raise CEError("enable_cfg_parallel_calls: the batch split (enable_cfg_parallel) is on: the two CFG splits are exclusive, "
                      "disable it first")

    def region_bytes(world):
        if world != 2:
            raise CEError(f"enable_cfg_parallel_calls: a CFG pair has two calls: the group must have 2 ranks, not {world}")
        return cfg_calls_region_bytes(model, batch, frames, height, width)

    return _enable_split(model, "enable_cfg_parallel_calls", group, disable_cfg_parallel_calls, region_bytes,
                         configure_cfg_parallel_calls)


def cfg_calls_region_bytes(model, batch: int, frames: int, height: int, width: int) -> int:
    """Bytes of the peer region each of the two ranks needs for calls of this geometry (ce_dit_cp_region_bytes)."""
    from . import _lib
    from ._lib import CEError

    n = _lib.lib().ce_dit_cp_region_bytes(model._ensure_handle(), batch, frames, height, width)
    if n < 0:
        raise CEError(f"call-pair split: invalid geometry (batch {batch}, 1 to 8; frames {frames}, height {height}, width {width})")
    return int(n)


def configure_cfg_parallel_calls(model, rank: int, region_ptrs: Sequence[int], region_bytes: int, state: Dict) -> None:
    """Hand rank `rank`'s table of the two peer-region addresses (as seen from this process) to the model's C handle
    (ce_dit_cp_configure) and switch the call-pair split on.  `state` is kept as `model._cp_state` (with "rank", "world" and "bytes"
    added) and holds what disable_cfg_parallel_calls releases, as for configure_sequence_parallel.  The next call is the first of a
    pair."""
    _configure_peer_regions(model, "ce_dit_cp_configure", rank, region_ptrs, region_bytes, state, "_cp_state")
    model._cp_pair = None
    model._invalidate("results")


def disable_cfg_parallel_calls(model) -> None:
    """Back to computing every call on this GPU; releases what enable_cfg_parallel_calls allocated and opened.  A pair whose second
    call never came is dropped with a warning."""
    if not _release_peer_regions(model, "ce_dit_cp_configure", "_cp_state"):
        return
    if model._cp_pair is not None:
        import warnings

        warnings.warn("disable_cfg_parallel_calls: the first call of a CFG pair is still open (its second call never came); "
                      "dropping it")
    model._cp_pair = None
    model._invalidate("results")


# ----------------------------------------------------------------------------------------------------------------------
# The VAE of one edit split over the ranks of a node (row bands, see include/chronoedit_b200.h, ce_vae_sp_*)
# ----------------------------------------------------------------------------------------------------------------------
def enable_vae_sequence_parallel(vae, height: int, width: int, group=None) -> int:
    """Split `vae.encode` / `vae.decode` of ONE edit over the ranks of `group` (one process per GPU of a node) by horizontal bands of
    rows: rank r owns latent rows [r h / world, (r + 1) h / world) and only the rows that cross the band edges (and the mid attention's
    input) travel, by peer stores over NVLink into the other ranks' regions.  Called with the SAME full inputs on every rank, encode and
    decode return the full result on every rank, bit-identical to the single-GPU call.

    `height` x `width` is the edit's pixel geometry: one configuration serves the encode of any 1 + 4k frames at that size and the
    decode of any latent frame count at height / 8 x width / 8.  Allocates this rank's peer region (ce_ipc_alloc), exchanges the CUDA
    IPC handles through torch.distributed and configures the handle (ce_vae_sp_configure).  Returns the region size in bytes.
    The split is built for the bf16 VAE only: an fp32 VAE is refused before anything is allocated."""
    _refuse_fp32_vae(vae)
    return _enable_split(vae, "enable_vae_sequence_parallel", group, disable_vae_sequence_parallel,
                         lambda world: vae_sp_region_bytes(vae, height, width, world), configure_vae_sequence_parallel)


def _refuse_fp32_vae(vae) -> None:
    from ._lib import CEError

    if vae.dtype == torch.float32:
        raise CEError("the VAE split over GPUs is built for the bf16 VAE only; this VAE was loaded in fp32")


def vae_sp_region_bytes(vae, height: int, width: int, world: int) -> int:
    """Bytes of the peer region every rank needs for pixel geometry height x width (ce_vae_sp_region_bytes)."""
    from . import _lib
    from ._lib import check

    n = _lib.lib().ce_vae_sp_region_bytes(vae._ensure_handle(), height, width, world)
    if n < 0:
        check(int(n))
    return int(n)


def configure_vae_sequence_parallel(vae, rank: int, region_ptrs: Sequence[int], region_bytes: int, state: Dict) -> None:
    """Hand rank `rank`'s table of peer-region addresses (one per rank, as seen from this process) to the VAE's C handle
    (ce_vae_sp_configure).  `state` is kept as `vae._sp_state` and holds what disable_vae_sequence_parallel releases: the own region
    under "own" (ce_ipc_free, after a barrier on the process group under "group") and the opened peer mappings under "opened"
    (ce_ipc_close)."""
    _refuse_fp32_vae(vae)
    _configure_peer_regions(vae, "ce_vae_sp_configure", rank, region_ptrs, region_bytes, state)


def disable_vae_sequence_parallel(vae) -> None:
    """Back to the single-GPU VAE; releases what enable_vae_sequence_parallel allocated and opened."""
    _release_peer_regions(vae, "ce_vae_sp_configure")
