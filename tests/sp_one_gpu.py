"""Shared harness of the one-GPU split tests (test_gpu_seqpar_one_gpu.py, test_gpu_vae_seqpar_one_gpu.py): `world` handles of one
process play the ranks, each driven from its own host thread on its own stream, with ordinary device allocations as peer regions and
the host barrier between the exchanges.  Each region carries a guard band of a byte pattern that the split must never write."""
import gc
import threading
import time

import pytest
import torch

GUARD = 64 << 10        # bytes of pattern after every region
PATTERN = 0xA5
BARRIER_MS = 60000      # host barrier timeout of the bit-equality runs
SHORT_MS = 2000         # of the refusal tests: a refusal that regressed times out at the first barrier


def run_ranks(fn, world, timeout):
    """fn(r) for every rank r at once, each from its own thread on its own stream; returns the results.  A thread's exception is
    raised here."""
    torch.cuda.synchronize()
    outs, errs = [None] * world, [None] * world

    def work(r):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                outs[r] = fn(r)
            s.synchronize()
        except BaseException as e:   # noqa: BLE001 -- re-raised in the test's thread
            errs[r] = e

    threads = [threading.Thread(target=work, args=(r,), daemon=True, name=f"rank-{r}") for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout)
    stuck = [t.name for t in threads if t.is_alive()]
    assert not stuck, f"rank threads still running after {timeout} s: {stuck}"
    for r, e in enumerate(errs):
        if e is not None:
            raise AssertionError(f"rank {r} failed: {e!r}") from e
    return outs


def guarded_regions(n, world, device):
    """One peer region of `n` bytes per rank, followed by a guard band, all filled with the pattern."""
    return [torch.full((n + GUARD,), PATTERN, dtype=torch.uint8, device=device) for _ in range(world)]


def assert_pattern_kept(regions, n, ranges):
    """Every region still holds the pattern in the (name, start, end) byte ranges and in its guard band after `n` bytes."""
    for r, region in enumerate(regions):
        for what, a, b in list(ranges) + [("guard band", n, n + GUARD)]:
            hit = (region[a:b] != PATTERN).nonzero()
            assert hit.numel() == 0, f"rank {r}'s region: {hit.numel()} bytes of its {what} [{a}, {b}) were written (first at {a + int(hit[0])})"


@pytest.fixture
def _clean_device():
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"  [{time.perf_counter() - t0:.1f} s, peak {torch.cuda.max_memory_reserved() / 2**30:.2f} GiB reserved]", flush=True)
    gc.collect()
    torch.cuda.empty_cache()
