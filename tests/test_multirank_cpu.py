"""tests/multirank.run_ranks without a GPU: gloo ranks on the CPU.  A failing rank fails the run with its message, a
rank that hangs fails it within the timeout and leaves no process behind, and two runs at once stay apart."""
import multiprocessing
import threading
import time

import pytest
import torch
import torch.distributed as dist

from multirank import run_ranks


def _gather(rank, world, tag):
    got = [None] * world
    dist.all_gather_object(got, (tag, rank))
    assert got == [(tag, r) for r in range(world)], got


def _fails_on_one_rank(rank, world, dev):
    assert dev == torch.device("cpu")
    _gather(rank, world, "fail")
    if rank == 1:
        raise ValueError("rank 1 refuses")
    return 1


def test_a_failing_rank_fails_the_run_with_its_message():
    with pytest.raises(AssertionError, match="ValueError: rank 1 refuses"):
        run_ranks(_fails_on_one_rank, 3, backend=None, timeout=120)


def _hangs_on_one_rank(rank, world, dev):
    if rank == 2:
        time.sleep(600)


def test_a_hanging_rank_fails_the_run_and_is_stopped():
    start = time.monotonic()
    with pytest.raises(AssertionError):
        run_ranks(_hangs_on_one_rank, 3, backend=None, timeout=30, join_timeout=2)
    assert time.monotonic() - start < 120
    assert multiprocessing.active_children() == []


def _meets_its_own_ranks(rank, world, dev, tag):
    _gather(rank, world, tag)
    time.sleep(2)  # both runs' groups are alive at once
    _gather(rank, world, tag)
    return 2


def test_two_runs_at_once_keep_their_own_groups():
    errors = []

    def run(tag):
        try:
            run_ranks(_meets_its_own_ranks, 2, tag, backend=None, timeout=120)
        except BaseException as e:  # noqa: BLE001  (reported by the main thread)
            errors.append(f"{tag}: {e!r}")

    threads = [threading.Thread(target=run, args=(tag,)) for tag in ("a", "b")]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert errors == []
    assert multiprocessing.active_children() == []
