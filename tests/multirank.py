"""Multi-process helpers shared by the tests of the compressed collectives.

run_ranks(worker, world, *args) starts `world` ranks, each a spawned process in its own torch.distributed group, and
calls worker(rank, world, dev, *args) in every rank.  The ranks meet through a file store in a fresh temporary
directory, so no test picks a port and two runs on one host cannot join each other's group.  The parent fails the
test unless every rank reports success and exits cleanly, and it never leaves a rank running.

The rest are the data and checks the multi-rank tests and the collectives' refusal tests share."""
from __future__ import annotations

import os
import queue
import shutil
import tempfile
import time

import numpy as np
import pytest
import torch

NAME = {torch.float16: "f16", torch.bfloat16: "bf16", torch.float32: "f32"}


def _rank_main(worker, rank, world, nccl, cuda, store, args, q):
    """One rank: set up the device and the group, run the worker, report (rank, "ok" or the error, checks made)."""
    import torch.distributed as dist

    msg, count = "ok", 0
    try:
        dev = torch.device("cpu")
        if cuda:
            dev = torch.device("cuda", rank if nccl else 0)
            torch.cuda.set_device(dev)
        dist.init_process_group("nccl" if nccl else "gloo", init_method=f"file://{store}", rank=rank,
                                world_size=world)
        count = worker(rank, world, dev, *args) or 0
    except BaseException as e:  # reported to the parent, which fails the test with it (pytest.fail is no Exception)
        msg = f"{type(e).__name__}: {e}"
    finally:
        q.put((rank, msg, count))
        if dist.is_initialized():
            dist.destroy_process_group()


def run_ranks(worker, world, *args, backend="auto", timeout=300, join_timeout=120):
    """Run worker(rank, world, dev, *args) on `world` spawned ranks; the worker is a module-level function that raises
    on a failed check and may return how many checks it made.

    backend "auto": NCCL with one GPU per rank when there are `world` GPUs, otherwise gloo with every rank on cuda:0;
    "gloo": gloo on cuda:0; None: gloo and no CUDA at all (dev is the CPU).  The ranks have `timeout` seconds to
    report and then `join_timeout` seconds each to exit; any rank still alive after that is terminated, then killed."""
    import torch.multiprocessing as mp

    nccl = backend == "auto" and torch.cuda.device_count() >= world
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    tmp = tempfile.mkdtemp(prefix="multirank-")
    store = os.path.join(tmp, "store")
    procs = [ctx.Process(target=_rank_main, args=(worker, r, world, nccl, backend is not None, store, args, q))
             for r in range(world)]
    res = {}
    try:
        for p in procs:
            p.start()
        deadline = time.monotonic() + timeout
        while len(res) < world:
            try:
                r, msg, count = q.get(timeout=max(0.0, deadline - time.monotonic()))
            except queue.Empty:
                break
            res[r] = (msg, count)
        for p in procs:
            p.join(timeout=join_timeout)
    finally:
        started = [p for p in procs if p.pid is not None]
        for p in started:
            if p.is_alive():
                p.terminate()
        for p in started:
            p.join(timeout=30)
            if p.is_alive():
                p.kill()
                p.join()
        shutil.rmtree(tmp, ignore_errors=True)
    name = ("nccl" if nccl else "gloo") + ("" if backend is None else " on CUDA")
    print(f"world {world}: backend {name}, checks per rank {[res.get(r, (None, 0))[1] for r in range(world)]}")
    assert sorted(res) == list(range(world)), (name, res)
    assert all(m == "ok" for m, _ in res.values()), (name, res)
    assert all(p.exitcode == 0 for p in procs), (name, [p.exitcode for p in procs])


def host_words(x):
    """Host raw words of a tensor (any device)."""
    x = x.detach().contiguous().cpu()
    return x.view(torch.int32 if x.element_size() == 4 else torch.int16).numpy().view(
        np.uint32 if x.element_size() == 4 else np.uint16)


def rank_data(dt, n, world, seed, widened=False):
    """Every rank's tensor (CPU, dtype dt), built so that the rank order of a sum shows in its bits: at one element a
    single rank holds 2^p (p = the type's precision) and every other rank holds 1 (or, for the fp16 fp32 sums, 2^15
    and 2^-9), so each later add of the small value is a tie that rounds away, while any other order adds the small
    values up first; +inf and -inf sit on different ranks, NaN on one rank, -0 on every rank, and +-max sit so that
    the rank-order sum overflows while other orders do not.  These take elements 0..7 of every 16."""
    xs = []
    for r in range(world):
        g = torch.Generator().manual_seed(seed + 31 * r)
        xs.append(torch.randn(n, generator=g, dtype=torch.float64) * (1 + r))
    if widened:  # sums in fp32 of 16-bit values
        big, small = (2.0 ** 15, 2.0 ** -9) if dt == torch.float16 else (2.0 ** 24, 1.0)
    else:
        big, small = {torch.float16: (2048.0, 1.0), torch.bfloat16: (256.0, 1.0),
                      torch.float32: (2.0 ** 24, 1.0)}[dt]
    top = torch.finfo(dt).max
    pos = torch.arange(n)
    for r in range(world):
        x = xs[r]
        k = pos % 16
        x[k == 0] = torch.where((pos[k == 0] // 16) % world == r, big, small).double()
        x[k == 1] = big if r == 0 else small
        if r == 0:
            x[k == 2] = float("inf")
        if r == world - 1:
            x[k == 2] = float("-inf")
        x[k == 3] = float("nan") if r == 1 else 1.5
        x[k == 4] = -0.0
        x[k == 5] = top if r < 2 else -top  # rank order: (max + max) = inf first
        x[k == 6] = float("inf") if r == 1 else -1.0
        x[k == 7] = -small if r == world - 1 else small
    return [x.to(dt) for x in xs]


class Untouchable:
    """Stands for an archive tensor: any use of it fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"the archive was touched ({name}) before the call was refused")


@pytest.fixture
def no_communication(monkeypatch):
    """Every torch.distributed call fails the test; returns the monkeypatch, so a test can give one name back."""
    import torch.distributed as dist

    def boom(*a, **k):
        raise AssertionError("communication before the refusal")

    for name in ("all_gather_into_tensor", "all_to_all_single", "all_gather", "all_reduce", "broadcast", "barrier",
                 "get_rank", "get_world_size", "get_backend", "is_initialized"):
        monkeypatch.setattr(dist, name, boom)
    return monkeypatch
