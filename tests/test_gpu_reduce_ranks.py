"""The compressed collectives at three and four ranks, where the rank order of the sum shows in the result: from
three ranks on, every reassociation of a bf16 / fp16 / fp32 fold can change its bits, and the decode-and-sum kernel
runs with two or more archives per group inside reduce_scatter_compressed.

Every rank builds every rank's data from one seed, so each checks its result against the float64 fold of
tests/reduce_reference.py over ranks in rank order and against torch's left fold.  The data is made so that the
order matters: at one element a single rank holds 2^p (p = the type's precision) and every other rank holds 1
(or, for the fp16 fp32 sums, 2^15 and 2^-9), so each later add of the small value is a tie that rounds away, while
any other order adds the small values up first; +inf and -inf sit on different ranks, NaN on one rank, -0 on every
rank, and +-max sit so that the rank-order sum overflows while other orders do not.

With torch.cuda.device_count() >= world every rank has its own GPU and NCCL; otherwise every rank runs on cuda:0
and the exchange goes through gloo."""
import os
import queue

import numpy as np
import pytest
import torch

from reduce_reference import assert_same_words, fold_ref

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16, torch.float32]
NAME = {torch.float16: "f16", torch.bfloat16: "bf16", torch.float32: "f32"}


def _words(x):
    """Host raw words of a tensor (any device)."""
    x = x.detach().contiguous().cpu()
    return x.view(torch.int32 if x.element_size() == 4 else torch.int16).numpy().view(
        np.uint32 if x.element_size() == 4 else np.uint16)


def rank_data(dt, n, world, seed, widened=False):
    """Every rank's tensor (CPU, dtype dt), with the order-dependent elements described in the module docstring."""
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


def torch_fold(ts, dt):
    acc = ts[0].to(dt)
    for x in ts[1:]:
        acc = acc + x.to(dt)
    return acc


def _worker(rank, world, port, backend, q):
    import torch.distributed as dist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    local = rank if backend == "nccl" else 0
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group(backend, rank=rank, world_size=world)
    msg = "ok"
    done = []
    try:
        import dietgpu_b200 as dg

        def check(got, ts_ref, at, ot, lo, hi, what):
            """got == the rank-order fold of ts_ref[:, lo:hi] (fold_ref and torch's fold)."""
            ref = fold_ref([_words(x[lo:hi]) for x in ts_ref], at, ot)
            assert_same_words(_words(got), ref, ot, f"{what} (float64 fold)")
            tf = torch_fold([x[lo:hi].to(dev) for x in ts_ref], torch.float32 if ot == "f32" else ts_ref[0].dtype)
            assert_same_words(_words(got), _words(tf), ot, f"{what} (torch fold)")
            done.append(what)

        # reduce_scatter_compressed: members 1, 3, 8; 16-bit sums and fp32 sums of 16-bit data; 16-bit wires for fp32
        for dt in DTYPES:
            for shard in (12289, 65536):
                n = world * shard
                cases = [(None, None)] + ([(torch.float32, None)] if dt != torch.float32 else
                                          [(None, torch.float16), (None, torch.bfloat16)])
                for reduce_dtype, wire in cases:
                    widened = reduce_dtype is not None or wire is not None
                    ts = rank_data(wire or dt, n, world, 100 + shard, widened=widened)
                    if wire is not None:  # fp32 inputs whose narrowing is ts (plus a part that rounds)
                        src = [x.float() + (x.float() * 2.0 ** -14 if wire == torch.float16 else 0.0) for x in ts]
                        ts = [x.to(wire) for x in src]
                    else:
                        src = ts
                    at = NAME[wire or dt]
                    ot = "f32" if widened else at
                    for members in (1, 3, 8):
                        got = dg.reduce_scatter_compressed(src[rank].to(dev), members=members,
                                                           reduce_dtype=reduce_dtype, wire_dtype=wire)
                        check(got, ts, at, ot, rank * shard, (rank + 1) * shard,
                              f"reduce_scatter {dt} n {n} members {members} reduce {reduce_dtype} wire {wire}")
        # all_reduce_compressed: n = 1, n < world, world * 8 * k, 300001
        for dt in DTYPES:
            for n in (1, world - 1, world * 8 * 1111, 300001):
                for reduce_dtype in ([None] if dt == torch.float32 else [None, torch.float32]):
                    widened = reduce_dtype is not None
                    ts = rank_data(dt, n, world, 200 + n, widened=widened)
                    for members in (1, 8):
                        got = dg.all_reduce_compressed(ts[rank].to(dev), members=members, reduce_dtype=reduce_dtype)
                        check(got, ts, NAME[dt], "f32" if widened else NAME[dt], 0, n,
                              f"all_reduce {dt} n {n} members {members} reduce {reduce_dtype}")
        # one pass of all_gather_compressed
        for stages in (1, 2, 3):
            for n in (0, 1, 4095, 300001):
                ts = rank_data(torch.bfloat16, n, world, 300 + n)
                got = dg.all_gather_compressed(ts[rank].to(dev), stages=stages)
                want = torch.cat(ts)
                assert np.array_equal(_words(got), _words(want)), f"all_gather stages {stages} n {n}"
                done.append(f"all_gather {stages} {n}")
        # one pass of all_to_all_compressed: per-pair lengths 0, 1 and 4097
        lens = (0, 1, 4097)
        for dt in DTYPES:
            def chunk(s, d):
                return rank_data(dt, lens[(s + 2 * d) % 3], 1, 400 + 10 * s + d)[0]

            got = dg.all_to_all_compressed([chunk(rank, d).to(dev) for d in range(world)])
            for s in range(world):
                assert np.array_equal(_words(got[s]), _words(chunk(s, rank))), f"all_to_all {dt} from {s}"
            done.append(f"all_to_all {dt}")
    except Exception as e:  # reported to the parent, which fails the test with it
        msg = f"{type(e).__name__}: {e}"
    finally:
        q.put((rank, msg, len(done)))
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [3, 4])
def test_reduce_collectives_in_rank_order(world):
    import torch.multiprocessing as mp

    backend = "nccl" if torch.cuda.device_count() >= world else "gloo"
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31200 + 2 * (os.getpid() % 200) + (world - 3)  # no other test uses 31200..31599
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, q)) for r in range(world)]
    res = {}
    try:
        for p in procs:
            p.start()
        for _ in range(world):
            try:
                r, msg, cnt = q.get(timeout=300)
            except queue.Empty:
                break
            res[r] = (msg, cnt)
        for p in procs:
            p.join(timeout=120)
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
    print(f"world {world}: backend {backend}, checks per rank {[res.get(r, (None, 0))[1] for r in range(world)]}")
    assert sorted(res) == list(range(world)), (backend, res)
    assert all(m == "ok" for m, _ in res.values()), (backend, res)
    assert all(p.exitcode == 0 for p in procs), (backend, [p.exitcode for p in procs])
