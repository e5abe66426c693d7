"""The compressed collectives at three and four ranks, where the rank order of the sum shows in the result: from
three ranks on, every reassociation of a bf16 / fp16 / fp32 fold can change its bits, and the decode-and-sum kernel
runs with two or more archives per group inside reduce_scatter_compressed.

Every rank builds every rank's data from one seed, so each checks its result against the float64 fold of
tests/reduce_reference.py over ranks in rank order and against torch's left fold.  The data is
tests/multirank.rank_data, made so that the order matters.

With torch.cuda.device_count() >= world every rank has its own GPU and NCCL; otherwise every rank runs on cuda:0
and the exchange goes through gloo."""
import numpy as np
import pytest
import torch

from multirank import NAME, host_words, rank_data, run_ranks
from reduce_reference import assert_same_words, fold_ref

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16, torch.float32]


def torch_fold(ts, dt):
    acc = ts[0].to(dt)
    for x in ts[1:]:
        acc = acc + x.to(dt)
    return acc


def _worker(rank, world, dev):
    import dietgpu_b200 as dg

    done = []

    def check(got, ts_ref, at, ot, lo, hi, what):
        """got == the rank-order fold of ts_ref[:, lo:hi] (fold_ref and torch's fold)."""
        ref = fold_ref([host_words(x[lo:hi]) for x in ts_ref], at, ot)
        assert_same_words(host_words(got), ref, ot, f"{what} (float64 fold)")
        tf = torch_fold([x[lo:hi].to(dev) for x in ts_ref], torch.float32 if ot == "f32" else ts_ref[0].dtype)
        assert_same_words(host_words(got), host_words(tf), ot, f"{what} (torch fold)")
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
            assert np.array_equal(host_words(got), host_words(want)), f"all_gather stages {stages} n {n}"
            done.append(f"all_gather {stages} {n}")
    # one pass of all_to_all_compressed: per-pair lengths 0, 1 and 4097
    lens = (0, 1, 4097)
    for dt in DTYPES:
        def chunk(s, d):
            return rank_data(dt, lens[(s + 2 * d) % 3], 1, 400 + 10 * s + d)[0]

        got = dg.all_to_all_compressed([chunk(rank, d).to(dev) for d in range(world)])
        for s in range(world):
            assert np.array_equal(host_words(got[s]), host_words(chunk(s, rank))), f"all_to_all {dt} from {s}"
        done.append(f"all_to_all {dt}")
    return len(done)


@pytest.mark.parametrize("world", [3, 4])
def test_reduce_collectives_in_rank_order(world):
    run_ranks(_worker, world, timeout=300)
