"""The sq_norm keyword of the compressed reduce-scatter and all-reduce on 2-4 ranks (gloo ranks sharing cuda:0 on a
one-GPU machine, NCCL with one GPU per rank where there are enough): same-type, widening, narrowing and sparse sums.

The reduce-scatter's value must equal the restatement (tests/sq_norm_reference.py) of the returned shard's `members`
pieces folded in member order, on every rank: the ranks whose decode-and-sum writes the final values take it in the
kernel, the last rank with ops.sq_norm.  The all-reduce's must be identical on every rank and equal the rank-order fold
of the shards' values."""
import numpy as np
import pytest
import torch

import sq_norm_reference as R
from multirank import run_ranks

pytestmark = pytest.mark.gpu


def _split(n, parts, quantum=8):
    from dietgpu_b200.collectives import _split as split

    return split(n, parts, quantum)


def _worker(rank, world, dev):
    import torch.distributed as dist

    import dietgpu_b200 as dg

    done = 0
    s = float(np.float32(0.75) / np.float32(world))
    for dt in (torch.float16, torch.bfloat16, torch.float32):
        n = world * 12289 + world * 5
        n -= n % world
        for variant in ("plain", "widen", "narrow", "sparse"):
            if dt == torch.float32 and variant in ("widen", "narrow"):
                continue
            kw = dict(members=3, scale_tensor=torch.tensor([s], device=dev))
            if variant in ("widen", "narrow"):
                kw["reduce_dtype"] = torch.float32
            if variant == "narrow":
                kw["out_dtype"] = dt
            if variant == "sparse":
                kw["sparse"] = True
            g = torch.Generator().manual_seed(700 + 31 * rank + done)
            x = torch.randn(n, generator=g) * (1 + rank)
            x[::5] = 0.0  # zeros for the sparse archives to elide
            x = x.to(dt).to(dev)
            tag = f"{dt} {variant} world {world}"
            sq = torch.full((1,), -1.0, dtype=torch.float64, device=dev)
            fi = torch.zeros(1, device=dev)
            res = dg.reduce_scatter_compressed(x, found_inf=fi, sq_norm=sq, **kw)
            ref = dg.reduce_scatter_compressed(x, found_inf=torch.zeros(1, device=dev), **kw)
            assert torch.equal(res.view(torch.int16 if res.element_size() == 2 else torch.int32),
                               ref.view(torch.int16 if ref.element_size() == 2 else torch.int32)), tag
            b = _split(res.numel(), 3)
            host = res.double().cpu().numpy()
            want = R.fold([R.sq_norm(host[b[i]:b[i + 1]]) for i in range(len(b) - 1)])
            assert R.same(float(sq), want), f"reduce_scatter {tag} rank {rank}: {float(sq)!r} != {want!r}"
            done += 1
            for m in (1, n // 2 + 1, n):
                xa = x[:m].contiguous()
                sq = torch.full((1,), -1.0, dtype=torch.float64, device=dev)
                full = dg.all_reduce_compressed(xa, sq_norm=sq, **kw)
                # identical on every rank
                every = [torch.empty(1, dtype=torch.float64) for _ in range(world)]
                dist.all_gather(every, sq.cpu())
                assert all(R.same(float(e), float(sq)) for e in every), f"all_reduce {tag} n {m}: {every}"
                # the rank-order fold of the shards' reduce-scatter values, over the zero-padded exchange
                per = -(-(-(-m // world)) // 8) * 8
                padded = np.zeros(world * per)
                padded[:m] = full.reshape(-1).double().cpu().numpy()
                bs = _split(per, 3)
                shards = [R.fold([R.sq_norm(padded[r * per + bs[i]: r * per + bs[i + 1]]) for i in range(len(bs) - 1)])
                          for r in range(world)]
                want = R.fold(shards)
                assert R.same(float(sq), want), f"all_reduce {tag} n {m} rank {rank}: {float(sq)!r} != {want!r}"
                done += 1
    return done


@pytest.mark.parametrize("world", [2, 3, 4])
def test_sq_norm_collectives(world):
    run_ranks(_worker, world, backend="gloo", timeout=600)


def test_world_of_one_and_empty():
    """Without a process group the collectives finish with torch: the norm is ops.sq_norm of the same pieces, folded
    in member order, and an empty tensor's is +0."""
    import dietgpu_b200 as dg

    x = (torch.randn(50001) * 3).to(torch.bfloat16).cuda()
    sc = torch.ones(1, device="cuda")
    for f in (dg.reduce_scatter_compressed, dg.all_reduce_compressed):
        sq = torch.empty(1, dtype=torch.float64, device="cuda")
        res = f(x, members=4, scale_tensor=sc, sq_norm=sq)
        b = _split(res.numel(), 4)
        host = res.reshape(-1).double().cpu().numpy()
        want = R.fold([R.sq_norm(host[b[i]:b[i + 1]]) for i in range(len(b) - 1)])
        assert R.same(float(sq), want), (f.__name__, float(sq), want)
        sq.fill_(-1.0)
        f(x[:0], scale_tensor=sc, sq_norm=sq)
        assert float(sq) == 0.0 and not bool(torch.signbit(sq))
