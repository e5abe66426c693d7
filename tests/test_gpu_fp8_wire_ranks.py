"""The fp8 wire of the compressed collectives on 2, 3 and 4 ranks (gloo, every rank on cuda:0):

    reduce_scatter_compressed(t, wire_dtype=T, wire_scale=s, ...) == the rank-order fold of q_r.float() * d
    all_gather_compressed(t, wire_dtype=T, wire_scale=s)          == cat([q_r for every rank r])

bit for bit on every rank, with q_r = ops.cast_fp8([t_r], T, s) (the cast pinned to torch's clamp-cast by
test_gpu_fp8_wire.py) and d = u / s, u being 1, np.float32(scale), np.float32(1 / world) or scale_tensor; found_inf
and sq_norm against their definitions on the returned shard."""
import numpy as np
import pytest
import torch

from multirank import run_ranks

pytestmark = pytest.mark.gpu

FP8 = (torch.float8_e4m3fn, torch.float8_e5m2)


def _tensor(rank, n, dtype, dev):
    g = torch.Generator(device="cpu").manual_seed(7000 + 13 * rank + n)
    x = torch.randn(n, generator=g) * (1 + rank)
    x[::101] = -0.0
    x[3::211] = 1e6 if rank == 0 else 1e-9  # saturates, and flushes to zero
    return x.to(dtype).to(dev)


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _worker(rank, world, dev):
    import dietgpu_b200 as dg
    from dietgpu_b200 import ops
    from dietgpu_b200.collectives import _split

    checks = 0
    n = world * 8 * 4099
    shard = n // world
    for dtype in (torch.float32, torch.bfloat16):
        ts = [_tensor(r, n, dtype, dev) for r in range(world)]
        t = ts[rank]
        for T in FP8:
            for sv in (None, 0.37):
                s = None if sv is None else torch.full((1,), sv, device=dev)
                qs = [ops.cast_fp8([x], T, s)[0] for x in ts]
                # all-gather: every rank's cast, in rank order
                got = dg.all_gather_compressed(t, wire_dtype=T, wire_scale=s, members=3)
                want = torch.cat(qs)
                assert got.dtype == T and torch.equal(got.view(torch.uint8), want.view(torch.uint8)), (dtype, T, sv)
                checks += 1
                for mode in ("plain", "average", "scale", "device"):
                    kw, u = {}, torch.ones(1, device=dev)
                    if mode == "average":
                        kw, u = dict(average=True), torch.full((1,), float(np.float32(1 / world)), device=dev)
                    elif mode == "scale":
                        kw, u = dict(scale=-2.5), torch.full((1,), -2.5, device=dev)
                    elif mode == "device":
                        u = torch.full((1,), 0.125, device=dev)
                        flag = torch.zeros(1, device=dev)
                        sq = torch.zeros(1, dtype=torch.float64, device=dev)
                        kw = dict(scale_tensor=u, found_inf=flag, sq_norm=sq)
                    d = u if s is None else u / s
                    for members in (1, 5):
                        res = dg.reduce_scatter_compressed(t, wire_dtype=T, wire_scale=s, members=members, **kw)
                        chunk = slice(rank * shard, (rank + 1) * shard)
                        want = qs[0][chunk].float() * d.reshape(())
                        for r in range(1, world):
                            want = want + qs[r][chunk].float() * d.reshape(())
                        assert _same(res, want), (dtype, T, sv, mode, members)
                        checks += 1
                        if mode == "device":
                            assert float(flag) == 0.0
                            bounds = _split(shard, members, 8)
                            parts = ops.sq_norm([res[bounds[i]:bounds[i + 1]] for i in range(len(bounds) - 1)])
                            acc = parts[0:1].clone()
                            for i in range(1, parts.numel()):
                                acc += parts[i:i + 1]
                            assert torch.equal(sq.view(torch.int64), acc.view(torch.int64)), (dtype, T, sv, members)
                            checks += 1
                # an infinite dequantisation scale sets the flag on every rank
                flag = torch.zeros(1, device=dev)
                dg.reduce_scatter_compressed(t, wire_dtype=T, wire_scale=s,
                                             scale_tensor=torch.full((1,), float("inf"), device=dev), found_inf=flag)
                assert float(flag) == 1.0
                checks += 1
    return checks


@pytest.mark.parametrize("world", [2, 3, 4])
def test_fp8_wire_ranks(world):
    run_ranks(_worker, world, backend="gloo", timeout=900)
