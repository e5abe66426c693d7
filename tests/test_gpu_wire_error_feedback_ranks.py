"""Error feedback in the compressed collectives, on 2 and 3 ranks (run_ranks: NCCL with a GPU per rank, else gloo with
every rank on cuda:0).

    reduce_scatter_compressed(t, wire_dtype=w, error_feedback=e, **kw) == reduce_scatter_compressed(t + e, wire_dtype=w, **kw)
    all_gather_compressed(t, wire_dtype=w, error_feedback=e)           == all_gather_compressed(t + e, wire_dtype=w)

bit for bit on every rank, and e ends as torch.where(w.isfinite(), y - w.float(), 0) with y = t + e, w = y.to(w)
over the whole tensor, own chunk included."""
import pytest
import torch

from multirank import run_ranks

pytestmark = pytest.mark.gpu

WIRES = (torch.float16, torch.bfloat16)


def _bits(t):
    return t.view(torch.int32 if t.element_size() == 4 else torch.int16)


def _residual(t, e, w):
    y = t + e
    q = y.to(w)
    return torch.where(q.isfinite(), y - q.float(), 0)


def _rank_tensors(rank, n, dev):
    g = torch.Generator(device="cpu").manual_seed(4000 + 17 * rank + n)
    x = torch.randn(n, generator=g) * (1 + rank)
    x[::97] = float("nan") if rank == 1 else 0.0
    x[5::89] = -0.0
    x[7::211] = float("inf") if rank == 0 else 1.0
    e = torch.randn(n, generator=g) * 2 ** -9
    e[::13] = 0.0
    e[3::101] = -0.0
    return x.to(dev), e.to(dev)


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _identities(rank, world, dev):
    import dietgpu_b200 as dg

    checks = 0
    for w in WIRES:
        for n in (world * 8 * 4099, world * 300000):
            t, e0 = _rank_tensors(rank, n, dev)
            t[9::4001] = 70000.0  # every chunk: +inf in fp16, finite in bf16
            want_e = _residual(t, e0, w)
            shard = n // world
            kws = [dict(), dict(reduce_dtype=torch.float32), dict(out_dtype=w), dict(average=True)]
            for members in (1, 6):
                for kw in kws:
                    e = e0.clone()
                    got = dg.reduce_scatter_compressed(t, members=members, wire_dtype=w, error_feedback=e, **kw)
                    want = dg.reduce_scatter_compressed(t + e0, members=members, wire_dtype=w, **kw)
                    assert _same(got, want), f"reduce_scatter {w} {n} {members} {kw}"
                    assert torch.equal(_bits(e), _bits(want_e)), f"residual {w} {n} {members} {kw}"
                    for d in range(world):  # every chunk got its new residual, own chunk included
                        assert not torch.equal(_bits(e[d * shard:(d + 1) * shard]), _bits(e0[d * shard:(d + 1) * shard])), \
                            f"chunk {d} kept its old residual"
                    checks += 2
                # the device-side keywords: scale, non-finite flag and squared norm together
                s = torch.full((1,), 0.25, device=dev)
                flags = [torch.zeros(1, device=dev) for _ in range(2)]
                norms = [torch.zeros(1, dtype=torch.float64, device=dev) for _ in range(2)]
                e = e0.clone()
                got = dg.reduce_scatter_compressed(t, members=members, wire_dtype=w, error_feedback=e, scale_tensor=s,
                                                   found_inf=flags[0], sq_norm=norms[0], out_dtype=w)
                want = dg.reduce_scatter_compressed(t + e0, members=members, wire_dtype=w, scale_tensor=s,
                                                    found_inf=flags[1], sq_norm=norms[1], out_dtype=w)
                assert _same(got, want), f"reduce_scatter {w} {n} {members} device keywords"
                assert torch.equal(flags[0], flags[1]), f"found_inf {w} {n} {members}"
                assert torch.equal(norms[0].view(torch.int64), norms[1].view(torch.int64)), f"sq_norm {w} {n} {members}"
                assert torch.equal(_bits(e), _bits(want_e)), f"residual {w} {n} {members} device keywords"
                # rank 0's +inf is in every chunk, so every shard is flagged
                assert float(flags[0]) == 1.0, "found_inf not set"
                if w == torch.float16:
                    # 70000 rounds to fp16 inf: its residual is +0, not -inf
                    assert bool((_bits(e[9::4001]) == 0).all()), "an fp16 overflow left a non-zero residual"
                checks += 1
                for stages in (1, 2, 3):
                    e = e0.clone()
                    got = dg.all_gather_compressed(t, members=members, stages=stages, wire_dtype=w, error_feedback=e)
                    want = dg.all_gather_compressed(t + e0, members=members, stages=stages, wire_dtype=w)
                    assert _same(got, want), f"all_gather {w} {n} {members} {stages}"
                    assert torch.equal(_bits(e), _bits(want_e)), f"all_gather residual {w} {n} {members} {stages}"
                    checks += 1
            # the two-phase fp32 all-reduce with a worker and a server error
            es0 = torch.randn(shard, device=dev) * 2 ** -9
            ew, es = e0.clone(), es0.clone()
            shard_sum = dg.reduce_scatter_compressed(t, wire_dtype=w, error_feedback=ew)
            full = dg.all_gather_compressed(shard_sum, wire_dtype=w, error_feedback=es)
            want_shard = dg.reduce_scatter_compressed(t + e0, wire_dtype=w)
            assert _same(full, dg.all_gather_compressed(want_shard + es0, wire_dtype=w)), f"two phases {w} {n}"
            assert torch.equal(_bits(ew), _bits(want_e)), f"worker error {w} {n}"
            assert torch.equal(_bits(es), _bits(_residual(want_shard, es0, w))), f"server error {w} {n}"
            checks += 1
    return checks


def _drift(rank, world, dev):
    # a constant gradient bf16 cannot hold (1 + 2^-10 rounds to 1): the mean of the reduced values over many steps
    # stays a whole rounding error away without error feedback, and comes within a bf16 ulp / steps with it
    import dietgpu_b200 as dg

    g = torch.full((world * 4096,), 1 + 2 ** -10, device=dev)
    steps, ulp = 64, 2 ** -7
    for use_ef in (False, True):
        e = torch.zeros_like(g) if use_ef else None
        total = torch.zeros(4096, dtype=torch.float64, device=dev)
        for _ in range(steps):
            total += dg.reduce_scatter_compressed(g, wire_dtype=torch.bfloat16, average=True,
                                                  error_feedback=e).double()
        err = float((total / steps - (1 + 2 ** -10)).abs().max())
        if use_ef:
            assert err <= ulp / steps, err
            assert float(e.abs().max()) <= ulp / 2
        else:
            assert err >= 0.99 * 2 ** -10, err
    return 2


def _worker(rank, world, dev):
    return _identities(rank, world, dev) + _drift(rank, world, dev)


@pytest.mark.parametrize("world", [2, 3])
def test_collective_identities(world):
    run_ranks(_worker, world, timeout=900)


def test_single_process_takes_the_torch_path():
    import dietgpu_b200 as dg

    t, e0 = _rank_tensors(0, 40000, "cuda")
    for w in WIRES:
        e = e0.clone()
        got = dg.reduce_scatter_compressed(t, wire_dtype=w, error_feedback=e, reduce_dtype=torch.float32)
        assert _same(got, dg.reduce_scatter_compressed(t + e0, wire_dtype=w, reduce_dtype=torch.float32))
        assert torch.equal(_bits(e), _bits(_residual(t, e0, w)))
        e = e0.clone()
        got = dg.all_gather_compressed(t, wire_dtype=w, error_feedback=e)
        assert _same(got, dg.all_gather_compressed(t + e0, wire_dtype=w))
        assert torch.equal(_bits(e), _bits(_residual(t, e0, w)))
        empty = torch.empty(0, device="cuda")
        ee = torch.empty(0, device="cuda")
        assert dg.reduce_scatter_compressed(empty, wire_dtype=w, error_feedback=ee).numel() == 0
        assert dg.all_gather_compressed(empty, wire_dtype=w, error_feedback=ee).numel() == 0
