"""Compressed collectives (dietgpu_b200/collectives.py, SURVEY.md 8f-3) with TWO ranks: real codec kernels on
the GPU, real exchange between two processes.  On a box with >= 2 GPUs the ranks use NCCL, one GPU each; on a
single-GPU box both ranks share cuda:0 and talk over gloo (the packed archives are staged through host memory),
so the multi-rank path is exercised wherever the GPU tests run."""
import pytest
import torch

from multirank import run_ranks

pytestmark = pytest.mark.gpu


def _worker(rank, world, dev):
    import torch.distributed as dist

    import dietgpu_b200 as dg

    # peer-memory transport (NVLink pull by the decode kernel): needs one GPU per rank
    ws = dg.PeerWorkspace(32 << 20) if dist.get_backend() == "nccl" else None
    for dt, n in ((torch.bfloat16, 300001), (torch.float16, 70000), (torch.uint8, 123457)):
        def make(r):
            g = torch.Generator(device="cpu").manual_seed(1000 + r)
            if dt.is_floating_point:
                return torch.randn(n, generator=g).to(dt)
            return torch.randint(0, 40, (n,), generator=g, dtype=torch.int32).to(dt)

        mine = make(rank).to(dev)
        want = torch.cat([make(r) for r in range(world)]).to(dev)
        for stages in (1, 2, 3):
            got = dg.all_gather_compressed(mine, members=6, stages=stages)
            assert torch.equal(got.view(torch.uint8), want.view(torch.uint8)), f"all_gather {dt} stages {stages}"
        # all-to-all: rank r sends a different chunk (and a different LENGTH) to every destination
        def chunk(src, dst):
            g = torch.Generator(device="cpu").manual_seed(77 + 10 * src + dst)
            m = 50000 + 3001 * src + 17 * dst
            if dt.is_floating_point:
                return torch.randn(m, generator=g).to(dt)
            return torch.randint(0, 9, (m,), generator=g, dtype=torch.int32).to(dt)

        recv = dg.all_to_all_compressed([chunk(rank, d).to(dev) for d in range(world)])
        for s in range(world):
            assert torch.equal(recv[s].view(torch.uint8), chunk(s, rank).to(dev).view(torch.uint8)), \
                f"all_to_all {dt} from {s}"
        if ws is not None:
            for mode, stages in (("push", 1), ("push", 2), ("push", 3), ("pull", 2), ("direct", 1), ("auto", 2)):
                got = dg.all_gather_compressed(mine, members=6, peer=ws, peer_mode=mode, stages=stages)
                assert torch.equal(got.view(torch.uint8), want.view(torch.uint8)), f"{mode} {dt} stages {stages}"

            def reg(src, dst):  # regular all-to-all: one length
                g = torch.Generator(device="cpu").manual_seed(99 + 10 * src + dst)
                if dt.is_floating_point:
                    return torch.randn(40001, generator=g).to(dt)
                return torch.randint(0, 9, (40001,), generator=g, dtype=torch.int32).to(dt)

            for mode in ("pull", "direct"):
                recv = dg.all_to_all_compressed([reg(rank, d).to(dev) for d in range(world)], peer=ws, peer_mode=mode)
                for s in range(world):
                    assert torch.equal(recv[s].view(torch.uint8), reg(s, rank).to(dev).view(torch.uint8)), \
                        f"{mode} all_to_all {dt} from {s}"


def test_two_rank_compressed_collectives():
    run_ranks(_worker, 2, timeout=150)
