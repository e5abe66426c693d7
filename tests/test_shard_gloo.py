"""world_size-2 gloo test of the multi-GPU plumbing (host logic only): the batch shards by member with
no data-path collective; ranks only exchange the archive sizes."""
import pytest
import torch

from dietgpu_b200.collectives import exchange_archives, pack_offsets
from dietgpu_b200.shard import gather_sizes, shard_members, shard_range
from multirank import run_ranks


def test_shard_range_partitions():
    for n in (0, 1, 7, 64, 257):
        for world in (1, 2, 3, 8):
            seen = []
            for r in range(world):
                rr = shard_range(n, r, world)
                seen += list(rr)
                assert len(rr) in (n // world, n // world + 1)
            assert seen == list(range(n))
    with pytest.raises(ValueError):
        shard_range(4, 2, 2)
    assert shard_members(list("abcde"), 1, 2) == ["d", "e"]


def _worker(rank, world, dev, n):
    mine = shard_range(n, rank, world)
    # each rank "compresses" its members: fake sizes that encode the member index
    local = torch.tensor([1000 + 16 * i for i in mine], dtype=torch.int32)
    allsz = gather_sizes(local, n)
    assert allsz.tolist() == [1000 + 16 * i for i in range(n)], allsz.tolist()


@pytest.mark.parametrize("n", [7, 64])
def test_gather_sizes_world2(n):
    run_ranks(_worker, 2, n, backend=None, timeout=120, join_timeout=60)


def test_pack_offsets():
    offs, total = pack_offsets([0, 1, 16, 17, 4096])
    assert offs == [0, 0, 16, 32, 64] and total == 64 + 4096


def _archive(rank, i, size):
    g = torch.Generator().manual_seed(1000 * rank + i)
    return torch.randint(0, 256, (size,), dtype=torch.uint8, generator=g)


def _exchange_worker(rank, world, dev, sizes):
    rows = [_archive(rank, i, s) for i, s in enumerate(sizes[rank])]
    got = exchange_archives(rows)
    assert len(got) == world
    for w in range(world):
        assert len(got[w]) == len(sizes[w])
        for i, s in enumerate(sizes[w]):
            assert got[w][i].numel() == s and torch.equal(got[w][i], _archive(w, i, s)), (w, i)


@pytest.mark.parametrize("sizes", [[[160, 48, 4112], [16, 70000, 32]], [[32], [1616]]])
def test_exchange_archives_world2(sizes):
    # variable-size archives, different totals per rank: sizes all-gather + padded payload all-gather
    run_ranks(_exchange_worker, 2, sizes, backend=None, timeout=120, join_timeout=60)


def test_exchange_archives_single_process():
    rows = [_archive(0, i, s) for i, s in enumerate([16, 4096])]
    got = exchange_archives(rows)
    assert len(got) == 1 and all(torch.equal(a, b) for a, b in zip(got[0], rows))
    with pytest.raises(ValueError):
        exchange_archives([])
