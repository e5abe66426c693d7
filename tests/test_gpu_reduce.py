"""Decode-and-sum (dgb_float_decompress_reduce / ops.decompress_data_reduce) and the reducing collectives built on
it.  Decoding is lossless, so the reference of every group is the torch left fold of the ORIGINAL tensors in
archive order; results must match it bit for bit, with NaN compared as "both NaN"."""
import re

import numpy as np
import pytest
import torch

from codec_helpers import assert_guard_intact, codec_options, guarded_out
from multirank import run_ranks

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16, torch.float32]
SIZES = [0, 1, 31, 33, 4095, 4096, 4097, 8209, 300001]
WIDTHS = [1, 2, 3, 4, 5, 8, 9, 17]


def _bits(t):
    return t.view(torch.int32 if t.element_size() == 4 else torch.int16)


def assert_same(got, want, what):
    assert got.shape == want.shape, what
    nan = torch.isnan(got) & torch.isnan(want)
    bad = (_bits(got) != _bits(want)) & ~nan
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} element(s) differ, first at {int(bad.nonzero()[0])}"


def fold(xs, init=None):
    acc = xs[0].clone() if init is None else init.clone()
    for x in (xs[1:] if init is None else xs):
        acc = acc + x
    return acc


def data(n, dtype, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(n, generator=g) * scale
    return x.to(dtype).cuda()


def compress(ts, pb=10, dtype=None):
    from dietgpu_b200 import ops

    comp, sizes, _ = ops.compress_data(True, ts, prob_bits=pb)
    hs = sizes.cpu().tolist()
    return [comp[i, :hs[i]] for i in range(len(ts))]


def reduce(groups_in, outs, accumulate=False, pb=10, status=None):
    from dietgpu_b200 import ops

    return ops.decompress_data_reduce(groups_in, outs, accumulate, None, status, prob_bits=pb)


def run_groups(dtype, pb, accumulate, width, sizes, seed=0, offsets=None):
    """One call over len(sizes) groups; checks every group against the fold and the guard bands."""
    xs = [[data(n, dtype, seed + 1000 * g + j, scale=1.0 + j) for j in range(width)] for g, n in enumerate(sizes)]
    arch = compress([x for grp in xs for x in grp], pb)
    groups_in = [arch[g * width:(g + 1) * width] for g in range(len(sizes))]
    bufs, outs, spans, inits = [], [], [], []
    for g, n in enumerate(sizes):
        b, v, span = guarded_out(n, dtype, (g * 3 + 1) % 8 if offsets is None else offsets[g])
        init = data(n, dtype, 77 + g)
        if accumulate:
            v.copy_(init)
        bufs.append(b)
        outs.append(v)
        spans.append(span)
        inits.append(init)
    st = torch.zeros(len(sizes) * width, dtype=torch.uint8, device="cuda")
    reduce(groups_in, outs, accumulate, pb, st)
    torch.cuda.synchronize()
    assert bool(st.all())
    for g in range(len(sizes)):
        want = fold(xs[g], inits[g] if accumulate else None)
        assert_same(outs[g], want, f"{dtype} pb {pb} acc {accumulate} W {width} group {g} n {sizes[g]}")
        assert_guard_intact(bufs[g], *spans[g], f"group {g}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("pb", [9, 10, 11])
@pytest.mark.parametrize("accumulate", [False, True])
def test_bit_exact_against_fold(dtype, pb, accumulate):
    for w in WIDTHS:
        run_groups(dtype, pb, accumulate, w, SIZES, seed=w)


@pytest.mark.parametrize("groups,width", [(1, 1), (64, 1), (65, 1), (70, 1), (8, 8), (13, 5), (3, 17)])
@pytest.mark.parametrize("inline", [1, 0])
def test_group_counts(groups, width, inline):
    with codec_options(inline_members=inline):
        run_groups(torch.bfloat16, 10, True, width, [4097 + 517 * (g % 7) for g in range(groups)], seed=groups)


def test_output_offsets_zero_to_seven():
    for dtype in DTYPES:
        run_groups(dtype, 10, False, 3, [8209] * 8, seed=5, offsets=list(range(8)))


def test_value_edges():
    for dtype in DTYPES:
        big = 65504.0 if dtype == torch.float16 else 3.0e38
        tiny = torch.finfo(dtype).tiny  # smallest normal; halves of it are subnormal
        a = torch.tensor([1.5, -0.0, 0.0, -0.0, float("inf"), big, tiny / 2, tiny / 4, -tiny / 2, 3.0], dtype=dtype)
        b = torch.tensor([-1.5, -0.0, -0.0, 0.0, float("-inf"), big, tiny / 4, tiny / 4, tiny / 4, float("nan")],
                         dtype=dtype)
        a, b = a.repeat(1000).cuda(), b.repeat(1000).cuda()
        arch = compress([a, b])
        out = torch.empty_like(a)
        reduce([arch], [out])
        want = a + b
        assert_same(out, want, f"{dtype} edges")
        o = _bits(out)[:10].cpu()
        assert int(o[0]) == 0 and int(o[1]) == int(_bits(torch.tensor([-0.0], dtype=dtype))[0])  # +0, -0
        assert int(o[2]) == 0 and int(o[3]) == 0
        assert bool(torch.isnan(out[4])) and bool(torch.isnan(out[9]))
        assert bool(torch.isinf(out[5]))  # the largest finite value twice overflows
        assert float(out[6]) != 0.0 and float(out[8]) != 0.0  # subnormal results are kept
    # W = 1 without accumulate is a plain decode: NaN payloads and -0 survive bit for bit
    for dtype in DTYPES:
        it = torch.int32 if dtype == torch.float32 else torch.int16
        pat = ([0x7fc00123, 0x7f800001, -0x7ff0000, -2147483648, 5] if dtype == torch.float32
               else [0x7e01, 0x7c01, -0x0201, -32768, 5])
        x = torch.tensor(pat * 999, dtype=it).view(dtype).cuda()
        out = torch.empty_like(x)
        reduce([compress([x])], [out])
        assert torch.equal(_bits(out), _bits(x))


def test_canonical_archives_give_the_same_result():
    xs = [data(300001, torch.bfloat16, 40 + j) for j in range(5)]
    a = compress(xs)
    with codec_options(encode_canonical=1):
        b = compress(xs)
    o1, o2 = torch.empty_like(xs[0]), torch.empty_like(xs[0])
    reduce([a], [o1])
    reduce([b], [o2])
    assert torch.equal(_bits(o1), _bits(o2))
    assert_same(o1, fold(xs), "canonical")


def test_two_calls_identical():
    xs = [data(1 << 20, torch.float32, 50 + j) for j in range(9)]
    arch = compress(xs)
    o1, o2 = torch.empty_like(xs[0]), torch.empty_like(xs[0])
    reduce([arch], [o1])
    reduce([arch], [o2])
    assert torch.equal(_bits(o1), _bits(o2))


def test_invalid_groups_are_not_written():
    from dietgpu_b200 import ops

    n = 10000
    dt = torch.bfloat16
    width = 3
    xs = [[data(n, dt, 900 + 10 * g + j) for j in range(width)] for g in range(6)]
    arch = compress([x for grp in xs for x in grp])
    groups_in = [arch[g * width:(g + 1) * width] for g in range(6)]
    bad = [
        compress([data(n, torch.float16, 1)])[0],            # another float type
        compress([data(n, dt, 2)], pb=9)[0],                  # other probBits
        compress([data(n - 1, dt, 3)])[0],                    # one word short
        compress([data(n + 1, dt, 4)])[0],                    # one word long
    ]
    corrupt = arch[4 * width + 1].clone()
    corrupt[0] ^= 0xff                                         # magic
    bad.append(corrupt)
    for g, a in enumerate(bad):
        groups_in[g] = list(groups_in[g])
        groups_in[g][1] = a
    bufs, outs, spans = [], [], []
    for g in range(6):
        b, v, span = guarded_out(n, dt, g)
        bufs.append(b)
        outs.append(v)
        spans.append(span)
    st = torch.full((6 * width,), 7, dtype=torch.uint8, device="cuda")
    ops.decompress_data_reduce(groups_in, outs, False, None, st)
    torch.cuda.synchronize()
    want_st = [1] * (6 * width)
    for g in range(5):
        want_st[g * width + 1] = 0
    assert st.cpu().tolist() == want_st
    for g in range(5):
        assert bool((bufs[g] == bufs[g][0]).all()), f"invalid group {g} was written"
    assert_same(outs[5], fold(xs[5]), "valid group")
    assert_guard_intact(bufs[5], *spans[5], "valid group")
    # every pass takes the same decision: the invalid archive sits in a later pass
    xs9 = [data(n, dt, 300 + j) for j in range(9)]
    a9 = compress(xs9)
    a9[7] = bad[2]
    out = torch.full((n,), 3.0, dtype=dt, device="cuda")
    st9 = torch.zeros(9, dtype=torch.uint8, device="cuda")
    ops.decompress_data_reduce([a9], [out], True, None, st9)
    assert st9.cpu().tolist() == [1] * 7 + [0, 1]
    assert bool((out == 3.0).all())


@pytest.mark.parametrize("groups,width", [(2, 3), (26, 5)])
def test_graph_capture(groups, width):
    n = 20000
    dt = torch.float16
    cols = 64 << 10
    rows = torch.zeros(groups * width, cols, dtype=torch.uint8, device="cuda")

    def load(seed):
        xs = [[data(n, dt, seed + 100 * g + j) for j in range(width)] for g in range(groups)]
        arch = compress([x for grp in xs for x in grp])
        for i, a in enumerate(arch):
            rows[i, :a.numel()].copy_(a)
        return xs, [a.numel() for a in arch]

    xs, lens = load(1)
    init = [data(n, dt, 5 + g) for g in range(groups)]
    outs = [torch.empty(n, dtype=dt, device="cuda") for _ in range(groups)]
    ins = [[rows[g * width + j, :lens[g * width + j]] for j in range(width)] for g in range(groups)]
    scratch = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    from dietgpu_b200 import ops

    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for o, i in zip(outs, init):
            o.copy_(i)
        ops.decompress_data_reduce(ins, outs, True, scratch)  # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        ops.decompress_data_reduce(ins, outs, True, scratch)
    for seed in (2, 3):
        xs, lens2 = load(seed * 1000)
        # each archive is read only up to its own header's sizes, so new contents fit the captured rows as long as
        # they are no longer than the row
        for o, i in zip(outs, init):
            o.copy_(i)
        g.replay()
        torch.cuda.synchronize()
        for k in range(groups):
            assert_same(outs[k], fold(xs[k], init[k]), f"replay seed {seed} group {k}")


def test_profiler_sees_every_instantiation():
    # in a fresh process: in a long-lived one the GPU's timestamps drift against the host clock that bounds the
    # profiler's window, and every record of a window can fall outside it
    run_ranks(_profiler_sees_every_instantiation, 1, backend="gloo")


def _profiler_sees_every_instantiation(rank, world, dev):
    from torch.profiler import ProfilerActivity, profile

    work = []
    for dtype in DTYPES:
        for pb in (9, 10, 11):
            xs = [data(5000, dtype, 11 + j) for j in range(2)]
            work.append(([compress(xs, pb)], [torch.empty_like(xs[0])], pb))
    # the first kernel of a profiler session can be missing from its trace when an earlier session ran in the same
    # process, so a throwaway kernel goes first and every instantiation is launched three times
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device="cuda").add_(1)
        for _ in range(3):
            for ins, outs, pb in work:
                reduce(ins, outs, False, pb)
        torch.cuda.synchronize()
    names = {re.sub(r"\s", "", e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    for kind in (1, 2, 3):
        for pb in (9, 10, 11):
            assert any(f"decodeReduceKernel<{kind},{pb}>" in k for k in names), (kind, pb, sorted(names))


def test_large_bf16_8x8x2mi():
    groups, width, n = 8, 8, 2 << 20
    xs = [[data(n, torch.bfloat16, 7000 + 10 * g + j) for j in range(width)] for g in range(groups)]
    arch = compress([x for grp in xs for x in grp])
    outs = [torch.empty(n, dtype=torch.bfloat16, device="cuda") for _ in range(groups)]
    st = torch.zeros(groups * width, dtype=torch.uint8, device="cuda")
    reduce([arch[g * width:(g + 1) * width] for g in range(groups)], outs, False, 10, st)
    assert bool(st.all())
    for g in range(groups):
        assert_same(outs[g], fold(xs[g]), f"group {g}")


def test_argument_errors():
    from dietgpu_b200 import ops

    x = data(100, torch.bfloat16, 1)
    a = compress([x])
    with pytest.raises(ValueError):
        ops.decompress_data_reduce([a], [torch.empty(100, dtype=torch.float64, device="cuda")])
    with pytest.raises(RuntimeError):
        ops.decompress_data_reduce([a, a + [a[0]]], [torch.empty_like(x), torch.empty_like(x)])
    with pytest.raises(RuntimeError):
        ops.decompress_data_reduce([a], [torch.empty_like(x), torch.empty_like(x)])
    with pytest.raises(RuntimeError):
        ops.decompress_data_reduce([a], [torch.empty_like(x)], out_status=torch.zeros(2, dtype=torch.uint8, device="cuda"))


# ---- two ranks ------------------------------------------------------------------------------------------------

def _worker(rank, world, dev):
    import dietgpu_b200 as dg

    def same(a, b):
        nan = torch.isnan(a) & torch.isnan(b)
        return a.shape == b.shape and not bool(((_bits(a) != _bits(b)) & ~nan).any())

    for dt in DTYPES:
        for n in (2 * 40000, 300001):
            ts = []
            for r in range(world):
                g = torch.Generator(device="cpu").manual_seed(500 + r + n)
                x = torch.randn(n, generator=g) * (1 + r)
                x[::97] = float("nan") if r == 1 else 0.0
                x[5::89] = -0.0
                ts.append(x.to(dt).to(dev))
            want = fold(ts)
            for members in (1, 6):
                if n % world == 0:
                    got = dg.reduce_scatter_compressed(ts[rank], members=members)
                    shard = n // world
                    assert same(got, want[rank * shard:(rank + 1) * shard]), f"reduce_scatter {dt} {n} {members}"
                got = dg.all_reduce_compressed(ts[rank].view(-1, 1) if n % 2 else ts[rank], members=members)
                assert same(got.reshape(-1), want), f"all_reduce {dt} {n} {members}"
    for bad in (torch.zeros(16, dtype=torch.uint8, device=dev), torch.zeros(16, dtype=torch.float64, device=dev),
                torch.zeros(15, dtype=torch.bfloat16, device=dev)):
        with pytest.raises(ValueError):
            dg.reduce_scatter_compressed(bad)
    for bad in (torch.zeros(16, dtype=torch.uint8, device=dev), torch.zeros(16, dtype=torch.float64, device=dev)):
        with pytest.raises(ValueError):
            dg.all_reduce_compressed(bad)


def test_two_rank_reduce_collectives():
    run_ranks(_worker, 2, timeout=300)
