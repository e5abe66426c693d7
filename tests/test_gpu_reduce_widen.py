"""Widening decode-and-sum (dgb_float_decompress_reduce_to / ops.decompress_data_reduce(archive_dtype=...)) and the
reducing collectives' reduce_dtype=torch.float32.  fp16 / bf16 archives are summed into fp32 outputs; decoding is
lossless, so the reference of every group is torch's fp32 left fold of the ORIGINAL 16-bit tensors in archive order,
acc = x0.float(); acc = acc + x1.float(); ...  Results must match it bit for bit, with NaN compared as "both NaN"."""
import itertools
import re
import time

import pytest
import torch

from codec_helpers import assert_guard_intact, codec_options, guarded_out
from multirank import run_ranks

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
SIZES = [0, 1, 31, 33, 4095, 4096, 4097, 8209, 300001]
WIDTHS = [1, 2, 3, 4, 5, 8, 9, 17]


def _bits(t):
    return t.view(torch.int32 if t.element_size() == 4 else torch.int16)


def assert_same(got, want, what):
    assert got.dtype == want.dtype and got.shape == want.shape, what
    nan = torch.isnan(got) & torch.isnan(want)
    bad = (_bits(got) != _bits(want)) & ~nan
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} element(s) differ, first at {int(bad.nonzero()[0])}"


def fold32(xs, init=None):
    """torch's fp32 left fold of the widened inputs, starting from `init` (fp32) when given."""
    acc = xs[0].float() if init is None else init.clone()
    for x in (xs[1:] if init is None else xs):
        acc = acc + x.float()
    return acc


def data(n, dtype, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(n, generator=g) * scale
    return x.to(dtype).cuda()


def compress(ts, pb=10, sparse=False):
    from dietgpu_b200 import ops

    comp, sizes, _ = ops.compress_data(True, ts, prob_bits=pb, sparse=sparse)
    hs = sizes.cpu().tolist()
    return [comp[i, :hs[i]] for i in range(len(ts))]


def reduce32(groups_in, outs, archive_dtype, accumulate=False, pb=10, status=None, temp=None):
    from dietgpu_b200 import ops

    return ops.decompress_data_reduce(groups_in, outs, accumulate, temp, status, prob_bits=pb,
                                      archive_dtype=archive_dtype)


def run_groups(dtype, pb, accumulate, width, sizes, seed=0, offsets=None):
    """One call over len(sizes) groups into fp32 outputs; checks every group against the fp32 fold and the guards."""
    xs = [[data(n, dtype, seed + 1000 * g + j, scale=1.0 + j) for j in range(width)] for g, n in enumerate(sizes)]
    arch = compress([x for grp in xs for x in grp], pb)
    groups_in = [arch[g * width:(g + 1) * width] for g in range(len(sizes))]
    bufs, outs, spans, inits = [], [], [], []
    for g, n in enumerate(sizes):
        b, v, span = guarded_out(n, torch.float32, (g * 3 + 1) % 8 if offsets is None else offsets[g])
        init = data(n, torch.float32, 77 + g)
        if accumulate:
            v.copy_(init)
        bufs.append(b)
        outs.append(v)
        spans.append(span)
        inits.append(init)
    st = torch.zeros(len(sizes) * width, dtype=torch.uint8, device="cuda")
    reduce32(groups_in, outs, dtype, accumulate, pb, st)
    torch.cuda.synchronize()
    assert bool(st.all())
    for g in range(len(sizes)):
        want = fold32(xs[g], inits[g] if accumulate else None)
        assert_same(outs[g], want, f"{dtype} pb {pb} acc {accumulate} W {width} group {g} n {sizes[g]}")
        assert_guard_intact(bufs[g], *spans[g], f"group {g}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("pb", [9, 10, 11])
@pytest.mark.parametrize("accumulate", [False, True])
def test_bit_exact_against_fp32_fold(dtype, pb, accumulate):
    for w in WIDTHS:
        run_groups(dtype, pb, accumulate, w, SIZES, seed=w)


@pytest.mark.parametrize("groups,width", [(1, 1), (64, 1), (65, 1), (70, 1), (8, 8), (13, 5), (3, 17)])
@pytest.mark.parametrize("inline", [1, 0])
def test_group_counts(groups, width, inline):
    with codec_options(inline_members=inline):
        run_groups(torch.bfloat16, 10, True, width, [4097 + 517 * (g % 7) for g in range(groups)], seed=groups)


def test_output_offsets_zero_to_seven():
    for dtype in DTYPES:
        for acc in (False, True):
            run_groups(dtype, 10, acc, 3, [8209] * 8, seed=5, offsets=list(range(8)))


def test_value_edges():
    for dtype in DTYPES:
        big = torch.finfo(dtype).max
        tiny = torch.finfo(dtype).tiny  # smallest normal; halves of it are subnormal
        a = torch.tensor([1.5, -0.0, 0.0, -0.0, float("inf"), big, tiny / 2, tiny / 4, -tiny / 2, 3.0, float("inf"),
                          -big], dtype=dtype)
        b = torch.tensor([-1.5, -0.0, -0.0, 0.0, float("-inf"), big, tiny / 4, tiny / 4, tiny / 4, float("nan"),
                          float("inf"), -big], dtype=dtype)
        a, b = a.repeat(1000).cuda(), b.repeat(1000).cuda()
        arch = compress([a, b])
        out = torch.empty(a.numel(), dtype=torch.float32, device="cuda")
        reduce32([arch], [out], dtype)
        assert_same(out, fold32([a, b]), f"{dtype} edges")
        o = _bits(out)[:12].cpu()
        assert int(o[0]) == 0 and int(o[1]) == -2 ** 31  # +0, -0
        assert int(o[2]) == 0 and int(o[3]) == 0
        assert bool(torch.isnan(out[4])) and bool(torch.isnan(out[9]))  # Inf - Inf, NaN
        assert float(out[10]) == float("inf")
        assert bool(torch.isinf((a + b)[5]))  # the 16-bit maximum twice overflows in the 16-bit sum ...
        if dtype == torch.float16:  # ... and is finite in fp32 for fp16 (bf16 has fp32's exponent range)
            assert float(out[5]) == 2 * float(big) and float(out[11]) == -2 * float(big)
        else:
            assert float(out[5]) == float("inf") and float(out[11]) == float("-inf")
        assert float(out[6]) == float(tiny) * 0.75 and float(out[8]) == -float(tiny) * 0.25  # subnormals kept


@pytest.mark.parametrize("accumulate", [False, True])
def test_signed_zeros_in_every_pairing(accumulate):
    combos = list(itertools.product([0.0, -0.0], repeat=3))  # (init, x0, x1)
    for dtype in DTYPES:
        init = torch.tensor([c[0] for c in combos] * 3000, dtype=torch.float32).cuda()
        x0 = torch.tensor([c[1] for c in combos] * 3000, dtype=dtype).cuda()
        x1 = torch.tensor([c[2] for c in combos] * 3000, dtype=dtype).cuda()
        out = init.clone()
        reduce32([compress([x0, x1])], [out], dtype, accumulate)
        assert_same(out, fold32([x0, x1], init if accumulate else None), f"{dtype} zeros acc {accumulate}")


def test_plain_widening_decode_of_every_bit_pattern():
    # W = 1 without accumulate: every 16-bit pattern, in two orders, decodes to x.float() (-0, infinities and
    # subnormals bit for bit; NaN as NaN)
    for dtype in DTYPES:
        pats = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
        for x in (pats, pats.flip(0)):
            x = x.repeat(3).view(dtype).cuda()
            out = torch.empty(x.numel(), dtype=torch.float32, device="cuda")
            reduce32([compress([x])], [out], dtype)
            assert_same(out, x.float(), f"{dtype} patterns")


def test_sums_are_fp32():
    n = 100000
    xs = [data(n, torch.bfloat16, 60 + j, scale=1.0 + j) for j in range(17)]
    out = torch.empty(n, dtype=torch.float32, device="cuda")
    reduce32([compress(xs)], [out], torch.bfloat16)
    assert_same(out, fold32(xs), "fp32 fold")
    acc16 = xs[0]
    for x in xs[1:]:
        acc16 = acc16 + x
    differ = int((_bits(out) != _bits(acc16.float())).sum())
    assert differ > n // 2, f"only {differ} of {n} elements differ from the bf16 fold"


def _raw(fn, ft, out_ft, groups_in, outs, accumulate, status):
    from dietgpu_b200 import capi

    L = capi.lib()
    ins = [a for grp in groups_in for a in grp]
    need = L.dgb_float_decompress_temp_bytes(ft, len(ins), 0)
    temp = torch.empty(need + 256, dtype=torch.uint8, device="cuda")
    ptr = temp.data_ptr() + (-temp.data_ptr()) % 256
    args = (len(groups_in), len(groups_in[0]), capi.ptr_array([a.data_ptr() for a in ins]),
            capi.ptr_array([o.data_ptr() for o in outs]), capi.u32_array([o.numel() for o in outs]), int(accumulate),
            status.data_ptr(), torch.cuda.current_stream().cuda_stream)
    if fn == "reduce":
        rc = L.dgb_float_decompress_reduce(ptr, need, ft, 10, *args)
    else:
        rc = L.dgb_float_decompress_reduce_to(ptr, need, ft, out_ft, 10, *args)
    assert rc == capi.OK
    torch.cuda.synchronize()


@pytest.mark.parametrize("accumulate", [False, True])
def test_equal_types_match_the_same_type_call(accumulate):
    from dietgpu_b200 import capi

    types = {torch.float16: capi.FLOAT16, torch.bfloat16: capi.BFLOAT16, torch.float32: capi.FLOAT32}
    for dtype, ft in types.items():
        groups, width, n = 3, 6, 9001
        xs = [data(n, dtype, 30 + j) for j in range(groups * width)]
        arch = compress(xs)
        groups_in = [arch[g * width:(g + 1) * width] for g in range(groups)]
        groups_in[1][4] = compress([data(n + 1, dtype, 3)])[0]  # one invalid archive, in the second pass
        init = data(n, dtype, 99)
        res = {}
        for fn in ("reduce", "reduce_to"):
            outs = [init.clone() for _ in range(groups)]
            st = torch.full((groups * width,), 7, dtype=torch.uint8, device="cuda")
            _raw(fn, ft, ft, groups_in, outs, accumulate, st)
            res[fn] = (outs, st.cpu().tolist())
        assert res["reduce"][1] == res["reduce_to"][1]
        assert res["reduce"][1] == [1] * width + [1, 1, 1, 1, 0, 1] + [1] * width
        for a, b in zip(res["reduce"][0], res["reduce_to"][0]):
            assert torch.equal(_bits(a), _bits(b)), dtype


def test_invalid_groups_are_not_written():
    from dietgpu_b200 import ops

    n = 10000
    dt = torch.bfloat16
    width = 3
    xs = [[data(n, dt, 900 + 10 * g + j) for j in range(width)] for g in range(7)]
    arch = compress([x for grp in xs for x in grp])
    groups_in = [list(arch[g * width:(g + 1) * width]) for g in range(7)]
    relu = torch.relu(data(n, dt, 5))
    bad = [
        compress([data(n, torch.float32, 1)])[0],             # an fp32 archive given as bf16
        compress([relu], sparse=True)[0],                     # a sparse bf16 archive
        compress([data(n, dt, 2)], pb=9)[0],                  # other probBits
        compress([data(n - 1, dt, 3)])[0],                    # one word short
        compress([data(n + 1, dt, 4)])[0],                    # one word long
        compress([data(n, torch.float16, 6)])[0],             # fp16 given as bf16
    ]
    for g, a in enumerate(bad):
        groups_in[g][1] = a
    bufs, outs, spans = [], [], []
    for g in range(7):
        b, v, span = guarded_out(n, torch.float32, g)
        bufs.append(b)
        outs.append(v)
        spans.append(span)
    st = torch.full((7 * width,), 7, dtype=torch.uint8, device="cuda")
    ops.decompress_data_reduce(groups_in, outs, False, None, st, archive_dtype=dt)
    torch.cuda.synchronize()
    want_st = [1] * (7 * width)
    for g in range(6):
        want_st[g * width + 1] = 0
    assert st.cpu().tolist() == want_st
    for g in range(6):
        assert bool((bufs[g] == bufs[g][0]).all()), f"invalid group {g} was written"
    assert_same(outs[6], fold32(xs[6]), "valid group")
    assert_guard_intact(bufs[6], *spans[6], "valid group")
    # the invalid archive in a later pass: nothing is written by any pass
    xs9 = [data(n, dt, 300 + j) for j in range(9)]
    a9 = compress(xs9)
    a9[7] = bad[3]
    out = torch.full((n,), 3.0, dtype=torch.float32, device="cuda")
    st9 = torch.zeros(9, dtype=torch.uint8, device="cuda")
    ops.decompress_data_reduce([a9], [out], True, None, st9, archive_dtype=dt)
    assert st9.cpu().tolist() == [1] * 7 + [0, 1]
    assert bool((out == 3.0).all())


@pytest.mark.parametrize("dtype", DTYPES)
def test_graph_capture(dtype):
    from dietgpu_b200 import ops

    groups, width, n = 6, 5, 20000
    cols = 64 << 10
    rows = torch.zeros(groups * width, cols, dtype=torch.uint8, device="cuda")

    def load(seed):
        xs = [[data(n, dtype, seed + 100 * g + j) for j in range(width)] for g in range(groups)]
        arch = compress([x for grp in xs for x in grp])
        for i, a in enumerate(arch):
            rows[i, :a.numel()].copy_(a)
        return xs, [a.numel() for a in arch]

    xs, lens = load(1)
    init = [data(n, torch.float32, 5 + g) for g in range(groups)]
    outs = [torch.empty(n, dtype=torch.float32, device="cuda") for _ in range(groups)]
    ins = [[rows[g * width + j, :lens[g * width + j]] for j in range(width)] for g in range(groups)]
    scratch = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for o, i in zip(outs, init):
            o.copy_(i)
        ops.decompress_data_reduce(ins, outs, True, scratch, archive_dtype=dtype)  # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        ops.decompress_data_reduce(ins, outs, True, scratch, archive_dtype=dtype)
    for seed in (2, 3):
        xs, _ = load(seed * 1000)  # new contents, no longer than the captured rows
        for o, i in zip(outs, init):
            o.copy_(i)
        g.replay()
        torch.cuda.synchronize()
        for k in range(groups):
            assert_same(outs[k], fold32(xs[k], init[k]), f"replay seed {seed} group {k}")


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
            work.append(([compress(xs, pb)], [torch.empty(5000, dtype=torch.float32, device="cuda")], dtype, pb))
    # a throwaway kernel goes first (the first kernel of a session can be missing from its trace) and every
    # instantiation is launched three times, well inside the profiler's window: in a long-lived process the GPU
    # timestamps drift against the host clock and records near the window's edges are dropped
    # (test_gpu_weighted_reduce.py)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(1.0)
        torch.ones(1, device="cuda").add_(1)
        for _ in range(3):
            for ins, outs, dtype, pb in work:
                reduce32(ins, outs, dtype, False, pb)
        torch.cuda.synchronize()
        time.sleep(1.0)
    names = {re.sub(r"\s", "", e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    for kind in (33, 34):  # fp16 | widen, bf16 | widen
        for pb in (9, 10, 11):
            assert any(f"decodeReduceKernel<{kind},{pb}>" in k for k in names), (kind, pb, sorted(names))


def test_large_bf16_8x8x2mi():
    groups, width, n = 8, 8, 2 << 20
    xs = [[data(n, torch.bfloat16, 7000 + 10 * g + j) for j in range(width)] for g in range(groups)]
    arch = compress([x for grp in xs for x in grp])
    outs = [torch.empty(n, dtype=torch.float32, device="cuda") for _ in range(groups)]
    st = torch.zeros(groups * width, dtype=torch.uint8, device="cuda")
    reduce32([arch[g * width:(g + 1) * width] for g in range(groups)], outs, torch.bfloat16, False, 10, st)
    assert bool(st.all())
    for g in range(groups):
        assert_same(outs[g], fold32(xs[g]), f"group {g}")


def test_argument_errors():
    from dietgpu_b200 import ops

    x = data(100, torch.bfloat16, 1)
    a = compress([x])
    f32 = torch.empty(100, dtype=torch.float32, device="cuda")
    bad = [
        (torch.empty(100, dtype=torch.bfloat16, device="cuda"), torch.float32),   # fp32 archives into bf16
        (torch.empty(100, dtype=torch.bfloat16, device="cuda"), torch.float16),   # fp16 archives into bf16
        (torch.empty(100, dtype=torch.float16, device="cuda"), torch.bfloat16),   # bf16 archives into fp16
        (f32, torch.float64),                                                     # float64 archives
        (torch.empty(100, dtype=torch.float64, device="cuda"), torch.bfloat16),   # float64 outputs
        (torch.empty(100, dtype=torch.float64, device="cuda"), torch.float64),
        (torch.empty(100, dtype=torch.float64, device="cuda"), None),
    ]
    for out, adt in bad:
        with pytest.raises(ValueError):
            ops.decompress_data_reduce([a], [out], archive_dtype=adt)
    # archive_dtype equal to the outputs' dtype is the same-type call
    o1, o2 = torch.empty_like(x), torch.empty_like(x)
    ops.decompress_data_reduce([a], [o1])
    ops.decompress_data_reduce([a], [o2], archive_dtype=torch.bfloat16)
    assert torch.equal(_bits(o1), _bits(o2)) and torch.equal(_bits(o1), _bits(x))


# ---- two ranks ------------------------------------------------------------------------------------------------

def _worker(rank, world, dev):
    import dietgpu_b200 as dg

    def same(a, b):
        nan = torch.isnan(a) & torch.isnan(b)
        return a.dtype == b.dtype and a.shape == b.shape and not bool(((_bits(a) != _bits(b)) & ~nan).any())

    for dt in DTYPES:
        for n in (2 * 40000, 300001):
            ts = []
            for r in range(world):
                g = torch.Generator(device="cpu").manual_seed(700 + r + n)
                x = torch.randn(n, generator=g) * (1 + r)
                x[::97] = float("nan") if r == 1 else 0.0
                x[5::89] = -0.0
                ts.append(x.to(dt).to(dev))
            want = fold32(ts)
            for members in (1, 6):
                if n % world == 0:
                    shard = n // world
                    got = dg.reduce_scatter_compressed(ts[rank], members=members, reduce_dtype=torch.float32)
                    assert same(got, want[rank * shard:(rank + 1) * shard]), f"reduce_scatter {dt} {n} {members}"
                    a = dg.reduce_scatter_compressed(ts[rank], members=members, reduce_dtype=dt)
                    b = dg.reduce_scatter_compressed(ts[rank], members=members)
                    assert same(a, b), f"reduce_scatter reduce_dtype={dt} {n} {members}"
                t = ts[rank].view(-1, 1) if n % 2 else ts[rank]
                got = dg.all_reduce_compressed(t, members=members, reduce_dtype=torch.float32)
                assert got.shape == t.shape and same(got.reshape(-1), want), f"all_reduce {dt} {n} {members}"
                a = dg.all_reduce_compressed(t, members=members, reduce_dtype=dt)
                b = dg.all_reduce_compressed(t, members=members)
                assert same(a, b), f"all_reduce reduce_dtype={dt} {n} {members}"
    for t, rdt in ((torch.zeros(16, dtype=torch.float32, device=dev), torch.float16),
                   (torch.zeros(16, dtype=torch.float32, device=dev), torch.bfloat16),
                   (torch.zeros(16, dtype=torch.bfloat16, device=dev), torch.float64),
                   (torch.zeros(16, dtype=torch.float16, device=dev), torch.bfloat16),
                   (torch.zeros(16, dtype=torch.bfloat16, device=dev), torch.float16)):
        for fn in (dg.reduce_scatter_compressed, dg.all_reduce_compressed):
            with pytest.raises(ValueError):
                fn(t, reduce_dtype=rdt)


def test_two_rank_reduce_collectives_fp32():
    run_ranks(_worker, 2, timeout=300)
