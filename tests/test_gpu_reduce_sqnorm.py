"""Squared norms: ops.decompress_data_reduce(sq_norm=) on the 14 device-scale kinds (dgb_float_decompress_reduce_
scaled_dev_norm and _narrow_norm) and the standalone ops.sq_norm (dgb_float_sq_norm).

Every call is compared with the same call without sq_norm (outputs and found_inf bit for bit), and its norms with
ops.sq_norm of the outputs and with the numpy restatement tests/sq_norm_reference.py, bit for bit (a NaN matches any
NaN), at probBits 9-11, W = 1..9 (one, two and three kernel launches), with and without accumulate, on groups of 0,
1, 33, 4095, 4097 and 70001 words (partial last rows and blocks, an empty group).  The crafted order pins of the
restatement must come out as it predicts, a group with an invalid archive keeps its sentinel, a CUDA graph replay
reads the current scale, and both stream branches of the block decoder (staged and read from global memory) agree."""
import numpy as np
import pytest
import torch

import sq_norm_reference as R
from dietgpu_b200 import capi

pytestmark = pytest.mark.gpu

SIZES = [0, 1, 33, 4095, 4097, 70001]
SCALE = float(np.float32(-0.37))
# (archive dtype, sparse, output dtype, narrowing): the ten device-scale kinds and the four narrowing ones
KINDS = {
    "f16": (torch.float16, False, torch.float16, False),
    "bf16": (torch.bfloat16, False, torch.bfloat16, False),
    "f32": (torch.float32, False, torch.float32, False),
    "f16s": (torch.float16, True, torch.float16, False),
    "bf16s": (torch.bfloat16, True, torch.bfloat16, False),
    "f32s": (torch.float32, True, torch.float32, False),
    "f16-f32": (torch.float16, False, torch.float32, False),
    "bf16-f32": (torch.bfloat16, False, torch.float32, False),
    "f16s-f32": (torch.float16, True, torch.float32, False),
    "bf16s-f32": (torch.bfloat16, True, torch.float32, False),
    "f16-narrow": (torch.float16, False, torch.float16, True),
    "bf16-narrow": (torch.bfloat16, False, torch.bfloat16, True),
    "f16s-narrow": (torch.float16, True, torch.float16, True),
    "bf16s-narrow": (torch.bfloat16, True, torch.bfloat16, True),
}


def _words(dt, n, seed, j):
    g = torch.Generator().manual_seed(seed * 131 + j)
    x = torch.randn(n, generator=g) * (1 + j)
    if n > 64:
        x[64::3] = 0.0  # zeros for the sparse kinds to elide
    return x.to(dt)


def _archives(xs, pb, sparse):
    from dietgpu_b200 import ops

    comp, sizes, _ = ops.compress_data(True, xs, prob_bits=pb, sparse=sparse)
    hs = sizes.cpu().tolist()
    return [comp[i, :hs[i]].clone() for i in range(len(xs))]


def _bits(t):
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _same(a, b, what):
    ok = (_bits(a) == _bits(b)) | (a.isnan() & b.isnan())
    assert bool(ok.all()), f"{what}: {int((~ok).sum())} of {a.numel()} differ"


def _expect(norms, outs, what):
    """norms equal ops.sq_norm of the outputs and the restatement, bit for bit."""
    from dietgpu_b200 import ops

    _same(norms, ops.sq_norm(outs), f"{what}: against ops.sq_norm")
    got = norms.cpu().numpy()
    for g, o in enumerate(outs):
        want = R.sq_norm(o.double().cpu().numpy())
        assert R.same(got[g], want), f"{what}: group {g} ({o.numel()} words): {got[g]!r} != {want!r}"


class Case:
    def __init__(self, kind, pb, widths, sizes=SIZES, seed=0):
        self.adt, self.sparse, self.odt, self.narrow = KINDS[kind]
        self.pb, self.sizes = pb, sizes
        self.all = [_archives([_words(self.adt, n, seed + g, j).cuda() for j in range(widths)], pb, self.sparse)
                    for g, n in enumerate(sizes)]

    def call(self, width, accumulate, scale, inits, sq_norm=None, found_inf=None, status=None, temp=None):
        from dietgpu_b200 import ops

        kw = dict(prob_bits=self.pb, archive_dtype=self.adt, sparse=self.sparse, scale_tensor=scale,
                  found_inf=found_inf, sq_norm=sq_norm)
        outs = [torch.full((n,), float("nan"), dtype=self.odt, device="cuda") for n in self.sizes]
        if self.narrow:
            kw["reduce_dtype"] = torch.float32
            kw["acc"] = [i.clone() for i in inits] if accumulate else None
        elif accumulate:
            outs = [i.to(self.odt) for i in inits]
        ops.decompress_data_reduce([a[:width] for a in self.all], outs, accumulate, temp, status, **kw)
        return outs


def _inits(sizes, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(n, generator=g) * 3).cuda() for n in sizes]


@pytest.mark.parametrize("pb", [9, 10, 11])
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_norm_is_the_restatement_and_leaves_the_sum_alone(kind, pb):
    case = Case(kind, pb, 9, seed=pb)
    for width in range(1, 10):
        for accumulate in (False, True):
            inits = _inits(case.sizes, width)
            sc = torch.full((1,), SCALE, device="cuda")
            fa, fb = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
            want = case.call(width, accumulate, sc, inits, found_inf=fa)
            norms = torch.full((len(case.sizes),), -1.0, dtype=torch.float64, device="cuda")
            st = torch.zeros(len(case.sizes) * width, dtype=torch.uint8, device="cuda")
            got = case.call(width, accumulate, sc, inits, sq_norm=norms, found_inf=fb, status=st)
            what = f"{kind} pb={pb} W={width} accumulate={accumulate}"
            assert bool(st.all()), what
            for g, (a, b) in enumerate(zip(got, want)):
                _same(a, b, f"{what} group {g}")
            assert float(fa) == float(fb), what
            _expect(norms, got, what)
            assert float(norms[0]) == 0.0 and not bool(torch.signbit(norms[0])), f"{what}: the empty group"


@pytest.mark.parametrize("slot", ["8", "worst"])
@pytest.mark.parametrize("kind", ["bf16", "f32s", "f16s-f32", "bf16s-narrow"])
def test_both_stream_branches(kind, slot):
    """decode_slot_words = 8 sends nearly every block through the global-memory stream; the worst case stages all."""
    case = Case(kind, 11, 5, seed=21)
    sc = torch.full((1,), SCALE, device="cuda")
    base = torch.empty(len(case.sizes), dtype=torch.float64, device="cuda")
    want = case.call(5, False, sc, None, sq_norm=base)
    capi.set_option("decode_slot_words", 8 if slot == "8" else 256 * 11 + 8)
    try:
        norms = torch.empty_like(base)
        got = case.call(5, False, sc, None, sq_norm=norms)
    finally:
        capi.set_option("decode_slot_words", 0)
    for a, b in zip(got, want):
        _same(a, b, f"{kind} slot {slot}")
    _same(norms, base, f"{kind} slot {slot}")
    _expect(norms, got, f"{kind} slot {slot}")


PINS = {torch.float16: (2.0 ** 15, 2.0 ** -12), torch.bfloat16: (2.0 ** 27, 1.0), torch.float32: (2.0 ** 27, 1.0)}


@pytest.mark.parametrize("kind", ["f16", "bf16", "f32", "bf16s", "f16-narrow"])
def test_order_pins(kind):
    """The rows, lanes and blocks pins of the restatement: the kernels' value is the one the documented order gives,
    which its obvious alternatives do not (tests/test_sq_norm_cpu.py)."""
    from dietgpu_b200 import ops

    adt, sparse, odt, narrow = KINDS[kind]
    big, small = PINS[adt]
    for name, x in (("rows", R.pin_rows(big, small)), ("lanes", R.pin_lanes(big, small)),
                    ("blocks", R.pin_blocks(big, small))):
        xt = torch.from_numpy(x).to(adt).cuda()
        arch = _archives([xt], 10, sparse)
        out = torch.empty(xt.numel(), dtype=odt, device="cuda")
        norms = torch.empty(1, dtype=torch.float64, device="cuda")
        kw = dict(reduce_dtype=torch.float32) if narrow else {}
        ops.decompress_data_reduce([arch], [out], archive_dtype=adt, sparse=sparse,
                                   scale_tensor=torch.ones(1, device="cuda"), sq_norm=norms, **kw)
        want = R.sq_norm(x)
        assert R.same(float(norms), want), (kind, name, float(norms), want)
        assert R.same(float(ops.sq_norm([xt])), want), (kind, name)


@pytest.mark.parametrize("kind", ["bf16", "f32s", "bf16s-narrow"])
@pytest.mark.parametrize("width", [1, 6])
def test_invalid_group_keeps_the_sentinel(kind, width):
    adt = KINDS[kind][0]
    case = Case(kind, 10, width, sizes=[4097, 9000], seed=3)
    wrong = _archives([_words(adt, 4096, 5, 0).cuda()], 10, KINDS[kind][1])[0]  # 4096 words for a 4097-word group
    case.all[0][width - 1] = wrong
    norms = torch.full((2,), 12345.5, dtype=torch.float64, device="cuda")
    st = torch.zeros(2 * width, dtype=torch.uint8, device="cuda")
    outs = case.call(width, False, torch.ones(1, device="cuda"), None, sq_norm=norms, status=st)
    assert st.cpu().tolist() == [1] * (width - 1) + [0] + [1] * width
    assert float(norms[0]) == 12345.5
    _expect(norms[1:], outs[1:], f"{kind} W={width} valid group")


def test_graph_replay_reads_the_current_scale():
    from dietgpu_b200 import ops

    case = Case("bf16s-narrow", 10, 6, sizes=[4097, 70001], seed=4)
    sc = torch.full((1,), SCALE, device="cuda")
    norms = torch.empty(2, dtype=torch.float64, device="cuda")
    acc = [torch.empty(n, device="cuda") for n in case.sizes]
    outs = [torch.empty(n, dtype=torch.bfloat16, device="cuda") for n in case.sizes]
    temp = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    kw = dict(archive_dtype=torch.bfloat16, sparse=True, reduce_dtype=torch.float32, acc=acc, scale_tensor=sc,
              sq_norm=norms)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):  # warm up outside the capture
        ops.decompress_data_reduce(case.all, outs, False, temp, **kw)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.decompress_data_reduce(case.all, outs, False, temp, **kw)
    for s in (0.25, -3.0, 1e30):
        sc.fill_(s)
        norms.fill_(-1.0)
        graph.replay()
        eager = torch.empty(2, dtype=torch.float64, device="cuda")
        want = case.call(6, False, torch.full((1,), s, device="cuda"), None, sq_norm=eager)
        _same(norms, eager, f"replay with scale {s}")
        for a, b in zip(outs, want):
            _same(a, b, f"replay with scale {s}")


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16, torch.float32])
def test_standalone_norm(dt):
    from dietgpu_b200 import ops

    g = torch.Generator().manual_seed(5)
    base = (torch.randn(300000, generator=g) * 7).to(dt).cuda()
    base[100] = 0.0
    # unaligned sizes and starts (element-aligned views at odd offsets), an empty tensor, one block and many
    ts = [base[:0], base[1:2], base[3:36], base[5:4100], base[7:8200], base[11:70012], base[13:290013]]
    got = ops.sq_norm(ts)
    assert got.dtype == torch.float64 and got.shape == (len(ts),)
    for i, t in enumerate(ts):
        want = R.sq_norm(t.double().cpu().numpy())
        assert R.same(float(got[i]), want), (dt, i, float(got[i]), want)
    out = torch.full((len(ts),), -1.0, dtype=torch.float64, device="cuda")
    assert ops.sq_norm(ts, out=out) is out
    _same(out, got, "out=")
    # a non-finite word gives a non-finite norm
    bad = base[:5000].clone()
    bad[4321] = float("inf")
    assert float(ops.sq_norm([bad])) == float("inf")
    bad[17] = float("nan")
    assert np.isnan(float(ops.sq_norm([bad])))
