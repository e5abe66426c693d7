"""Narrowing decode-and-sum (ops.decompress_data_reduce(reduce_dtype=torch.float32) into float16 / bfloat16 outputs,
dgb_float_decompress_reduce_narrow).

The reference is the existing path: the widening call (archive_dtype=dtype into float32 outputs, with the same scale,
scale_tensor and accumulated init) followed by torch's CUDA .to(dtype).  Every output is compared with it bit for bit
(a NaN stands for any NaN: the two roundings may pick different NaN payloads), on every archive kind (dense and
sparse fp16 / bf16), at probBits 9-11, for W = 1..9 (one, two and three kernel passes), with and without accumulate,
unscaled, host-scaled and device-scaled, and on groups of 0, 1, 4095, 4096, 4097 and 70001 words.  The words hold
sums that tie at the 16-bit rounding, fp16 sums that are finite in fp32 and round to inf, subnormal results, NaN and
-0 + -0.  found_inf must be set exactly when a stored 16-bit word is inf or NaN."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = {"f16": torch.float16, "bf16": torch.bfloat16}
SIZES = [0, 1, 4095, 4096, 4097, 70001]
SCALE = float(np.float32(-0.37))


def _words(dt, n, seed, j):
    """Archive j's words: N(0, 1) scaled per archive, with crafted elements at the front of every group."""
    g = torch.Generator().manual_seed(seed * 131 + j)
    x = torch.randn(n, generator=g, dtype=torch.float32) * (1 + j)
    if dt == torch.float16:
        tie, small, top = 2.0 ** -11, 2.0 ** -24, 65504.0
    else:
        tie, small, top = 2.0 ** -8, 2.0 ** -133, float(torch.finfo(torch.bfloat16).max)
    special = [
        1.0 if j == 0 else (tie if j == 1 else 0.0),        # 1 + half an ulp: a tie that rounds to even
        top if j == 0 else (16.0 if j == 1 else 0.0),        # fp16: 65504 + 16 = 65520, finite in fp32, inf in fp16
        3 * small if j == 0 else (-small if j == 1 else 0.0),  # a subnormal result
        float("nan") if j == 2 else 1.0,                     # NaN in one archive
        -0.0,                                                # -0 + -0 + ... = -0
        float("inf") if j == 1 else 0.5,
        -0.0 if j % 2 else 0.0,                              # signed zeros (sparse kinds elide both)
    ]
    k = min(n, len(special))
    x[:k] = torch.tensor(special[:k])
    if n > 64:
        x[64::3] = 0.0  # zeros for the sparse kinds to elide
    return x.to(dt)


def _archives(xs, pb, sparse):
    from dietgpu_b200 import ops

    comp, sizes, _ = ops.compress_data(True, xs, prob_bits=pb, sparse=sparse)
    hs = sizes.cpu().tolist()
    return [comp[i, :hs[i]].clone() for i in range(len(xs))]


def _same(a, b, what):
    """Bit equality of two 16-bit tensors, any NaN matching any NaN."""
    wa, wb = a.view(torch.int16), b.view(torch.int16)
    ok = (wa == wb) | (a.isnan() & b.isnan())
    assert bool(ok.all()), f"{what}: {int((~ok).sum())} of {a.numel()} differ, first at {int((~ok).nonzero()[0])}"


def _init(n, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(n, generator=g) * 3
    if n > 4:
        a[:4] = torch.tensor([-0.0, 65000.0, float("nan"), 1e-40])
    return a.cuda()


class Case:
    """G groups of W archives of one kind, with the widening reference computed for a scale mode."""

    def __init__(self, t, sparse, pb, width, sizes=SIZES, seed=0):
        self.dt, self.sparse, self.pb, self.width, self.sizes = DTYPES[t], sparse, pb, width, sizes
        self.groups = []
        for g, n in enumerate(sizes):
            xs = [_words(self.dt, n, seed + g, j).cuda() for j in range(width)]
            self.groups.append(_archives(xs, pb, sparse))

    def call(self, mode, accumulate, acc=None, outs=None, found_inf=None, status=None, scale_tensor=None):
        from dietgpu_b200 import ops

        kw = dict(prob_bits=self.pb, archive_dtype=self.dt, sparse=self.sparse)
        if mode == "host":
            kw["scale"] = SCALE
        elif mode == "dev":
            kw["scale_tensor"] = scale_tensor if scale_tensor is not None else torch.full((1,), SCALE, device="cuda")
            kw["found_inf"] = found_inf
        outs = outs if outs is not None else [torch.full((n,), float("nan"), dtype=self.dt, device="cuda")
                                              for n in self.sizes]
        ops.decompress_data_reduce(self.groups, outs, accumulate, None, status, reduce_dtype=torch.float32, acc=acc,
                                   **kw)
        return outs

    def reference(self, mode, accumulate, inits):
        from dietgpu_b200 import ops

        kw = dict(prob_bits=self.pb, archive_dtype=self.dt, sparse=self.sparse)
        if mode != "none":
            kw["scale"] = SCALE  # the device-scale call equals the host-scaled one (test_gpu_weighted_reduce_devscale)
        outs = [i.clone() if accumulate else torch.empty(n, device="cuda") for i, n in zip(inits, self.sizes)]
        ops.decompress_data_reduce(self.groups, outs, accumulate, **kw)
        return [o.to(self.dt) for o in outs]


@pytest.mark.parametrize("mode", ["none", "host", "dev"])
@pytest.mark.parametrize("pb", [9, 10, 11])
@pytest.mark.parametrize("t,sparse", [("f16", False), ("bf16", False), ("f16", True), ("bf16", True)],
                         ids=["f16", "bf16", "f16-sparse", "bf16-sparse"])
def test_equals_widening_then_to(t, sparse, pb, mode):
    for width in range(1, 10):
        case = Case(t, sparse, pb, width, seed=width)
        for accumulate in (False, True):
            inits = [_init(n, 7 * g + width) for g, n in enumerate(case.sizes)]
            want = case.reference(mode, accumulate, inits)
            acc = [i.clone() for i in inits] if accumulate else None
            flag = torch.zeros(1, device="cuda") if mode == "dev" else None
            st = torch.zeros(len(case.sizes) * width, dtype=torch.uint8, device="cuda")
            got = case.call(mode, accumulate, acc=acc, found_inf=flag, status=st)
            torch.cuda.synchronize()
            what = f"{t} sparse={sparse} pb={pb} {mode} W={width} accumulate={accumulate}"
            assert bool(st.all()), what
            for g, (a, b) in enumerate(zip(got, want)):
                _same(a, b, f"{what} group {g} ({case.sizes[g]} words)")
            if flag is not None:
                bad = any(bool((~torch.isfinite(o)).any()) for o in want if o.numel())
                assert float(flag) == (1.0 if bad else 0.0), what


@pytest.mark.parametrize("t,sparse", [("f16", False), ("bf16", True)])
def test_fp32_sum_that_rounds_to_inf_sets_the_flag(t, sparse):
    """A finite float32 sum whose 16-bit rounding is inf raises found_inf: the check sees the stored word."""
    from dietgpu_b200 import ops

    dt = DTYPES[t]
    top = 65504.0 if dt == torch.float16 else float(torch.finfo(torch.bfloat16).max)
    step = 16.0 if dt == torch.float16 else 2.0 ** 119  # half an ulp of the largest finite value
    xs = [torch.full((5000,), top, dtype=dt, device="cuda"), torch.zeros(5000, dtype=dt, device="cuda")]
    xs[1][1234] = step
    arch = _archives(xs, 10, sparse)
    out = torch.empty(5000, dtype=dt, device="cuda")
    flag = torch.zeros(1, device="cuda")
    ops.decompress_data_reduce([arch], [out], archive_dtype=dt, sparse=sparse, reduce_dtype=torch.float32,
                               scale_tensor=torch.ones(1, device="cuda"), found_inf=flag)
    wide = torch.empty(5000, device="cuda")
    ops.decompress_data_reduce([arch], [wide], archive_dtype=dt, sparse=sparse)
    assert bool(torch.isfinite(wide).all())
    assert bool(torch.isinf(out[1234])) and bool(torch.isfinite(out[:1234]).all())
    assert float(flag) == 1.0
    flag.zero_()
    xs[1][1234] = 0.0
    ops.decompress_data_reduce([_archives(xs, 10, sparse)], [out], archive_dtype=dt, sparse=sparse,
                               reduce_dtype=torch.float32, scale_tensor=torch.ones(1, device="cuda"), found_inf=flag)
    assert float(flag) == 0.0


@pytest.mark.parametrize("width", [1, 3, 6])
@pytest.mark.parametrize("t,sparse", [("bf16", False), ("f16", True)])
def test_invalid_archive_leaves_acc_and_out_untouched(t, sparse, width):
    from dietgpu_b200 import ops

    dt = DTYPES[t]
    sizes = [4097, 9000]
    case = Case(t, sparse, 10, width, sizes=sizes, seed=3)
    wrong = _archives([_words(dt, 4096, 5, 0).cuda()], 10, sparse)[0]  # 4096 words where the group holds 4097
    groups = [list(case.groups[0]), list(case.groups[1])]
    groups[0][width - 1] = wrong
    case.groups = groups
    for accumulate in (False, True):
        inits = [_init(n, 11) for n in sizes]
        acc = [i.clone() for i in inits]
        outs = [torch.full((n,), 7.0, dtype=dt, device="cuda") for n in sizes]
        st = torch.zeros(2 * width, dtype=torch.uint8, device="cuda")
        flag = torch.zeros(1, device="cuda")
        case.call("dev", accumulate, acc=acc, outs=outs, found_inf=flag, status=st)
        torch.cuda.synchronize()
        want_st = [1] * (2 * width)
        want_st[width - 1] = 0
        assert st.cpu().tolist() == want_st
        assert bool((outs[0] == 7.0).all()), "the invalid group's output was written"
        assert torch.equal(acc[0].view(torch.int32), inits[0].view(torch.int32)), "the invalid group's acc was written"
        # the valid group is summed as usual
        ref = Case.reference(case, "dev", accumulate, inits)
        _same(outs[1], ref[1], f"valid group, accumulate={accumulate}")


def test_single_archive_needs_no_accumulator():
    """W = 1 without accumulate stores round(term) without any float32 buffer, and a W > 1 call without acc takes a
    temporary: both equal the widening call followed by .to()."""
    for width in (1, 2, 5):
        case = Case("bf16", False, 11, width, sizes=[4097, 70001], seed=9)
        for mode in ("none", "host", "dev"):
            got = case.call(mode, False)
            want = case.reference(mode, False, [None, None])
            for a, b in zip(got, want):
                _same(a, b, f"W={width} {mode}")


def test_graph_replays_read_the_current_scale():
    from dietgpu_b200 import ops

    case = Case("f16", True, 10, 6, sizes=[4097, 70001], seed=4)
    sc = torch.full((1,), SCALE, device="cuda")
    flag = torch.zeros(1, device="cuda")
    acc = [torch.empty(n, device="cuda") for n in case.sizes]
    outs = [torch.empty(n, dtype=torch.float16, device="cuda") for n in case.sizes]
    temp = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):  # warm up outside the capture
        ops.decompress_data_reduce(case.groups, outs, False, temp, reduce_dtype=torch.float32, acc=acc,
                                   archive_dtype=torch.float16, sparse=True, scale_tensor=sc, found_inf=flag)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.decompress_data_reduce(case.groups, outs, False, temp, reduce_dtype=torch.float32, acc=acc,
                                   archive_dtype=torch.float16, sparse=True, scale_tensor=sc, found_inf=flag)
    for s in (0.25, -3.0, 1e30):
        sc.fill_(s)
        flag.zero_()
        for o in outs:
            o.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        want = []
        for g in case.groups:
            w = torch.empty(case.sizes[len(want)], device="cuda")
            ops.decompress_data_reduce([g], [w], archive_dtype=torch.float16, sparse=True, scale=s)
            want.append(w.to(torch.float16))
        for a, b in zip(outs, want):
            _same(a, b, f"replay with scale {s}")
        bad = any(bool((~torch.isfinite(w)).any()) for w in want)
        assert float(flag) == (1.0 if bad else 0.0), s
