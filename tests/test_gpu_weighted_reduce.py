"""Scaled decode-and-sum (ops.decompress_data_reduce(scale=), dgb_float_decompress_reduce_scaled) and averaging in
the compressed reduce-scatter and all-reduce.

Every case is compared with two references: torch's fold on the GPU, term(x) = (x.float() * s32).to(out dtype) with
s32 a float32 CUDA tensor and one torch add per archive (identical bits, or NaN against NaN), and the float64 fold of
tests/scaled_reference.py.  The archives are the corpora of test_gpu_reduce_edges.py (dense: blocks above the slot,
the 256 * probBits-word worst case, empty streams, full-range words with NaN, +-inf and subnormals) and of
test_gpu_reduce_sparse.py (sparse: ReLU, all +-0, +-0 in every pairing, zero and nonzero blocks, NaN / +-inf /
subnormals among zeros), so both stream branches of decodeReduceBlock run under every scaled writer, and the
scales 3 and 2^15 overflow words that are finite unscaled.  Outputs sit in guard-banded buffers.

The module's name sorts after every other GPU module, so in a single-process run of the suite it runs last.  The
profiler checks of the other modules (test_gpu_reduce*.py, test_gpu_sparse*.py, ...) find their kernels in
torch.profiler's trace, and the profiler drops GPU records whose timestamps have drifted outside its capture window;
that drift grows with the age of the process, and after minutes of GPU work it drops the first records of a
session.  A module of this length run ahead of them would shift their sessions minutes later and make them miss
launches."""
import re
import time

import numpy as np
import pytest
import torch

from codec_helpers import assert_guard_intact, codec_options, guarded_out
from multirank import NAME, host_words, rank_data, run_ranks
from reduce_reference import assert_same_words
from scaled_reference import SCALES, scaled_fold_ref
import test_gpu_reduce_edges as E
import test_gpu_reduce_sparse as S

pytestmark = pytest.mark.gpu

TORCH = {"f16": torch.float16, "bf16": torch.bfloat16, "f32": torch.float32}
PAIRS = [("f16", "f16"), ("bf16", "bf16"), ("f32", "f32"), ("f16", "f32"), ("bf16", "f32")]
CASES = [(at, ot, sp) for sp in (False, True) for at, ot in PAIRS]
CASE_IDS = [f"{'sparse-' if sp else ''}{at}-{ot}" for at, ot, sp in CASES]
WIDTHS = [1, 2, 4, 5, 9]
SOME = [float(np.float32(1 / 3)), -0.25, 2.0 ** 15]  # the scales every width runs (W = 5 runs all of SCALES)


def kernel_kind(at, ot, sparse):
    k = ({"f16": 5, "bf16": 6, "f32": 8} if sparse else {"f16": 1, "bf16": 2, "f32": 3})[at]
    return k | (0x20 if ot != at else 0) | 0x80


def _it_of(x):
    return torch.int32 if x.element_size() == 4 else torch.int16


def same_dev(got, want):
    """Per element on the device: identical bits, or both NaN."""
    return (got.view(_it_of(got)) == want.view(_it_of(want))) | (torch.isnan(got) & torch.isnan(want))


def torch_fold(xs, ot, s, init=None):
    """torch's scaled fold on the GPU: acc = term(x_0) (or init, unscaled); acc = acc + term(x_j)."""
    s32 = torch.tensor(s, dtype=torch.float32, device="cuda")
    T = TORCH[ot]
    acc = init.clone() if init is not None else (xs[0].float() * s32).to(T)
    for x in (xs if init is not None else xs[1:]):
        acc = acc + (x.float() * s32).to(T)
    return acc


# ---- corpus: the dense and the sparse decode-and-sum corpora --------------------------------------------------------

_DEV = {}


def corpus(at, pb, sparse):
    """(sizes, {(g, j): archive}, {(g, j): host words}, {(g, j): device words}, block check, dense archives)."""
    if sparse:
        arch, words, sizes = S.archives(at, pb), S.corpus(at), S.SIZES
        archives = {k: v[0] for k, v in arch.items()}
        dense = {k: v[1] for k, v in arch.items()}
        blocks = {k: v[2] for k, v in arch.items()}
    else:
        arch, words, sizes = E.library_archives(at, pb), E.corpus(at), E.SIZES
        archives = {k: v[0] for k, v in arch.items()}
        dense = None
        blocks = {k: v[1] for k, v in arch.items()}
    key = (at, sparse)
    if key not in _DEV:
        _DEV.clear()
        _DEV[key] = {k: E.device_words(w, at) for k, w in words.items()}
    return sizes, archives, words, _DEV[key], blocks, dense


def check_branches(at, pb, sparse, sizes, blocks, w, accumulate, what):
    """Dense: the blocks of this call's store and of its add writer each reach both stream branches, the worst case
    and empty streams (test_gpu_reduce_edges.py); sparse: the call's blocks reach both stream branches
    (test_gpu_reduce_sparse.py)."""
    gs = [g for g, n in enumerate(sizes) if n > 0]
    if sparse:
        S.assert_both_branches([blocks[g, j] for g in gs for j in range(w)], S.DEFAULT_SLOT, what)
        return
    store = [] if accumulate else [blocks[g, 0] for g in gs]
    add = [blocks[g, j] for g in gs for j in range(0 if accumulate else 1, w)]
    for kind, bws in (("store", store), ("add", add)):
        if not bws:
            continue
        E.assert_paths_covered(bws, pb, f"{what} {kind} writer")


def scaled_sum(at, ot, pb, sparse, groups, sizes, s, accumulate, inits, what, status_ok=True):
    """One scaled call into fresh guard-banded outputs; returns (outputs, buffers, spans)."""
    from dietgpu_b200 import ops

    bufs, outs, spans = [], [], []
    for g, n in enumerate(sizes):
        b, v, span = guarded_out(n, TORCH[ot], (3 * g + 1) % 8)
        if accumulate:
            v.copy_(inits[g])
        bufs.append(b)
        outs.append(v)
        spans.append(span)
    st = torch.zeros(sum(len(grp) for grp in groups), dtype=torch.uint8, device="cuda")
    ops.decompress_data_reduce(groups, outs, accumulate, None, st, prob_bits=pb, archive_dtype=TORCH[at],
                               sparse=sparse, scale=s)
    torch.cuda.synchronize()
    if status_ok:
        assert bool(st.all()), f"{what}: status {st.cpu().tolist()}"
    for g in range(len(sizes)):
        assert_guard_intact(bufs[g], *spans[g], f"{what} group {g}")
    return outs, bufs


def _inits(ot, sizes, seed):
    return [E.device_words(E.init_words(ot, n, seed + g), ot) for g, n in enumerate(sizes)]


@pytest.mark.parametrize("pb", [9, 10, 11])
@pytest.mark.parametrize("at,ot,sparse", CASES, ids=CASE_IDS)
def test_corpus(at, ot, sparse, pb):
    """Every width, with and without accumulate, against torch's GPU fold; W = 5 at every scale of SCALES, also
    against the float64 fold.  s = 1 equals the unscaled call, and sparse archives equal dense ones of the same
    words (s < 0 included, where elided +0 words turn into -0)."""
    sizes, arch, words, dev, blocks, dense = corpus(at, pb, sparse)
    G = range(len(sizes))
    for accumulate in (False, True):
        inits = _inits(ot, sizes, 7 * pb) if accumulate else [None] * len(sizes)
        for w in WIDTHS:
            what = f"{at}->{ot} sparse {sparse} pb {pb} acc {accumulate} W {w}"
            check_branches(at, pb, sparse, sizes, blocks, w, accumulate, what)
            groups = [[arch[g, j] for j in range(w)] for g in G]
            for s in (SCALES if w == 5 else SOME):
                outs, bufs = scaled_sum(at, ot, pb, sparse, groups, sizes, s, accumulate, inits, f"{what} s {s}")
                for g in G:
                    want = torch_fold([dev[g, j] for j in range(w)], ot, s, inits[g])
                    ok = same_dev(outs[g], want)
                    assert bool(ok.all()), f"{what} s {s} group {g}: {int((~ok).sum())} element(s) differ from torch"
                    if w == 5:
                        init_h = E.to_host_words(inits[g], ot) if accumulate else None
                        assert_same_words(E.to_host_words(outs[g], ot),
                                          scaled_fold_ref([words[g, j] for j in range(w)], at, ot, s, init_h),
                                          ot, f"{what} s {s} group {g} (float64)")
                if sparse and (w == 5 or s < 0):
                    dgroups = [[dense[g, j] for j in range(w)] for g in G]
                    _, dbufs = scaled_sum(at, ot, pb, False, dgroups, sizes, s, accumulate, inits,
                                          f"{what} s {s} dense")
                    for g in G:
                        assert torch.equal(bufs[g], dbufs[g]), f"{what} s {s} group {g}: sparse != dense"
            if w in (5, 9):
                from dietgpu_b200 import ops

                _, one = scaled_sum(at, ot, pb, sparse, groups, sizes, 1.0, accumulate, inits, f"{what} s 1")
                plain = []
                for g, n in enumerate(sizes):
                    b, v, _ = guarded_out(n, TORCH[ot], (3 * g + 1) % 8)
                    if accumulate:
                        v.copy_(inits[g])
                    plain.append((b, v))
                ops.decompress_data_reduce(groups, [v for _, v in plain], accumulate, prob_bits=pb,
                                           archive_dtype=TORCH[at], sparse=sparse)
                torch.cuda.synchronize()
                for g in G:
                    assert torch.equal(one[g], plain[g][0]), f"{what} group {g}: scale 1 != the unscaled call"


MODES = {"slot8": dict(decode_slot_words=1), "slot_max": dict(decode_slot_words=4096),
         "inline0": dict(inline_members=0)}


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("at,ot,sparse", CASES, ids=CASE_IDS)
def test_forced_slots_and_scratch_tables(at, ot, sparse, mode):
    """The slot forced to 8 words (every non-empty block from global memory) and to the worst case (every block
    staged), and member tables read from scratch, under the scaled store and add writers, across the 4-archive
    pass."""
    pb = 10
    sizes, arch, words, dev, _, _ = corpus(at, pb, sparse)
    G = range(len(sizes))
    for accumulate in (False, True):
        inits = _inits(ot, sizes, 3) if accumulate else [None] * len(sizes)
        for w in (5, 9):
            groups = [[arch[g, j] for j in range(w)] for g in G]
            for s in SOME:
                what = f"{at}->{ot} sparse {sparse} {mode} acc {accumulate} W {w} s {s}"
                with codec_options(**MODES[mode]):
                    outs, _ = scaled_sum(at, ot, pb, sparse, groups, sizes, s, accumulate, inits, what)
                for g in G:
                    ok = same_dev(outs[g], torch_fold([dev[g, j] for j in range(w)], ot, s, inits[g]))
                    assert bool(ok.all()), f"{what} group {g}"


def test_invalid_archive_leaves_the_group_unwritten():
    from dietgpu_b200 import ops

    sizes, arch, _, _, _, _ = corpus("bf16", 10, False)
    g = 6  # 4097 elements
    good = [arch[g, j] for j in range(3)]
    wrong = arch[g + 1, 0]  # another word count
    b, v, span = guarded_out(sizes[g], torch.bfloat16, 1)
    before = b.clone()
    st = torch.full((3,), 7, dtype=torch.uint8, device="cuda")
    ops.decompress_data_reduce([[good[0], wrong, good[2]]], [v], False, None, st, scale=0.5)
    torch.cuda.synchronize()
    assert st.cpu().tolist() == [1, 0, 1]
    assert torch.equal(b, before)


# ---- every new kernel runs -----------------------------------------------------------------------------------------

def test_profiler_sees_every_instantiation():
    # in a fresh process: in a long-lived one the GPU's timestamps drift against the host clock that bounds the
    # profiler's window, and every record of a window can fall outside it
    run_ranks(_profiler_sees_every_instantiation, 1, backend="gloo")


def _profiler_sees_every_instantiation(rank, world, dev):
    from torch.profiler import ProfilerActivity, profile

    from dietgpu_b200 import ops

    work = []
    for at, ot, sp in CASES:
        for pb in (9, 10, 11):
            dev = [E.device_words(S.shape_words(at, "relu", 5000, 11 + j), at) for j in range(2)]
            work.append(([S.compress(dev, pb, sp)], [torch.empty(5000, dtype=TORCH[ot], device="cuda")], at, pb, sp))
    torch.cuda.synchronize()
    # The profiler drops GPU records whose timestamps fall outside its capture window, and in a long-lived process the
    # GPU timestamps drift by milliseconds against the host clock (the profiler's own log counts them as
    # "Out-of-range").  The launches therefore start well after the window opens and end well before it closes.
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(1.0)
        torch.ones(1, device="cuda").add_(1)  # the first kernel of a session can be missing from its trace
        for _ in range(3):
            for ins, outs, at, pb, sp in work:
                ops.decompress_data_reduce(ins, outs, prob_bits=pb, archive_dtype=TORCH[at], sparse=sp, scale=0.5)
        torch.cuda.synchronize()
        time.sleep(1.0)
    names = {re.sub(r"\s", "", e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    kinds = sorted({kernel_kind(at, ot, sp) for at, ot, sp in CASES})
    assert kinds == [129, 130, 131, 133, 134, 136, 161, 162, 165, 166]
    for kind in kinds:
        for pb in (9, 10, 11):
            assert any(f"decodeReduceKernel<{kind},{pb}>" in k for k in names), (kind, pb, sorted(names))


# ---- CUDA graphs ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("at,ot,sparse", [("bf16", "bf16", False), ("f16", "f32", False), ("f32", "f32", True),
                                          ("bf16", "f32", True)], ids=["bf16", "f16-f32", "sparse-f32", "sparse-bf16-f32"])
def test_graph_capture_replays_the_captured_scale(at, ot, sparse):
    """A scaled call captured on a side stream replays on the current stream after the work queued in front of it
    (new archives copied into the captured rows, the outputs reset), with the scale it was captured with, even after
    an eager call with another scale."""
    from dietgpu_b200 import ops

    groups, width, n = 3, 6, 70001
    s_cap = float(np.float32(1 / 7))
    cols = int(ops.max_float_compressed_size(torch.empty(0, dtype=TORCH[at]), n)) + 64
    rows = torch.zeros(groups * width, cols, dtype=torch.uint8, device="cuda")

    def load(seed):
        xs = [E.device_words(S.shape_words(at, S.SHAPES[(seed + k) % len(S.SHAPES)], n, seed + k, k), at)
              for k in range(groups * width)]
        arch = S.compress(xs, 10, sparse)
        big = torch.randn(4096, 4096, device="cuda")
        big = big @ big  # work in front of the copies, on the same stream
        for i, a in enumerate(arch):
            rows[i, :a.numel()].copy_(a)
        return [xs[g * width:(g + 1) * width] for g in range(groups)]

    load(1)
    ins = [[rows[g * width + j, :cols] for j in range(width)] for g in range(groups)]
    init = [E.device_words(E.init_words(ot, n, 5 + g), ot) for g in range(groups)]
    outs = [torch.empty(n, dtype=TORCH[ot], device="cuda") for _ in range(groups)]
    st = torch.zeros(groups * width, dtype=torch.uint8, device="cuda")
    scratch = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.decompress_data_reduce(ins, outs, True, scratch, st, archive_dtype=TORCH[at], sparse=sparse,
                                   scale=s_cap)  # warm-up
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        ops.decompress_data_reduce(ins, outs, True, scratch, st, archive_dtype=TORCH[at], sparse=sparse, scale=s_cap)
    other = [torch.empty(n, dtype=TORCH[ot], device="cuda") for _ in range(groups)]
    for seed in (2, 3):
        xs = load(seed * 1000)  # new archives in the captured rows
        ops.decompress_data_reduce(ins, other, False, archive_dtype=TORCH[at], sparse=sparse, scale=3.0)
        for o, i in zip(outs, init):
            o.copy_(i)
        st.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert bool(st.all()), f"replay {seed}: status"
        for g in range(groups):
            ok = same_dev(outs[g], torch_fold(xs[g], ot, s_cap, init[g]))
            assert bool(ok.all()), f"replay seed {seed} group {g}"
            ok = same_dev(other[g], torch_fold(xs[g], ot, 3.0))
            assert bool(ok.all()), f"eager call between replays, seed {seed} group {g}"


# ---- collectives ----------------------------------------------------------------------------------------------------

def _term(x, acc, s):
    return (x.float() * torch.tensor(s, dtype=torch.float32, device=x.device)).to(acc)


def _worker(rank, world, dev):
    import dietgpu_b200 as dg

    done = []

    def check(got, ts_arch, acc, s, what):
        """got == the rank-order fold of term(t_r) (torch on the GPU and float64), t_r in the archive dtype."""
        want = _term(ts_arch[0].to(dev), acc, s)
        for x in ts_arch[1:]:
            want = want + _term(x.to(dev), acc, s)
        assert bool(same_dev(got, want).all()), f"{what}: differs from torch's fold"
        assert_same_words(host_words(got), scaled_fold_ref([host_words(x) for x in ts_arch],
                                                            NAME[ts_arch[0].dtype], NAME[acc], s),
                          NAME[acc], f"{what} (float64)")
        done.append(what)

    avg = float(np.float32(1 / world))
    for dt in (torch.float16, torch.bfloat16, torch.float32):
        variants = [(None, None)] + ([(torch.float32, None)] if dt != torch.float32 else
                                     [(None, torch.bfloat16), (None, torch.float16)])
        for reduce_dtype, wire in variants:
            for sparse in ((False, True) if wire is None else (False,)):
                for how in ("average", "scale"):
                    kw = dict(average=True) if how == "average" else dict(scale=-0.3)
                    s = avg if how == "average" else -0.3
                    tag = f"{dt} reduce {reduce_dtype} wire {wire} sparse {sparse} {how}"
                    widened = reduce_dtype is not None
                    n = world * 12289 if world > 1 else 12289
                    ts = rank_data(dt, n, world, 500 + len(done), widened=widened)
                    acc = torch.float32 if (widened or wire is not None) else dt
                    arch_dt = wire or dt
                    got = dg.reduce_scatter_compressed(ts[rank].to(dev), members=3, reduce_dtype=reduce_dtype,
                                                       wire_dtype=wire, sparse=sparse, **kw)
                    lo, hi = rank * (n // world), (rank + 1) * (n // world)
                    check(got, [t[lo:hi].to(arch_dt) for t in ts], acc, s, f"reduce_scatter {tag}")
                    if wire is None:
                        for m in (1, 30001):
                            tm = rank_data(dt, m, world, 900 + m, widened=widened)
                            got = dg.all_reduce_compressed(tm[rank].to(dev), members=3, reduce_dtype=reduce_dtype,
                                                           sparse=sparse, **kw)
                            check(got, tm, acc, s, f"all_reduce {tag} n {m}")
                            if dt == torch.float16 and how == "average" and world > 1 and not widened:
                                # element 5 of every 16 is max, max, -max, ...: the rank-order fp16 sum
                                # overflows to inf, the average does not
                                k5 = got.view(-1)[5::16]
                                assert bool(torch.isfinite(k5).all()), f"{tag}: the average overflowed"
                                plain = dg.all_reduce_compressed(tm[rank].to(dev), members=3)
                                assert bool(torch.isinf(plain.view(-1)[5::16]).all()), f"{tag}: plain sum"
    return len(done)


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_scaled_collectives(world):
    run_ranks(_worker, world, backend="gloo", timeout=600)
