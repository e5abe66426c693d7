"""Device-scale decode-and-sum (ops.decompress_data_reduce(scale_tensor=, found_inf=),
dgb_float_decompress_reduce_scaled_dev) and the scale_tensor / found_inf keywords of the compressed reduce-scatter
and all-reduce.

Every output is compared bit for bit with the host-scaled call (scale=float(s)) on the same archives and inits, in
guard-banded buffers, and with the float64 fold of tests/scaled_reference.py; every flag is compared with torch's
isfinite over the elements the call wrote.  The corpora are those of test_gpu_weighted_reduce.py, which reach both
stream branches of decodeReduceBlock under every writer and hold NaN, +-inf and words that overflow when scaled.
Crafted archives place one inf or NaN at the first element, at the last element of a partial row, in the last block,
in archive 0, a middle archive or the last one, and only in the accumulated init; NaN-filled guard bands, partial rows
and groups left unwritten around finite sums must not set the flag.

The module's name sorts after test_gpu_weighted_reduce.py, so in a single-process run of the suite it runs after every
other GPU module that reads torch.profiler's trace; its own profiler check comes first in the module.  The profiler
drops GPU records whose timestamps have drifted outside its capture window, the drift grows with the age of the
process, and this module's minutes of GPU work run ahead of a check without wide margins around its window would
make that check miss launches (test_gpu_weighted_reduce.py)."""
import re
import time

import numpy as np
import pytest
import torch

from codec_helpers import assert_guard_intact, codec_options, guarded_out
from multirank import rank_data, run_ranks
from reduce_reference import assert_same_words
from scaled_reference import SCALES, scaled_fold_ref
import test_gpu_reduce_edges as E
import test_gpu_reduce_sparse as S
import test_gpu_weighted_reduce as W

pytestmark = pytest.mark.gpu

TORCH = W.TORCH
CASES, CASE_IDS = W.CASES, W.CASE_IDS
WIDTHS = [1, 2, 4, 5, 9]
NAN_BYTE = 0xFF  # 0xFFFF and 0xFFFFFFFF are NaN in fp16, bf16 and fp32


def _flag(v=0.0):
    return torch.full((1,), v, dtype=torch.float32, device="cuda")


def _scale(s):
    return torch.tensor([s], dtype=torch.float32, device="cuda")


def _bufs(sizes, ot, inits, accumulate):
    bufs, outs, spans = [], [], []
    for g, n in enumerate(sizes):
        b, v, span = guarded_out(n, TORCH[ot], (3 * g + 1) % 8)
        if accumulate:
            v.copy_(inits[g])
        bufs.append(b)
        outs.append(v)
        spans.append(span)
    return bufs, outs, spans


def dev_sum(at, ot, pb, sparse, groups, sizes, s, accumulate, inits, what, flag=0.0, with_flag=True):
    """One device-scale call into fresh guard-banded outputs; returns (outputs, buffers, flag value or None)."""
    from dietgpu_b200 import ops

    bufs, outs, spans = _bufs(sizes, ot, inits, accumulate)
    st = torch.zeros(sum(len(grp) for grp in groups), dtype=torch.uint8, device="cuda")
    fi = _flag(flag) if with_flag else None
    ops.decompress_data_reduce(groups, outs, accumulate, None, st, prob_bits=pb, archive_dtype=TORCH[at],
                               sparse=sparse, scale_tensor=_scale(s), found_inf=fi)
    torch.cuda.synchronize()
    assert bool(st.all()), f"{what}: status {st.cpu().tolist()}"
    for g in range(len(sizes)):
        assert_guard_intact(bufs[g], *spans[g], f"{what} group {g}")
    return outs, bufs, (float(fi.item()) if with_flag else None)


def non_finite(outs):
    return any(bool((~torch.isfinite(o)).any()) for o in outs if o.numel())


# ---- every new kernel runs, and no host-scaled one on this path -----------------------------------------------------

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
    sc, fi = _scale(0.5), _flag()
    torch.cuda.synchronize()
    # launches start well after the profiler's window opens and end well before it closes (test_gpu_weighted_reduce)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(1.0)
        torch.ones(1, device="cuda").add_(1)  # the first kernel of a session can be missing from its trace
        for _ in range(3):
            for ins, outs, at, pb, sp in work:
                ops.decompress_data_reduce(ins, outs, prob_bits=pb, archive_dtype=TORCH[at], sparse=sp,
                                           scale_tensor=sc, found_inf=fi)
        torch.cuda.synchronize()
        time.sleep(1.0)
    names = {re.sub(r"\s", "", e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    kinds = sorted({W.kernel_kind(at, ot, sp) | 0x100 for at, ot, sp in CASES})
    assert kinds == [385, 386, 387, 389, 390, 392, 417, 418, 421, 422]
    for kind in kinds:
        for pb in (9, 10, 11):
            assert any(f"decodeReduceDevScaleKernel<{kind},{pb}>" in k for k in names), (kind, pb, sorted(names))
    assert not any("decodeReduceKernel<" in k for k in names), sorted(names)


# ---- equivalence with the host-scaled call --------------------------------------------------------------------------

@pytest.mark.parametrize("pb", [9, 10, 11])
@pytest.mark.parametrize("at,ot,sparse", CASES, ids=CASE_IDS)
def test_corpus_equals_the_host_scaled_call(at, ot, sparse, pb):
    """Every width, with and without accumulate, at every scale of SCALES: the outputs equal the host-scaled call's
    bytes (guard bands included) and the float64 fold, and the flag is set exactly when an output is inf or NaN."""
    sizes, arch, words, _, blocks, _ = W.corpus(at, pb, sparse)
    G = range(len(sizes))
    for accumulate in (False, True):
        inits = W._inits(ot, sizes, 7 * pb) if accumulate else [None] * len(sizes)
        init_h = [E.to_host_words(i, ot) for i in inits] if accumulate else [None] * len(sizes)
        for w in WIDTHS:
            what = f"{at}->{ot} sparse {sparse} pb {pb} acc {accumulate} W {w}"
            W.check_branches(at, pb, sparse, sizes, blocks, w, accumulate, what)
            groups = [[arch[g, j] for j in range(w)] for g in G]
            for s in SCALES:
                outs, bufs, fl = dev_sum(at, ot, pb, sparse, groups, sizes, s, accumulate, inits, f"{what} s {s}")
                _, hbufs = W.scaled_sum(at, ot, pb, sparse, groups, sizes, s, accumulate, inits, f"{what} s {s} host")
                for g in G:
                    assert torch.equal(bufs[g], hbufs[g]), f"{what} s {s} group {g}: != the host-scaled call"
                    assert_same_words(E.to_host_words(outs[g], ot),
                                      scaled_fold_ref([words[g, j] for j in range(w)], at, ot, s, init_h[g]),
                                      ot, f"{what} s {s} group {g} (float64)")
                assert fl == (1.0 if non_finite(outs) else 0.0), f"{what} s {s}: flag {fl}"


@pytest.mark.parametrize("mode", list(W.MODES))
@pytest.mark.parametrize("at,ot,sparse", CASES, ids=CASE_IDS)
def test_forced_slots_and_scratch_tables(at, ot, sparse, mode):
    pb = 10
    sizes, arch, _, _, _, _ = W.corpus(at, pb, sparse)
    G = range(len(sizes))
    for accumulate in (False, True):
        inits = W._inits(ot, sizes, 3) if accumulate else [None] * len(sizes)
        for w in (1, 5, 9):
            groups = [[arch[g, j] for j in range(w)] for g in G]
            for s in W.SOME + [float("inf")]:
                what = f"{at}->{ot} sparse {sparse} {mode} acc {accumulate} W {w} s {s}"
                with codec_options(**W.MODES[mode]):
                    outs, bufs, fl = dev_sum(at, ot, pb, sparse, groups, sizes, s, accumulate, inits, what)
                    _, hbufs = W.scaled_sum(at, ot, pb, sparse, groups, sizes, s, accumulate, inits, what)
                for g in G:
                    assert torch.equal(bufs[g], hbufs[g]), f"{what} group {g}"
                assert fl == (1.0 if non_finite(outs) else 0.0), f"{what}: flag {fl}"


# ---- the flag on crafted archives -----------------------------------------------------------------------------------

N = 2 * 4096 + 45  # three blocks, the last ending in a partial row
SPECIAL = {"f16": {"inf": 0x7C00, "nan": 0x7E00, "max": 0x7BFF},
           "bf16": {"inf": 0x7F80, "nan": 0x7FC0, "max": 0x7F7F},
           "f32": {"inf": 0x7F800000, "nan": 0x7FC00000, "max": 0x7F7FFFFF}}
SPOTS = {"first": 0, "last": N - 1, "last_block": 2 * 4096 + 3}
FLAG_CASES = [("bf16", "bf16", False), ("f16", "f16", False), ("f32", "f32", False), ("f16", "f32", False),
              ("bf16", "bf16", True), ("f32", "f32", True), ("bf16", "f32", True)]
FLAG_IDS = [f"{'sparse-' if sp else ''}{a}-{o}" for a, o, sp in FLAG_CASES]


def _finite_words(t, n, seed, zeros=False):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(n).astype(np.float32)
    if zeros:
        x[rng.random(n) < 0.5] = 0.0
        x[1::9] = -0.0
    return torch.from_numpy(x).to(TORCH[t]).view(torch.int32 if t == "f32" else torch.int16).numpy().view(
        E.WORD[t]).copy()


def _archives(at, words, sparse, pb=10):
    xs = [E.device_words(w, at) for w in words]
    return S.compress(xs, pb, sparse)


def _dev_and_host(at, ot, sparse, words, s, init=None, flag=0.0, n=N):
    """Device-scale call with a flag (and without one) against the host-scaled call; returns the flag."""
    arch = _archives(at, words, sparse)
    acc = init is not None
    inits = [E.device_words(init, ot)] if acc else [None]
    what = f"{at}->{ot} sparse {sparse} W {len(words)} s {s}"
    outs, bufs, fl = dev_sum(at, ot, 10, sparse, [arch], [n], s, acc, inits, what, flag=flag)
    _, nbufs, _ = dev_sum(at, ot, 10, sparse, [arch], [n], s, acc, inits, what, with_flag=False)
    _, hbufs = W.scaled_sum(at, ot, 10, sparse, [arch], [n], s, acc, inits, what)
    assert torch.equal(bufs[0], hbufs[0]), f"{what}: != the host-scaled call"
    assert torch.equal(bufs[0], nbufs[0]), f"{what}: found_inf=None changed the output"
    return fl


@pytest.mark.parametrize("at,ot,sparse", FLAG_CASES, ids=FLAG_IDS)
def test_finite_sums_leave_the_flag(at, ot, sparse):
    for w in (1, 4, 9):
        words = [_finite_words(at, N, 10 * w + j, zeros=sparse) for j in range(w)]
        for s in (1.0, -0.25, 0.0):
            assert _dev_and_host(at, ot, sparse, words, s) == 0.0, (w, s)
            assert _dev_and_host(at, ot, sparse, words, s, flag=1.0) == 1.0, (w, s)  # never cleared
        init = _finite_words(ot, N, 99)
        assert _dev_and_host(at, ot, sparse, words, 0.5, init=init) == 0.0


@pytest.mark.parametrize("at,ot,sparse", FLAG_CASES, ids=FLAG_IDS)
def test_one_non_finite_word_sets_the_flag(at, ot, sparse):
    for w in (1, 3, 9):
        for j in sorted({0, w // 2, w - 1}):  # archive 0 (the first pass of W = 9), a middle one, the last one
            for spot, i in SPOTS.items():
                for kind in ("inf", "nan"):
                    words = [_finite_words(at, N, 10 * w + k, zeros=sparse) for k in range(w)]
                    words[j][i] = SPECIAL[at][kind]
                    fl = _dev_and_host(at, ot, sparse, words, 0.5)
                    assert fl == 1.0, f"W {w} archive {j} {spot} {kind}: flag {fl}"


@pytest.mark.parametrize("at,ot,sparse", FLAG_CASES, ids=FLAG_IDS)
def test_non_finite_terms_set_the_flag(at, ot, sparse):
    w = 3
    base = [_finite_words(at, N, 40 + k, zeros=sparse) for k in range(w)]
    # only the accumulated init
    for spot, i in SPOTS.items():
        init = _finite_words(ot, N, 7)
        init[i] = SPECIAL[ot]["nan"]
        assert _dev_and_host(at, ot, sparse, base, 0.5, init=init) == 1.0, f"init {spot}"
    # inf * 0, and an infinite or NaN scale on finite words
    words = [b.copy() for b in base]
    words[1][SPOTS["last"]] = SPECIAL[at]["inf"]
    assert _dev_and_host(at, ot, sparse, words, 0.0) == 1.0, "inf * 0"
    for s in (float("inf"), float("-inf"), float("nan")):
        assert _dev_and_host(at, ot, sparse, base, s) == 1.0, f"scale {s}"
    # a fold that overflows: max + max in the 16-bit type (and, widened or fp32, max * 3 in fp32)
    words = [b.copy() for b in base]
    words[0][SPOTS["last_block"]] = SPECIAL[at]["max"]
    words[1][SPOTS["last_block"]] = SPECIAL[at]["max"]
    s = 1.0 if ot != "f32" or at == "f32" else 2.0 ** 127
    assert _dev_and_host(at, ot, sparse, words, s) == 1.0, "overflow"
    if sparse:  # an elided +-0 times an infinite scale is NaN
        zeros = [np.zeros(N, E.WORD[at]) for _ in range(w)]
        zeros[1][::3] = 0x8000 if at != "f32" else 0x80000000
        assert _dev_and_host(at, ot, sparse, zeros, float("inf")) == 1.0, "0 * inf"
        assert _dev_and_host(at, ot, sparse, zeros, 1.0) == 0.0, "0 * 1"


def test_fp16_max_plus_max():
    words = [np.full(N, 0x7BFF, np.uint16), np.full(N, 0x7BFF, np.uint16)]  # 65504 + 65504 = inf in fp16
    assert _dev_and_host("f16", "f16", False, words, 1.0) == 1.0
    assert _dev_and_host("f16", "f32", False, words, 1.0) == 0.0  # 131008 in fp32
    assert _dev_and_host("f16", "f16", True, words, 1.0) == 1.0


@pytest.mark.parametrize("at,ot,sparse", FLAG_CASES, ids=FLAG_IDS)
def test_unwritten_elements_do_not_count(at, ot, sparse):
    """Finite sums in NaN-filled buffers: outputs that end mid-row, and a group left unwritten because one of its
    archives is invalid, next to the written one in the same buffer, keep the flag at 0."""
    from dietgpu_b200 import ops

    w = 3
    for n in (N, 45, 4096 + 1):
        words = [_finite_words(at, n, 70 + k, zeros=sparse) for k in range(w)]
        good = _archives(at, words, sparse)
        wrong = _archives(at, [_finite_words(at, n + 8, 3, zeros=sparse)], sparse)[0]  # another word count
        es = torch.empty(0, dtype=TORCH[ot]).element_size()
        buf = torch.full(((2 * n + 4096) * es,), NAN_BYTE, dtype=torch.uint8, device="cuda")
        v = buf.view(TORCH[ot])
        o0, o1 = v[2048:2048 + n], v[2048 + n:2048 + 2 * n]  # adjacent outputs
        st = torch.zeros(2 * w, dtype=torch.uint8, device="cuda")
        fi = _flag()
        ops.decompress_data_reduce([good, [good[0], wrong, good[2]]], [o0, o1], False, None, st,
                                   archive_dtype=TORCH[at], sparse=sparse, scale_tensor=_scale(0.5), found_inf=fi)
        torch.cuda.synchronize()
        assert st.cpu().tolist() == [1] * w + [1, 0, 1]
        assert bool(torch.isnan(o1).all()), f"n {n}: the invalid group was written"
        assert bool(torch.isfinite(o0).all())
        assert float(fi.item()) == 0.0, f"n {n}: unwritten NaN words set the flag"
        head, tail = buf[:2048 * es], buf[(2048 + 2 * n) * es:]
        assert bool((head == NAN_BYTE).all()) and bool((tail == NAN_BYTE).all())


def test_no_groups_leaves_everything():
    from dietgpu_b200 import capi

    fi = _flag(0.25)
    rc = capi.lib().dgb_float_decompress_reduce_scaled_dev(None, 0, capi.BFLOAT16, capi.BFLOAT16, 10, 0, 1, None,
                                                           None, None, 0, _scale(2.0).data_ptr(), fi.data_ptr(),
                                                           None, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert rc == capi.OK and float(fi.item()) == 0.25


# ---- CUDA graphs: a replay reads the scale's current value ----------------------------------------------------------

@pytest.mark.parametrize("groups", [6, 130])
@pytest.mark.parametrize("at,ot,sparse", [("bf16", "bf16", False), ("f16", "f32", False), ("f32", "f32", True),
                                          ("bf16", "f32", True)], ids=["bf16", "f16-f32", "sparse-f32",
                                                                       "sparse-bf16-f32"])
def test_graph_replays_read_the_current_scale(at, ot, sparse, groups):
    """Captured with W = 2 (6 groups: member table in the kernel parameters; 130: in scratch).  Between replays the
    scale is rewritten with fill_ and by a kernel on the same stream, the flag is reset, and each replay equals the
    host-scaled call with the new value; its flag follows that replay's result."""
    from dietgpu_b200 import ops

    width, n = 2, 5003
    xs = [E.device_words(_finite_words(at, n, 500 + k, zeros=sparse), at) for k in range(groups * width)]
    arch = S.compress(xs, 10, sparse)
    ins = [[arch[g * width + j] for j in range(width)] for g in range(groups)]
    outs = [torch.empty(n, dtype=TORCH[ot], device="cuda") for _ in range(groups)]
    st = torch.zeros(groups * width, dtype=torch.uint8, device="cuda")
    scratch = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    sc, fi = _scale(0.5), _flag()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.decompress_data_reduce(ins, outs, False, scratch, st, archive_dtype=TORCH[at], sparse=sparse,
                                   scale_tensor=sc, found_inf=fi)  # warm-up
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        ops.decompress_data_reduce(ins, outs, False, scratch, st, archive_dtype=TORCH[at], sparse=sparse,
                                   scale_tensor=sc, found_inf=fi)
    num, den = _scale(3.0), _scale(7.0)
    for how, s in (("fill", 0.25), ("kernel", float(np.float32(3.0) / np.float32(7.0))), ("fill", float("inf")),
                   ("fill", -2.0), ("kernel", float(np.float32(3.0) / np.float32(7.0)))):
        if how == "fill":
            sc.fill_(s)
        else:
            big = torch.randn(2048, 2048, device="cuda")
            big = big @ big  # work in front of the rewrite, on the same stream
            torch.div(num, den, out=sc)
        fi.zero_()
        st.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert bool(st.all()), f"replay {how} {s}: status"
        want = [torch.empty(n, dtype=TORCH[ot], device="cuda") for _ in range(groups)]
        ops.decompress_data_reduce(ins, want, False, archive_dtype=TORCH[at], sparse=sparse, scale=s)
        torch.cuda.synchronize()
        for g in range(groups):
            assert torch.equal(outs[g].view(W._it_of(outs[g])), want[g].view(W._it_of(want[g]))), \
                f"replay {how} {s} group {g}"
        assert float(fi.item()) == (1.0 if non_finite(outs) else 0.0), f"replay {how} {s}: flag"
        assert (float(fi.item()) == 1.0) == (s == float("inf")), f"replay {how} {s}: flag {float(fi.item())}"


# ---- collectives ----------------------------------------------------------------------------------------------------

def _randn(dt, n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, generator=g).to(dt)


def _bits_equal(a, b):
    return torch.equal(a.view(W._it_of(a)), b.view(W._it_of(b)))


def _worker(rank, world, dev):
    import dietgpu_b200 as dg

    done = []
    s = float(np.float32(-0.3) / np.float32(world))
    for dt in (torch.float16, torch.bfloat16, torch.float32):
        variants = [(None, None)] + ([(torch.float32, None)] if dt != torch.float32 else
                                     [(None, torch.bfloat16), (None, torch.float16)])
        for reduce_dtype, wire in variants:
            for sparse in ((False, True) if wire is None else (False,)):
                tag = f"{dt} reduce {reduce_dtype} wire {wire} sparse {sparse}"
                kw2 = dict(members=3, reduce_dtype=reduce_dtype, sparse=sparse)  # all_reduce_compressed's
                kw = dict(kw2, wire_dtype=wire)
                n = world * 12289 if world > 1 else 12289
                ts = rank_data(dt, n, world, 700 + len(done), widened=reduce_dtype is not None)
                x = ts[rank].to(dev)
                # equivalence: == scale=float(s), with the flag set exactly where the shard is non-finite
                fi = torch.zeros(1, device=dev)
                got = dg.reduce_scatter_compressed(x, scale_tensor=torch.tensor([s], device=dev), found_inf=fi,
                                                   **kw)
                want = dg.reduce_scatter_compressed(x, scale=s, **kw)
                assert _bits_equal(got, want), f"reduce_scatter {tag}"
                assert float(fi.item()) == float(bool((~torch.isfinite(got)).any())), f"reduce_scatter {tag} flag"
                done.append(tag)
                if wire is None:
                    for m in (1, 30001):
                        tm = rank_data(dt, m, world, 900 + m, widened=reduce_dtype is not None)
                        fi = torch.zeros(1, device=dev)
                        got = dg.all_reduce_compressed(tm[rank].to(dev), scale_tensor=torch.tensor([s], device=dev),
                                                       found_inf=fi, **kw2)
                        want = dg.all_reduce_compressed(tm[rank].to(dev), scale=s, **kw2)
                        assert _bits_equal(got, want), f"all_reduce {tag} n {m}"
                        assert float(fi.item()) == float(bool((~torch.isfinite(got)).any())), \
                            f"all_reduce {tag} n {m} flag"
                        done.append(tag)
                # the flag: one non-finite word in rank r's chunk for destination d
                n = world * 4104
                shard = n // world
                base = _randn(dt, n, 31 * rank + 5)
                for flag0 in (0.0, 1.0):  # a finite run leaves the flag as it was
                    fi = torch.full((1,), flag0, device=dev)
                    dg.reduce_scatter_compressed(base.to(dev), scale_tensor=torch.tensor([s], device=dev),
                                                 found_inf=fi, **kw)
                    assert float(fi.item()) == flag0, f"{tag}: finite reduce_scatter, flag {flag0}"
                    if wire is None:
                        fi = torch.full((1,), flag0, device=dev)
                        dg.all_reduce_compressed(base.to(dev), scale_tensor=torch.tensor([s], device=dev),
                                                 found_inf=fi, **kw2)
                        assert float(fi.item()) == flag0, f"{tag}: finite all_reduce, flag {flag0}"
                for d in range(world):
                    for r in sorted({d, (d + 1) % world}):
                        x = base.clone()
                        if rank == r:
                            x[d * shard + 4097] = float("inf") if d % 2 == 0 else float("nan")
                        fi = torch.zeros(1, device=dev)
                        dg.reduce_scatter_compressed(x.to(dev), scale_tensor=torch.tensor([s], device=dev),
                                                     found_inf=fi, **kw)
                        assert float(fi.item()) == (1.0 if rank == d else 0.0), \
                            f"{tag}: reduce_scatter, bad word from {r} for {d}, flag on {rank}"
                        if wire is None:
                            fi = torch.zeros(1, device=dev)
                            dg.all_reduce_compressed(x.to(dev), scale_tensor=torch.tensor([s], device=dev),
                                                     found_inf=fi, **kw2)
                            assert float(fi.item()) == 1.0, f"{tag}: all_reduce, bad word from {r} for {d}"
                        done.append(tag)
    return len(done)


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_devscale_collectives(world):
    run_ranks(_worker, world, backend="gloo", timeout=600)
