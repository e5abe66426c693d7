"""Sparse decode-and-sum (ops.decompress_data_reduce(sparse=True), dgb_float_decompress_reduce_sparse) and sparse
archives on the wire of the compressed collectives.

The reference of every case is the dense path: the same words compressed dense and summed by
ops.decompress_data_reduce, which tests/test_gpu_reduce_edges.py pins to the float64 fold of
tests/reduce_reference.py.  Outputs sit in guard-banded, sentinel-filled buffers, and the sparse and the dense call
must leave the two buffers identical byte for byte (-0 and NaN payloads included, guards untouched).

The corpus mixes, inside every group, archives whose words are ReLU outputs, all +0, all -0, +-0 in every pairing
(with a few other words), blocks of only zeros next to blocks without any, no zeros at all, full-range words (no
two symbols are free, so nothing is elided and +-0 words are stored) and NaN / +-inf / subnormals among zeros.
Every call parses its archives' block tables and fails unless blocks were decoded through both stream branches of
decodeReduceBlock (staged in the warp's slot, or read from global memory)."""
import re

import numpy as np
import pytest
import torch

from codec_helpers import assert_guard_intact, codec_options, guarded_out, to_dev_bytes
from multirank import NAME, host_words, rank_data, run_ranks
from oracle import oracle as O
from reduce_reference import WORD, assert_same_words, fold_ref
import sparse32_oracle as SP32
import sparse_oracle as SP
from test_gpu_reduce_edges import device_words, init_words

pytestmark = pytest.mark.gpu

TORCH = {"f16": torch.float16, "bf16": torch.bfloat16, "f32": torch.float32}
SPARSE_TYPE = {"f16": 5, "bf16": 6, "f32": 8}
PAIRS = [("f16", "f16"), ("bf16", "bf16"), ("f32", "f32"), ("f16", "f32"), ("bf16", "f32")]
PAIR_IDS = [f"{a}-{o}" for a, o in PAIRS]
SIZES = [0, 1, 31, 33, 4095, 4096, 4097, 65537, 300001]
SHAPES = ("relu", "pos0", "neg0", "signs", "blocks", "nozero", "full", "special")
NEG0 = {"f16": 0x8000, "bf16": 0x8000, "f32": 0x80000000}
DEFAULT_SLOT = 1536  # decoderSmem's float slot, in u16 words
MODES = {"default": {}, "slot8": dict(decode_slot_words=1), "slot_max": dict(decode_slot_words=4096)}


# ---- corpus --------------------------------------------------------------------------------------------------

def _to_words(x32, t):
    """Host words of type t of a float32 array (torch's round-to-nearest-even cast)."""
    if t == "f32":
        return x32.astype(np.float32).view(np.uint32).copy()
    return torch.from_numpy(x32.astype(np.float32)).to(TORCH[t]).view(torch.int16).numpy().view(np.uint16).copy()


def _no_zero(w, t):
    w[(w & ~np.array(NEG0[t], WORD[t])) == 0] = _to_words(np.ones(1, np.float32), t)[0]
    return w


def shape_words(t, shape, n, seed, j=0):
    rng = np.random.default_rng(seed)
    wt = WORD[t]
    x = rng.standard_normal(n).astype(np.float32)
    if shape == "relu":
        w = _to_words(np.maximum(x, 0), t)
        w[(w == 0) & (rng.random(n) < 0.1)] = NEG0[t]
        return w
    if shape == "pos0":
        return np.zeros(n, wt)
    if shape == "neg0":
        return np.full(n, NEG0[t], wt)
    if shape == "signs":
        # +-0 whose sign is bit j % 4 of the element index: at every element of a group the archives' zeros meet in
        # every pairing; one element in eight holds another value
        i = np.arange(n)
        w = np.where((i >> (j % 4)) & 1, NEG0[t], 0).astype(wt)
        other = i % 8 == 7
        w[other] = _no_zero(_to_words(x, t), t)[other]
        return w
    if shape == "blocks":
        w = _no_zero(_to_words(x, t), t)
        blk = np.arange(n) // 4096
        z = blk % 2 == j % 2
        w[z] = np.where(rng.random(int(z.sum())) < 0.5, NEG0[t], 0).astype(wt)
        return w
    if shape == "nozero":
        return _no_zero(_to_words(x * [1.0, 1e-3, 1e3][seed % 3], t), t)
    if shape == "full":
        if t == "f32":
            w = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
            w[::37] = 0
            w[5::41] = NEG0[t]
            return w
        return np.resize(rng.permutation(1 << 16).astype(np.uint16), n)
    assert shape == "special"
    w = _to_words(x, t)
    nan = {"f16": 0x7E01, "bf16": 0x7FC1, "f32": 0x7FC00123}[t]
    inf = {"f16": 0x7C00, "bf16": 0x7F80, "f32": 0x7F800000}[t]
    sub = {"f16": 0x83FF, "bf16": 0x807F, "f32": 0x807FFFFF}[t]
    w[0::3] = 0
    w[1::7] = NEG0[t]
    w[2::11] = nan
    w[4::13] = inf
    w[5::17] = inf | NEG0[t]
    w[6::19] &= np.array(sub, wt)  # subnormals of either sign
    w[8::23] = 1
    return w


_WORDS = {}


def corpus(t):
    """{(group, archive): words} for every size of SIZES and archive index 0..8; shape SHAPES[(g + j) % 8]."""
    if t not in _WORDS:
        _WORDS[t] = {(g, j): shape_words(t, SHAPES[(g + j) % len(SHAPES)], n, 1000 * g + j + 11, j)
                     for g, n in enumerate(SIZES) for j in range(9)}
    return _WORDS[t]


def compress(ts, pb, sparse, checksum=False):
    from dietgpu_b200 import ops

    comp, sizes, _ = ops.compress_data(True, ts, checksum, prob_bits=pb, sparse=sparse)
    hs = sizes.cpu().tolist()
    return [comp[i, :hs[i]].clone() for i in range(len(ts))]


def sparse_block_words(arch, t):
    """(stream words, stream offset) of every block of a sparse archive (device or host bytes)."""
    a = arch.cpu().numpy() if torch.is_tensor(arch) else np.asarray(arch)
    ans = SP32.ans_part(a) if t == "f32" else SP.ans_part(a)
    bw = O.parse_ans(ans)["block_words"]
    return (bw[:, 0] & 0xFFFF).astype(np.int64), bw[:, 1].astype(np.int64)


_ARCH = {}


def archives(t, pb):
    """{(g, j): (sparse archive, dense archive, (block words, offsets))} of the corpus."""
    key = (t, pb)
    if key not in _ARCH:
        words = corpus(t)
        out = {}
        for g in range(len(SIZES)):
            dev = [device_words(words[g, j], t) for j in range(9)]
            sp, de = compress(dev, pb, True), compress(dev, pb, False)
            for j in range(9):
                out[g, j] = (sp[j], de[j], sparse_block_words(sp[j], t))
        _ARCH.clear()  # one (type, pb) at a time keeps device memory small
        _ARCH[key] = out
    return _ARCH[key]


def assert_both_branches(blocks, slot, what):
    """blocks: (words, offsets) of every archive a call decodes; the slot as decoderSmem rounds it."""
    staged = any(bool(((w <= slot) & (o % 8 == 0)).any()) for w, o in blocks)
    direct = any(bool(((w > slot) | (o % 8 != 0)).any()) for w, o in blocks)
    assert staged, f"{what}: no block went through the staged stream"
    assert direct, f"{what}: no block went through the global-memory stream"


# ---- the sum, sparse against dense -----------------------------------------------------------------------------

def sum_both(at, ot, pb, sparse_groups, dense_groups, sizes, accumulate, what, seed=0, expect_status=None,
             offsets=None):
    """Sums the sparse groups with sparse=True and the dense groups with the dense call into twin guard-banded
    buffers, and checks that the two buffers are byte-identical, the guards intact and the archives unchanged.
    expect_status: the sparse call's status per archive (default all 1); groups with a 0 must stay unwritten.
    Returns the sparse outputs."""
    from dietgpu_b200 import ops

    bufs, outs, spans = {"s": [], "d": []}, {"s": [], "d": []}, []
    for g, n in enumerate(sizes):
        off = (3 * g + 1) % 8 if offsets is None else offsets[g]
        init = device_words(init_words(ot, n, seed + g), ot) if accumulate else None
        for k in ("s", "d"):
            b, v, span = guarded_out(n, TORCH[ot], off)
            if init is not None:
                v.copy_(init)
            bufs[k].append(b)
            outs[k].append(v)
        spans.append(span)
    before = [b.clone() for b in bufs["s"]]
    arch_before = [a.clone() for grp in sparse_groups for a in grp]
    nst = sum(len(grp) for grp in sparse_groups)
    st_s = torch.full((nst,), 7, dtype=torch.uint8, device="cuda")
    st_d = torch.zeros(nst, dtype=torch.uint8, device="cuda")
    ops.decompress_data_reduce(sparse_groups, outs["s"], accumulate, None, st_s, prob_bits=pb,
                               archive_dtype=TORCH[at], sparse=True)
    ops.decompress_data_reduce(dense_groups, outs["d"], accumulate, None, st_d, prob_bits=pb,
                               archive_dtype=TORCH[at])
    torch.cuda.synchronize()
    want_st = [1] * nst if expect_status is None else list(expect_status)
    assert st_s.cpu().tolist() == want_st, f"{what}: status {st_s.cpu().tolist()} != {want_st}"
    for a, b in zip([a for grp in sparse_groups for a in grp], arch_before):
        assert torch.equal(a, b), f"{what}: an archive changed"
    k0 = 0
    for g in range(len(sizes)):
        w = len(sparse_groups[g])
        valid = all(want_st[k0:k0 + w])
        k0 += w
        if valid:
            assert bool(st_d[k0 - w:k0].all()), f"{what}: dense reference group {g} failed"
            assert torch.equal(bufs["s"][g], bufs["d"][g]), \
                f"{what} group {g} n {sizes[g]}: sparse sum differs from the dense sum"
            assert_guard_intact(bufs["s"][g], *spans[g], f"{what} group {g}")
        else:
            assert torch.equal(bufs["s"][g], before[g]), f"{what}: invalid group {g} was written"
    return outs["s"]


# ---- corpus under every writer, pass and stream branch ----------------------------------------------------------

@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("pb", [9, 10, 11])
@pytest.mark.parametrize("at,ot", PAIRS, ids=PAIR_IDS)
def test_corpus(at, ot, pb, mode):
    arch = archives(at, pb)
    slot = {"default": DEFAULT_SLOT, "slot8": 8, "slot_max": 256 * pb + 8}[mode]
    groups = range(len(SIZES))
    for accumulate in (False, True):
        for w in range(1, 10):
            what = f"{at}->{ot} pb {pb} {mode} acc {accumulate} W {w}"
            blocks = [arch[g, j][2] for g in groups for j in range(w) if SIZES[g] > 0]
            if mode == "slot_max":
                assert not any(bool((b[0] > slot).any()) for b in blocks)
            else:
                assert_both_branches(blocks, slot, what)
            with codec_options(**MODES[mode]):
                sum_both(at, ot, pb, [[arch[g, j][0] for j in range(w)] for g in groups],
                         [[arch[g, j][1] for j in range(w)] for g in groups], SIZES, accumulate, what,
                         seed=17 * w + pb)


def test_type8_windows_advance():
    """Type 8 streams a block's kept words in windows of 512; a full block of nonzero words needs eight."""
    arch = archives("f32", 10)
    words = corpus("f32")
    full = [(g, j) for (g, j) in arch if SIZES[g] >= 4096
            and int(((words[g, j][:4096] & 0x7FFFFFFF) != 0).sum()) > 1536]
    assert len(full) >= 9, full
    # ... and the W = 9 sums of the corpus above include them; here the same archives sum with themselves
    g, j = full[0]
    a, d = arch[g, j][0], arch[g, j][1]
    for acc in (False, True):
        sum_both("f32", "f32", 10, [[a, a, a]], [[d, d, d]], [SIZES[g]], acc, f"type 8 windows acc {acc}")


def test_signed_zero_pairings():
    """Groups made of the 'signs' shape only: at each element -0 + +0, -0 + -0, +0 + -0 and +0 + +0 all occur."""
    n = 40000
    for at, ot in PAIRS:
        words = [shape_words(at, "signs", n, 5 + j, j) for j in range(6)]
        sgn = np.stack([(w & np.array(NEG0[at], WORD[at])) != 0 for w in words])
        zero = np.stack([(w & ~np.array(NEG0[at], WORD[at])) == 0 for w in words])
        both = zero[0] & zero[1]
        for a, b in ((False, False), (True, False), (True, True), (False, True)):
            assert bool((both & (sgn[0] == a) & (sgn[1] == b)).any())
        dev = [device_words(w, at) for w in words]
        sp, de = compress(dev, 10, True), compress(dev, 10, False)
        for w in (2, 3, 6):
            for acc in (False, True):
                got = sum_both(at, ot, 10, [sp[:w]], [de[:w]], [n], acc, f"signs {at}->{ot} W {w} acc {acc}")
                if not acc:
                    h = got[0].view(torch.int32 if ot == "f32" else torch.int16).cpu().numpy().view(WORD[ot])
                    assert_same_words(h, fold_ref(words[:w], at, ot), ot, f"signs {at}->{ot} W {w} fold")


# ---- group counts: inline and uploaded member tables -------------------------------------------------------------

@pytest.mark.parametrize("groups", [1, 6, 65, 130])
def test_group_counts(groups):
    width = 5
    for at, ot in PAIRS:
        sizes = [4097 + 517 * (g % 7) for g in range(groups)]
        words = [[shape_words(at, SHAPES[(g + j) % len(SHAPES)], n, 31 * g + j, j) for j in range(width)]
                 for g, n in enumerate(sizes)]
        dev = [device_words(w, at) for grp in words for w in grp]
        sp, de = compress(dev, 10, True), compress(dev, 10, False)
        sg = [sp[g * width:(g + 1) * width] for g in range(groups)]
        dg_ = [de[g * width:(g + 1) * width] for g in range(groups)]
        for acc in (False, True):
            sum_both(at, ot, 10, sg, dg_, sizes, acc, f"G {groups} {at}->{ot} acc {acc}", seed=groups)


# ---- invalid archives ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("at,ot", PAIRS, ids=PAIR_IDS)
def test_invalid_groups_are_not_written(at, ot):
    n, width = 9000, 3
    words = [shape_words(at, "relu", n, 70 + j) for j in range(width)]
    dev = [device_words(w, at) for w in words]
    sp, de = compress(dev, 10, True), compress(dev, 10, False)
    other = "bf16" if at == "f16" else "f16"  # type 5 archives given as 6 and the other way round
    wrong_type = compress([device_words(shape_words(other, "relu", n, 80), other)], 10, True)[0]
    f32_as_16 = compress([device_words(shape_words("f32", "relu", n, 81), "f32")], 10, True)[0]
    f16_as_32 = compress([device_words(shape_words("f16", "relu", n, 82), "f16")], 10, True)[0]
    other_pb = compress(dev[:1], 9, True)[0]
    short = compress([device_words(words[0][:n - 1], at)], 10, True)[0]
    long = compress([device_words(np.concatenate([words[0], words[0][:1]]), at)], 10, True)[0]
    bad = {"dense": de[1], "other pb": other_pb, "one word short": short, "one word long": long,
           "type 8 as 5 / 6" if at != "f32" else "type 5 as 8": f32_as_16 if at != "f32" else f16_as_32}
    if at != "f32":
        bad["type 5 as 6" if at == "bf16" else "type 6 as 5"] = wrong_type
    sparse_groups, dense_groups, status = [], [], []
    for k, (name, a) in enumerate(bad.items()):
        # a valid group before every invalid one; the bad archive sits at position k % width
        sparse_groups.append(list(sp))
        dense_groups.append(list(de))
        status += [1] * width
        grp = list(sp)
        grp[k % width] = a
        sparse_groups.append(grp)
        dense_groups.append(list(de))
        status += [0 if j == k % width else 1 for j in range(width)]
    sizes = [n] * len(sparse_groups)
    for acc in (False, True):
        sum_both(at, ot, 10, sparse_groups, dense_groups, sizes, acc, f"invalid {at}->{ot} acc {acc}",
                 expect_status=status)


# ---- other producers ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("pb", [9, 10, 11])
@pytest.mark.parametrize("t", ["f16", "bf16", "f32"])
def test_every_producer_sums_the_same(t, pb):
    from test_gpu_variants import VARIANTS

    words = corpus(t)
    groups = [6, 8]  # 65537 and 300001 elements
    width = 5
    hw = [[words[g, j] for j in range(width)] for g in groups]
    sizes = [SIZES[g] for g in groups]
    dev = [device_words(w, t) for grp in hw for w in grp]
    dense = compress(dev, pb, False)
    dgroups = [dense[k * width:(k + 1) * width] for k in range(len(groups))]
    outs = [t] if t == "f32" else [t, "f32"]

    def check(arch, what):
        sg = [arch[k * width:(k + 1) * width] for k in range(len(groups))]
        for ot in outs:
            sum_both(t, ot, pb, sg, dgroups, sizes, False, f"{what} -> {ot}")

    for name, opts, role in VARIANTS:
        if role == "dec":
            continue
        for checksum in (False, True):
            with codec_options(**opts):
                arch = compress(dev, pb, True, checksum)
            check(arch, f"{t} pb {pb} {name} checksum {checksum}")
    for checksum in (False, True):
        if t == "f32":
            arch = [to_dev_bytes(SP32.compress(w, pb, checksum)) for grp in hw for w in grp]
        else:
            arch = [to_dev_bytes(SP.compress(w, SPARSE_TYPE[t], pb, checksum)) for grp in hw for w in grp]
        check(arch, f"{t} pb {pb} CPU restatement checksum {checksum}")


# ---- W = 1 is a plain decode -------------------------------------------------------------------------------------

@pytest.mark.parametrize("at,ot", PAIRS, ids=PAIR_IDS)
def test_single_archive_is_the_sparse_decode(at, ot):
    from dietgpu_b200 import ops

    words = corpus(at)
    arch = archives(at, 10)
    for g, n in enumerate(SIZES):
        a = arch[g, 0][0]
        dec = torch.empty(n, dtype=TORCH[at], device="cuda")
        ops.decompress_data(True, [a], [dec], sparse=True)
        out = torch.empty(n, dtype=TORCH[ot], device="cuda")
        ops.decompress_data_reduce([[a]], [out], archive_dtype=TORCH[at], sparse=True)
        want = dec if ot == at else dec.float()
        it = torch.int32 if ot == "f32" else torch.int16
        if at == ot:
            assert torch.equal(out.view(it), want.view(it)), f"{at}->{ot} n {n}"
        else:  # a NaN stays a NaN (the widening keeps its payload's top bits, like torch's cast)
            same = (out.view(it) == want.view(it)) | (torch.isnan(out) & torch.isnan(want))
            assert bool(same.all()), f"{at}->{ot} n {n}"
        assert np.array_equal(dec.view(torch.int32 if at == "f32" else torch.int16).cpu().numpy().view(WORD[at]),
                              words[g, 0])


# ---- CUDA graphs ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("groups", [6, 130])
@pytest.mark.parametrize("at,ot", [("bf16", "f32"), ("f32", "f32"), ("f16", "f16")])
def test_graph_capture(at, ot, groups):
    from dietgpu_b200 import ops

    width, n = 3, 5000
    cols = (64 << 10) if at == "f32" else (32 << 10)
    rows = torch.zeros(groups * width, cols, dtype=torch.uint8, device="cuda")

    def load(seed):
        words = [[shape_words(at, SHAPES[(seed + g + j) % len(SHAPES)], n, seed + 100 * g + j, j)
                  for j in range(width)] for g in range(groups)]
        dev = [device_words(w, at) for grp in words for w in grp]
        arch = compress(dev, 10, True)
        for i, a in enumerate(arch):
            assert a.numel() <= cols
            rows[i, :a.numel()].copy_(a)
        dense = compress(dev, 10, False)
        return [arch[g * width:(g + 1) * width] for g in range(groups)], \
               [dense[g * width:(g + 1) * width] for g in range(groups)]

    load(1)
    ins = [[rows[g * width + j, :cols] for j in range(width)] for g in range(groups)]
    init = [device_words(init_words(ot, n, 5 + g), ot) for g in range(groups)]
    outs = [torch.empty(n, dtype=TORCH[ot], device="cuda") for _ in range(groups)]
    st = torch.zeros(groups * width, dtype=torch.uint8, device="cuda")
    scratch = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.decompress_data_reduce(ins, outs, True, scratch, st, archive_dtype=TORCH[at], sparse=True)  # warm-up
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        ops.decompress_data_reduce(ins, outs, True, scratch, st, archive_dtype=TORCH[at], sparse=True)
    for seed in (2, 3):
        _, dense = load(seed * 1000)  # new archives in the captured rows
        for o, i in zip(outs, init):
            o.copy_(i)
        st.zero_()
        graph.replay()
        want = [i.clone() for i in init]
        ops.decompress_data_reduce(dense, want, True, archive_dtype=TORCH[at])
        torch.cuda.synchronize()
        assert bool(st.all()), f"replay {seed}: status"
        it = torch.int32 if ot == "f32" else torch.int16
        for k in range(groups):
            assert torch.equal(outs[k].view(it), want[k].view(it)), f"replay seed {seed} group {k}"


# ---- every new kernel runs -----------------------------------------------------------------------------------------

def test_profiler_sees_every_instantiation():
    # in a fresh process: in a long-lived one the GPU's timestamps drift against the host clock that bounds the
    # profiler's window, and every record of a window can fall outside it
    run_ranks(_profiler_sees_every_instantiation, 1, backend="gloo")


def _profiler_sees_every_instantiation(rank, world, dev):
    from torch.profiler import ProfilerActivity, profile

    from dietgpu_b200 import ops

    work = []
    for at, ot in PAIRS:
        for pb in (9, 10, 11):
            dev = [device_words(shape_words(at, "relu", 5000, 11 + j), at) for j in range(2)]
            work.append(([compress(dev, pb, True)], [torch.empty(5000, dtype=TORCH[ot], device="cuda")], at, pb))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device="cuda").add_(1)  # the first kernel of a session can be missing from its trace
        for _ in range(3):
            for ins, outs, at, pb in work:
                ops.decompress_data_reduce(ins, outs, prob_bits=pb, archive_dtype=TORCH[at], sparse=True)
        torch.cuda.synchronize()
    names = {re.sub(r"\s", "", e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    for kind in (5, 6, 8, 5 | 0x20, 6 | 0x20):
        for pb in (9, 10, 11):
            assert any(f"decodeReduceKernel<{kind},{pb}>" in k for k in names), (kind, pb, sorted(names))


# ---- collectives ------------------------------------------------------------------------------------------------

def sparse_rank_data(dt, n, world, seed, pruned, widened=False):
    """tests/multirank.rank_data (order-dependent elements, +-0, NaN, +-inf in elements 0..7 of every 16) with the
    other elements ReLU'd, or 90 % of them pruned to +-0."""
    xs = rank_data(dt, n, world, seed, widened=widened)
    pos = torch.arange(n)
    out = []
    for r, x in enumerate(xs):
        x = x.clone()
        free = pos % 16 >= 8
        if pruned:
            g = torch.Generator().manual_seed(seed + 7 * r)
            u = torch.rand(n, generator=g)
            x[free & (u < 0.45)] = 0.0
            x[free & (u >= 0.45) & (u < 0.9)] = -0.0
        else:
            x[free & (x < 0)] = 0.0
        out.append(x)
    return out


def _worker(rank, world, dev):
    import torch.distributed as dist

    import dietgpu_b200 as dg

    done = []
    sent = [0]
    a2a_calls = []

    # count the payload bytes this rank sends (the size exchanges are int tensors and not counted), and the
    # all_to_all_single calls by the dtype they send
    real_gather, real_a2a = dist.all_gather_into_tensor, dist.all_to_all_single

    def gather(out, inp, *a, **k):
        if inp.dtype == torch.uint8:
            sent[0] += inp.numel()
        return real_gather(out, inp, *a, **k)

    def a2a(out, inp, *a, **k):
        a2a_calls.append(inp.dtype)
        if inp.dtype == torch.uint8:
            sent[0] += inp.numel()
        return real_a2a(out, inp, *a, **k)

    dist.all_gather_into_tensor, dist.all_to_all_single = gather, a2a

    def run(f):
        sent[0] = 0
        r = f()
        return r, sent[0]

    def exchange(f, what):
        """f() makes one per-destination exchange: the int64 size table, then the uint8 payload."""
        a2a_calls.clear()
        r = f()
        assert a2a_calls == [torch.int64, torch.uint8], f"{what}: all_to_all_single sent {a2a_calls}"
        return r

    def same(a, b, what):
        assert np.array_equal(host_words(a), host_words(b)), what
        done.append(what)

    for dt in (torch.float16, torch.bfloat16, torch.float32):
        for pruned in (False, True):
            for members in (1, 6):
                tag = f"{dt} pruned {pruned} members {members}"
                n = world * 12289
                ts = sparse_rank_data(dt, n, world, 100 + members, pruned)
                x = ts[rank].to(dev)
                got, b_s = run(lambda: dg.all_gather_compressed(x, members=members, sparse=True))
                want, b_d = run(lambda: dg.all_gather_compressed(x, members=members))
                same(got, want, f"all_gather {tag}")
                same(got, torch.cat(ts), f"all_gather {tag} (inputs)")
                assert b_s < b_d, f"all_gather {tag}: {b_s} sparse bytes sent, {b_d} dense"
                chunks = [x[d * 12289:(d + 1) * 12289 - d] for d in range(world)]
                got = exchange(lambda: dg.all_to_all_compressed(chunks, sparse=True), f"all_to_all {tag}")
                want = exchange(lambda: dg.all_to_all_compressed(chunks), f"all_to_all {tag}")
                for s in range(world):
                    same(got[s], want[s], f"all_to_all {tag} from {s}")
                for reduce_dtype in ([None] if dt == torch.float32 else [None, torch.float32]):
                    widened = reduce_dtype is not None
                    ts = sparse_rank_data(dt, n, world, 200 + members, pruned, widened)
                    x = ts[rank].to(dev)
                    at = NAME[dt]
                    ot = "f32" if widened else at
                    what = f"reduce_scatter {tag} reduce {reduce_dtype}"
                    got, b_s = run(lambda: exchange(lambda: dg.reduce_scatter_compressed(
                        x, members=members, reduce_dtype=reduce_dtype, sparse=True), what))
                    want, b_d = run(lambda: exchange(lambda: dg.reduce_scatter_compressed(
                        x, members=members, reduce_dtype=reduce_dtype), what))
                    same(got, want, what)
                    lo, hi = rank * (n // world), (rank + 1) * (n // world)
                    assert_same_words(host_words(got), fold_ref([host_words(t[lo:hi]) for t in ts], at, ot),
                                      ot, f"{what} (rank-order fold)")
                    assert b_s < b_d, f"{what}: {b_s} sparse bytes sent, {b_d} dense"
                    for m in (1, 300001):
                        tm = sparse_rank_data(dt, m, world, 300 + m, pruned, widened)
                        xm = tm[rank].to(dev)
                        got = dg.all_reduce_compressed(xm, members=members, reduce_dtype=reduce_dtype,
                                                       sparse=True)
                        want = dg.all_reduce_compressed(xm, members=members, reduce_dtype=reduce_dtype)
                        what = f"all_reduce {tag} n {m} reduce {reduce_dtype}"
                        same(got, want, what)
                        assert_same_words(host_words(got), fold_ref([host_words(t) for t in tm], at, ot), ot,
                                          f"{what} (rank-order fold)")
                        zero = np.all(np.stack([(host_words(t) & ~np.array(
                            0x80000000 if t.element_size() == 4 else 0x8000, host_words(t).dtype)) == 0
                            for t in tm]), axis=0)
                        gw = host_words(got)
                        assert np.all((gw[zero] & ~np.array(0x80000000 if got.element_size() == 4 else 0x8000,
                                                            gw.dtype)) == 0), f"{what}: zeros"
    return len(done)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_sparse_collectives(world):
    run_ranks(_worker, world, backend="gloo", timeout=600)
