"""The narrowing decode-and-sum (decodeReduceNarrowKernel, dgb_float_decompress_reduce_narrow) and the squared norms
(decodeReduceNormKernel and sqNormFoldKernel, dgb_float_decompress_reduce_scaled_dev_norm / _narrow_norm; the
standalone floatSqNormKernel, dgb_float_sq_norm) on the edge corpora of the other decode-and-sum families, against
the float64 fold.

References: every narrowing output equals tests/scaled_reference.narrow_fold_ref (the fp32 fold rounded once to 16
bits) word for word, and the widening call into fp32 followed by torch's .to() (NaN payloads aside); every other
output equals scaled_fold_ref.  Every norm equals sq_norm_reference.sq_norm of the *expected* words, so a writer that
stores one word and squares another fails, and ops.sq_norm of the outputs.  Buffers: outputs, the fp32 accumulators
and the norm vector sit inside sentinel-filled buffers whose bytes around them must survive; a W = 1 call without
accumulate must not touch its accumulator at all.

Coverage: the corpora are those of test_gpu_weighted_reduce.corpus (dense: over-slot blocks, the 256 * probBits-word
worst case, empty streams, full-range words with NaN, +-inf and subnormals; sparse: both stream branches).  The
narrowing and the norm are done by the writer of archive W - 1 alone, so every group lists the corpus's archives in
reverse (order()): its last archive is the corpus's archive 0, whose shape cycles through all of them across the
groups, and every corpus call asserts from the parsed block tables which blocks that writer sees, for the W = 1
store form and for the add form.

Also: the slot forced to 8 words and to the worst case and member tables in scratch (next to the narrowing table and
the norm's block partials), 70 groups, 65 archives, groups of 1 Mi + 1 and 2 Mi words at nonzero partial offsets with
empty groups around them (the fold's strided path), scratch of exactly the returned size, a graph replayed after an
intruder call of the same family, and the standalone norm at every element offset, over 1000 tensors, around 256
blocks and past one wave of its grid.

The module's name sorts after every other GPU module, so in a single-process run of the suite it runs last and the
profiler checks of the other modules keep their place in the process; its own profiler check comes first, with the
same margins around its window (test_gpu_weighted_reduce.py)."""
import re
import time

import numpy as np
import pytest
import torch

from codec_helpers import SENTINEL, assert_guard_intact, codec_options, guarded_out
from multirank import run_ranks
from reduce_reference import assert_same_words, to_f64
from scaled_reference import SCALES, narrow_fold_ref, scaled_fold_ref
import sq_norm_reference as R
import test_gpu_reduce_edges as E
import test_gpu_reduce_sparse as S
import test_gpu_weighted_reduce as W

pytestmark = pytest.mark.gpu

TORCH = W.TORCH
WIDTHS = [1, 2, 4, 5, 9]
NARROW_CASES = [("f16", False), ("bf16", False), ("f16", True), ("bf16", True)]
NARROW_IDS = ["f16", "bf16", "sparse-f16", "sparse-bf16"]
NARROW_MODES = ["none", "host", "dev"]
NORM_SCALES = [1.0, -0.25, float(np.float32(1 / 3)), 2.0 ** 15, float("inf"), float("nan")]
# norm kinds: (archive type, sparse, output type, narrowing): the ten device-scale pairs and the four narrowing ones
NORM_KINDS = {
    "f16": ("f16", False, "f16", False), "bf16": ("bf16", False, "bf16", False), "f32": ("f32", False, "f32", False),
    "f16s": ("f16", True, "f16", False), "bf16s": ("bf16", True, "bf16", False), "f32s": ("f32", True, "f32", False),
    "f16-f32": ("f16", False, "f32", False), "bf16-f32": ("bf16", False, "f32", False),
    "f16s-f32": ("f16", True, "f32", False), "bf16s-f32": ("bf16", True, "f32", False),
    "f16-narrow": ("f16", False, "f16", True), "bf16-narrow": ("bf16", False, "bf16", True),
    "f16s-narrow": ("f16", True, "f16", True), "bf16s-narrow": ("bf16", True, "bf16", True),
}
NORM_SENTINEL = -12345.5


def narrow_kind(t, sparse, mode):
    """decodeReduceNarrowKernel's KIND: archive kind | kWidenF32 | kNarrowOut (| kScaled (| kDevScale))."""
    k = ({"f16": 5, "bf16": 6} if sparse else {"f16": 1, "bf16": 2})[t]
    return k | 0x20 | 0x400 | {"none": 0, "host": 0x80, "dev": 0x180}[mode]


def norm_kind(name):
    """decodeReduceNormKernel's KIND: the device-scale kind (| kWidenF32 | kNarrowOut) | kSqNorm."""
    at, sparse, ot, narrow = NORM_KINDS[name]
    return W.kernel_kind(at, ot, sparse) | 0x100 | 0x800 | (0x420 if narrow else 0)


def _scale(s):
    return torch.tensor([s], dtype=torch.float32, device="cuda")


def _flag():
    return torch.zeros(1, dtype=torch.float32, device="cuda")


# ---- a: every instantiation runs, and no kernel of another family on these paths ------------------------------------

def test_profiler_sees_every_instantiation():
    # in a fresh process: in a long-lived one the GPU's timestamps drift against the host clock that bounds the
    # profiler's window, and every record of a window can fall outside it
    run_ranks(_profiler_sees_every_instantiation, 1, backend="gloo")


def _profiler_sees_every_instantiation(rank, world, dev):
    from torch.profiler import ProfilerActivity, profile

    from dietgpu_b200 import ops

    narrow, norm = [], []
    for t, sp in NARROW_CASES:
        for pb in (9, 10, 11):
            dev = [E.device_words(S.shape_words(t, "relu", 5000, 11 + j), t) for j in range(2)]
            arch = S.compress(dev, pb, sp)
            for mode in NARROW_MODES:
                narrow.append((arch, t, sp, pb, mode, torch.empty(5000, dtype=TORCH[t], device="cuda"),
                               torch.empty(5000, dtype=torch.float32, device="cuda")))
    for name, (at, sp, ot, nw) in NORM_KINDS.items():
        for pb in (9, 10, 11):
            dev = [E.device_words(S.shape_words(at, "relu", 5000, 21 + j), at) for j in range(2)]
            norm.append((S.compress(dev, pb, sp), at, sp, ot, nw, pb, torch.empty(5000, dtype=TORCH[ot], device="cuda"),
                         torch.empty(5000, dtype=torch.float32, device="cuda")))
    plain = [[E.device_words(E.init_words(t, 9000, 3), t)] for t in ("f16", "bf16", "f32")]
    sc, fi, sq = _scale(0.5), _flag(), torch.empty(1, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    # launches start well after the profiler's window opens and end well before it closes (test_gpu_weighted_reduce)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(1.0)
        torch.ones(1, device="cuda").add_(1)  # the first kernel of a session can be missing from its trace
        for _ in range(3):
            for arch, t, sp, pb, mode, out, acc in narrow:
                kw = {"host": dict(scale=0.5), "dev": dict(scale_tensor=sc, found_inf=fi), "none": {}}[mode]
                ops.decompress_data_reduce([arch], [out], prob_bits=pb, archive_dtype=TORCH[t], sparse=sp,
                                           reduce_dtype=torch.float32, acc=[acc], **kw)
            for arch, at, sp, ot, nw, pb, out, acc in norm:
                kw = dict(reduce_dtype=torch.float32, acc=[acc]) if nw else {}
                ops.decompress_data_reduce([arch], [out], prob_bits=pb, archive_dtype=TORCH[at], sparse=sp,
                                           scale_tensor=sc, found_inf=fi, sq_norm=sq, **kw)
            for ts in plain:
                ops.sq_norm(ts)
        torch.cuda.synchronize()
        time.sleep(1.0)
    names = {re.sub(r"\s", "", e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    nk = sorted({narrow_kind(t, sp, m) for t, sp in NARROW_CASES for m in NARROW_MODES})
    assert nk == [1057, 1058, 1061, 1062, 1185, 1186, 1189, 1190, 1441, 1442, 1445, 1446]
    qk = sorted({norm_kind(n) for n in NORM_KINDS})
    assert qk == [2433, 2434, 2435, 2437, 2438, 2440, 2465, 2466, 2469, 2470, 3489, 3490, 3493, 3494]
    for name, kinds in (("decodeReduceNarrowKernel", nk), ("decodeReduceNormKernel", qk)):
        for kind in kinds:
            for pb in (9, 10, 11):
                assert any(f"{name}<{kind},{pb}>" in k for k in names), (name, kind, pb, sorted(names))
    assert any("sqNormFoldKernel" in k for k in names), sorted(names)
    for k in (1, 2, 3):
        assert any(f"floatSqNormKernel<{k}>" in n for n in names), (k, sorted(names))
    assert not any("decodeReduceDevScaleKernel<" in k or "decodeReduceKernel<" in k for k in names), sorted(names)


# ---- the calls and their checks ---------------------------------------------------------------------------------------

def order(w):
    """The corpus archive indices of a width-w group, in call order: archive 0 last.  Archive j of corpus group g has
    shape SHAPES[(g + j) % len(SHAPES)], so the writer of archive W - 1 sees shape SHAPES[g % len(SHAPES)] in group g
    at every width: the worst case in the 262144-word group, over-slot blocks, empty streams; in the corpus's own order
    that writer would miss the worst case at W = 2."""
    return list(range(w - 1, -1, -1))


def check_last_writer(pb, sparse, blocks, gs, idx, accumulate, what):
    """The blocks the writer of archive W - 1 decodes (groups gs, call order idx): dense, an over-slot block, a
    256 * pb-word block and an empty-stream archive (test_gpu_reduce_edges); sparse, both stream branches."""
    form = "store" if len(idx) == 1 and not accumulate else "add"
    last = [blocks[g, idx[-1]] for g in gs]
    if sparse:
        S.assert_both_branches(last, S.DEFAULT_SLOT, f"{what}: the {form} writer of archive W - 1")
    else:
        E.assert_paths_covered(last, pb, f"{what}: the {form} writer of archive W - 1")


class Call:
    """One decode-and-sum into guard-banded buffers, with its standard checks done: every status 1, every guard band
    intact, and (W = 1 without accumulate) a narrowing call's accumulators untouched.

    narrow: 16-bit outputs of the archive type and fp32 accumulators, always passed; mode: "none", "host" (scale=s)
    or "dev" (scale_tensor, found_inf); sq: the norms, a G-element view with a sentinel element on either side."""

    def __init__(self, at, ot, sparse, narrow, pb, groups, sizes, mode, s, accumulate, inits, what, sq=False,
                 temp=None):
        from dietgpu_b200 import ops

        w = len(groups[0])
        self.what = what
        self.bufs, self.outs, spans = [], [], []
        self.abufs, accs, aspans = [], [], []
        for g, n in enumerate(sizes):
            b, v, span = guarded_out(n, TORCH[ot], (3 * g + 1) % 8)
            if accumulate and not narrow:
                v.copy_(E.device_words(inits[g], ot))
            self.bufs.append(b)
            self.outs.append(v)
            spans.append(span)
            if narrow:
                b, v, span = guarded_out(n, torch.float32, (5 * g + 2) % 8)
                if accumulate:
                    v.copy_(E.device_words(inits[g], "f32"))
                self.abufs.append(b)
                accs.append(v)
                aspans.append(span)
        kw = dict(prob_bits=pb, archive_dtype=TORCH[at], sparse=sparse)
        if narrow:
            kw.update(reduce_dtype=torch.float32, acc=accs)
        fi = None
        if mode == "host":
            kw["scale"] = s
        elif mode == "dev":
            fi = _flag()
            kw.update(scale_tensor=_scale(s), found_inf=fi)
        self.normbuf = None
        if sq:
            self.normbuf = torch.full((len(sizes) + 2,), NORM_SENTINEL, dtype=torch.float64, device="cuda")
            kw["sq_norm"] = self.normbuf[1:-1]
        st = torch.zeros(sum(len(grp) for grp in groups), dtype=torch.uint8, device="cuda")
        self.used = ops.decompress_data_reduce(groups, self.outs, accumulate, temp, st, **kw)
        torch.cuda.synchronize()
        assert bool(st.all()), f"{what}: status {st.cpu().tolist()}"
        for g in range(len(sizes)):
            assert_guard_intact(self.bufs[g], *spans[g], f"{what} group {g}")
            if narrow:
                assert_guard_intact(self.abufs[g], *aspans[g], f"{what} group {g} acc")
                if w == 1 and not accumulate:
                    assert bool((self.abufs[g] == SENTINEL).all()), f"{what} group {g}: W = 1 wrote its acc"
        self.flag = None if fi is None else float(fi.item())
        self.norms = None
        if sq:
            nb = self.normbuf.cpu().numpy()
            assert nb[0] == NORM_SENTINEL and nb[-1] == NORM_SENTINEL, f"{what}: a sentinel of the norms was written"
            self.norms = nb[1:-1]

    def check(self, ot, want, what=None):
        """want: (expected words per group, expected norms or None, any expected word non-finite)."""
        from dietgpu_b200 import ops

        what = what or self.what
        words, norms, bad = want
        for g, o in enumerate(self.outs):
            assert_same_words(E.to_host_words(o, ot), words[g], ot, f"{what} group {g} (float64)")
        if self.flag is not None:
            assert self.flag == (1.0 if bad else 0.0), f"{what}: found_inf {self.flag}, non-finite {bad}"
        if self.norms is not None:
            again = ops.sq_norm(self.outs).cpu().numpy()
            for g in range(len(self.outs)):
                assert R.same(self.norms[g], norms[g]), \
                    f"{what} group {g} ({self.outs[g].numel()} words): norm {self.norms[g]!r} != {norms[g]!r}"
                assert R.same(self.norms[g], again[g]), f"{what} group {g}: norm != ops.sq_norm of the outputs"
                if self.outs[g].numel() == 0:
                    assert self.norms[g] == 0.0 and not np.signbit(self.norms[g]), f"{what} group {g}: empty"


def expect(at, ot, narrow, hw, s, inits, norms):
    """(expected words per group, their norms when asked, any non-finite word): the float64 folds of host words hw
    (groups of lists, call order), s None for the unscaled narrowing sum."""
    words = []
    for g, grp in enumerate(hw):
        init = None if inits is None else inits[g]
        words.append(narrow_fold_ref(grp, at, s, init) if narrow else scaled_fold_ref(grp, at, ot, s, init))
    nq = [R.sq_norm(to_f64(w, ot)) for w in words] if norms else None
    bad = any(not bool(np.isfinite(to_f64(w, ot)).all()) for w in words)
    return words, nq, bad


_REF = {}


def cached(owner, key, make):
    """The references of one test (owner) at a time, shared by its probBits: the corpus words do not depend on it."""
    if _REF.get("owner") != owner:
        _REF.clear()
        _REF["owner"] = owner
    if key not in _REF:
        _REF[key] = make()
    return _REF[key]


def scale_key(s):
    """A cache key that tells the scales apart as the kernels do: 0.0 and -0.0 are equal floats but not equal scales."""
    return None if s is None else np.float32(s).tobytes()


def _inits(t, sizes, seed):
    return [E.init_words(t, n, seed + g) for g, n in enumerate(sizes)]


# ---- b: the narrowing sums on the corpus ------------------------------------------------------------------------------

def widen_then_to(t, sparse, pb, groups, sizes, mode, s, accumulate, inits):
    """The widening call (same archives, scale and fp32 init) into fp32 outputs, then torch's .to(t)."""
    from dietgpu_b200 import ops

    wide = [E.device_words(i, "f32") if accumulate else torch.empty(n, dtype=torch.float32, device="cuda")
            for i, n in zip(inits or [None] * len(sizes), sizes)]
    kw = {"none": {}, "host": dict(scale=s), "dev": dict(scale_tensor=_scale(s))}[mode] if s is not None else {}
    ops.decompress_data_reduce(groups, wide, accumulate, prob_bits=pb, archive_dtype=TORCH[t], sparse=sparse, **kw)
    return [x.to(TORCH[t]) for x in wide]


@pytest.mark.parametrize("pb", [9, 10, 11])
@pytest.mark.parametrize("t,sparse", NARROW_CASES, ids=NARROW_IDS)
def test_narrowing_corpus(t, sparse, pb):
    """Unscaled, host-scaled at SOME and device-scaled (every scale of SCALES at W = 5, SOME otherwise), every width,
    with and without accumulate: the float64 fold, the widening call then .to(), guards, untouched accumulators and
    the flag."""
    sizes, arch, words, _, blocks, _ = W.corpus(t, pb, sparse)
    G = range(len(sizes))
    gs = [g for g in G if sizes[g] > 0]
    for accumulate in (False, True):
        for w in WIDTHS:
            idx = order(w)
            what = f"{t} sparse {sparse} pb {pb} acc {accumulate} W {w}"
            check_last_writer(pb, sparse, blocks, gs, idx, accumulate, what)
            groups = [[arch[g, j] for j in idx] for g in G]
            hw = [[words[g, j] for j in idx] for g in G]
            inits = _inits("f32", sizes, 31 * w) if accumulate else None
            runs = [("none", None)] + [("host", s) for s in W.SOME] + [("dev", s) for s in (SCALES if w == 5 else W.SOME)]
            for mode, s in runs:
                tag = f"{what} {mode} s {s}"
                want = cached(("narrow", t, sparse), (w, accumulate, scale_key(s)),
                              lambda: expect(t, t, True, hw, s, inits, False))
                c = Call(t, t, sparse, True, pb, groups, sizes, mode, s, accumulate, inits, tag)
                c.check(t, want)
                ref = widen_then_to(t, sparse, pb, groups, sizes, mode, s, accumulate, inits)
                for g in G:
                    ok = W.same_dev(c.outs[g], ref[g])
                    assert bool(ok.all()), f"{tag} group {g}: {int((~ok).sum())} word(s) != the widening call then .to()"


# ---- c: the squared norms on the corpus -------------------------------------------------------------------------------

_EMPTY = {}


def empty_archive(at, pb, sparse):
    key = (at, pb, sparse)
    if key not in _EMPTY:
        _EMPTY.clear()
        _EMPTY[key] = S.compress([torch.empty(0, dtype=TORCH[at], device="cuda")], pb, sparse)[0]
    return _EMPTY[key]


def norm_layout(n):
    """Corpus group indices with a 0-word group (None) in the middle and one at the end."""
    return list(range(n // 2)) + [None] + list(range(n // 2, n)) + [None]


@pytest.mark.parametrize("pb", [9, 10, 11])
@pytest.mark.parametrize("kind", sorted(NORM_KINDS))
def test_norm_corpus(kind, pb):
    """Every width, with and without accumulate, at 1, -0.25, fp32(1/3), 2^15, inf and NaN: outputs, guards and the
    flag identical to the call without sq_norm and equal to the float64 fold; every norm that of the expected words,
    and of ops.sq_norm of the outputs."""
    at, sparse, ot, narrow = NORM_KINDS[kind]
    sizes0, arch, words, _, blocks, _ = W.corpus(at, pb, sparse)
    layout = norm_layout(len(sizes0))
    sizes = [0 if g is None else sizes0[g] for g in layout]
    empty = empty_archive(at, pb, sparse)
    gs = [g for g in range(len(sizes0)) if sizes0[g] > 0]
    it = "f32" if narrow else ot
    for accumulate in (False, True):
        inits = _inits(it, sizes, 7) if accumulate else None
        for w in WIDTHS:
            idx = order(w)
            what = f"{kind} pb {pb} acc {accumulate} W {w}"
            check_last_writer(pb, sparse, blocks, gs, idx, accumulate, what)
            groups = [[empty] * w if g is None else [arch[g, j] for j in idx] for g in layout]
            hw = [[np.zeros(0, E.WORD[at])] * w if g is None else [words[g, j] for j in idx] for g in layout]
            for s in NORM_SCALES:
                tag = f"{what} s {s}"
                want = cached(("norm", kind), (w, accumulate, scale_key(s)), lambda: expect(at, ot, narrow, hw, s, inits, True))
                c = Call(at, ot, sparse, narrow, pb, groups, sizes, "dev", s, accumulate, inits, tag, sq=True)
                plain = Call(at, ot, sparse, narrow, pb, groups, sizes, "dev", s, accumulate, inits, f"{tag} no sq")
                for g in range(len(sizes)):
                    assert torch.equal(c.bufs[g], plain.bufs[g]), f"{tag} group {g}: sq_norm changed the output"
                assert c.flag == plain.flag, f"{tag}: sq_norm changed found_inf"
                c.check(ot, want)


# ---- d: forced slots and member tables in scratch ---------------------------------------------------------------------

def _kinds(family):
    """(archive type, output type, sparse, narrowing, scale mode, sq) of every kernel kind of a family."""
    if family == "narrow":
        return [(t, t, sp, True, m, False) for t, sp in NARROW_CASES for m in NARROW_MODES]
    return [(at, ot, sp, nw, "dev", True) for at, sp, ot, nw in NORM_KINDS.values()]


@pytest.mark.parametrize("mode", list(W.MODES))
@pytest.mark.parametrize("family", ["narrow", "norm"])
def test_forced_slots_and_scratch_tables(family, mode):
    """Every kind at probBits 10, W = 1, 5 and 9, with and without accumulate, with the slot forced to 8 words (every
    non-empty block from global memory), to the worst case (every block staged), and with member tables in scratch:
    the same bytes and norms as the default options."""
    pb = 10
    for at, ot, sparse, narrow, smode, sq in sorted(_kinds(family), key=lambda k: (k[0], k[2])):
        sizes, arch, _, _, _, _ = W.corpus(at, pb, sparse)
        s = None if smode == "none" else W.SOME[0]
        for accumulate in (False, True):
            inits = _inits("f32" if narrow else ot, sizes, 3) if accumulate else None
            for w in (1, 5, 9):
                groups = [[arch[g, j] for j in order(w)] for g in range(len(sizes))]
                what = f"{at}->{ot} sparse {sparse} narrow {narrow} {smode} {mode} acc {accumulate} W {w}"
                base = Call(at, ot, sparse, narrow, pb, groups, sizes, smode, s, accumulate, inits, what, sq=sq)
                with codec_options(**W.MODES[mode]):
                    got = Call(at, ot, sparse, narrow, pb, groups, sizes, smode, s, accumulate, inits, what, sq=sq)
                for g in range(len(sizes)):
                    assert torch.equal(got.bufs[g], base.bufs[g]), f"{what} group {g}"
                assert got.flag == base.flag, what
                if sq:
                    assert all(R.same(a, b) for a, b in zip(got.norms, base.norms)), f"{what}: norms"


# ---- e: many groups, many archives, large groups ----------------------------------------------------------------------

def shaped_groups(at, sparse, sizes, w, seed):
    """Host words [g][j]: the corpus shapes, shape (g + j) in group g's archive j."""
    out = []
    for g, n in enumerate(sizes):
        grp = []
        for j in range(w):
            if sparse:
                grp.append(S.shape_words(at, S.SHAPES[(g + j) % len(S.SHAPES)], n, seed + 100 * g + j, j))
            else:
                grp.append(E._shape_words(at, E.SHAPES[(g + j) % len(E.SHAPES)], n, seed + 100 * g + j))
        out.append(grp)
    return out


def compress_groups(at, sparse, pb, hw):
    flat = S.compress([E.device_words(x, at) for grp in hw for x in grp], pb, sparse)
    w = len(hw[0])
    return [flat[g * w:(g + 1) * w] for g in range(len(hw))]


SIZES70 = ([0, 1, 4097] + E.SIZES) * 6  # 78 sizes: 0, 1, 4097 and the corpus sizes, repeated
LARGE = [(1 << 20) + 1, 5, 0, 2 << 20, 4097, 0]  # 257 and 512 blocks at nonzero partial offsets, empty groups


@pytest.mark.parametrize("kind", sorted(NORM_KINDS))
def test_many_groups_and_large_groups(kind):
    """70 groups at W = 1 and 2 (member tables in scratch; 70 partial offsets and, narrowing, a 70-entry output
    table), one group of 65 archives, and groups of 1 Mi + 1 and 2 Mi words next to small and empty ones, whose
    partials the fold sums with its strided loop from a nonzero offset."""
    at, sparse, ot, narrow = NORM_KINDS[kind]
    it = "f32" if narrow else ot
    pb = 10
    s = -0.25
    cases = [(SIZES70[:70], 1, False), (SIZES70[:70], 2, False), (SIZES70[:70], 2, True), ([70001], 65, False),
             (LARGE, 2, False), (LARGE, 1, True)]
    for k, (sizes, w, accumulate) in enumerate(cases):
        what = f"{kind} G {len(sizes)} W {w} acc {accumulate} sizes {sorted(set(sizes))[-1]}"
        hw = shaped_groups(at, sparse, sizes, w, 1000 * k)
        groups = compress_groups(at, sparse, pb, hw)
        inits = _inits(it, sizes, 11 * k) if accumulate else None
        c = Call(at, ot, sparse, narrow, pb, groups, sizes, "dev", s, accumulate, inits, what, sq=True)
        plain = Call(at, ot, sparse, narrow, pb, groups, sizes, "dev", s, accumulate, inits, f"{what} no sq")
        for g in range(len(sizes)):
            assert torch.equal(c.bufs[g], plain.bufs[g]), f"{what} group {g}: sq_norm changed the output"
        assert c.flag == plain.flag, what
        c.check(ot, expect(at, ot, narrow, hw, s, inits, True))


# ---- f: scratch of exactly the returned size --------------------------------------------------------------------------

def _exact_temp(need, lead=37):
    """temp_mem of need + 256 bytes (the alignment pad) at an odd offset inside a larger sentinel-filled buffer;
    returns (buffer, temp_mem, offset of the aligned scratch in the buffer)."""
    big = torch.full((need + 256 + 2 * 1024,), SENTINEL, dtype=torch.uint8, device="cuda")
    temp = big[1024 + lead:1024 + lead + need + 256]
    return big, temp, 1024 + lead + (-temp.data_ptr()) % 256


def _assert_scratch_kept(big, start, need, what):
    head, tail = big[:start], big[start + need:]
    assert bool((head == SENTINEL).all()), f"{what}: scratch written before the aligned start"
    assert bool((tail == SENTINEL).all()), f"{what}: {int((tail != SENTINEL).sum())} byte(s) written past the " \
                                           f"{need} bytes of scratch"


@pytest.mark.parametrize("kind", ["bf16-narrow", "f16s-narrow", "f32", "bf16s-f32"])
def test_exact_scratch(kind):
    from dietgpu_b200 import capi

    at, sparse, ot, narrow = NORM_KINDS[kind]
    it = "f32" if narrow else ot
    L = capi.lib()
    ft = ({"f16": capi.FLOAT16_SPARSE, "bf16": capi.BFLOAT16_SPARSE, "f32": capi.FLOAT32_SPARSE} if sparse else
          {"f16": capi.FLOAT16, "bf16": capi.BFLOAT16, "f32": capi.FLOAT32})[at]
    sizes = SIZES70[:70]
    for w, accumulate in ((2, False), (1, False), (2, True)):
        hw = shaped_groups(at, sparse, sizes, w, 77 + w)
        groups = compress_groups(at, sparse, 10, hw)
        inits = _inits(it, sizes, 5) if accumulate else None
        want = expect(at, ot, narrow, hw, 0.5, inits, True)
        what = f"{kind} W {w} acc {accumulate}"
        # the norm call
        need = L.dgb_float_decompress_reduce_norm_temp_bytes(ft, len(sizes), w, capi.u32_array(sizes))
        big, temp, start = _exact_temp(need)
        c = Call(at, ot, sparse, narrow, 10, groups, sizes, "dev", 0.5, accumulate, inits, f"{what} norm", sq=True,
                 temp=temp)
        assert c.used == need, (c.used, need)
        torch.cuda.synchronize()
        _assert_scratch_kept(big, start, need, f"{what} norm")
        c.check(ot, want)
        # the call without the norm (narrowing, or device-scale)
        need = L.dgb_float_decompress_temp_bytes(ft, len(sizes) * w, 0)
        big, temp, start = _exact_temp(need, lead=101)
        c = Call(at, ot, sparse, narrow, 10, groups, sizes, "dev", 0.5, accumulate, inits, f"{what} plain", temp=temp)
        assert c.used == need, (c.used, need)
        _assert_scratch_kept(big, start, need, f"{what} plain")
        c.check(ot, want)
        if narrow:
            c = Call(at, ot, sparse, narrow, 10, groups, sizes, "none", None, accumulate, inits, f"{what} unscaled",
                     temp=temp)
            _assert_scratch_kept(big, start, need, f"{what} unscaled")
            c.check(ot, expect(at, ot, narrow, hw, None, inits, False))


@pytest.mark.parametrize("t", ["f16", "bf16", "f32"])
def test_exact_scratch_of_the_standalone_norm(t):
    from dietgpu_b200 import capi, ops

    sizes = [0, 1, 4097, 70001, 0, 300001, 33, 0]
    ts = [E.device_words(_finite_words(t, n, 9 + i), t) for i, n in enumerate(sizes)]
    need = capi.lib().dgb_float_sq_norm_temp_bytes(len(sizes), capi.u32_array(sizes))
    big, temp, start = _exact_temp(need, lead=3)
    got = ops.sq_norm(ts, temp_mem=temp).cpu().numpy()
    torch.cuda.synchronize()
    _assert_scratch_kept(big, start, need, f"{t} sq_norm")
    for i, x in enumerate(ts):
        assert R.same(got[i], R.sq_norm(x.double().cpu().numpy())), (t, i)


# ---- g: a graph replayed after an intruder call of the same family ----------------------------------------------------

@pytest.mark.parametrize("kind", ["bf16-narrow", "f16s-narrow"])
def test_graph_replay_after_an_intruder(kind):
    """A narrowing + norm call of 70 groups at W = 2 (scratch member table, narrowing table, 70 partial offsets)
    captured on a side stream after a warm-up.  Before each replay an eager call of the same family with other group
    counts and sizes rebuilds every host-side table; the replay, with the scale rewritten by fill_, equals an eager
    call on the captured shape, outputs and norms, and the intruder's results stay as they were."""
    from dietgpu_b200 import ops

    at, sparse, ot, _ = NORM_KINDS[kind]
    T = TORCH[at]
    sizes = SIZES70[3:73]
    hw = shaped_groups(at, sparse, sizes, 2, 5)
    groups = compress_groups(at, sparse, 10, hw)
    sc = _scale(0.5)
    outs = [torch.empty(n, dtype=T, device="cuda") for n in sizes]
    accs = [torch.empty(n, dtype=torch.float32, device="cuda") for n in sizes]
    norms = torch.empty(len(sizes), dtype=torch.float64, device="cuda")
    temp = torch.empty(32 << 20, dtype=torch.uint8, device="cuda")
    kw = dict(archive_dtype=T, sparse=sparse, reduce_dtype=torch.float32, acc=accs, scale_tensor=sc, sq_norm=norms)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.decompress_data_reduce(groups, outs, False, temp, **kw)  # warm-up
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        ops.decompress_data_reduce(groups, outs, False, temp, **kw)

    isizes = [4097, 0, 70001, 1, 12345, 0, 262144]
    ihw = shaped_groups(at, sparse, isizes, 3, 9)
    igroups = compress_groups(at, sparse, 10, ihw)
    for s in (0.25, -3.0, float(np.float32(1 / 3))):
        intr = Call(at, at, sparse, True, 10, igroups, isizes, "dev", 7.0, False, None, f"intruder before {s}",
                    sq=True)
        ikeep = [b.clone() for b in intr.bufs]
        sc.fill_(s)
        norms.fill_(-1.0)
        for o in outs:
            o.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        eager = Call(at, at, sparse, True, 10, groups, sizes, "dev", s, False, None, f"eager {s}", sq=True)
        for g in range(len(sizes)):
            ok = W.same_dev(outs[g], eager.outs[g])
            assert bool(ok.all()), f"replay with scale {s} group {g}: != the eager call"
        got = norms.cpu().numpy()
        assert all(R.same(a, b) for a, b in zip(got, eager.norms)), f"replay with scale {s}: norms"
        eager.check(at, expect(at, at, True, hw, s, None, True), f"eager {s}")
        for g in range(len(isizes)):
            assert torch.equal(intr.bufs[g], ikeep[g]), f"replay with scale {s}: the intruder's group {g} changed"
        intr.check(at, expect(at, at, True, ihw, 7.0, None, True), f"intruder at {s}")


# ---- h: the standalone norm -------------------------------------------------------------------------------------------

def _placed(words, t, off):
    x = E.device_words(words, t)
    base = torch.empty(x.numel() + 8, dtype=x.dtype, device="cuda")
    v = base[off:off + x.numel()]
    v.copy_(x)
    return v


def _assert_norms(ts, what, want=None):
    """ops.sq_norm(ts) equals the restatement bit for bit (want: the expected norms, else from the tensors)."""
    from dietgpu_b200 import ops

    got = ops.sq_norm(ts).cpu().numpy()
    for i, x in enumerate(ts):
        w = R.sq_norm(x.double().cpu().numpy()) if want is None else want[i]
        assert R.same(got[i], w), f"{what} tensor {i} ({x.numel()} words): {got[i]!r} != {w!r}"


@pytest.mark.parametrize("t", ["f16", "bf16", "f32"])
def test_standalone_norm_on_the_corpora(t):
    """Every shape of both corpora at element offsets 0-7, in one call per offset."""
    dense, sparse = E.corpus(t), S.corpus(t)
    hs = [dense[g, j] for g in range(len(E.SIZES)) for j in range(4)]
    hs += [sparse[g, j] for g in range(len(S.SIZES)) for j in range(len(S.SHAPES))]
    want = [R.sq_norm(to_f64(h, t)) for h in hs]
    assert any(np.isfinite(v) and v > 0 for v in want) and any(not np.isfinite(v) for v in want)
    for off in range(8):
        _assert_norms([_placed(h, t, off) for h in hs], f"{t} offset {off}", want)


def _finite_words(t, n, seed):
    """N(0, 1) at a per-tensor scale, with +-0 and (fp16 / bf16) subnormals: a finite norm that every word moves."""
    rng = np.random.default_rng(seed)
    x = torch.from_numpy(rng.standard_normal(n).astype(np.float32) * np.float32(2.0 ** int(rng.integers(-8, 8))))
    w = x.to(TORCH[t]).view(torch.int32 if t == "f32" else torch.int16).numpy().view(E.WORD[t]).copy()
    w[3::11] = 0
    w[5::13] = 0x8000 if t != "f32" else 0x80000000
    w[7::17] = 0x0003 if t != "f32" else 0x00000005
    return w


@pytest.mark.parametrize("t", ["f16", "bf16", "f32"])
def test_standalone_norm_many_tensors_and_block_edges(t):
    """1000 tensors in one call with empty ones interleaved and last; sizes around the fold's 256 partials."""
    rng = np.random.default_rng(4)
    sizes = [0 if i % 7 == 3 else int(rng.integers(1, 9000)) for i in range(999)] + [0]
    host = [_finite_words(t, n, i) for i, n in enumerate(sizes)]
    _assert_norms([E.device_words(h, t) for h in host], f"{t} 1000 tensors", [R.sq_norm(to_f64(h, t)) for h in host])
    edges = [256 * 4096 - 1, 256 * 4096, 256 * 4096 + 1, 257 * 4096]
    ts = [E.device_words(_finite_words(t, n, 3 + i), t) for i, n in enumerate(edges)]
    ts.append(ts[2].clone())
    ts[-1][5 * 4096 + 7] = float("inf")
    _assert_norms(ts, f"{t} around 256 blocks")


def test_standalone_norm_past_one_wave():
    """40 Mi fp32 words: 10240 blocks, past the grid's smCount * 8 CTAs of 8 warps, so warps take a second block."""
    n = 40 << 20
    g = torch.Generator(device="cuda").manual_seed(12)
    x = torch.randn(n, generator=g, device="cuda") * torch.rand(n // 4096, 1, generator=g, device="cuda").repeat(
        1, 4096).reshape(-1)
    _assert_norms([x, x[4096 * 9000:]], "40 Mi words")
