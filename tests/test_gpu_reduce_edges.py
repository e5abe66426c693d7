"""Decode-and-sum (ops.decompress_data_reduce) against the float64 fold of tests/reduce_reference.py, on the
inputs that reach every branch of decodeReduceKernel:

  - a block's stream is staged in the warp's shared-memory slot by TMA when it fits the slot (1536 words by
    default) and is read from global memory otherwise; both branches run under the store writer (archive 0 of a
    non-accumulating call) and the add writer (every later archive), for every archive / output type pair;
  - blocks whose stream is empty (one-symbol archives, pdf = 2^probBits) and the 256 * probBits-word worst case;
  - the first launch and the later launches of the kReducePass = 4 archives per launch;
  - the slot size forced down to 8 words and up to the worst case, and member tables read from scratch;
  - every 16-bit pair through the fp16 / bf16 adds and their widened fp32 form;
  - archives from every encoder variant, with checksums, from the CPU oracle and from the narrowing compress.

The corpus of one (archive type, probBits) mixes four shapes inside every group, so consecutive archives of one
block alternate between the two stream branches and between LUTs:
  worst     a constant archive except block min(5, last) whose coded symbols occur nowhere else; at 262144 and
            300001 elements every symbol of that block normalises to pdf 1 and the block costs 256 * pb words
  empty     one value everywhere (+0, -0, 1.0 or a NaN payload): every block codes to 0 words
  over      full-range words (a shuffled arange of every 16-bit pattern, random fp32 words with NaN, +-inf and
            subnormals): uniform exponents, about 2048 words per full block
  ordinary  randn at different scales
Every call checks which blocks its archives hold (the host parses the block tables), so a change to the slot
size or to the corpus that leaves a branch unexercised fails here instead of passing quietly."""
import time

import numpy as np
import pytest
import torch

from codec_helpers import KINDS, assert_guard_intact, codec_options, guarded_out, to_dev_bytes
from oracle import oracle as O
from reduce_reference import WORD, assert_same_words, fold_ref, pair_operands

pytestmark = pytest.mark.gpu

PAIRS = [("f16", "f16"), ("bf16", "bf16"), ("f32", "f32"), ("f16", "f32"), ("bf16", "f32")]
SIZES = [1, 31, 33, 511, 513, 4095, 4097, 65537, 262144, 300001]
WIDTHS = [1, 2, 4, 5, 9]
SHAPES = ("worst", "empty", "over", "ordinary")
TORCH = {"f16": torch.float16, "bf16": torch.bfloat16, "f32": torch.float32}
DEFAULT_SLOT = 1536  # decoderSmem's float slot, in u16 words
MODES = {"default": {}, "slot8": dict(decode_slot_words=1), "slot_max": dict(decode_slot_words=4096),
         "inline0": dict(inline_members=0)}


# ---- corpus --------------------------------------------------------------------------------------------------

def _shape_words(t, shape, n, seed):
    rng = np.random.default_rng(seed)
    wt = WORD[t]
    if shape == "over":
        if t == "f32":
            w = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
            w[::101] = 0x7FC00123
            w[7::103] = 0xFF800000
            w[9::107] = 0x7F800000
            w[3::109] &= np.uint32(0x807FFFFF)  # subnormals
            return w
        perm = rng.permutation(1 << 16).astype(np.uint16)
        return np.resize(perm, n)
    if shape == "empty":
        one = {"f16": (0x0000, 0x8000, 0x3C00, 0x7E01), "bf16": (0x0000, 0x8000, 0x3F80, 0x7FC1),
               "f32": (0, 0x80000000, 0x3F800000, 0x7FC00123)}[t][seed % 4]
        return np.full(n, one, wt)
    if shape == "worst":
        base = {"f16": 0x3C00, "bf16": 0x3F80, "f32": 0x3F800000}[t]
        s0 = base >> {"f16": 8, "bf16": 7, "f32": 23}[t]
        w = np.full(n, base, wt)
        if n == 0:
            return w
        nb = -(-n // 4096)
        k = min(5, nb - 1)
        m = min(4096, n - 4096 * k)
        sym = rng.integers(0, 255, m)
        sym = np.where(sym >= s0, sym + 1, sym).astype(np.uint64)
        if t == "f16":
            blk = (sym << 8) | rng.integers(0, 256, m, dtype=np.uint64)
        elif t == "bf16":
            blk = (rng.integers(0, 2, m, dtype=np.uint64) << 15) | (sym << 7) | rng.integers(0, 128, m, dtype=np.uint64)
        else:
            blk = ((rng.integers(0, 2, m, dtype=np.uint64) << 31) | (sym << 23)
                   | rng.integers(0, 1 << 23, m, dtype=np.uint64))
        w[4096 * k:4096 * k + m] = blk.astype(wt)
        return w
    scale = [2.0 ** -12, 1.0, 2.0 ** 9][seed % 3] if t == "f16" else [1e-30, 1.0, 1e30][seed % 3]
    x = torch.from_numpy(rng.standard_normal(n)) * scale
    return x.to(TORCH[t]).view(torch.int32 if t == "f32" else torch.int16).numpy().view(wt)


_WORDS = {}


def corpus(t):
    """{(group, archive): words} for every size of SIZES and archive index 0..8; shape SHAPES[(g + j) % 4]."""
    if t not in _WORDS:
        _WORDS[t] = {(g, j): _shape_words(t, SHAPES[(g + j) % 4], n, 1000 * g + j + 7)
                     for g, n in enumerate(SIZES) for j in range(max(WIDTHS))}
    return _WORDS[t]


def device_words(w, t):
    return torch.from_numpy(w.view(np.int32 if t == "f32" else np.int16).copy()).view(TORCH[t]).cuda()


def block_words(arch_host, t):
    """Stream words of every block of a float archive (host bytes)."""
    a = np.ascontiguousarray(arch_host).view(np.uint8)
    n = int(a[4:8].view(np.uint32)[0])
    ans = a[16 + O.float_noncomp_bytes(KINDS[t][0], n):]
    return (O.parse_ans(ans)["block_words"][:, 0] & 0xFFFF).astype(np.int64)


def compress_lib(ts, pb, checksum=False, archive_dtype=None):
    from dietgpu_b200 import ops

    comp, sizes, _ = ops.compress_data(True, ts, checksum, prob_bits=pb, archive_dtype=archive_dtype)
    hs = sizes.cpu().tolist()
    return [comp[i, :hs[i]] for i in range(len(ts))]


_ARCH = {}


def library_archives(t, pb):
    """{(g, j): (device archive, block words)} of the corpus, from the library's default encoder."""
    key = (t, pb)
    if key not in _ARCH:
        words = corpus(t)
        out = {}
        for g in range(len(SIZES)):
            js = range(max(WIDTHS))
            arch = compress_lib([device_words(words[g, j], t) for j in js], pb)
            for j, a in zip(js, arch):
                out[g, j] = (a, block_words(a.cpu().numpy(), t))
        _ARCH.clear()  # one (type, pb) at a time keeps device memory small
        _ARCH[key] = out
    return _ARCH[key]


def init_words(t, n, seed):
    """Accumulate inits of type t: randn with NaN, +-0, +-inf, subnormals and (fp32) values no 16-bit type holds."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(n).astype(np.float32)
    if t == "f32":
        x[2::5] = np.float32(1.0 + 2.0 ** -20) * np.float32(2.0) ** rng.integers(-20, 20, x[2::5].size)
        x[4::17] = np.float32(1e-40)
        x[6::17] = np.float32(-3e-42)
    x[0::7] = np.nan
    x[1::11] = 0.0
    x[3::11] = -0.0
    x[5::13] = np.inf
    x[8::13] = -np.inf
    w = x.view(np.uint32)
    if t == "f32":
        return w.copy()
    h = torch.from_numpy(x).to(TORCH[t]).view(torch.int16).numpy().view(np.uint16).copy()
    h[9::19] = 0x0001 if t == "f16" else 0x0003  # subnormals of the 16-bit type
    h[10::19] = 0x83FF if t == "f16" else 0x807F
    return h


def to_host_words(v, t):
    return v.view(torch.int32 if t == "f32" else torch.int16).cpu().numpy().view(WORD[t])


def reduce_and_check(at, ot, pb, groups, words, accumulate, what, seed=0):
    """groups: list of lists of device archives (one group per output); words: the matching host words.
    Sums them into guard-banded outputs and checks every group against fold_ref."""
    from dietgpu_b200 import ops

    bufs, outs, spans, inits = [], [], [], []
    for g, grp in enumerate(words):
        n = grp[0].size
        b, v, span = guarded_out(n, TORCH[ot], (g * 3 + 1) % 8)
        init = None
        if accumulate:
            init = init_words(ot, n, seed + g)
            v.copy_(device_words(init, ot))
        bufs.append(b)
        outs.append(v)
        spans.append(span)
        inits.append(init)
    st = torch.zeros(sum(len(grp) for grp in groups), dtype=torch.uint8, device="cuda")
    ops.decompress_data_reduce(groups, outs, accumulate, None, st, prob_bits=pb, archive_dtype=TORCH[at])
    torch.cuda.synchronize()
    assert bool(st.all()), f"{what}: status {st.cpu().tolist()}"
    got = []
    for g, grp in enumerate(words):
        h = to_host_words(outs[g], ot)
        assert_same_words(h, fold_ref(grp, at, ot, inits[g]), ot, f"{what} group {g} n {grp[0].size}")
        assert_guard_intact(bufs[g], *spans[g], f"{what} group {g}")
        got.append(h)
    return got


def assert_paths_covered(bws, pb, what):
    """bws: block-word arrays of the archives one writer kind decodes in a call."""
    assert any(int(b.max(initial=0)) > DEFAULT_SLOT for b in bws), f"{what}: no block above the slot"
    assert any(int(b.max(initial=0)) == 256 * pb for b in bws), f"{what}: no {256 * pb}-word block"
    assert any(b.size > 0 and int(b.max()) == 0 for b in bws), f"{what}: no archive of empty streams"


# ---- a, b, c: the corpus under every writer kind, pass and slot mode --------------------------------------------

@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("pb", [9, 10, 11])
@pytest.mark.parametrize("at,ot", PAIRS, ids=[f"{a}-{o}" for a, o in PAIRS])
def test_corpus(at, ot, pb, mode):
    arch = library_archives(at, pb)
    words = corpus(at)
    for accumulate in (False, True):
        for w in WIDTHS:
            what = f"{at}->{ot} pb {pb} {mode} acc {accumulate} W {w}"
            store = [arch[g, 0][1] for g in range(len(SIZES))] if not accumulate else []
            add = [arch[g, j][1] for g in range(len(SIZES)) for j in range(0 if accumulate else 1, w)]
            for kind, bws in (("store", store), ("add", add)):
                if bws:
                    assert_paths_covered(bws, pb, f"{what} {kind} writer")
            groups = [[arch[g, j][0] for j in range(w)] for g in range(len(SIZES))]
            hw = [[words[g, j] for j in range(w)] for g in range(len(SIZES))]
            with codec_options(**MODES[mode]):
                reduce_and_check(at, ot, pb, groups, hw, accumulate, what, seed=17 * w + pb)


# ---- d: every 16-bit pair -----------------------------------------------------------------------------------------

def _assert_same_dev(got, want, what):
    it = torch.int32 if got.element_size() == 4 else torch.int16
    nan = torch.isnan(got) & torch.isnan(want)
    bad = (got.view(it) != want.view(it)) & ~nan
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} element(s) differ, first at {int(bad.nonzero()[0])}"


@pytest.mark.parametrize("t", ["f16", "bf16"])
def test_every_16bit_pair(t):
    """x0[i] = i & 0xffff, x1[i] = i >> 16 over all 2^32 pairs, in 64 chunks of 2^26: W = 2 sums in t and in fp32
    against torch's device adds, and the pairs with the pair_operands b set against fold_ref."""
    from dietgpu_b200 import ops

    T = TORCH[t]
    chunk = 1 << 26
    pb = 10
    x0 = torch.arange(1 << 16, dtype=torch.int32, device="cuda").to(torch.int16).repeat(chunk >> 16).view(T)
    a0 = compress_lib([x0], pb)[0]
    b_set = pair_operands(t)
    a_all = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    out16 = torch.empty(chunk, dtype=T, device="cuda")
    out32 = torch.empty(chunk, dtype=torch.float32, device="cuda")
    checked = 0
    t0 = time.time()
    for c in range(64):
        hi = (c << 10) + torch.arange(1024, dtype=torch.int32, device="cuda")
        x1 = hi.to(torch.int16).repeat_interleave(1 << 16).view(T)
        a1 = compress_lib([x1], pb)[0]
        ops.decompress_data_reduce([[a0, a1]], [out16], prob_bits=pb)
        ops.decompress_data_reduce([[a0, a1]], [out32], prob_bits=pb, archive_dtype=T)
        f0, f1 = x0.float(), x1.float()
        _assert_same_dev(out16, (f0 + f1).to(T), f"{t} chunk {c}")
        _assert_same_dev(out32, f0 + f1, f"{t} -> f32 chunk {c}")
        del f0, f1
        mine = b_set[(b_set >> 10) == c]
        if mine.size:
            idx = torch.from_numpy(((mine.astype(np.int64) & 1023) << 16)).cuda()
            sel = (idx[:, None] + torch.arange(1 << 16, device="cuda")[None, :]).reshape(-1)
            aa = np.tile(a_all, mine.size)
            bb = np.repeat(mine, 1 << 16)
            assert_same_words(to_host_words(out16[sel], t), fold_ref([aa, bb], t, t), t, f"{t} b set chunk {c}")
            assert_same_words(to_host_words(out32[sel], "f32"), fold_ref([aa, bb], t, "f32"), "f32",
                              f"{t} -> f32 b set chunk {c}")
            checked += mine.size
        del x1, a1, hi
    assert checked == b_set.size
    print(f"every {t} pair: {time.time() - t0:.1f} s")


# ---- e: every archive producer sums the same way ------------------------------------------------------------------

PRODUCER_GROUPS = [8, 6]  # 262144 (the 64-block worst case is archive 0) and 4097 elements; five archives each


@pytest.mark.parametrize("pb", [9, 10, 11])
@pytest.mark.parametrize("t", ["f16", "bf16", "f32"])
def test_every_producer_sums_the_same(t, pb):
    from test_gpu_variants import VARIANTS

    words = corpus(t)
    width = 5
    hw = [[words[g, j] for j in range(width)] for g in PRODUCER_GROUPS]
    outs_types = [t] if t == "f32" else [t, "f32"]
    dev = [[device_words(w, t) for w in grp] for grp in hw]

    def sums(groups, ref_words, what):
        return {ot: reduce_and_check(t, ot, pb, groups, ref_words, False, f"{what} -> {ot}") for ot in outs_types}

    def split(flat):
        return [flat[k * width:(k + 1) * width] for k in range(len(PRODUCER_GROUPS))]

    first = None
    for name, opts, role in VARIANTS:
        if role == "dec":
            continue
        for checksum in (False, True):
            with codec_options(**opts):
                arch = compress_lib([x for grp in dev for x in grp], pb, checksum)
            got = sums(split(arch), hw, f"{t} pb {pb} {name} checksum {checksum}")
            if first is None:
                first = got
            for ot in outs_types:
                for g in range(len(PRODUCER_GROUPS)):
                    assert np.array_equal(got[ot][g], first[ot][g]), f"{name} checksum {checksum} -> {ot} group {g}"
    for checksum in (False, True):
        arch = [to_dev_bytes(O.float_compress(KINDS[t][0], w, pb, checksum)) for grp in hw for w in grp]
        got = sums(split(arch), hw, f"{t} pb {pb} oracle checksum {checksum}")
        for ot in outs_types:
            for g in range(len(PRODUCER_GROUPS)):
                assert np.array_equal(got[ot][g], first[ot][g]), f"oracle checksum {checksum} -> {ot} group {g}"
    if t != "f32":
        # the narrowing compress of the exact fp32 values: the archives are those of x.to(T), which differs from the
        # words only in NaN payloads
        xs = [x.float() for grp in dev for x in grp]
        narrowed = [to_host_words(x.to(TORCH[t]), t) for x in xs]
        for checksum in (False, True):
            arch = compress_lib(xs, pb, checksum, archive_dtype=TORCH[t])
            got = sums(split(arch), split(narrowed), f"{t} pb {pb} narrowing checksum {checksum}")
            for ot in outs_types:
                for g in range(len(PRODUCER_GROUPS)):
                    assert_same_words(got[ot][g], first[ot][g], ot, f"narrowing checksum {checksum} -> {ot} group {g}")


# ---- f: one archive in several places, groups of 0 to 2 Mi elements ----------------------------------------------

@pytest.mark.parametrize("t", ["f16", "bf16", "f32"])
def test_repeated_archives_and_group_sizes(t):
    words = corpus(t)
    arch = library_archives(t, 10)
    a, b, c = arch[7, 0][0], arch[7, 1][0], arch[7, 2][0]
    wa, wb, wc = words[7, 0], words[7, 1], words[7, 2]
    for ot in ([t] if t == "f32" else [t, "f32"]):
        for accumulate in (False, True):
            reduce_and_check(t, ot, 10, [[a, a, b], [b, a, a], [a, c, a]], [[wa, wa, wb], [wb, wa, wa], [wa, wc, wa]],
                             accumulate, f"{t} -> {ot} repeated archive acc {accumulate}")
    rng = np.random.default_rng(3)
    sizes = [0, 1, 4096, 2 << 20, 0, 12345]
    hw = []
    for g, n in enumerate(sizes):
        grp = [_shape_words(t, SHAPES[(g + j) % 4], n, 50 * g + j) for j in range(3)]
        grp[rng.integers(0, 3)] = _shape_words(t, "over", n, 99 + g)
        hw.append(grp)
    archs = compress_lib([device_words(w, t) for grp in hw for w in grp], 10)
    groups = [archs[3 * g:3 * g + 3] for g in range(len(sizes))]
    for ot in ([t] if t == "f32" else [t, "f32"]):
        for accumulate in (False, True):
            reduce_and_check(t, ot, 10, groups, hw, accumulate, f"{t} -> {ot} sizes 0..2Mi acc {accumulate}")
