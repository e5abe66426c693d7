"""Error feedback (kinds 0xC1 / 0xC2: dgb_float_compress_to_ef, ops.compress_data(error_feedback=)) pinned to the
numpy contract and the CPU oracle, on the narrowing edge corpus and on crafted members, under every encoder option
that selects another kernel or code path, with guard-banded inputs, residuals, archive rows and scratch.  It is the
one encoder that writes caller memory besides the archive: the residual e of every member, in place.

Reference of a member: ef_reference.np_step(x, e) gives the expected residuals e' bit for bit and the expected 16-bit
words w.  The CPU keeps NaN payloads and the device does not, so a NaN y expects the one word torch's CUDA cast gives
a NaN, after checking that every NaN payload of the member casts to that word.  Then the archive equals
oracle_archive(w) (byte for byte under encode_canonical=1, by O.assert_same_float otherwise) and decodes to w, and
torch's device expression (test_gpu_wire_error_feedback.torch_step) gives the same words and residuals.

Buffers: every input and residual passed to a kernel sits at element offset 0-3 inside an int32 buffer of its own with
32 words (128 B) of guard on either side (a partial row that strays reaches at most 31 words past a member's end);
input and residual share their address modulo 16.  The guards hold a NaN pattern, so a stray residual store (+0 for a
NaN y) shows.  After each call every input buffer is as it was, every residual guard holds its pattern, and every
archive row (prefilled with SENTINEL) still holds SENTINEL from the reported size to its end.

The module's name sorts after every other GPU module, so in a single-process run of the suite it runs last.  Its
profiler check, like every other one of the suite, runs in a fresh process (multirank.run_ranks with one rank)."""
import re
import time

import numpy as np
import pytest
import torch

from codec_helpers import GUARD, KINDS, SENTINEL, assert_pdf_matches, codec_options, guarded_decode, oracle_archive
from ef_reference import _widen, np_step
from multirank import run_ranks
from oracle import oracle as O
from test_gpu_narrow import FAMILIES, SIZES, TYPES, family
from test_gpu_variants import VARIANTS
from test_gpu_wire_error_feedback import residual_pool, torch_step

pytestmark = pytest.mark.gpu

EF_GUARD = 32            # words of guard on either side of every input and residual buffer (128 B)
NAN_GUARD = 0x7FA5A5A5   # the guard word: a NaN
EF_KINDS = {torch.float16: 193, torch.bfloat16: 194}  # 0x80 | 0x40 | the archive type
MANT = {torch.float16: 10, torch.bfloat16: 7}          # stored mantissa bits of the archive type
MAX_EXP = {torch.float16: 30, torch.bfloat16: 254}     # largest finite biased exponent


def _bits(t):
    return t.view(torch.int32 if t.element_size() == 4 else torch.int16)


def _dev(u32):
    return torch.from_numpy(np.ascontiguousarray(u32, np.uint32).view(np.int32)).cuda()


def _host_u32(t):
    return t.view(torch.int32).cpu().numpy().view(np.uint32)


def _host_u16(t):
    return t.view(torch.int16).cpu().numpy().view(np.uint16)


# ---- guarded buffers ------------------------------------------------------------------------------------------------

class Guarded:
    """n float32 words at element offset `off` (0-3) inside an int32 buffer of NAN_GUARD words with at least EF_GUARD
    words on either side; the buffer starts 256 B aligned, so the words sit at 4 * off B modulo 16."""

    def __init__(self, n, off, words=None):
        self.buf = torch.full((n + 2 * EF_GUARD + 4,), NAN_GUARD, dtype=torch.int32, device="cuda")
        assert self.buf.data_ptr() % 16 == 0
        self.lo, self.hi = EF_GUARD + off, EF_GUARD + off + n
        self.view = self.buf[self.lo:self.hi].view(torch.float32)
        if words is not None:
            self.view.view(torch.int32).copy_(words if isinstance(words, torch.Tensor) else _dev(words))

    def guards_intact(self):
        return bool((self.buf[:self.lo] == NAN_GUARD).all()) and bool((self.buf[self.hi:] == NAN_GUARD).all())


def place(xh, eh, offsets):
    """Every member in buffers of its own: (input buffers, residual buffers, input views, residual views)."""
    xb = [Guarded(x.size, o, x) for x, o in zip(xh, offsets)]
    eb = [Guarded(e.size, o, e) for e, o in zip(eh, offsets)]
    return xb, eb, [b.view for b in xb], [b.view for b in eb]


def place_touching(xh, eh, off):
    """Every member back to back in one input buffer and one residual buffer (both at element offset off)."""
    xb = Guarded(sum(x.size for x in xh), off, np.concatenate(xh))
    eb = Guarded(sum(e.size for e in eh), off, np.concatenate(eh))
    cut = np.concatenate([[0], np.cumsum([x.size for x in xh])])
    xs = [xb.view[int(a):int(b)] for a, b in zip(cut[:-1], cut[1:])]
    es = [eb.view[int(a):int(b)] for a, b in zip(cut[:-1], cut[1:])]
    return [xb], [eb], xs, es


# ---- the reference ----------------------------------------------------------------------------------------------------

_NAN_WORD = {}


def nan_word(dtype):
    if dtype not in _NAN_WORD:
        _NAN_WORD[dtype] = int(_host_u16(torch.tensor([float("nan")], device="cuda").to(dtype))[0])
    return _NAN_WORD[dtype]


def words16(wf, dtype):
    """The 16-bit words of float32 values that are exactly words of the archive type (not NaN)."""
    if dtype == torch.float16:
        return wf.astype(np.float16).view(np.uint16)
    return (wf.view(np.uint32) >> 16).astype(np.uint16)


def expected(xh, eh, dtype):
    """(w, e') of a member by np_step: uint16 words and uint32 residual bits."""
    y, wf, res = np_step(xh.view(np.float32), eh.view(np.float32), dtype)
    nan = np.isnan(y)
    w = words16(np.where(nan, np.float32(0), wf), dtype).copy()
    if nan.any():
        casts = _host_u16(torch.from_numpy(y[nan]).cuda().to(dtype))
        assert (casts == nan_word(dtype)).all(), f"NaN payloads cast to {sorted(set(casts.tolist()))[:4]} on the device"
        w[nan] = nan_word(dtype)
    return w, res.view(np.uint32).copy()


# ---- one call and its checks ------------------------------------------------------------------------------------------

def ef_call(xs, es, dtype, pb, checksum, temp=None):
    """compress_data(error_feedback=) into sentinel-prefilled rows of cols + GUARD bytes: (rows, host sizes)."""
    from dietgpu_b200 import ops

    n = len(xs)
    cols = ops.max_float_compressed_size(torch.empty(0, dtype=dtype), max(max(x.numel() for x in xs), 1))
    assert cols % 16 == 0
    comp = torch.full((n, cols + GUARD), SENTINEL, dtype=torch.uint8, device="cuda")
    _, sizes, _ = ops.compress_data(True, xs, checksum, temp, comp, None, prob_bits=pb, archive_dtype=dtype,
                                    error_feedback=es)
    return comp, sizes.cpu().tolist()


def assert_rows_clean(comp, hs, what):
    stray = [i for i in range(len(hs)) if not bool((comp[i, hs[i]:] == SENTINEL).all())]
    assert not stray, f"{what}: bytes written past the archive size in rows {stray[:8]}"


def check_archives(comp, hs, ws, dtype, pb, checksum, canonical, what):
    """Every member's archive against the oracle's archive of its expected words; decodes to them."""
    kind = TYPES[dtype]
    ft = KINDS[kind][0]
    host = comp[:, :max(hs) if hs else 0].cpu().numpy()
    for i, w in enumerate(ws):
        want = oracle_archive(kind, w, pb, checksum)
        assert hs[i] == want.size, f"{what} member {i} ({w.size} words): size {hs[i]} != oracle {want.size}"
        if canonical:
            assert np.array_equal(host[i, :hs[i]], want), f"{what} member {i}: canonical archive != the oracle's"
        else:
            O.assert_same_float(host[i, :hs[i]], want, ft, f"{what} member {i} vs oracle")
    rows = [comp[i, :hs[i]] for i in range(len(ws))]
    expect = [torch.from_numpy(w.view(np.int16)).cuda().view(dtype) for w in ws]
    guarded_decode(True, rows, [w.size for w in ws], dtype, pb, checksum, expect, what)
    return host


def run_checked(xh, eh, placed, dtype, pb, checksum, opts=None, what="", plain=None, temp=None):
    """One EF call on placed buffers holding xh / eh (host uint32 words), with every check of the module docstring.
    plain: the residuals are all -0 ("x": y = x, so the archives must also equal the plain narrowing compress of x) or
    all +0 ("y": y = x with -0 turned +0, the plain narrowing compress of torch's x + e)."""
    from dietgpu_b200 import ops

    opts = dict(opts or {})
    canonical = opts.get("encode_canonical", 0) == 1
    xb, eb, xs, es = placed
    ref = [expected(x, e, dtype) for x, e in zip(xh, eh)]
    # torch's expression, computed on the device before the call overwrites the residuals
    tw, tr = [], []
    for x, e in zip(xs, es):
        y, r = torch_step(x, e.clone(), dtype)
        tw.append(_host_u16(y.to(dtype)))
        tr.append(_host_u32(r))
    before = [b.buf.clone() for b in xb]
    if plain == "y":
        ys = [Guarded(x.numel(), (x.data_ptr() % 16) // 4, _bits(x + e)).view for x, e in zip(xs, es)]
    with codec_options(**opts):
        comp, hs = ef_call(xs, es, dtype, pb, checksum, temp)
        if plain:
            pc, phs = ef_call_plain(xs if plain == "x" else ys, dtype, pb, checksum)
    torch.cuda.synchronize()
    for k, b in enumerate(xb):
        assert torch.equal(b.buf, before[k]), f"{what}: an input buffer changed (input or guard)"
    for k, b in enumerate(eb):
        assert b.guards_intact(), f"{what}: residual buffer {k}: a guard word was written"
    assert_rows_clean(comp, hs, what)
    for i, (w, r) in enumerate(ref):
        got = _host_u32(es[i])
        bad = np.flatnonzero(got != r)
        assert bad.size == 0, f"{what} member {i}: residual != np_step at {bad[:8].tolist()} " \
                              f"(got {[hex(v) for v in got[bad[:4]]]}, want {[hex(v) for v in r[bad[:4]]]})"
        assert np.array_equal(tr[i], r), f"{what} member {i}: torch's residual != np_step"
        assert np.array_equal(tw[i], w), f"{what} member {i}: torch's cast of y != np_step's words"
    host = check_archives(comp, hs, [w for w, _ in ref], dtype, pb, checksum, canonical, what)
    if plain:
        assert phs == hs, f"{what}: sizes {hs} != the plain narrowing compress's {phs}"
        ph = pc[:, :max(hs) if hs else 0].cpu().numpy()
        for i in range(len(xs)):
            if canonical:
                assert np.array_equal(host[i, :hs[i]], ph[i, :hs[i]]), f"{what} member {i}: != plain narrowing"
            else:
                O.assert_same_float(host[i, :hs[i]], ph[i, :hs[i]], KINDS[TYPES[dtype]][0],
                                    f"{what} member {i} vs plain narrowing")
    return comp, hs


def ef_call_plain(xs, dtype, pb, checksum):
    from dietgpu_b200 import ops

    comp, sizes, _ = ops.compress_data(True, xs, checksum, prob_bits=pb, archive_dtype=dtype)
    return comp, sizes.cpu().tolist()


def run_separate(xh, eh, offsets, dtype, pb, checksum, opts=None, what="", plain=None):
    return run_checked(xh, eh, place(xh, eh, offsets), dtype, pb, checksum, opts, what, plain)


# ---- the kernel list (first: the profiler's window must not see another module's work) ---------------------------------

def test_profiler_sees_every_ef_instantiation():
    # in a fresh process: in a long-lived one the GPU's timestamps drift against the host clock that bounds the
    # profiler's window, and every record of a window can fall outside it
    run_ranks(_profiler_sees_every_ef_instantiation, 1, backend="gloo")


def _profiler_sees_every_ef_instantiation(rank, world, dev):
    """statsFloatEfKernel<193|194>, encodeKernelFastEf<false|true, 193|194> and encodeKernelEf<193|194> run; the fused
    and staged options fall back to them (no fused or staged kernel runs), and no plain narrowing kernel runs."""
    from torch.profiler import ProfilerActivity, profile

    from dietgpu_b200 import ops

    sizes = [70001, 4096, 33]
    xs = [torch.randn(n, device="cuda") for n in sizes]
    runs = [dict(), dict(encode_wide_table=0), dict(encode_wide_table=1), dict(encode_canonical=1),
            dict(encode_fused=1), dict(encode_fused=1, fused_stage=1), dict(stats_stage=1)]
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(1.0)
        torch.ones(1, device="cuda").add_(1)  # the first kernel of a session can be missing from its trace
        for _ in range(3):
            for opts in runs:
                with codec_options(**opts):
                    for dtype in TYPES:
                        es = [torch.zeros(n, device="cuda") for n in sizes]
                        ops.compress_data(True, xs, True, archive_dtype=dtype, error_feedback=es)
        torch.cuda.synchronize()
        time.sleep(1.0)
    names = {re.sub(r"\s", "", e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    for kind in EF_KINDS.values():
        for want in (f"statsFloatEfKernel<{kind}>", f"encodeKernelFastEf<false,{kind}>",
                     f"encodeKernelFastEf<true,{kind}>", f"encodeKernelEf<{kind}>"):
            assert any(want in k for k in names), (want, sorted(names))
    assert not any("encodeFusedKernel" in k or "statsFloatStagedKernel" in k for k in names), sorted(names)
    for kind in (65, 66):  # the narrowing kinds without error feedback
        for never in (f"statsFloatKernel<{kind}>", f"encodeKernelFast<false,{kind}>", f"encodeKernelFast<true,{kind}>",
                      f"encodeKernel<{kind}>"):
            assert not any(never in k for k in names), (never, sorted(names))


# ---- the edge corpus --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", list(TYPES))
@pytest.mark.parametrize("pb", [9, 10, 11])
@pytest.mark.parametrize("checksum", [False, True])
def test_edge_corpus(dtype, pb, checksum):
    """Every test_gpu_narrow family at test_gpu_narrow.SIZES, four members per size at element offsets 0-3, with
    residuals from residual_pool (signed zeros, 3e4, inf, NaN), all +0 and all -0, canonical and not.  With -0
    residuals y = x, so the archives also equal the plain narrowing compress's of x; with +0 ones y is x with -0 turned
    +0 (-0 + +0 = +0), and they equal the plain narrowing compress's of torch's x + e."""
    sizes = [n for n in SIZES for _ in range(4)]
    offsets = [off for _ in SIZES for off in range(4)]
    for fi, name in enumerate(FAMILIES):
        pool = family(name, seed=pb)
        xh = [pool[:n] for n in sizes]
        for res in ("pool", "+0", "-0"):
            eh = [residual_pool(max(n, 1), 1000 * fi + 7 * i + pb)[:n] if res == "pool" else
                  np.full(n, 0 if res == "+0" else 0x80000000, np.uint32) for i, n in enumerate(sizes)]
            for canonical in (0, 1):
                run_separate(xh, eh, offsets, dtype, pb, checksum, dict(encode_canonical=canonical),
                             f"{dtype} pb {pb} checksum {checksum} {name} e {res} canonical {canonical}",
                             plain={"pool": None, "+0": "y", "-0": "x"}[res])


# ---- option variants --------------------------------------------------------------------------------------------------

ENC_VARIANTS = [(name, opts, role) for name, opts, role in VARIANTS if role in ("enc", "exact")]
VARIANT_SIZES = [0, 1, 2, 3, 31, 33, 4095, 4097, 8209, 65537, 300001, 5, 4096, 70001]


@pytest.mark.parametrize("dtype", list(TYPES))
@pytest.mark.parametrize("name,opts,role", ENC_VARIANTS, ids=[v[0] for v in ENC_VARIANTS])
def test_option_variants(dtype, name, opts, role):
    """Every encoder-role option set of test_gpu_variants at probBits 10 with checksum; the canonical one byte for
    byte against the oracle."""
    assert (role == "exact") == (opts.get("encode_canonical", 0) == 1)
    n = len(VARIANT_SIZES)
    xh = [family(FAMILIES[i % len(FAMILIES)], s, seed=31 + i) for i, s in enumerate(VARIANT_SIZES)]
    eh = [residual_pool(max(s, 1), 500 + i)[:s] for i, s in enumerate(VARIANT_SIZES)]
    run_separate(xh, eh, [i % 4 for i in range(n)], dtype, 10, True, opts, f"{dtype} {name}")


# ---- crafted members --------------------------------------------------------------------------------------------------

def widen(w, dtype):
    """float32 values of uint16 words of the archive type"""
    return _widen(w.view(np.float16) if dtype == torch.float16 else w, dtype)


def ulp16(w, dtype):
    """float64 spacing above |w| (finite, below the largest finite word)."""
    mag = (w & 0x7FFF).astype(np.uint16)
    return (widen(mag + 1, dtype).astype(np.float64) - widen(mag, dtype).astype(np.float64))


def ulp32(f):
    return np.spacing(np.abs(f).astype(np.float32)).astype(np.float64)


def sign_of(w):
    return np.where(w & 0x8000, -1.0, 1.0)


def random_words(rng, n, dtype, exp_lo=1, exp_hi=None):
    """Finite words of the archive type with biased exponents in [exp_lo, exp_hi]."""
    m = MANT[dtype]
    exp_hi = MAX_EXP[dtype] - 1 if exp_hi is None else exp_hi
    e = rng.integers(exp_lo, exp_hi + 1, n).astype(np.uint32)
    return ((rng.integers(0, 2, n).astype(np.uint32) << 15) | (e << m) |
            rng.integers(0, 1 << m, n).astype(np.uint32)).astype(np.uint16)


def as_f32_bits(v64):
    """float64 values that are exact float32 values -> uint32 bits (asserted exact)."""
    f = v64.astype(np.float32)
    assert np.array_equal(f.astype(np.float64), v64), "not exact in float32"
    return f.view(np.uint32)


def carry(w, dtype, rng, k_max=3):
    """x = widen(w), e = d with d a few float32 ulps of x (sign of w for +-0): round(y) = w and e' = d."""
    wf = widen(w, dtype).astype(np.float64)
    k = rng.integers(1, k_max + 1, w.size)
    s = np.where((w & 0x7FFF) == 0, sign_of(w), rng.choice([-1.0, 1.0], w.size))
    d = s * k * ulp32(wf)
    x, e = as_f32_bits(wf), as_f32_bits(d)
    ww, r = expected(x, e, dtype)
    assert np.array_equal(ww, w) and np.array_equal(r, e), "carry: round(y) != w or e' != d"
    return x, e


def cross(w, dtype, rng):
    """d away from zero, past half a 16-bit ulp by a few float32 ulps: round(y) is the next word out, e' = d - ulp."""
    wf = widen(w, dtype).astype(np.float64)
    s, u = sign_of(w), ulp16(w, dtype)
    d = s * (u / 2 + rng.integers(1, 4, w.size) * ulp32(wf))
    x, e = as_f32_bits(wf), as_f32_bits(d)
    ww, r = expected(x, e, dtype)
    assert np.array_equal(ww, w + 1), "cross: round(y) is not the next word"
    assert np.array_equal(r.view(np.float32).astype(np.float64), d - s * u), "cross: e' != d - ulp"
    return x, e


def ties(w, dtype):
    """d = half an ulp away from zero (mantissa != 0 also toward zero): ties to even."""
    wf = widen(w, dtype).astype(np.float64)
    s, u = sign_of(w), ulp16(w, dtype)
    away = np.arange(w.size) % 2 == 0
    inner = (w & ((1 << MANT[dtype]) - 1)) != 0
    toward = ~away & inner
    d = np.where(toward, -s * u / 2, s * u / 2)
    x, e = as_f32_bits(wf), as_f32_bits(d)
    ww, _ = expected(x, e, dtype)
    odd = (w & 1) == 1
    want = np.where(odd, np.where(toward, w - 1, w + 1), w).astype(np.uint16)
    assert np.array_equal(ww, want), "ties: not to even"
    return x, e


def binade_bottom(dtype, rng, n):
    """Words with a zero stored mantissa whose exponent has a normal binade below it."""
    m = MANT[dtype]
    e = rng.integers(2, MAX_EXP[dtype], n).astype(np.uint32)
    return ((rng.integers(0, 2, n).astype(np.uint32) << 15) | (e << m)).astype(np.uint16)


def coded_symbol(w, dtype):
    return ((w >> 7) & 0xFF) if dtype == torch.bfloat16 else (w >> 8)


def symbol_changing(w, dtype):
    """w at the bottom of its binade: x = widen(w) - delta, e = delta (toward zero, 3/4 of the lower binade's ulp), so
    round(x) is the word below w, with another coded symbol, while round(y) = w and e' = +0."""
    wf = widen(w, dtype).astype(np.float64)
    s = sign_of(w)
    delta = 0.75 * (ulp16(w, dtype) / 2)  # the binade below has half the spacing
    x, e = as_f32_bits(wf - s * delta), as_f32_bits(s * delta)
    ww, r = expected(x, e, dtype)
    assert np.array_equal(ww, w) and (r == 0).all(), "symbol-changing: round(y) != w or e' != +0"
    wx, _ = expected(x, np.zeros_like(x), dtype)
    assert np.array_equal(wx, w - 1) and (coded_symbol(wx, dtype) != coded_symbol(w, dtype)).all()
    return x, e


def head_tail_member(dtype, rng, off, n):
    """A member of n < 512 words at element offset off whose statistics head and tail words (the scalar paths) are all
    symbol-changing; every coded symbol of y also occurs (at least twice) in the vector body."""
    head = (4 - off) % 4
    tail = (n - head) % 4
    assert head + tail > 0 and n < 512
    edge = list(range(head)) + list(range(n - tail, n))
    bw = binade_bottom(dtype, rng, len(edge))
    body_idx = np.setdiff1d(np.arange(n), edge)
    w = random_words(rng, n, dtype)
    # the edge words' symbols twice each in the body, and some body words symbol-changing too (the vector path)
    w[body_idx[:2 * len(edge)]] = np.repeat(bw, 2)
    w[body_idx[2 * len(edge):2 * len(edge) + 8]] = binade_bottom(dtype, rng, 8)
    w[edge] = bw
    x, e = carry(w, dtype, rng)
    sc = np.concatenate([edge, body_idx[2 * len(edge):2 * len(edge) + 8]])
    sx, se = symbol_changing(w[sc], dtype)
    x[sc], e[sc] = sx, se
    body_syms = set(coded_symbol(w[body_idx], dtype).tolist())
    assert set(coded_symbol(w, dtype).tolist()) <= body_syms
    return x, e


def carry_member(dtype, rng, n):
    """Carries, crossings past half an ulp and ties with even and odd kept bits, interleaved."""
    w = random_words(rng, n, dtype, exp_lo=1, exp_hi=MAX_EXP[dtype] - 1)
    w[::5] &= 0x8000 | (0xFFFF ^ ((1 << MANT[dtype]) - 1))  # some words at the bottom of their binade
    w[1::17] = (w[1::17] & 0x8000)  # +-0
    w[2::19] = (w[2::19] & 0x8000) | rng.integers(1, 1 << MANT[dtype], w[2::19].size).astype(np.uint16)  # subnormal
    x, e = carry(w, dtype, rng)
    c = (np.arange(n) % 7 == 3) & ((w & 0x7FFF) != 0)  # past half an ulp of +-0 is not exact in float32
    x[c], e[c] = cross(w[c], dtype, rng)
    t = np.arange(n) % 7 == 5
    x[t], e[t] = ties(w[t], dtype)
    return x, e


def worst_case_member(dtype, rng, pb):
    """64 blocks of words with one dominant coded symbol, except block 5 made of the other symbols only (each about 16
    times in 262144 words: pdf 1), which costs 256 * pb stream words (test_gpu_variants builds it for bytes).  Symbols
    of NaN words are left out (a NaN y takes the one NaN word); the infinities are x = inf, e = +0."""
    n = 64 * 4096
    syms = np.arange(256)
    if dtype == torch.bfloat16:
        dom, nan_syms = 127, []
        mk = lambda s, r: ((r.integers(0, 2, s.size) << 15) | (s << 7) |  # noqa: E731
                           np.where(s == 255, 0, r.integers(0, 1 << 7, s.size))).astype(np.uint16)
    else:
        dom, nan_syms = 0x3C, [0x7D, 0x7E, 0x7F, 0xFD, 0xFE, 0xFF]
        mk = lambda s, r: ((s << 8) | np.where((s & 0x7F) == 0x7C, 0, r.integers(0, 256, s.size))).astype(np.uint16)  # noqa: E731
    rare = np.setdiff1d(syms, [dom] + nan_syms)
    s = np.full(n, dom)
    s[5 * 4096:6 * 4096] = rare[rng.integers(0, rare.size, 4096)]
    w = mk(s, rng)
    assert set(coded_symbol(w[5 * 4096:6 * 4096], dtype).tolist()) <= set(rare.tolist())
    inf = (w & 0x7FFF) == (0x7F80 if dtype == torch.bfloat16 else 0x7C00)
    x = np.empty(n, np.uint32)
    e = np.zeros(n, np.uint32)
    x[inf] = widen(w[inf], dtype).view(np.uint32)
    x[~inf], e[~inf] = carry(w[~inf], dtype, rng)
    return x, e


def block_words(archive, dtype):
    a = np.ascontiguousarray(archive)
    n = int(a[4:8].view(np.uint32)[0])
    p = O.parse_ans(a[16 + O.float_noncomp_bytes(KINDS[TYPES[dtype]][0], n):])
    return p["block_words"][:, 0] & 0xFFFF


@pytest.mark.parametrize("dtype", list(TYPES))
@pytest.mark.parametrize("slot", ["default", "enc_slot_min"])
def test_crafted_members(dtype, slot):
    """At probBits 11: carries, crossings and ties at every offset; members shorter than 2^pb words with
    symbol-changing head and tail words (a count of round(x) instead of round(x + e) changes the pdf); the worst-case
    block at offset 0 (no scalar head or tail) with the slot forced to its minimum or not."""
    pb = 11
    rng = np.random.default_rng(11 + (dtype == torch.float16))
    xh, eh, offs = [], [], []
    for off in range(4):
        for n in (1, 2, 3, 7, 33, 4099, 20011):
            x, e = carry_member(dtype, rng, n)
            xh.append(x), eh.append(e), offs.append(off)
    for off in (1, 2, 3):
        for q in (6, 31, 126):  # a head of 4 - off words and a tail of 3
            x, e = head_tail_member(dtype, rng, off, 4 - off + 4 * q + 3)
            xh.append(x), eh.append(e), offs.append(off)
    for n in (30, 130, 509):  # offset 0: only a tail
        x, e = head_tail_member(dtype, rng, 0, n)
        xh.append(x), eh.append(e), offs.append(0)
    x, e = worst_case_member(dtype, rng, pb)
    xh.append(x), eh.append(e), offs.append(0)
    opts = dict(encode_slot_words=1) if slot == "enc_slot_min" else {}
    for checksum in (False, True):
        for canonical in (0, 1):
            what = f"{dtype} {slot} checksum {checksum} canonical {canonical}"
            comp, hs = run_separate(xh, eh, offs, dtype, pb, checksum, dict(opts, encode_canonical=canonical), what)
            bw = block_words(comp[-1, :hs[-1]].cpu().numpy(), dtype)
            assert int(bw[5]) == 256 * pb and int(bw.max()) == 256 * pb, f"{what}: worst-case block {bw[4:7]}"


# ---- touching and shared buffers, empty members -----------------------------------------------------------------------

TOUCH_SIZES = [1, 2, 3, 4095, 4097, 33, 5, 4096, 7, 65537, 1, 8209, 3, 300001, 2, 31, 4099, 6, 1, 12345, 3, 70001, 9,
               4093]


@pytest.mark.parametrize("opts", [dict(parts=2, first_part_pct=10, last_part_pct=200),
                                  dict(parts=4, first_part_pct=200, last_part_pct=10),
                                  dict(parts=8, first_part_pct=200, last_part_pct=200),
                                  dict(parts=1)], ids=["parts2", "parts4", "parts8", "parts1"])
@pytest.mark.parametrize("inline", [1, 0])
def test_touching_buffers(opts, inline):
    """Inputs and residuals back to back in one buffer each (member boundaries inside 16 B vectors), under unequal
    sub-batches, where one part's statistics pass runs beside another part's coder."""
    for dtype in TYPES:
        for off in (0, 3):
            xh = [family(FAMILIES[i % len(FAMILIES)], n, seed=70 + i) for i, n in enumerate(TOUCH_SIZES)]
            eh = [residual_pool(n, 900 + i) for i, n in enumerate(TOUCH_SIZES)]
            run_checked(xh, eh, place_touching(xh, eh, off), dtype, 10, True, dict(opts, inline_members=inline),
                        f"{dtype} touching at {off} {opts} inline {inline}")


def test_shared_inputs():
    """One input listed for three members (each with its own residual buffer), beside other members."""
    for dtype in TYPES:
        for canonical in (0, 1):
            x = family("normal_1", 20011, seed=4)
            xh = [x, family("ties", 4097, seed=5), x, x, family("carry", 33, seed=6)]
            eh = [residual_pool(s.size, 60 + i) for i, s in enumerate(xh)]
            offs = [1, 2, 1, 1, 3]
            xb, eb, xs, es = place(xh, eh, offs)
            xs[2] = xs[3] = xs[0]
            run_checked(xh, eh, ([xb[0], xb[1], xb[4]], eb, xs, es), dtype, 10, True, dict(encode_canonical=canonical),
                        f"{dtype} shared input canonical {canonical}")


def _raw_ef(ft, xs, sizes, errs, rows, out_sizes, pb, checksum, temp_ptr, temp_bytes):
    from dietgpu_b200 import capi

    return capi.lib().dgb_float_compress_to_ef(
        temp_ptr, temp_bytes, capi.FLOAT32, ft, pb, int(checksum), len(sizes), capi.ptr_array(xs),
        capi.u32_array(sizes), capi.ptr_array(errs), capi.ptr_array([r.data_ptr() for r in rows]),
        out_sizes.data_ptr(), torch.cuda.current_stream().cuda_stream)


def _exact_temp(need, lead):
    """temp_mem of exactly `need` bytes at a 256 B aligned start inside a larger sentinel-filled buffer."""
    big = torch.full((need + 256 + 2048,), SENTINEL, dtype=torch.uint8, device="cuda")
    start = 1024 + lead
    start += (-(big.data_ptr() + start)) % 256
    return big, start


def _check_raw(ft, dtype, xh, eh, off, empty_ptrs, pb, checksum, canonical, temp_lead=0, what=""):
    """dgb_float_compress_to_ef with exactly dgb_float_compress_temp_bytes of scratch; empty members pass a NULL
    residual (and input, when empty_ptrs says so)."""
    from dietgpu_b200 import capi, ops

    L = capi.lib()
    n = len(xh)
    xb, eb, xs, es = place(xh, eh, [off(i) for i in range(n)])
    sizes = [x.size for x in xh]
    ref = [expected(x, e, dtype) for x, e in zip(xh, eh)]
    need = L.dgb_float_compress_temp_bytes(ft, n, max(sizes))
    big, start = _exact_temp(need, temp_lead)
    cols = ops.max_float_compressed_size(torch.empty(0, dtype=dtype), max(max(sizes), 1))
    comp = torch.full((n, cols + GUARD), SENTINEL, dtype=torch.uint8, device="cuda")
    osz = torch.zeros(n, dtype=torch.int32, device="cuda")
    xp = [x.data_ptr() if s or not empty_ptrs else 0 for x, s in zip(xs, sizes)]
    ep = [e.data_ptr() if s else 0 for e, s in zip(es, sizes)]
    before = [b.buf.clone() for b in xb]
    with codec_options(encode_canonical=canonical):
        rc = _raw_ef(ft, xp, sizes, ep, [comp[i] for i in range(n)], osz, pb, checksum, big.data_ptr() + start, need)
    assert rc == capi.OK, (what, rc)
    torch.cuda.synchronize()
    head, tail = big[:start], big[start + need:]
    assert bool((head == SENTINEL).all()) and bool((tail == SENTINEL).all()), f"{what}: scratch written outside"
    for k, b in enumerate(xb):
        assert torch.equal(b.buf, before[k]), f"{what}: input buffer {k} changed"
    for k, b in enumerate(eb):
        assert b.guards_intact(), f"{what}: residual buffer {k}: a guard word was written"
    hs = osz.cpu().tolist()
    assert_rows_clean(comp, hs, what)
    for i, (w, r) in enumerate(ref):
        assert np.array_equal(_host_u32(es[i]), r), f"{what} member {i}: residual != np_step"
    check_archives(comp, hs, [w for w, _ in ref], dtype, pb, checksum, canonical, what)


def test_empty_members_with_null_residuals():
    from dietgpu_b200 import capi

    sizes = [0, 4097, 0, 1, 0, 33, 0]
    for dtype, ft in ((torch.float16, capi.FLOAT16), (torch.bfloat16, capi.BFLOAT16)):
        xh = [family(FAMILIES[i % len(FAMILIES)], n, seed=i) for i, n in enumerate(sizes)]
        eh = [residual_pool(max(n, 1), 40 + i)[:n] for i, n in enumerate(sizes)]
        for canonical in (0, 1):
            for null_in in (False, True):
                _check_raw(ft, dtype, xh, eh, lambda i: i % 4, null_in, 10, True, canonical,
                           what=f"{dtype} empty members canonical {canonical} null inputs {null_in}")


@pytest.mark.parametrize("members", [1, 64, 65, 256])
def test_exact_scratch(members):
    """Scratch of exactly dgb_float_compress_temp_bytes: the residual table in the kernel parameters (up to 64
    members, not canonical) or in the scratch (beyond 64 members, and canonical)."""
    from dietgpu_b200 import capi

    sizes = [(i * 7919 + 1) % 20011 for i in range(members)]
    for dtype, ft in ((torch.float16, capi.FLOAT16), (torch.bfloat16, capi.BFLOAT16)):
        xh = [family(FAMILIES[i % len(FAMILIES)], n, seed=200 + i) for i, n in enumerate(sizes)]
        eh = [residual_pool(max(n, 1), 300 + i)[:n] for i, n in enumerate(sizes)]
        for canonical in (0, 1):
            _check_raw(ft, dtype, xh, eh, lambda i: (3 * i + 1) % 4, False, 10, False, canonical, temp_lead=37 + members,
                       what=f"{dtype} {members} members canonical {canonical}")


# ---- steps: eager and replayed from one captured graph ----------------------------------------------------------------

STEP_SIZES = [1, 33, 4097, 20011, 70001]


def test_steps_eager_and_graph_equal_the_numpy_chain():
    """8 steps e_{k+1} = np_step(x_k, e_k): eager calls and replays of one captured call, each step's archives equal
    to the oracle's archives of its words and its residuals to the chain's."""
    from dietgpu_b200 import ops

    steps, n = 8, len(STEP_SIZES)
    offs = [i % 4 for i in range(n)]
    for dtype in TYPES:
        xk = [[family(FAMILIES[(i + k) % len(FAMILIES)], s, seed=100 * k + i) for i, s in enumerate(STEP_SIZES)]
              for k in range(steps)]
        e0 = [residual_pool(s, 77 + i) for i, s in enumerate(STEP_SIZES)]
        # eager
        xb, eb, xs, es = place(xk[0], e0, offs)
        chain = [e.copy() for e in e0]
        for k in range(steps):
            for i in range(n):
                xs[i].view(torch.int32).copy_(_dev(xk[k][i]))
            run_checked(xk[k], chain, (xb, eb, xs, es), dtype, 10, True, {}, f"{dtype} eager step {k}")
            chain = [expected(x, e, dtype)[1] for x, e in zip(xk[k], chain)]
        # one captured call, replayed
        gx, ge, gxs, ges = place(xk[0], e0, offs)
        cols = ops.max_float_compressed_size(torch.empty(0, dtype=dtype), max(STEP_SIZES))
        comp = torch.full((n, cols + GUARD), SENTINEL, dtype=torch.uint8, device="cuda")
        sizes = torch.zeros(n, dtype=torch.int32, device="cuda")
        scratch = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):  # warm-up outside the capture
            ops.compress_data(True, gxs, True, scratch, comp, sizes, archive_dtype=dtype, error_feedback=ges)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            ops.compress_data(True, gxs, True, scratch, comp, sizes, archive_dtype=dtype, error_feedback=ges)
        chain = [e.copy() for e in e0]
        for i in range(n):
            ges[i].view(torch.int32).copy_(_dev(e0[i]))
        for k in range(steps):
            what = f"{dtype} replay {k}"
            for i in range(n):
                gxs[i].view(torch.int32).copy_(_dev(xk[k][i]))
            ref = [expected(x, e, dtype) for x, e in zip(xk[k], chain)]
            comp.fill_(SENTINEL)
            graph.replay()
            torch.cuda.synchronize()
            hs = sizes.cpu().tolist()
            assert all(b.guards_intact() for b in gx + ge), f"{what}: a guard word was written"
            for i in range(n):
                assert np.array_equal(_host_u32(gxs[i]), xk[k][i]), f"{what} member {i}: the input changed"
                assert np.array_equal(_host_u32(ges[i]), ref[i][1]), f"{what} member {i}: residual != the chain"
            assert_rows_clean(comp, hs, what)
            check_archives(comp, hs, [w for w, _ in ref], dtype, 10, True, False, what)
            chain = [r for _, r in ref]
        del graph


# ---- a member past 4 GiB of float32 input -----------------------------------------------------------------------------

LARGE = (1 << 30) + 3 * 4096 + 5
CHUNK = 1 << 26


def _hash(lo, hi, salt):
    v = torch.arange(lo, hi, dtype=torch.int64, device="cuda")
    h = (v * 0x9E3779B1 + salt) & 0xFFFFFFFF
    h = ((h ^ (h >> 16)) * 0x85EBCA6B) & 0xFFFFFFFF
    h = ((h ^ (h >> 13)) * 0xC2B2AE35) & 0xFFFFFFFF
    return h ^ (h >> 16)


def _f32(u):
    return torch.where(u >= 1 << 31, u - (1 << 32), u).to(torch.int32).view(torch.float32)


def large_chunk(lo, hi):
    """x and e of words [lo, hi) of the large member, from a counter hash: x at exponents 2^-15 .. 2^16 (fp16
    subnormals to fp16 overflow) with +-inf and NaN every 4099th / 8191st word, e from 2^-31 to 2^-8 and +0."""
    h, g = _hash(lo, hi, 1), _hash(lo, hi, 2)
    x = (h & 0x807FFFFF) | (((h >> 23) % 32 + 112) << 23)
    idx = torch.arange(lo, hi, device="cuda")
    x = torch.where(idx % 4099 == 7, (h & 0x80000000) | 0x7F800000, x)
    x = torch.where(idx % 8191 == 11, 0x7FC00000 | (h & 0x3FF), x)
    e = (g & 0x807FFFFF) | (((g >> 23) % 24 + 96) << 23)
    e = torch.where(g % 7 == 0, torch.zeros_like(e), e)
    return _f32(x), _f32(e)


def test_large_member_past_4_gib_of_input():
    """One member of 2^30 + 3 * 4096 + 5 words per archive type (4 GiB + 48 KiB of float32 input and as much of
    residuals), canonical, with checksum, through the C ABI (ops refuses tensors past 4 GiB - 1 bytes): every residual
    and decoded word against torch's expression chunk by chunk, the archive byte for byte against the canonical
    compress of the words, the pdf against normalize(bincount)."""
    from dietgpu_b200 import capi, ops

    pb, n = 10, LARGE
    for dtype in TYPES:
        kind = TYPES[dtype]
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.time()
        xb, eb = Guarded(n, 0), Guarded(n, 0)
        for lo in range(0, n, CHUNK):
            hi = min(n, lo + CHUNK)
            x, e = large_chunk(lo, hi)
            xb.view[lo:hi].copy_(x)
            eb.view[lo:hi].copy_(e)
            del x, e
        ft = {torch.float16: capi.FLOAT16, torch.bfloat16: capi.BFLOAT16}[dtype]
        cols = ops.max_float_compressed_size(torch.empty(0, dtype=dtype), n)
        comp = torch.full((1, cols + GUARD), SENTINEL, dtype=torch.uint8, device="cuda")
        osz = torch.zeros(1, dtype=torch.int32, device="cuda")
        need = capi.lib().dgb_float_compress_temp_bytes(ft, 1, n)
        temp = torch.empty(need + 256, dtype=torch.uint8, device="cuda")
        with codec_options(encode_canonical=1):
            rc = _raw_ef(ft, [xb.view.data_ptr()], [n], [eb.view.data_ptr()], [comp[0]], osz, pb, True,
                         temp.data_ptr() + (-temp.data_ptr()) % 256, need)
        assert rc == capi.OK, rc
        torch.cuda.synchronize()
        del temp
        hs = [v & 0xFFFFFFFF for v in osz.cpu().tolist()]  # uint32 sizes in an int32 tensor: this one is past 2 GiB
        assert xb.guards_intact() and eb.guards_intact(), f"{dtype}: a guard word was written"
        assert_rows_clean(comp, hs, f"{dtype} large")
        w = torch.empty(n, dtype=dtype, device="cuda")
        for lo in range(0, n, CHUNK):
            hi = min(n, lo + CHUNK)
            x, e = large_chunk(lo, hi)
            assert torch.equal(_bits(xb.view[lo:hi]), _bits(x)), f"{dtype}: the input changed in [{lo}, {hi})"
            y, r = torch_step(x, e, dtype)
            bad = _bits(eb.view[lo:hi]) != _bits(r)
            assert not bool(bad.any()), f"{dtype}: residual differs at word {lo + int(bad.nonzero()[0])}"
            w[lo:hi] = y.to(dtype)
            del x, e, y, r, bad
        row = comp[0, :hs[0]]
        with codec_options(encode_canonical=1):
            want, wsz, _ = ops.compress_data(True, [w], True, prob_bits=pb)
        wsz = int(wsz[0]) & 0xFFFFFFFF
        assert wsz == hs[0], f"{dtype}: size {hs[0]} != the canonical compress of the words {wsz}"
        assert torch.equal(row, want[0, :hs[0]]), f"{dtype}: archive != the canonical compress of the words"
        del want
        assert_pdf_matches(row.cpu().numpy(), w, kind, pb, f"{dtype} large")
        guarded_decode(True, [row], [n], dtype, pb, True, [w], f"{dtype} large")
        peak = torch.cuda.max_memory_allocated() / 2 ** 30
        print(f"\n{dtype}: {n} words, archive {hs[0]} B, {time.time() - t0:.1f} s, peak {peak:.1f} GiB allocated")
        del xb, eb, comp, row, w
        torch.cuda.empty_cache()
