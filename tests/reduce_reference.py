"""Float64 reference of decode-and-sum's left fold, on raw words (numpy only, no device).

fold_ref(words_list, archive_type, out_type, init=None) returns the raw words of
    acc = init (or x_0);  acc = round_out(acc + x_j) for every later x_j, left to right,
where the types are "f16", "bf16" or "f32" (u16 words for the 16-bit types, u32 for fp32), out_type is the
archive type or "f32" (the widening sum), and init holds out_type words.

Every element is decoded exactly to float64 and every add is one float64 add followed by a rounding to the
output type: round-to-nearest-even, subnormals kept, overflow to +-inf, the sign of zero kept (numpy's casts
from float64 do all of that; bf16 goes float64 -> float32 -> bf16 by integer round-to-nearest-even on the bits).

Why this is one correctly rounded add per step, which is what add.rn.f16, add.rn.bf16 and __fadd_rn compute:
  - the exact sum a + b of two output-type values is rounded first to 53 bits, then (bf16 only) to 24 bits,
    then to the output's 11, 8 or 24 bits;
  - a + b of two p-bit values rounded to q >= 2p + 2 bits and then to p bits equals a + b rounded to p bits
    directly (double rounding is innocuous for +, -, *, / and sqrt when q >= 2p + 2).  float64 has 53 >= 2*24 + 2
    bits for fp32 and bf16 (whose values are 24-bit values too), 53 >= 2*11 + 2 for fp16, and float32 has
    24 >= 2*8 + 2 for bf16;
  - below the output's smallest normal the precision shrinks, but there a + b is a multiple of the smallest
    subnormal smaller than the smallest normal, so it is exact in every format of the chain: no rounding happens;
  - float64's range holds every sum; float32's holds every bf16 sum below the point where bf16 rounds to inf.
Infinities and NaN follow IEEE in float64 and survive every cast as infinities and NaN.

NaN payloads are not part of the contract: compare results with same_words / assert_same_words, which accept
any two NaNs and require every other bit pattern, -0 included, to be equal.
"""
from __future__ import annotations

import numpy as np

TYPES = ("f16", "bf16", "f32")
WORD = {"f16": np.uint16, "bf16": np.uint16, "f32": np.uint32}


def to_f64(words, t):
    """The exact float64 values of raw words of type t."""
    w = np.ascontiguousarray(words).view(WORD[t]).reshape(-1)
    with np.errstate(invalid="ignore"):  # signalling NaNs are quietened, which is all a NaN needs
        if t == "f16":
            return w.view(np.float16).astype(np.float64)
        if t == "bf16":
            return (w.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
        return w.view(np.float32).astype(np.float64)


def f32_to_bf16_words(x32):
    """float32 -> bf16 words, round-to-nearest-even on the bits; NaN stays a (quiet) NaN."""
    u = np.ascontiguousarray(x32, np.float32).view(np.uint32)
    r = ((u + np.uint32(0x7FFF) + ((u >> np.uint32(16)) & np.uint32(1))) >> np.uint32(16)).astype(np.uint16)
    nan = np.isnan(x32)
    return np.where(nan, (u >> np.uint32(16)).astype(np.uint16) | np.uint16(0x0040), r)


def round_to(x64, t):
    """Raw words of t nearest to float64 values (see the module docstring)."""
    with np.errstate(over="ignore", invalid="ignore"):
        if t == "f16":
            return x64.astype(np.float16).view(np.uint16)
        x32 = x64.astype(np.float32)
    if t == "bf16":
        return f32_to_bf16_words(x32)
    return x32.view(np.uint32)


def fold_ref(words_list, archive_type, out_type, init=None):
    """Raw out_type words of the left fold of words_list (archive_type words), after `init` when given."""
    assert archive_type in TYPES and out_type in (archive_type, "f32"), (archive_type, out_type)
    if init is None:
        acc = to_f64(words_list[0], archive_type)  # exact in out_type too (widening is exact)
        rest = words_list[1:]
    else:
        acc = to_f64(init, out_type)
        rest = words_list
    for w in rest:
        with np.errstate(invalid="ignore"):
            acc = to_f64(round_to(acc + to_f64(w, archive_type), out_type), out_type)
    return round_to(acc, out_type)


def _int(words, t):
    return np.ascontiguousarray(words).view(WORD[t]).reshape(-1)


def same_words(got, want, t):
    """Per element: both NaN, or identical bits."""
    g, w = _int(got, t), _int(want, t)
    return (g == w) | (np.isnan(to_f64(g, t)) & np.isnan(to_f64(w, t)))


def assert_same_words(got, want, t, what):
    g, w = _int(got, t), _int(want, t)
    assert g.shape == w.shape, f"{what}: shape {g.shape} != {w.shape}"
    ok = same_words(g, w, t)
    if not bool(ok.all()):
        i = int(np.flatnonzero(~ok)[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} element(s) differ, first at {i}: "
                             f"got {int(g[i]):#x}, want {int(w[i]):#x}")


def pair_operands(t):
    """The b operands the exhaustive pair tests pair with every 16-bit a: every exponent code with both signs
    (a few mantissas each, including 0 and all ones, which make ties), the subnormals, +-0, +-max, +-inf and two
    NaN payloads.  1024 or more values, deterministic."""
    assert t in ("f16", "bf16")
    mbits = 10 if t == "f16" else 7
    ebits = 15 - mbits
    per = 16 if t == "f16" else 2
    rng = np.random.default_rng(1234 if t == "f16" else 4321)
    fixed = [0, 1, 1 << (mbits - 1), (1 << mbits) - 1]
    vals = []
    for s in (0, 1):
        for e in range(1 << ebits):
            ms = [fixed[(e + k) % 4] for k in range(min(4, per // 2))]
            ms +=[int(m) for m in rng.integers(0, 1 << mbits, per - len(ms))]
            vals += [(s << 15) | (e << mbits) | m for m in ms]
    top = ((1 << ebits) - 1) << mbits  # +inf
    vals += [0x0000, 0x8000, 0x0001, 0x8001, (1 << mbits) - 1, 0x8000 | ((1 << mbits) - 1),  # zeros, subnormals
             1 << mbits, 0x8000 | (1 << mbits),                                           # smallest normals
             top - 1, 0x8000 | (top - 1), top, 0x8000 | top,                               # +-max, +-inf
             top | 1, 0x8000 | top | (1 << (mbits - 1)) | 5]                               # two NaN payloads
    return np.unique(np.array(vals, dtype=np.uint16))
