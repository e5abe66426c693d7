"""Float64 reference of the scaled decode-and-sum (dgb_float_decompress_reduce_scaled), on raw words, built on
tests/reduce_reference.py (to_f64, round_to, fold_ref).

term_ref(words, archive_type, out_type, s) returns the raw out_type words of s(x), the term the scaled writers add:
  - s is rounded once to float32 (np.float32(s)), as every caller's scale is;
  - the word's exact value times that float32 is exact in float64: the significands need at most 24 + 24 = 48 of
    float64's 53 bits, and every product of two float32 magnitudes lies between 2^-298 and 2^256, inside float64's
    normal range;
  - the exact product is rounded once to float32 (mul.rn.f32), and for a 16-bit out_type that float32 is rounded
    again to the 16-bit type (cvt.rn.f16.f32 / cvt.rn.bf16.f32).  The contract rounds twice here, so the reference
    does too; one direct rounding of the exact product to 16 bits could differ from it.
Infinities, NaN (0 * inf, s = NaN) and the sign of zero (s < 0 turns +0 into -0) follow IEEE in float64 and survive
the casts.

scaled_fold_ref(words_list, archive_type, out_type, s, init=None) is the left fold of the terms with the output
type's adds (fold_ref), after init when given; init is the running value taken in by accumulate and is not scaled.

narrow_fold_ref(words_list, t, s, init32) is the narrowing decode-and-sum (dgb_float_decompress_reduce_narrow): the
fp32 fold of the fp16 / bf16 words (scaled_fold_ref into "f32", or fold_ref for the unscaled sum, s = None), after
the fp32 running sums init32 when given, rounded once to t.  The fp32 sum is exact in float64, so round_to rounds it
once, as cvt.rn.f16.f32 / cvt.rn.bf16.f32 do.
"""
from __future__ import annotations

import numpy as np

from reduce_reference import fold_ref, round_to, to_f64

# the scales the tests run: exact ones, inexact reciprocals, a negative one, tiny and large ones, zeros and non-finite
SCALES = [1.0, 0.5, float(np.float32(1 / 3)), float(np.float32(1 / 7)), -0.25, 2.0 ** -24, 3.0, 2.0 ** 15, 0.0,
          -0.0, float("inf"), float("nan")]
SCALE_IDS = ["1", "0.5", "1/3", "1/7", "-0.25", "2^-24", "3", "2^15", "0", "-0", "inf", "nan"]


def term_ref(words, archive_type, out_type, s):
    """Raw out_type words of s(x) for raw archive_type words (see the module docstring)."""
    assert out_type in (archive_type, "f32"), (archive_type, out_type)
    s64 = np.float64(np.float32(s))
    with np.errstate(invalid="ignore", over="ignore"):
        p = to_f64(words, archive_type) * s64
    w32 = round_to(p, "f32")
    return w32 if out_type == "f32" else round_to(to_f64(w32, "f32"), out_type)


def scaled_fold_ref(words_list, archive_type, out_type, s, init=None):
    """Raw out_type words of init (unscaled, when given) + s(x_0) + s(x_1) + ..., left to right."""
    return fold_ref([term_ref(w, archive_type, out_type, s) for w in words_list], out_type, out_type, init)


def narrow_fold_ref(words_list, t, s=None, init32=None):
    """Raw t words of round_t((init32 or term(x_0)) + term(x_1) + ... in fp32), term unscaled when s is None."""
    assert t in ("f16", "bf16"), t
    f32 = fold_ref(words_list, t, "f32", init32) if s is None else scaled_fold_ref(words_list, t, "f32", s, init32)
    return round_to(to_f64(f32, "f32"), t)
