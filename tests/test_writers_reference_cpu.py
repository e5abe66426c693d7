"""The float64 reference of the narrowing decode-and-sum, tests/scaled_reference.narrow_fold_ref, against torch on the
CPU: the fp32 left fold acc = acc + x.float() (or the scaled terms x.float() * s32, s32 a float32 tensor), after an
fp32 init when given, followed by .to(float16 / bfloat16).  tests/test_gpu_writers_narrow_norm.py compares the
narrowing kernels with it, so it must be the contract of include/dietgpu_b200.h itself: one fp32 add per archive and
one rounding to 16 bits at the end, including ties with even and odd kept bits, an fp16 sum of 65520 that rounds to
inf, subnormal results, NaN and -0 + -0."""
import numpy as np
import pytest
import torch

from reduce_reference import assert_same_words
from scaled_reference import SCALE_IDS, SCALES, narrow_fold_ref
import test_gpu_reduce_edges as E
import test_gpu_reduce_sparse as S

TORCH = {"f16": torch.float16, "bf16": torch.bfloat16}
IDT = {"f16": torch.int16, "bf16": torch.int16, "f32": torch.int32}
NPI = {"f16": np.int16, "bf16": np.int16, "f32": np.int32}
NPW = {"f16": np.uint16, "bf16": np.uint16, "f32": np.uint32}


def _tensor(words, t):
    return torch.from_numpy(np.ascontiguousarray(words).view(NPW[t]).view(NPI[t]).copy()).view(
        TORCH.get(t, torch.float32))


def _words(x, t):
    return x.contiguous().view(IDT[t]).numpy().view(NPW[t])


def torch_narrow(words_list, t, s=None, init32=None):
    """torch's CPU fold in fp32 of the 16-bit words (scaled terms when s is not None), rounded once to t."""
    s32 = None if s is None else torch.tensor(s, dtype=torch.float32)
    xs = [_tensor(w, t) for w in words_list]

    def term(x):
        return x.float() if s32 is None else x.float() * s32

    if init32 is not None:
        acc = _tensor(init32, "f32").clone()
        rest = xs
    else:
        acc = term(xs[0])
        rest = xs[1:]
    for x in rest:
        acc = acc + term(x)
    return _words(acc.to(TORCH[t]), t)


def _random_words(t, n, seed):
    """Every 16-bit pattern in random order (NaN payloads, +-inf, subnormals, +-0), then N(0, 1) at three scales."""
    rng = np.random.default_rng(seed)
    perm = rng.permutation(1 << 16).astype(np.uint16)
    x = torch.from_numpy(rng.standard_normal(n).astype(np.float32) * np.float32([1e-3, 1.0, 3e3][seed % 3]))
    return np.concatenate([perm, _words(x.to(TORCH[t]), t)])


def _init32(n, seed):
    return E.init_words("f32", n, seed)


@pytest.mark.parametrize("s", [None] + SCALES, ids=["unscaled"] + SCALE_IDS)
@pytest.mark.parametrize("t", ["f16", "bf16"])
def test_random_words_match_torch(t, s):
    n = 20000
    words = [_random_words(t, n, 7 * j + 1) for j in range(5)]
    size = words[0].size
    for w in (1, 2, 5):
        for init in (None, _init32(size, w)):
            got = narrow_fold_ref(words[:w], t, s, init)
            assert_same_words(got, torch_narrow(words[:w], t, s, init), t,
                              f"{t} scale {s} W {w} init {init is not None}")


@pytest.mark.parametrize("t", ["f16", "bf16"])
def test_corpus_shapes_match_torch(t):
    """The dense and the sparse decode-and-sum corpora (worst, empty, over, ordinary; ReLU, +-0 pairings, zero
    blocks, full-range words and specials), unscaled and at two scales, with and without an fp32 init."""
    for shapes, make in ((E.SHAPES, lambda sh, n, sd, j: E._shape_words(t, sh, n, sd)),
                         (S.SHAPES, lambda sh, n, sd, j: S.shape_words(t, sh, n, sd, j))):
        for n in (1, 33, 4097, 65537):
            words = [make(shapes[(k + n) % len(shapes)], n, 100 * k + n, k) for k in range(len(shapes))]
            for s in (None, -0.25, 2.0 ** 15):
                for init in (None, _init32(n, n)):
                    assert_same_words(narrow_fold_ref(words, t, s, init), torch_narrow(words, t, s, init), t,
                                      f"{t} n {n} scale {s} init {init is not None}")


# ---- crafted sums: (archive words, fp32 init or None, scale or None, expected 16-bit word) -------------------------

def _w(t, *vals):
    return _words(torch.tensor(vals, dtype=torch.float32).to(TORCH[t]), t)


def _f32(*vals):
    return np.array(vals, np.float32).view(np.uint32)


def _cases(t):
    mb = 10 if t == "f16" else 7  # kept mantissa bits
    tie = 2.0 ** -(mb + 1)  # half an ulp of 1.0
    one = 0x3C00 if t == "f16" else 0x3F80
    tiny = 2.0 ** -24 if t == "f16" else 2.0 ** -133  # the smallest subnormal
    top = 65504.0 if t == "f16" else float(torch.finfo(torch.bfloat16).max)
    half_ulp_top = 16.0 if t == "f16" else 2.0 ** 119
    inf = 0x7C00 if t == "f16" else 0x7F80
    return {
        # 1 + half an ulp: a tie whose kept bits are even stays at 1; (1 + ulp) + half an ulp rounds up to 1 + 2 ulp
        "tie even": ([_w(t, 1.0), _w(t, tie)], None, None, one),
        "tie odd": ([_w(t, 1.0 + 2 * tie), _w(t, tie)], None, None, one + 2),
        # just below and just above that tie (2^-20 is exact in both types, and the fp32 sums are exact)
        "below tie": ([_w(t, 1.0), _w(t, tie), _w(t, -2.0 ** -20)], None, None, one),
        "above tie": ([_w(t, 1.0), _w(t, tie), _w(t, 2.0 ** -20)], None, None, one + 1),
        # the largest finite value plus half its ulp: finite in fp32, inf in the 16-bit type (fp16: 65520)
        "to inf": ([_w(t, top), _w(t, half_ulp_top)], None, None, inf),
        "to -inf": ([_w(t, -top), _w(t, -half_ulp_top)], None, None, 0x8000 | inf),
        "below inf": ([_w(t, top), _w(t, half_ulp_top / 2)], None, None, inf - 1),
        # subnormal results: 3 tiny - tiny = 2 tiny, and fp32 inits half-way between subnormals
        "subnormal": ([_w(t, 3 * tiny), _w(t, -tiny)], None, None, 0x0002),
        "subnormal tie even": ([_w(t, 0.0)], _f32(tiny / 2), None, 0x0000),
        "subnormal tie odd": ([_w(t, 0.0)], _f32(3 * tiny / 2), None, 0x0002),
        "subnormal scaled": ([_w(t, 3 * tiny), _w(t, tiny)], None, 0.5, 0x0002),
        # NaN in any archive, and inf - inf
        "nan": ([_w(t, 1.0), _w(t, float("nan")), _w(t, 2.0)], None, None, None),
        "inf - inf": ([_w(t, float("inf")), _w(t, float("-inf"))], None, None, None),
        # signed zeros: -0 + -0 = -0, -0 + +0 = +0, +0 * -0.25 = -0
        "-0 + -0": ([_w(t, -0.0), _w(t, -0.0), _w(t, -0.0)], None, None, 0x8000),
        "-0 + +0": ([_w(t, -0.0), _w(t, 0.0)], None, None, 0x0000),
        "+0 scaled negative": ([_w(t, 0.0), _w(t, 0.0)], None, -0.25, 0x8000),
        "-0 init": ([_w(t, -0.0)], _f32(-0.0), None, 0x8000),
    }


@pytest.mark.parametrize("t", ["f16", "bf16"])
def test_crafted_sums(t):
    for name, (words, init, s, want) in _cases(t).items():
        got = narrow_fold_ref(words, t, s, init)
        assert_same_words(got, torch_narrow(words, t, s, init), t, f"{t} {name}: against torch")
        if want is None:
            assert np.isnan(_tensor(got, t).float().numpy()).all(), f"{t} {name}: {got} is not NaN"
        else:
            assert int(got[0]) == want, f"{t} {name}: {int(got[0]):#06x} != {want:#06x}"


def test_one_rounding_differs_from_a_rounding_per_add():
    """The narrowing sum rounds once; the same-type 16-bit fold rounds after every add.  1 + 3 * (half an ulp) in
    three adds: each add of half an ulp to 1 ties back to 1 in fp16, while the fp32 sum rounds to 1 + 2 ulp."""
    from reduce_reference import fold_ref

    h = 2.0 ** -11
    words = [_w("f16", 1.0), _w("f16", h), _w("f16", h), _w("f16", h)]
    assert int(fold_ref(words, "f16", "f16")[0]) == 0x3C00
    assert int(narrow_fold_ref(words, "f16")[0]) == 0x3C02
