"""CPU tests of the scaled decode-and-sum: the argument checks of dgb_float_decompress_reduce_scaled and
ops.decompress_data_reduce(scale=), the collectives' scale / average refusals (all of them before any CUDA call or any
communication), and the float64 reference of tests/scaled_reference.py against torch's and numpy's CPU arithmetic."""
import ctypes as C

import numpy as np
import pytest
import torch

from dietgpu_b200 import capi
from multirank import Untouchable, no_communication  # noqa: F401  (no_communication is a fixture)
from reduce_reference import assert_same_words, f32_to_bf16_words, fold_ref, to_f64
from scaled_reference import SCALE_IDS, SCALES, scaled_fold_ref, term_ref

FAKE = 1 << 20  # never dereferenced: every call below fails (or returns) before it touches memory
ALLOWED = {(1, 1), (2, 2), (3, 3), (1, 3), (2, 3), (5, 1), (6, 2), (8, 3), (5, 3), (6, 3)}
TORCH = {"f16": torch.float16, "bf16": torch.bfloat16, "f32": torch.float32}
IDT = {"f16": torch.int16, "bf16": torch.int16, "f32": torch.int32}
NPW = {"f16": np.uint16, "bf16": np.uint16, "f32": np.uint32}


def _call(ft=capi.BFLOAT16, out_ft=capi.BFLOAT16, pb=10, groups=1, width=1, ins="ok", outs="ok", sizes="ok",
          scale=0.5):
    n = max(1, groups * width)
    in_arr = capi.ptr_array([FAKE] * n) if ins == "ok" else None
    out_arr = capi.ptr_array([FAKE] * max(1, groups)) if outs == "ok" else None
    size_arr = capi.u32_array([100] * max(1, groups)) if sizes == "ok" else None
    return capi.lib().dgb_float_decompress_reduce_scaled(None, 0, ft, out_ft, pb, groups, width, in_arr, out_arr,
                                                         size_arr, 0, scale, None, None)


@pytest.mark.parametrize("ft", range(10))
def test_type_pairs(ft):
    for out_ft in range(10):
        rc = _call(ft=ft, out_ft=out_ft)
        if (ft, out_ft) in ALLOWED:
            # the pair passes; the call then stops at the missing scratch
            assert rc == capi.ERR_TEMP_TOO_SMALL, (ft, out_ft, rc)
        else:
            assert rc == capi.ERR_INVALID_ARG, (ft, out_ft, rc)


@pytest.mark.parametrize("scale", [float("nan"), float("inf"), -0.0, 1.0])
def test_any_scale_passes_the_checks(scale):
    assert _call(scale=scale) == capi.ERR_TEMP_TOO_SMALL


@pytest.mark.parametrize("pb", [8, 12])
def test_prob_bits_out_of_range_are_rejected(pb):
    assert _call(pb=pb) == capi.ERR_INVALID_ARG


def test_empty_groups_are_rejected():
    assert _call(width=0) == capi.ERR_INVALID_ARG


@pytest.mark.parametrize("which", ["ins", "outs", "sizes"])
def test_null_arrays_are_rejected(which):
    assert _call(**{which: None}) == capi.ERR_INVALID_ARG


def test_no_groups_is_ok():
    assert _call(groups=0) == capi.OK
    assert _call(groups=0, ins=None, outs=None, sizes=None) == capi.OK
    assert _call(ft=capi.FLOAT32_SPARSE, out_ft=capi.FLOAT32, groups=0) == capi.OK
    # ... but only for an allowed pair
    assert _call(ft=capi.FLOAT32, out_ft=capi.BFLOAT16, groups=0) == capi.ERR_INVALID_ARG
    assert _call(ft=capi.FLOAT64, out_ft=capi.FLOAT64, groups=0) == capi.ERR_INVALID_ARG


@pytest.mark.parametrize("ft,out_ft", [(1, 3), (2, 3), (3, 3), (5, 3), (6, 3), (8, 3)])
def test_misaligned_fp32_output_is_rejected(ft, out_ft):
    # a 2 B aligned output is fine for 16-bit sums, not for fp32 ones; the check happens before any CUDA call
    rc = capi.lib().dgb_float_decompress_reduce_scaled(FAKE, 1 << 20, ft, out_ft, 10, 1, 1, capi.ptr_array([FAKE]),
                                                       capi.ptr_array([FAKE + 2]), capi.u32_array([100]), 0, 0.5,
                                                       None, None)
    assert rc == capi.ERR_INVALID_ARG


def test_signature_is_declared():
    f = capi.lib().dgb_float_decompress_reduce_scaled
    assert f.restype is C.c_int and len(f.argtypes) == 14 and f.argtypes[11] is C.c_float
    assert "dgb_float_decompress_reduce_scaled" in capi.SYMBOLS


# ---- ops.decompress_data_reduce(scale=) -----------------------------------------------------------------------------

@pytest.mark.parametrize("scale", [torch.tensor(0.5), "0.5", True, 1j, [0.5]])
def test_ops_refuses_non_real_scales_first(scale):
    from dietgpu_b200 import ops

    out = torch.empty(4, dtype=torch.bfloat16)  # a CPU tensor: any device work would fail differently
    with pytest.raises(TypeError, match="scale"):
        ops.decompress_data_reduce([[Untouchable()]], [out], scale=scale)


@pytest.mark.parametrize("sparse", [False, True])
@pytest.mark.parametrize("archive_dtype,out_dtype", [
    (torch.float32, torch.float16), (torch.float16, torch.bfloat16), (torch.float64, torch.float64),
    (torch.int32, torch.float32)])
def test_ops_refuses_bad_pairs_first(archive_dtype, out_dtype, sparse):
    from dietgpu_b200 import ops

    out = torch.empty(4, dtype=out_dtype)
    with pytest.raises(ValueError):
        ops.decompress_data_reduce([[Untouchable()]], [out], archive_dtype=archive_dtype, sparse=sparse, scale=0.5)


# ---- the collectives' refusals --------------------------------------------------------------------------------------

@pytest.mark.parametrize("scale", [0.5, 1.0, float("nan")])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
def test_collectives_refuse_average_with_scale(dtype, scale, no_communication):
    import dietgpu_b200 as dg

    t = torch.zeros(64, dtype=dtype)
    with pytest.raises(ValueError, match="average"):
        dg.reduce_scatter_compressed(t, scale=scale, average=True)
    with pytest.raises(ValueError, match="average"):
        dg.all_reduce_compressed(t, scale=scale, average=True)
    with pytest.raises(ValueError, match="average"):
        dg.reduce_scatter_compressed(t, scale=scale, average=True, sparse=True)
    with pytest.raises(ValueError, match="average"):
        dg.all_reduce_compressed(t, scale=scale, average=True, reduce_dtype=torch.float32)


@pytest.mark.parametrize("scale", [torch.tensor(0.5), "0.5", True])
def test_collectives_refuse_non_real_scales(scale, no_communication):
    import dietgpu_b200 as dg

    t = torch.zeros(64, dtype=torch.bfloat16)
    with pytest.raises(TypeError, match="scale"):
        dg.reduce_scatter_compressed(t, scale=scale)
    with pytest.raises(TypeError, match="scale"):
        dg.all_reduce_compressed(t, scale=scale)


def test_collectives_keep_their_other_refusals(no_communication):
    import dietgpu_b200 as dg

    with pytest.raises(ValueError, match="sparse"):
        dg.reduce_scatter_compressed(torch.zeros(64, dtype=torch.float64), scale=0.5, sparse=True)
    with pytest.raises(ValueError, match="wire_dtype"):
        dg.reduce_scatter_compressed(torch.zeros(64), average=True, wire_dtype=torch.bfloat16, sparse=True)


# ---- the float64 reference against torch's and numpy's CPU arithmetic ------------------------------------------------

def _torch_term(words, at, ot, s):
    x = torch.from_numpy(np.ascontiguousarray(words).view(NPW[at]).astype(NPW[at]).view(
        np.int16 if at != "f32" else np.int32)).view(TORCH[at])
    r = (x.float() * torch.tensor(s, dtype=torch.float32)).to(TORCH[ot])
    return r.view(IDT[ot]).numpy().view(NPW[ot])


@pytest.mark.parametrize("s", SCALES, ids=SCALE_IDS)
@pytest.mark.parametrize("at", ["f16", "bf16"])
def test_term_of_every_16_bit_word_matches_torch(at, s):
    words = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    for ot in (at, "f32"):
        assert_same_words(term_ref(words, at, ot, s), _torch_term(words, at, ot, s), ot, f"{at}->{ot} scale {s}")


def _f32_words(n, seed):
    rng = np.random.default_rng(seed)
    w = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    edge = np.array([0, 0x80000000, 1, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x00800000, 0x7F7FFFFF, 0xFF7FFFFF,
                     0x7F800000, 0xFF800000, 0x7FC00000, 0x7F800001, 0x3F800000, 0x3F800001, 0x4B000000,
                     0x33800000, 0x0C000000], np.uint32)
    return np.concatenate([edge, w, rng.standard_normal(n).astype(np.float32).view(np.uint32)])


@pytest.mark.parametrize("s", SCALES, ids=SCALE_IDS)
def test_term_of_fp32_words_matches_numpy(s):
    words = _f32_words(1 << 20, 17)
    with np.errstate(all="ignore"):
        want = (words.view(np.float32) * np.float32(s)).view(np.uint32)
    assert_same_words(term_ref(words, "f32", "f32", s), want, "f32", f"scale {s}")
    assert_same_words(term_ref(words, "f32", "f32", s), _torch_term(words, "f32", "f32", s), "f32", f"torch {s}")


def _direct(x64, t):
    """One round-to-nearest-even of float64 values to t (normal results only): the rounding the contract does not
    do for 16-bit same-type terms."""
    if t == "f16":
        return x64.astype(np.float16).view(np.uint16)
    u = x64.view(np.uint64)  # round float64's 52 fraction bits to bf16's 7
    r = (u + np.uint64((1 << 44) - 1) + ((u >> np.uint64(45)) & np.uint64(1))) >> np.uint64(45) << np.uint64(45)
    return f32_to_bf16_words(r.view(np.float64).astype(np.float32))


@pytest.mark.parametrize("at", ["f16", "bf16"])
def test_double_rounding_is_kept(at):
    # scales s = fp32(tie / x) put x * s within half an fp32 ulp of a 16-bit tie: the fp32 product (the contract,
    # and torch) lands on the tie and rounds to even, one direct rounding of the exact product may not.  The
    # reference must follow the contract wherever the two differ, and they must differ somewhere.
    mbits = 10 if at == "f16" else 7
    ties = 1 + (2 * np.arange(1 << mbits) + 1) * 2.0 ** -(mbits + 1)
    hits = 0
    for x in (3.0, 5.0, 7.0, 11.0, 13.0):
        xw = torch.tensor([x], dtype=TORCH[at]).view(IDT[at]).numpy().view(NPW[at])
        for s in (ties / x).astype(np.float32):
            got = term_ref(xw, at, at, float(s))
            if int(got[0]) != int(_direct(to_f64(xw, at) * np.float64(s), at)[0]):
                hits += 1
                assert_same_words(got, _torch_term(xw, at, at, float(s)), at, f"x {x} scale {s}")
    assert hits > 0


@pytest.mark.parametrize("s", SCALES, ids=SCALE_IDS)
@pytest.mark.parametrize("at,ot", [("f16", "f16"), ("bf16", "bf16"), ("f32", "f32"), ("f16", "f32"), ("bf16", "f32")])
def test_fold_matches_torch(at, ot, s):
    rng = np.random.default_rng(5)
    n = 4099
    words = []
    for j in range(9):
        x = rng.standard_normal(n).astype(np.float32) * np.float32([1, 1e3, 1e-3, 6e4, 1e-6][j % 5])
        x[::7] = [0.0, -0.0, np.inf, -np.inf, np.nan][j % 5]
        words.append(torch.from_numpy(x).to(TORCH[at]).view(IDT[at]).numpy().view(NPW[at]))
    init = torch.from_numpy(rng.standard_normal(n).astype(np.float32)).to(TORCH[ot])
    s32 = torch.tensor(s, dtype=torch.float32)
    xs = [torch.from_numpy(w.view(np.int16 if at != "f32" else np.int32)).view(TORCH[at]) for w in words]
    for use_init in (False, True):
        acc = init.clone() if use_init else (xs[0].float() * s32).to(TORCH[ot])
        for x in (xs if use_init else xs[1:]):
            acc = acc + (x.float() * s32).to(TORCH[ot])
        got = scaled_fold_ref(words, at, ot, s, init.view(IDT[ot]).numpy().view(NPW[ot]) if use_init else None)
        assert_same_words(got, acc.view(IDT[ot]).numpy().view(NPW[ot]), ot, f"{at}->{ot} init {use_init} scale {s}")


def test_scale_one_is_the_plain_fold():
    rng = np.random.default_rng(9)
    words = [rng.integers(0, 1 << 16, 5000, dtype=np.uint32).astype(np.uint16) for _ in range(5)]
    for at, ot in (("f16", "f16"), ("bf16", "bf16"), ("f16", "f32"), ("bf16", "f32")):
        assert_same_words(scaled_fold_ref(words, at, ot, 1.0), fold_ref(words, at, ot), ot, f"{at}->{ot}")
