"""CPU tests of dgb_float_decompress_reduce_to's argument checks: every malformed call returns its error code before
any CUDA call, so these run without a device."""
import ctypes as C

import pytest

from dietgpu_b200 import capi

FAKE = 1 << 20  # never dereferenced: every call below fails (or returns) before it touches memory
ALLOWED = {(1, 1), (2, 2), (3, 3), (1, 3), (2, 3)}


def _call(ft=capi.BFLOAT16, out_ft=capi.FLOAT32, pb=10, groups=1, width=1, ins="ok", outs="ok", sizes="ok"):
    n = max(1, groups * width)
    in_arr = capi.ptr_array([FAKE] * n) if ins == "ok" else None
    out_arr = capi.ptr_array([FAKE] * max(1, groups)) if outs == "ok" else None
    size_arr = capi.u32_array([100] * max(1, groups)) if sizes == "ok" else None
    return capi.lib().dgb_float_decompress_reduce_to(None, 0, ft, out_ft, pb, groups, width, in_arr, out_arr,
                                                     size_arr, 0, None, None)


@pytest.mark.parametrize("ft", range(10))
def test_type_pairs(ft):
    for out_ft in range(10):
        rc = _call(ft=ft, out_ft=out_ft)
        if (ft, out_ft) in ALLOWED:
            # the pair passes; the call then stops at the missing scratch
            assert rc == capi.ERR_TEMP_TOO_SMALL, (ft, out_ft, rc)
        else:
            assert rc == capi.ERR_INVALID_ARG, (ft, out_ft, rc)


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
    assert _call(ft=capi.FLOAT16, groups=0) == capi.OK


def test_misaligned_fp32_output_is_rejected():
    # a 2 B aligned output is fine for bf16 sums, not for fp32 ones; the check happens before any CUDA call
    rc = capi.lib().dgb_float_decompress_reduce_to(FAKE, 1 << 20, capi.BFLOAT16, capi.FLOAT32, 10, 1, 1,
                                                   capi.ptr_array([FAKE]), capi.ptr_array([FAKE + 2]),
                                                   capi.u32_array([100]), 0, None, None)
    assert rc == capi.ERR_INVALID_ARG


def test_signature_is_declared():
    f = capi.lib().dgb_float_decompress_reduce_to
    assert f.restype is C.c_int and len(f.argtypes) == 13
    assert "dgb_float_decompress_reduce_to" in capi.SYMBOLS
