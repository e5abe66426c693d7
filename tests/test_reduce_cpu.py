"""CPU tests of dgb_float_decompress_reduce's argument checks: every malformed call returns its error code before
any CUDA call, so these run without a device."""
import ctypes as C

import pytest

from dietgpu_b200 import capi

FAKE = 1 << 20  # never dereferenced: every call below fails (or returns) before it touches memory


def _call(ft=capi.BFLOAT16, pb=10, groups=1, width=1, ins="ok", outs="ok", sizes="ok"):
    n = max(1, groups * width)
    in_arr = capi.ptr_array([FAKE] * n) if ins == "ok" else None
    out_arr = capi.ptr_array([FAKE] * max(1, groups)) if outs == "ok" else None
    size_arr = capi.u32_array([100] * max(1, groups)) if sizes == "ok" else None
    return capi.lib().dgb_float_decompress_reduce(None, 0, ft, pb, groups, width, in_arr, out_arr, size_arr, 0,
                                                  None, None)


def test_no_groups_is_ok():
    assert _call(groups=0) == capi.OK
    assert _call(groups=0, ins=None, outs=None, sizes=None) == capi.OK


@pytest.mark.parametrize("ft", [0, 4, 5, 6, 7, 8, 9])
def test_other_float_types_are_rejected(ft):
    assert _call(ft=ft) == capi.ERR_INVALID_ARG


@pytest.mark.parametrize("pb", [8, 12])
def test_prob_bits_out_of_range_are_rejected(pb):
    assert _call(pb=pb) == capi.ERR_INVALID_ARG


def test_empty_groups_are_rejected():
    assert _call(width=0) == capi.ERR_INVALID_ARG


@pytest.mark.parametrize("which", ["ins", "outs", "sizes"])
def test_null_arrays_are_rejected(which):
    assert _call(**{which: None}) == capi.ERR_INVALID_ARG


def test_signature_is_declared():
    f = capi.lib().dgb_float_decompress_reduce
    assert f.restype is C.c_int and len(f.argtypes) == 12
    assert "dgb_float_decompress_reduce" in capi.SYMBOLS
