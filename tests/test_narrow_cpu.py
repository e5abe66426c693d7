"""CPU tests of dgb_float_compress_to's argument checks and of compress_data(archive_dtype=...)'s refusals: every
malformed call fails before any CUDA call, so these run without a device."""
import ctypes as C

import pytest
import torch

from dietgpu_b200 import capi

FAKE = 1 << 20  # never dereferenced: every call below fails before it touches memory
ALLOWED = {(1, 1), (2, 2), (3, 3), (3, 1), (3, 2)}


def _call(in_ft=capi.FLOAT32, ft=capi.BFLOAT16, pb=10, n=1, ins="ok", sizes="ok", outs="ok", in_ptr=FAKE):
    in_arr = capi.ptr_array([in_ptr] * n) if ins == "ok" else None
    size_arr = capi.u32_array([100] * n) if sizes == "ok" else None
    out_arr = capi.ptr_array([FAKE] * n) if outs == "ok" else None
    return capi.lib().dgb_float_compress_to(None, 0, in_ft, ft, pb, 0, n, in_arr, size_arr, out_arr, None, None)


@pytest.mark.parametrize("in_ft", range(10))
def test_type_pairs(in_ft):
    for ft in range(10):
        rc = _call(in_ft=in_ft, ft=ft)
        if (in_ft, ft) in ALLOWED:
            # the pair passes; the call then stops at the missing scratch
            assert rc == capi.ERR_TEMP_TOO_SMALL, (in_ft, ft, rc)
        else:
            assert rc == capi.ERR_INVALID_ARG, (in_ft, ft, rc)


@pytest.mark.parametrize("pb", [8, 12])
def test_prob_bits_out_of_range_are_rejected(pb):
    assert _call(pb=pb) == capi.ERR_INVALID_ARG
    assert _call(ft=capi.FLOAT16, pb=pb) == capi.ERR_INVALID_ARG


@pytest.mark.parametrize("which", ["ins", "sizes", "outs"])
def test_null_arrays_are_rejected(which):
    assert _call(**{which: None}) == capi.ERR_INVALID_ARG


def test_empty_batch_is_ok():
    assert _call(n=0, ins=None, sizes=None, outs=None) == capi.OK


def test_two_byte_aligned_fp32_input_is_rejected():
    # a 2 B aligned input is a valid fp16 / bf16 input but not a float32 one
    assert _call(in_ptr=FAKE + 2) == capi.ERR_INVALID_ARG
    assert _call(ft=capi.FLOAT16, in_ptr=FAKE + 2) == capi.ERR_INVALID_ARG
    assert _call(in_ft=capi.BFLOAT16, ft=capi.BFLOAT16, in_ptr=FAKE + 2) == capi.ERR_TEMP_TOO_SMALL


def test_scratch_is_the_archive_types():
    # narrowing takes dgb_float_compress_temp_bytes of the archive type, whose plan does not depend on the word size
    L = capi.lib()
    for n, mx in ((1, 100), (64, 2 << 20), (130, 4097)):
        assert L.dgb_float_compress_temp_bytes(capi.FLOAT16, n, mx) == L.dgb_float_compress_temp_bytes(capi.FLOAT32, n, mx)
        assert L.dgb_float_compress_temp_bytes(capi.BFLOAT16, n, mx) == L.dgb_float_compress_temp_bytes(capi.FLOAT32, n, mx)


def test_signature_is_declared():
    f = capi.lib().dgb_float_compress_to
    assert f.restype is C.c_int and len(f.argtypes) == 12
    assert "dgb_float_compress_to" in capi.SYMBOLS


@pytest.mark.parametrize("in_dtype,archive_dtype,kw", [
    (torch.float16, torch.bfloat16, {}),                     # fp16 -> bf16
    (torch.bfloat16, torch.float16, {}),
    (torch.float32, torch.float64, {}),                      # float64 archives
    (torch.float64, torch.float32, {}),                      # float64 inputs
    (torch.float64, torch.float16, {}),
    (torch.float32, torch.int8, {}),
    (torch.float32, torch.bfloat16, dict(sparse=True)),      # sparse together with narrowing
    (torch.float32, torch.float16, dict(sparse=True)),
    (torch.float32, torch.bfloat16, dict(as_float=False)),   # byte mode
])
def test_compress_data_refusals_before_the_device(in_dtype, archive_dtype, kw):
    from dietgpu_b200 import ops

    t = torch.zeros(16, dtype=in_dtype)  # a CPU tensor: a call that got past the dtype check would fail otherwise
    with pytest.raises(ValueError):
        ops.compress_data(kw.get("as_float", True), [t], archive_dtype=archive_dtype, sparse=kw.get("sparse", False))
