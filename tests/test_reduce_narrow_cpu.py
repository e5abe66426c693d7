"""CPU tests of the narrowing decode-and-sum: the argument checks of dgb_float_decompress_reduce_narrow, of
ops.decompress_data_reduce(reduce_dtype=, acc=) and of the collectives' out_dtype, all of which refuse before any
CUDA call, before any archive is read and before any communication."""
import ctypes as C

import pytest
import torch

from dietgpu_b200 import capi
from multirank import Untouchable, no_communication  # noqa: F401  (no_communication is a fixture)

FAKE = 1 << 20  # never dereferenced: every call below fails (or returns) before it touches memory
ALLOWED = {capi.FLOAT16, capi.BFLOAT16, capi.FLOAT16_SPARSE, capi.BFLOAT16_SPARSE}


def _call(ft=capi.BFLOAT16, pb=10, groups=1, width=2, acc=FAKE, accs=True, out=FAKE + 2, outs=True, accumulate=0,
          scale=None, scale_dev=None, found_inf=None, temp=None, temp_bytes=0):
    n = max(1, groups * width)
    g = max(1, groups)
    s = None if scale is None else C.c_float(scale)
    return capi.lib().dgb_float_decompress_reduce_narrow(
        temp, temp_bytes, ft, pb, groups, width, capi.ptr_array([FAKE] * n),
        capi.ptr_array([acc] * g) if accs else None, capi.ptr_array([out] * g) if outs else None,
        capi.u32_array([100] * g), accumulate, None if s is None else C.addressof(s), scale_dev, found_inf, None, None)


@pytest.mark.parametrize("ft", range(10))
def test_float_types(ft):
    for kw in (dict(), dict(scale=0.5), dict(scale_dev=FAKE), dict(scale_dev=FAKE, found_inf=FAKE + 4)):
        rc = _call(ft=ft, **kw)
        # an allowed type passes; the call then stops at the missing scratch
        assert rc == (capi.ERR_TEMP_TOO_SMALL if ft in ALLOWED else capi.ERR_INVALID_ARG), (ft, kw, rc)


@pytest.mark.parametrize("ft", [capi.FLOAT32, capi.FLOAT64, capi.FLOAT32_SPARSE])
def test_wide_types_are_rejected_before_anything(ft):
    assert _call(ft=ft, groups=0) == capi.ERR_INVALID_ARG
    assert _call(ft=ft, temp=FAKE, temp_bytes=1 << 30) == capi.ERR_INVALID_ARG


@pytest.mark.parametrize("pb", [8, 12])
def test_prob_bits_out_of_range_are_rejected(pb):
    assert _call(pb=pb) == capi.ERR_INVALID_ARG


@pytest.mark.parametrize("kw", [dict(scale=0.5, scale_dev=FAKE), dict(found_inf=FAKE), dict(scale=0.5, found_inf=FAKE),
                                dict(scale_dev=FAKE + 2), dict(scale_dev=FAKE, found_inf=FAKE + 2)])
def test_scale_arguments_are_rejected(kw):
    assert _call(**kw) == capi.ERR_INVALID_ARG
    # ... before anything else: with no groups, and with enough (fake) scratch
    assert _call(groups=0, **kw) == capi.ERR_INVALID_ARG
    assert _call(temp=FAKE, temp_bytes=1 << 30, **kw) == capi.ERR_INVALID_ARG


@pytest.mark.parametrize("width,accumulate", [(2, 0), (5, 0), (1, 1), (3, 1)])
def test_accumulator_is_required_where_it_is_read(width, accumulate):
    big = dict(temp=FAKE, temp_bytes=1 << 30, width=width, accumulate=accumulate)
    assert _call(acc=0, **big) == capi.ERR_INVALID_ARG
    assert _call(accs=False, **big) == capi.ERR_INVALID_ARG
    for misaligned in (FAKE + 1, FAKE + 2, FAKE + 3):
        assert _call(acc=misaligned, **big) == capi.ERR_INVALID_ARG


def test_accumulator_may_be_missing_when_it_is_not_read():
    # W = 1 without accumulate stores round(term) and reads no running sum: acc (the array or its entries) may be
    # NULL or anything else, which the entry's own checks let through; the call then stops at the missing scratch
    for kw in (dict(acc=0), dict(accs=False), dict(acc=FAKE + 1)):
        assert _call(width=1, **kw) == capi.ERR_TEMP_TOO_SMALL, kw


def test_output_is_checked():
    big = dict(temp=FAKE, temp_bytes=1 << 30)
    assert _call(out=0, **big) == capi.ERR_INVALID_ARG
    assert _call(out=FAKE + 1, **big) == capi.ERR_INVALID_ARG
    assert _call(outs=False, **big) == capi.ERR_INVALID_ARG
    assert _call(outs=False, width=1, accs=False, **big) == capi.ERR_INVALID_ARG
    assert _call(out=FAKE + 2) == capi.ERR_TEMP_TOO_SMALL  # 2 B aligned is enough for a 16-bit output


def test_no_groups_is_ok():
    assert _call(groups=0) == capi.OK
    assert _call(groups=0, accs=False, outs=False) == capi.OK
    assert _call(groups=0, scale_dev=FAKE, found_inf=FAKE) == capi.OK


def test_width_zero_is_rejected():
    assert _call(width=0) == capi.ERR_INVALID_ARG


def test_signature_is_declared():
    f = capi.lib().dgb_float_decompress_reduce_narrow
    assert f.restype is C.c_int and len(f.argtypes) == 16
    assert f.argtypes[2] is C.c_int and f.argtypes[4] is C.c_uint32 and f.argtypes[10] is C.c_int
    assert all(f.argtypes[i] is C.c_void_p for i in (6, 7, 8, 9, 11, 12, 13, 14, 15))
    assert "dgb_float_decompress_reduce_narrow" in capi.SYMBOLS


# ---- ops.decompress_data_reduce(reduce_dtype=, acc=) -----------------------------------------------------------------

def _f32(n=4, dtype=torch.float32):
    return torch.zeros(n, dtype=dtype)  # on the CPU: never the outputs' CUDA device


@pytest.mark.parametrize("out_dtype,kw,match", [
    (torch.bfloat16, dict(reduce_dtype=torch.float16), "reduce_dtype"),
    (torch.bfloat16, dict(reduce_dtype=torch.float64), "reduce_dtype"),
    (torch.float16, dict(reduce_dtype=torch.bfloat16), "reduce_dtype"),
    (torch.float32, dict(reduce_dtype=torch.float16), "reduce_dtype"),
    (torch.float32, dict(reduce_dtype=torch.float64, archive_dtype=torch.bfloat16), "reduce_dtype"),
    (torch.bfloat16, dict(reduce_dtype=torch.float32, archive_dtype=torch.float16), "archive|sums"),
    (torch.bfloat16, dict(reduce_dtype=torch.float32, accumulate=True), "needs acc"),
    (torch.bfloat16, dict(acc=[_f32()]), "acc needs"),
    (torch.float32, dict(acc=[_f32()], archive_dtype=torch.bfloat16), "acc needs"),
    (torch.float32, dict(acc=[_f32()], reduce_dtype=torch.float32, archive_dtype=torch.bfloat16), "acc needs"),
    (torch.bfloat16, dict(reduce_dtype=torch.float32, acc=[_f32(), _f32()]), "one tensor per group"),
    (torch.bfloat16, dict(reduce_dtype=torch.float32, acc=[_f32(dtype=torch.float64)]), "float32"),
    (torch.bfloat16, dict(reduce_dtype=torch.float32, acc=[_f32(dtype=torch.bfloat16)]), "float32"),
    (torch.bfloat16, dict(reduce_dtype=torch.float32, acc=[torch.zeros(8)[::2]]), "contiguous"),
    (torch.bfloat16, dict(reduce_dtype=torch.float32, acc=[_f32(5)]), "device|elements"),
    (torch.bfloat16, dict(reduce_dtype=torch.float32, acc=[_f32()]), "device"),
    (torch.bfloat16, dict(reduce_dtype=torch.float32, acc=[_f32()], accumulate=True), "device"),
    (torch.float16, dict(reduce_dtype=torch.float32, acc=[_f32()], sparse=True), "device"),
])
def test_ops_refuses_before_touching_archives(out_dtype, kw, match):
    from dietgpu_b200 import ops

    out = torch.empty(4, dtype=out_dtype)  # a CPU tensor: any device work would fail differently
    with pytest.raises(ValueError, match=match):
        ops.decompress_data_reduce([[Untouchable(), Untouchable()]], [out], **kw)


@pytest.mark.parametrize("reduce_dtype", [None, torch.bfloat16])
def test_ops_same_type_reduce_dtype_is_todays_call(reduce_dtype):
    # reduce_dtype None or the outputs' dtype reaches the existing entries (here: their output check, which a CPU
    # output fails with the RuntimeError it always raised)
    from dietgpu_b200 import ops

    with pytest.raises(RuntimeError, match="CUDA"):
        ops.decompress_data_reduce([[Untouchable()]], [torch.empty(4, dtype=torch.bfloat16)],
                                   reduce_dtype=reduce_dtype)


# ---- the collectives' refusals --------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype,kw", [
    (torch.bfloat16, dict(out_dtype=torch.float16)),  # a 16-bit sum cannot change type
    (torch.float16, dict(out_dtype=torch.bfloat16)),
    (torch.float16, dict(out_dtype=torch.float32)),
    (torch.bfloat16, dict(reduce_dtype=torch.float32, out_dtype=torch.float16)),  # not the archives' dtype
    (torch.float16, dict(reduce_dtype=torch.float32, out_dtype=torch.float64)),
    (torch.float32, dict(out_dtype=torch.bfloat16)),  # float32 archives: no narrowing decode
    (torch.float32, dict(out_dtype=torch.float16, wire_dtype=torch.bfloat16)),
    (torch.float32, dict(out_dtype=torch.float64)),
])
def test_collectives_refuse_out_dtype_before_communicating(dtype, kw, no_communication):
    import dietgpu_b200 as dg

    t = torch.zeros(64, dtype=dtype)
    with pytest.raises(ValueError, match="out_dtype"):
        dg.reduce_scatter_compressed(t, **kw)
    if "wire_dtype" not in kw:  # all_reduce_compressed has no wire dtype
        with pytest.raises(ValueError, match="out_dtype"):
            dg.all_reduce_compressed(t, **kw)


@pytest.mark.parametrize("kw", [dict(sparse=True), dict(average=True), dict(scale=0.5)])
def test_out_dtype_refusal_comes_with_the_other_keywords(kw, no_communication):
    import dietgpu_b200 as dg

    t = torch.zeros(64, dtype=torch.bfloat16)
    for f in (dg.reduce_scatter_compressed, dg.all_reduce_compressed):
        with pytest.raises(ValueError, match="out_dtype"):
            f(t, out_dtype=torch.float16, reduce_dtype=torch.float32, **kw)
