"""CPU tests of the device-scale decode-and-sum: the argument checks of dgb_float_decompress_reduce_scaled_dev, of
ops.decompress_data_reduce(scale_tensor=, found_inf=) and of the collectives' scale_tensor / found_inf keywords, all
of which refuse before any CUDA call, before any archive is read and before any communication."""
import ctypes as C

import pytest
import torch

from dietgpu_b200 import capi
from multirank import Untouchable, no_communication  # noqa: F401  (no_communication is a fixture)

FAKE = 1 << 20  # never dereferenced: every call below fails (or returns) before it touches memory
ALLOWED = {(1, 1), (2, 2), (3, 3), (1, 3), (2, 3), (5, 1), (6, 2), (8, 3), (5, 3), (6, 3)}


def _call(ft=capi.BFLOAT16, out_ft=capi.BFLOAT16, pb=10, groups=1, width=1, scale_dev=FAKE, found_inf=None,
          temp=None, temp_bytes=0, out=FAKE):
    n = max(1, groups * width)
    return capi.lib().dgb_float_decompress_reduce_scaled_dev(
        temp, temp_bytes, ft, out_ft, pb, groups, width, capi.ptr_array([FAKE] * n),
        capi.ptr_array([out] * max(1, groups)), capi.u32_array([100] * max(1, groups)), 0, scale_dev, found_inf, None,
        None)


@pytest.mark.parametrize("ft", range(10))
def test_type_pairs(ft):
    for out_ft in range(10):
        for found_inf in (None, FAKE + 4):
            rc = _call(ft=ft, out_ft=out_ft, found_inf=found_inf)
            if (ft, out_ft) in ALLOWED:
                # the pair passes; the call then stops at the missing scratch
                assert rc == capi.ERR_TEMP_TOO_SMALL, (ft, out_ft, found_inf, rc)
            else:
                assert rc == capi.ERR_INVALID_ARG, (ft, out_ft, found_inf, rc)


def test_float64_is_rejected():
    assert _call(ft=capi.FLOAT64, out_ft=capi.FLOAT64) == capi.ERR_INVALID_ARG
    assert _call(ft=capi.FLOAT64, out_ft=capi.FLOAT64, groups=0) == capi.ERR_INVALID_ARG


@pytest.mark.parametrize("pb", [8, 12])
def test_prob_bits_out_of_range_are_rejected(pb):
    assert _call(pb=pb) == capi.ERR_INVALID_ARG


@pytest.mark.parametrize("scale_dev", [None, FAKE + 1, FAKE + 2, FAKE + 3])
def test_null_or_misaligned_scale_is_rejected(scale_dev):
    assert _call(scale_dev=scale_dev) == capi.ERR_INVALID_ARG
    # ... before anything else: with no groups, and with enough (fake) scratch
    assert _call(scale_dev=scale_dev, groups=0) == capi.ERR_INVALID_ARG
    assert _call(scale_dev=scale_dev, temp=FAKE, temp_bytes=1 << 30) == capi.ERR_INVALID_ARG


@pytest.mark.parametrize("found_inf", [FAKE + 1, FAKE + 2, FAKE + 3])
def test_misaligned_flag_is_rejected(found_inf):
    assert _call(found_inf=found_inf) == capi.ERR_INVALID_ARG
    assert _call(found_inf=found_inf, groups=0) == capi.ERR_INVALID_ARG


@pytest.mark.parametrize("found_inf", [None, FAKE + 4])
def test_valid_arguments_reach_the_scratch_check(found_inf):
    assert _call(found_inf=found_inf) == capi.ERR_TEMP_TOO_SMALL
    assert _call(found_inf=found_inf, temp=FAKE, temp_bytes=16) == capi.ERR_TEMP_TOO_SMALL
    assert _call(ft=capi.FLOAT32_SPARSE, out_ft=capi.FLOAT32, found_inf=found_inf) == capi.ERR_TEMP_TOO_SMALL


def test_no_groups_is_ok():
    assert _call(groups=0) == capi.OK
    assert _call(groups=0, found_inf=FAKE) == capi.OK


def test_misaligned_fp32_output_is_rejected():
    # a 2 B aligned output is fine for 16-bit sums, not for fp32 ones; the check happens before any CUDA call
    assert _call(ft=capi.BFLOAT16, out_ft=capi.FLOAT32, temp=FAKE, temp_bytes=1 << 20, out=FAKE + 2) \
        == capi.ERR_INVALID_ARG


def test_signature_is_declared():
    f = capi.lib().dgb_float_decompress_reduce_scaled_dev
    assert f.restype is C.c_int and len(f.argtypes) == 15
    assert f.argtypes[10] is C.c_int and f.argtypes[11] is C.c_void_p and f.argtypes[12] is C.c_void_p
    assert "dgb_float_decompress_reduce_scaled_dev" in capi.SYMBOLS


# ---- ops.decompress_data_reduce(scale_tensor=, found_inf=) ----------------------------------------------------------

def _one(dtype=torch.float32, n=1):
    return torch.ones(n, dtype=dtype)  # on the CPU: never the outputs' CUDA device


@pytest.mark.parametrize("kw,match", [
    (dict(scale=0.5, scale_tensor=_one()), "not both"),
    (dict(found_inf=_one()), "found_inf needs scale_tensor"),
    (dict(scale=0.5, found_inf=_one()), "found_inf needs scale_tensor"),
    (dict(scale_tensor=0.5), "scale_tensor"),
    (dict(scale_tensor=_one(torch.float64)), "scale_tensor"),
    (dict(scale_tensor=_one(torch.float16)), "scale_tensor"),
    (dict(scale_tensor=_one(n=2)), "scale_tensor"),
    (dict(scale_tensor=_one(n=0)), "scale_tensor"),
    (dict(scale_tensor=_one()), "device"),
    (dict(scale_tensor=_one(), found_inf=_one(torch.int32)), "scale_tensor|found_inf"),
])
@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
def test_ops_refuses_before_touching_archives(kw, match, out_dtype):
    from dietgpu_b200 import ops

    out = torch.empty(4, dtype=out_dtype)  # a CPU tensor: any device work would fail differently
    with pytest.raises(ValueError, match=match):
        ops.decompress_data_reduce([[Untouchable()]], [out], **kw)


def test_ops_checks_the_flag_too():
    from dietgpu_b200 import ops

    out = torch.empty(4, dtype=torch.bfloat16)
    for bad in (_one(torch.float64), _one(n=2), _one(n=0), 1.0, _one()):
        with pytest.raises(ValueError, match="found_inf"):
            ops._check_flag_tensor("found_inf", bad, torch.device("cpu"))  # a CPU tensor is never accepted
    with pytest.raises(ValueError):
        ops.decompress_data_reduce([[Untouchable()]], [out], scale_tensor=_one(), found_inf=_one(n=2))


def test_ops_keeps_refusing_tensor_scales():
    from dietgpu_b200 import ops

    with pytest.raises(TypeError, match="scale"):
        ops.decompress_data_reduce([[Untouchable()]], [torch.empty(4)], scale=torch.tensor(0.5))


# ---- the collectives' refusals --------------------------------------------------------------------------------------

@pytest.mark.parametrize("kw,match", [
    (dict(scale=0.5, scale_tensor=_one()), "scale_tensor replaces"),
    (dict(average=True, scale_tensor=_one()), "scale_tensor replaces"),
    (dict(average=True, scale_tensor=_one(), found_inf=_one()), "scale_tensor replaces"),
    (dict(found_inf=_one()), "found_inf needs scale_tensor"),
    (dict(scale=0.5, found_inf=_one()), "found_inf needs scale_tensor"),
    (dict(average=True, found_inf=_one()), "found_inf needs scale_tensor"),
    (dict(scale_tensor=0.5), "scale_tensor"),
    (dict(scale_tensor=_one(torch.float64)), "scale_tensor"),
    (dict(scale_tensor=_one(n=3)), "scale_tensor"),
    (dict(scale_tensor=_one()), "device"),
])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
def test_collectives_refuse_before_communicating(dtype, kw, match, no_communication):
    import dietgpu_b200 as dg

    t = torch.zeros(64, dtype=dtype)
    with pytest.raises(ValueError, match=match):
        dg.reduce_scatter_compressed(t, **kw)
    with pytest.raises(ValueError, match=match):
        dg.all_reduce_compressed(t, **kw)
    with pytest.raises(ValueError, match=match):
        dg.reduce_scatter_compressed(t, sparse=True, **kw)
    with pytest.raises(ValueError, match=match):
        dg.all_reduce_compressed(t, reduce_dtype=torch.float32, **kw)


def test_collectives_keep_their_other_refusals(no_communication):
    import dietgpu_b200 as dg

    with pytest.raises(ValueError, match="average"):
        dg.reduce_scatter_compressed(torch.zeros(64), scale=0.5, average=True, scale_tensor=_one())
    with pytest.raises(TypeError, match="scale"):
        dg.all_reduce_compressed(torch.zeros(64), scale=torch.tensor(0.5))
