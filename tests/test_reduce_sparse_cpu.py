"""CPU tests of the sparse decode-and-sum's argument checks (dgb_float_decompress_reduce_sparse,
ops.decompress_data_reduce(sparse=True)) and of the collectives' sparse=True refusals: every one of them happens
before any CUDA call or any communication, so these run without a device."""
import ctypes as C

import pytest
import torch

from dietgpu_b200 import capi
from multirank import Untouchable, no_communication  # noqa: F401  (no_communication is a fixture)

FAKE = 1 << 20  # never dereferenced: every call below fails (or returns) before it touches memory
ALLOWED = {(5, 1), (6, 2), (8, 3), (5, 3), (6, 3)}


def _call(ft=capi.BFLOAT16_SPARSE, out_ft=capi.BFLOAT16, pb=10, groups=1, width=1, ins="ok", outs="ok", sizes="ok"):
    n = max(1, groups * width)
    in_arr = capi.ptr_array([FAKE] * n) if ins == "ok" else None
    out_arr = capi.ptr_array([FAKE] * max(1, groups)) if outs == "ok" else None
    size_arr = capi.u32_array([100] * max(1, groups)) if sizes == "ok" else None
    return capi.lib().dgb_float_decompress_reduce_sparse(None, 0, ft, out_ft, pb, groups, width, in_arr, out_arr,
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
    assert _call(ft=capi.FLOAT32_SPARSE, out_ft=capi.FLOAT32, groups=0) == capi.OK
    # ... but only for an allowed pair
    assert _call(ft=capi.BFLOAT16, out_ft=capi.BFLOAT16, groups=0) == capi.ERR_INVALID_ARG


@pytest.mark.parametrize("ft,out_ft", [(capi.FLOAT16_SPARSE, capi.FLOAT32), (capi.BFLOAT16_SPARSE, capi.FLOAT32),
                                       (capi.FLOAT32_SPARSE, capi.FLOAT32)])
def test_misaligned_fp32_output_is_rejected(ft, out_ft):
    # a 2 B aligned output is fine for 16-bit sums, not for fp32 ones; the check happens before any CUDA call
    rc = capi.lib().dgb_float_decompress_reduce_sparse(FAKE, 1 << 20, ft, out_ft, 10, 1, 1, capi.ptr_array([FAKE]),
                                                       capi.ptr_array([FAKE + 2]), capi.u32_array([100]), 0, None,
                                                       None)
    assert rc == capi.ERR_INVALID_ARG


def test_dense_entries_still_refuse_sparse_types():
    L = capi.lib()
    for ft in (capi.FLOAT16_SPARSE, capi.BFLOAT16_SPARSE, capi.FLOAT32_SPARSE):
        for out_ft in (1, 2, 3, ft):
            rc = L.dgb_float_decompress_reduce_to(None, 0, ft, out_ft, 10, 1, 1, capi.ptr_array([FAKE]),
                                                  capi.ptr_array([FAKE]), capi.u32_array([100]), 0, None, None)
            assert rc == capi.ERR_INVALID_ARG, (ft, out_ft)


def test_signature_is_declared():
    f = capi.lib().dgb_float_decompress_reduce_sparse
    assert f.restype is C.c_int and len(f.argtypes) == 13
    assert "dgb_float_decompress_reduce_sparse" in capi.SYMBOLS


# ---- ops.decompress_data_reduce(sparse=True) ------------------------------------------------------------------------

@pytest.mark.parametrize("archive_dtype,out_dtype", [
    (torch.float32, torch.float16), (torch.float32, torch.bfloat16), (torch.float16, torch.bfloat16),
    (torch.bfloat16, torch.float16), (torch.float64, torch.float64), (torch.float64, torch.float32),
    (torch.int32, torch.float32), (torch.uint8, torch.float16)])
def test_ops_refuses_bad_pairs_first(archive_dtype, out_dtype):
    from dietgpu_b200 import ops

    out = torch.empty(4, dtype=out_dtype)  # a CPU tensor: any device work would fail differently
    with pytest.raises(ValueError):
        ops.decompress_data_reduce([[Untouchable()]], [out], archive_dtype=archive_dtype, sparse=True)


# ---- the collectives' refusals --------------------------------------------------------------------------------------

def _allow_world_size_query(monkeypatch):
    """all_to_all_compressed checks its chunk count against the world size before its other arguments; outside a
    process group that is 1 and asks nothing of another process."""
    import torch.distributed as dist

    monkeypatch.setattr(dist, "is_initialized", lambda: False)


@pytest.mark.parametrize("dtype", [torch.float64, torch.int32, torch.uint8, torch.int16])
def test_collectives_refuse_other_dtypes(dtype, no_communication):
    import dietgpu_b200 as dg

    t = torch.zeros(64, dtype=dtype)
    with pytest.raises(ValueError, match="sparse"):
        dg.all_gather_compressed(t, sparse=True)
    with pytest.raises(ValueError, match="sparse"):
        dg.reduce_scatter_compressed(t, sparse=True)
    with pytest.raises(ValueError, match="sparse"):
        dg.all_reduce_compressed(t, sparse=True)
    _allow_world_size_query(no_communication)
    with pytest.raises(ValueError, match="sparse"):
        dg.all_to_all_compressed([t], sparse=True)


@pytest.mark.parametrize("wire", [torch.float16, torch.bfloat16])
def test_collectives_refuse_wire_dtype(wire, no_communication):
    import dietgpu_b200 as dg

    t = torch.zeros(64, dtype=torch.float32)
    with pytest.raises(ValueError, match="wire_dtype"):
        dg.all_gather_compressed(t, wire_dtype=wire, sparse=True)
    with pytest.raises(ValueError, match="wire_dtype"):
        dg.reduce_scatter_compressed(t, wire_dtype=wire, sparse=True)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
def test_collectives_refuse_peer_transports(dtype, no_communication):
    import dietgpu_b200 as dg

    t = torch.zeros(64, dtype=dtype)
    ws = object()  # never used: the refusal comes first
    with pytest.raises(ValueError, match="peer"):
        dg.all_gather_compressed(t, peer=ws, sparse=True)
    _allow_world_size_query(no_communication)
    with pytest.raises(ValueError, match="peer"):
        dg.all_to_all_compressed([t], peer=ws, sparse=True)
