"""CPU tests of the squared norm: the numpy restatement (tests/sq_norm_reference.py) against math.fsum and against the
orders it rules out, and the argument checks of the C entries, of ops.decompress_data_reduce(sq_norm=) / ops.sq_norm
and of the collectives' sq_norm keyword, all of which refuse before any CUDA call, before any archive is read and
before any communication."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import sq_norm_reference as R
from dietgpu_b200 import capi
from multirank import Untouchable, no_communication  # noqa: F401  (no_communication is a fixture)

FAKE = 1 << 20  # never dereferenced: every call below fails (or returns) before it touches memory
BIG = {"f16": (2.0 ** 15, 2.0 ** -12), "bf16": (2.0 ** 27, 1.0), "f32": (2.0 ** 27, 1.0)}


# ---- the restatement ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [1, 31, 33, 4095, 4096, 4097, 70001, 1 << 20])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
def test_restatement_is_the_exact_sum_to_rounding(n, dtype):
    g = torch.Generator().manual_seed(n)
    x = torch.randn(n, generator=g).to(dtype).double().numpy()
    exact = math.fsum((x * x).tolist())
    got = R.sq_norm(x)
    assert abs(got - exact) <= 1e-13 * exact, (got, exact)


def test_empty_group_is_plus_zero():
    v = R.sq_norm(np.zeros(0))
    assert v == 0.0 and not np.signbit(v)
    assert not np.signbit(R.sq_norm(np.array([-0.0, -0.0])))


def test_non_finite_words_give_a_non_finite_norm():
    assert np.isinf(R.sq_norm(np.array([1.0, -np.inf, 2.0])))
    assert np.isnan(R.sq_norm(np.array([1.0, np.nan, np.inf])))


def _sequential(x):
    s = 0.0
    for v in x:
        s = s + v * v
    return np.float64(s)


@pytest.mark.parametrize("t", sorted(BIG))
def test_rows_are_added_in_descending_order(t):
    big, small = BIG[t]
    x = R.pin_rows(big, small)
    got = R.sq_norm(x)
    assert got == big * big  # every small square is absorbed
    ascending = _sequential(x[0::R.LANES])  # lane 0's words in ascending row order
    assert ascending != got
    assert R.same(R.sq_norm(x), R.fold_group([R.butterfly(R.lane_sums(x))[0]]))


@pytest.mark.parametrize("t", sorted(BIG))
def test_lanes_are_combined_by_the_butterfly(t):
    big, small = BIG[t]
    x = R.pin_lanes(big, small)
    got = R.sq_norm(x)
    # the alternatives: lanes in order, lanes in reverse order
    assert got != _sequential(x)
    assert got != _sequential(x[::-1])
    if t != "f16":
        # big^2 + 1 -> big^2, + 2 -> big^2 (a tie to even), then + 4, + 8, + 16 exactly
        assert got == big * big + 28.0


@pytest.mark.parametrize("t", sorted(BIG))
def test_blocks_are_folded_in_the_documented_order(t):
    big, small = BIG[t]
    x = R.pin_blocks(big, small)
    q = R.block_partials(x)
    got = R.fold_group(q)
    assert got != _sequential(np.sqrt(q))  # blocks in order
    assert got != _sequential(np.sqrt(q[::-1]))  # blocks in reverse order
    assert got != R.fold(np.concatenate([q[:1], [R.fold(q[1:])]]))  # the small ones first


def test_fold_is_in_index_order():
    assert R.fold([2.0 ** 54, 1.0, 1.0, 1.0]) == 2.0 ** 54
    assert R.fold([1.0, 1.0, 1.0, 2.0 ** 54]) == 2.0 ** 54 + 4.0


# ---- the C entries ---------------------------------------------------------------------------------------------------

ALLOWED = {(1, 1), (2, 2), (3, 3), (1, 3), (2, 3), (5, 1), (6, 2), (8, 3), (5, 3), (6, 3)}


def _dev(ft=capi.BFLOAT16, out_ft=capi.BFLOAT16, groups=1, width=1, scale_dev=FAKE, found_inf=None,
         sq_norm=FAKE, temp=None, temp_bytes=0, pb=10):
    n = max(1, groups * width)
    return capi.lib().dgb_float_decompress_reduce_scaled_dev_norm(
        temp, temp_bytes, ft, out_ft, pb, groups, width, capi.ptr_array([FAKE] * n),
        capi.ptr_array([FAKE] * max(1, groups)), capi.u32_array([100] * max(1, groups)), 0, scale_dev, found_inf,
        sq_norm, None, None)


def _narrow(ft=capi.BFLOAT16, groups=1, width=2, scale_dev=FAKE, found_inf=None, sq_norm=FAKE, acc=FAKE,
            temp=None, temp_bytes=0):
    n = max(1, groups * width)
    return capi.lib().dgb_float_decompress_reduce_narrow_norm(
        temp, temp_bytes, ft, 10, groups, width, capi.ptr_array([FAKE] * n),
        capi.ptr_array([acc] * max(1, groups)), capi.ptr_array([FAKE] * max(1, groups)),
        capi.u32_array([100] * max(1, groups)), 0, scale_dev, found_inf, sq_norm, None, None)


def _plain(ft=capi.FLOAT32, groups=1, sq_norm=FAKE, ins=None, sizes=None, temp=None, temp_bytes=0):
    return capi.lib().dgb_float_sq_norm(
        temp, temp_bytes, ft, groups, capi.ptr_array(ins if ins is not None else [FAKE] * max(1, groups)),
        capi.u32_array(sizes if sizes is not None else [100] * max(1, groups)), sq_norm, None)


@pytest.mark.parametrize("ft", range(10))
def test_dev_norm_type_pairs(ft):
    for out_ft in range(10):
        rc = _dev(ft=ft, out_ft=out_ft)
        want = capi.ERR_TEMP_TOO_SMALL if (ft, out_ft) in ALLOWED else capi.ERR_INVALID_ARG
        assert rc == want, (ft, out_ft, rc)


@pytest.mark.parametrize("ft", range(10))
def test_narrow_norm_and_plain_types(ft):
    assert _narrow(ft=ft) == (capi.ERR_TEMP_TOO_SMALL if ft in (1, 2, 5, 6) else capi.ERR_INVALID_ARG)
    assert _plain(ft=ft) == (capi.ERR_TEMP_TOO_SMALL if ft in (1, 2, 3) else capi.ERR_INVALID_ARG)


@pytest.mark.parametrize("sq_norm", [None, FAKE + 1, FAKE + 4])
def test_null_or_misaligned_norm_is_rejected(sq_norm):
    for groups in (1, 0):
        assert _dev(sq_norm=sq_norm, groups=groups) == capi.ERR_INVALID_ARG
        assert _narrow(sq_norm=sq_norm, groups=groups) == capi.ERR_INVALID_ARG
        assert _plain(sq_norm=sq_norm, groups=groups) == capi.ERR_INVALID_ARG
    # ... before the scratch is looked at
    assert _dev(sq_norm=sq_norm, temp=FAKE, temp_bytes=1 << 30) == capi.ERR_INVALID_ARG
    assert _plain(sq_norm=sq_norm, temp=FAKE, temp_bytes=1 << 30) == capi.ERR_INVALID_ARG


@pytest.mark.parametrize("scale_dev", [None, FAKE + 2])
def test_null_or_misaligned_scale_is_rejected(scale_dev):
    for groups in (1, 0):
        assert _dev(scale_dev=scale_dev, groups=groups) == capi.ERR_INVALID_ARG
        assert _narrow(scale_dev=scale_dev, groups=groups) == capi.ERR_INVALID_ARG


def test_the_extended_entries_refusals_are_kept():
    assert _dev(found_inf=FAKE + 2) == capi.ERR_INVALID_ARG
    assert _dev(pb=12) == capi.ERR_INVALID_ARG
    assert _dev(width=0) == capi.ERR_INVALID_ARG
    assert _narrow(found_inf=FAKE + 1) == capi.ERR_INVALID_ARG
    assert _narrow(acc=0, temp=FAKE, temp_bytes=1 << 30) == capi.ERR_INVALID_ARG  # W > 1 reads acc
    assert _plain(ins=[0], temp=FAKE, temp_bytes=1 << 30) == capi.ERR_INVALID_ARG
    assert _plain(ins=[FAKE + 2], temp=FAKE, temp_bytes=1 << 30) == capi.ERR_INVALID_ARG  # fp32 needs 4 B
    assert _plain(ft=capi.FLOAT16, ins=[FAKE + 2]) == capi.ERR_TEMP_TOO_SMALL  # 2 B is enough for fp16
    assert _plain(ins=[0], sizes=[0]) == capi.ERR_TEMP_TOO_SMALL  # an empty group needs no pointer


def test_no_groups_is_ok():
    assert _dev(groups=0) == capi.OK
    assert _narrow(groups=0) == capi.OK
    assert _plain(groups=0) == capi.OK


def test_scratch_sizes():
    L = capi.lib()
    sizes = [0, 1, 4096, 4097, 70001]
    blocks = sum(-(-n // 4096) for n in sizes)
    plain = L.dgb_float_sq_norm_temp_bytes(len(sizes), capi.u32_array(sizes))
    assert plain >= 8 * blocks + 8 * len(sizes)
    for ft in (1, 2, 3, 5, 6, 8):
        base = L.dgb_float_decompress_temp_bytes(ft, len(sizes) * 3, 0)
        red = L.dgb_float_decompress_reduce_norm_temp_bytes(ft, len(sizes), 3, capi.u32_array(sizes))
        assert red >= base + 8 * blocks and red - base == plain - 256 * -(-8 * len(sizes) // 256)
    assert L.dgb_float_decompress_reduce_norm_temp_bytes(9, 1, 1, capi.u32_array([1])) == 0
    # a too small scratch is refused: the decode's own scratch is not enough
    need = L.dgb_float_decompress_temp_bytes(capi.BFLOAT16, 1, 0)
    assert _dev(temp=FAKE, temp_bytes=need - 256) == capi.ERR_TEMP_TOO_SMALL


def test_signatures_are_declared():
    L = capi.lib()
    for name, n in (("dgb_float_decompress_reduce_scaled_dev_norm", 16), ("dgb_float_decompress_reduce_narrow_norm", 16),
                    ("dgb_float_sq_norm", 8), ("dgb_float_decompress_reduce_norm_temp_bytes", 4),
                    ("dgb_float_sq_norm_temp_bytes", 2)):
        assert name in capi.SYMBOLS
        assert len(getattr(L, name).argtypes) == n, name
    assert L.dgb_float_decompress_reduce_scaled_dev_norm.restype is C.c_int
    assert L.dgb_float_sq_norm_temp_bytes.restype is C.c_size_t


# ---- ops ----------------------------------------------------------------------------------------------------------------

def _one(dtype=torch.float32, n=1):
    return torch.ones(n, dtype=dtype)  # on the CPU: never the outputs' CUDA device


@pytest.mark.parametrize("kw,match", [
    (dict(sq_norm=_one(torch.float64)), "sq_norm needs scale_tensor"),
    (dict(scale=0.5, sq_norm=_one(torch.float64)), "sq_norm needs scale_tensor"),
    (dict(scale=0.5, scale_tensor=_one(), sq_norm=_one(torch.float64)), "not both"),
    (dict(found_inf=_one(), sq_norm=_one(torch.float64)), "needs scale_tensor"),
])
@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
def test_ops_refuses_before_touching_archives(kw, match, out_dtype):
    from dietgpu_b200 import ops

    out = torch.empty(4, dtype=out_dtype)
    with pytest.raises(ValueError, match=match):
        ops.decompress_data_reduce([[Untouchable()]], [out], **kw)
    with pytest.raises(ValueError, match=match):
        ops.decompress_data_reduce([[Untouchable()]], [out], reduce_dtype=torch.float32, **kw)


@pytest.mark.parametrize("bad,match", [
    (1.0, "float64 CUDA tensor"),
    (_one(torch.float32), "float64"),
    (_one(torch.float64, 2), "1 element"),
    (_one(torch.float64, 0), "1 element"),
    (torch.zeros(2, 2, dtype=torch.float64)[:, 0][:1].expand(2), "1 element"),
    (_one(torch.float64), "device"),  # a CPU tensor
])
def test_ops_checks_the_norm_tensor(bad, match):
    """decompress_data_reduce and the collectives check sq_norm with this, after scale_tensor (which a CPU run can
    never pass), before any archive is read or any communication."""
    from dietgpu_b200 import ops

    with pytest.raises(ValueError, match=match):
        ops._check_sq_norm("sq_norm", bad, 1, torch.device("cuda", 0))


@pytest.mark.parametrize("ts", [
    [torch.zeros(4, dtype=torch.float64)],
    [torch.zeros(4, dtype=torch.int32)],
    [torch.zeros(4)],  # a CPU tensor
])
def test_ops_sq_norm_refuses_before_device_work(ts):
    from dietgpu_b200 import ops

    with pytest.raises(ValueError):
        ops.sq_norm(ts)


# ---- the collectives ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kw,match", [
    (dict(sq_norm=_one(torch.float64)), "sq_norm needs scale_tensor"),
    (dict(scale=0.5, sq_norm=_one(torch.float64)), "sq_norm needs scale_tensor"),
    (dict(average=True, sq_norm=_one(torch.float64)), "sq_norm needs scale_tensor"),
    (dict(found_inf=_one(), sq_norm=_one(torch.float64)), "needs scale_tensor"),
    (dict(scale_tensor=_one(), sq_norm=_one(torch.float64)), "device"),
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
