"""CPU tests of error feedback on the narrowing compress: dgb_float_compress_to_ef's argument checks,
compress_data(error_feedback=)'s and the collectives' refusals (every one before any device work or communication),
and the torch expression the GPU tests compare the kernels' residuals with, pinned against a numpy restatement of
the contract in include/dietgpu_b200.h:

    y = x + e (fp32, round to nearest)    w = round_T(y)    e' = y - float(w) if w is finite else +0
"""
import ctypes as C
import inspect

import numpy as np
import pytest
import torch

from dietgpu_b200 import capi
from ef_reference import np_step
from multirank import Untouchable, no_communication  # noqa: F401  (no_communication is a fixture)

FAKE = 1 << 20  # never dereferenced: every call below fails (or returns) before it touches memory


# ---- the contract, restated in numpy (ef_reference.np_step) ---------------------------------------------------------

def torch_step(x: torch.Tensor, e: torch.Tensor, dt):
    """The torch expression the library's residuals equal bit for bit"""
    y = x + e
    w = y.to(dt)
    return y, w.float(), torch.where(w.isfinite(), y - w.float(), 0)


def _bits(a) -> np.ndarray:
    a = a.numpy() if isinstance(a, torch.Tensor) else a
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _assert_same(x: np.ndarray, e: np.ndarray, dt):
    ny, nw, nr = np_step(x, e, dt)
    ty, tw, tr = torch_step(torch.from_numpy(x), torch.from_numpy(e), dt)
    assert np.array_equal(_bits(ty), _bits(ny))
    fin = np.isfinite(nw)
    assert np.array_equal(_bits(tw)[fin], _bits(nw)[fin])
    assert np.array_equal(np.isfinite(tw.numpy()), fin)
    assert np.array_equal(_bits(tr), _bits(nr))
    return ny, nw, nr


DTYPES = [torch.float16, torch.bfloat16]


@pytest.mark.parametrize("dt", DTYPES)
def test_torch_expression_is_the_contract_on_random_words(dt):
    rng = np.random.default_rng(3)
    # every exponent, both signs, plus residuals of the size a previous step leaves
    x = rng.integers(0, 1 << 32, 200000, dtype=np.uint64).astype(np.uint32).view(np.float32)
    e = (rng.standard_normal(200000) * np.exp2(rng.integers(-140, 20, 200000))).astype(np.float32)
    e[::7] = 0.0
    y, w, r = _assert_same(x, e, dt)
    # y - w is exact: the fp32 residual is the real difference (checked in fp64), and never inf or NaN
    fin = np.isfinite(w)
    assert np.array_equal(r[fin].astype(np.float64), y[fin].astype(np.float64) - w[fin].astype(np.float64))
    assert np.isfinite(r).all()
    assert (_bits(r)[~fin] == 0).all()


@pytest.mark.parametrize("dt", DTYPES)
def test_signed_zeros_and_exact_words(dt):
    x = np.array([-0.0, -0.0, 0.0, 1.0, -2.5, 0.0, 3.0], dtype=np.float32)
    e = np.array([0.0, -0.0, -0.0, 0.0, 0.0, 1.0, -0.0], dtype=np.float32)
    y, w, r = _assert_same(x, e, dt)
    # -0 + +0 = +0; -0 + -0 = -0, whose residual -0 - -0 is +0; y == w leaves +0
    assert _bits(y)[0] == 0 and _bits(y)[1] == 0x80000000
    assert (_bits(r) == 0).all()


def test_fp16_overflow_boundary():
    below = np.nextafter(np.float32(65520.0), np.float32(0.0))
    x = np.array([below, -below, 65520.0, -65520.0, 65504.0, 1e6], dtype=np.float32)
    y, w, r = _assert_same(x, np.zeros_like(x), torch.float16)
    # the largest float32 below 65520 rounds to 65504 and keeps its residual; 65520 rounds to inf with residual 0
    assert w[0] == 65504.0 and w[1] == -65504.0
    assert r[0] == below - np.float32(65504.0) and r[1] == -r[0] and r[0] > 0
    assert np.isinf(w[2]) and np.isinf(w[3]) and np.isinf(w[5])
    assert (_bits(r)[[2, 3, 5]] == 0).all() and r[4] == 0.0


@pytest.mark.parametrize("dt", DTYPES)
def test_non_finite_words_leave_a_zero_residual(dt):
    inf, nan = np.float32(np.inf), np.float32(np.nan)
    x = np.array([inf, -inf, nan, 1.0, 1.0, 1.0, inf], dtype=np.float32)
    e = np.array([0.0, 0.0, 0.0, inf, -inf, nan, -inf], dtype=np.float32)
    _, w, r = _assert_same(x, e, dt)
    assert not np.isfinite(w).any()
    assert (_bits(r) == 0).all()


@pytest.mark.parametrize("dt", DTYPES)
def test_subnormal_sums(dt):
    tiny = np.float32(1e-40)  # a float32 subnormal: fp16 rounds it to 0, bf16 to a bf16 subnormal
    x = np.array([tiny, -tiny, 3e-6, 6e-8, 1e-45, 2.0 ** -126], dtype=np.float32)
    e = np.array([tiny, 0.0, 1e-9, 0.0, 1e-45, -(2.0 ** -127)], dtype=np.float32)
    y, w, r = _assert_same(x, e, dt)
    assert y[0] == 2 * tiny and y[5] == np.float32(2.0 ** -127)  # subnormal sums are kept, not flushed
    if dt == torch.float16:
        assert w[0] == 0.0 and r[0] == y[0]  # the whole word is the residual
        assert 0 < abs(w[2]) < 6.2e-5  # an fp16 subnormal
    else:
        assert 0 < abs(w[0]) < 1.2e-38 and r[0] == y[0] - w[0]
    fin = np.isfinite(w)
    assert np.array_equal(r[fin].astype(np.float64), y[fin].astype(np.float64) - w[fin].astype(np.float64))


# ---- C ABI -----------------------------------------------------------------------------------------------------------

def _call(in_ft=capi.FLOAT32, ft=capi.BFLOAT16, pb=10, n=1, errs="ok", err_ptr=FAKE, in_ptr=FAKE, size=100):
    err_arr = capi.ptr_array([err_ptr] * n) if errs == "ok" else None
    return capi.lib().dgb_float_compress_to_ef(None, 0, in_ft, ft, pb, 0, n, capi.ptr_array([in_ptr] * n),
                                               capi.u32_array([size] * n), err_arr, capi.ptr_array([FAKE] * n),
                                               None, None)


@pytest.mark.parametrize("in_ft", range(10))
def test_capi_type_pairs(in_ft):
    for ft in range(10):
        rc = _call(in_ft=in_ft, ft=ft)
        if (in_ft, ft) in ((3, 1), (3, 2)):
            assert rc == capi.ERR_TEMP_TOO_SMALL, (in_ft, ft, rc)  # the pair passes; the call stops at the scratch
        else:
            assert rc == capi.ERR_INVALID_ARG, (in_ft, ft, rc)


@pytest.mark.parametrize("ft", [capi.FLOAT16, capi.BFLOAT16])
def test_capi_null_and_misaligned_residuals(ft):
    assert _call(ft=ft, errs=None) == capi.ERR_INVALID_ARG
    assert _call(ft=ft, errs=None, n=0) == capi.ERR_INVALID_ARG
    assert _call(ft=ft, err_ptr=0) == capi.ERR_INVALID_ARG
    for off in (4, 8, 12):
        assert _call(ft=ft, err_ptr=FAKE + off) == capi.ERR_INVALID_ARG
        assert _call(ft=ft, in_ptr=FAKE + off) == capi.ERR_INVALID_ARG
        # the same address modulo 16 is what the kernels need, not 16 B alignment
        assert _call(ft=ft, in_ptr=FAKE + off, err_ptr=2 * FAKE + 32 + off) == capi.ERR_TEMP_TOO_SMALL
    assert _call(ft=ft, err_ptr=2 * FAKE) == capi.ERR_TEMP_TOO_SMALL
    # an empty member reads neither its input nor its residual
    assert _call(ft=ft, err_ptr=0, in_ptr=0, size=0) == capi.ERR_TEMP_TOO_SMALL
    assert _call(ft=ft, n=0) == capi.OK


@pytest.mark.parametrize("pb", [8, 12])
def test_capi_prob_bits_out_of_range_are_rejected(pb):
    assert _call(pb=pb) == capi.ERR_INVALID_ARG


def test_capi_signature_is_declared():
    f = capi.lib().dgb_float_compress_to_ef
    assert f.restype is C.c_int and len(f.argtypes) == 13
    assert "dgb_float_compress_to_ef" in capi.SYMBOLS


# ---- compress_data(error_feedback=) ----------------------------------------------------------------------------------

class FakeCuda:
    """The metadata of a CUDA tensor at a chosen address: enough for every check, and any other use fails the
    test (so a call that got past its checks would fail loudly instead of touching a device)."""

    def __init__(self, numel, dtype=torch.float32, ptr=FAKE, shape=None, contiguous=True, index=0):
        self.dtype, self.is_cuda, self.device = dtype, True, torch.device("cuda", index)
        self.shape = torch.Size(shape if shape is not None else (numel,))
        self._numel, self._ptr, self._contiguous = numel, ptr, contiguous

    def numel(self):
        return self._numel

    def data_ptr(self):
        return self._ptr

    def element_size(self):
        return torch.empty(0, dtype=self.dtype).element_size()

    def is_contiguous(self):
        return self._contiguous

    def __getattr__(self, name):
        raise AssertionError(f"{name} of a tensor used before the call was refused")


class Reached(Exception):
    """A compress that passed every check got as far as allocating its output."""


@pytest.fixture(autouse=True)
def stop_before_the_device(monkeypatch):
    """A call with fake tensors that passed its checks stops where it would first allocate device memory, so no
    kernel can ever see a fake address."""
    from dietgpu_b200 import ops

    def stop(*a, **k):
        raise Reached()

    monkeypatch.setattr(ops, "_validate_out", stop)


def _compress(ts, errs, archive_dtype=torch.bfloat16, **kw):
    from dietgpu_b200 import ops

    return ops.compress_data(kw.pop("as_float", True), ts, archive_dtype=archive_dtype, error_feedback=errs, **kw)


@pytest.mark.parametrize("in_dtype,archive_dtype,kw", [
    (torch.float32, None, {}),                           # no narrowing
    (torch.float32, torch.float32, {}),                  # archive_dtype == the inputs' dtype
    (torch.bfloat16, torch.bfloat16, {}),
    (torch.float32, None, dict(as_float=False)),         # byte mode
    (torch.float32, None, dict(sparse=True)),            # sparse archives
])
def test_ops_error_feedback_needs_a_narrowing_compress(in_dtype, archive_dtype, kw):
    t = torch.zeros(16, dtype=in_dtype)  # a CPU tensor: a call that got past the refusal would fail differently
    with pytest.raises(ValueError, match="error_feedback needs a narrowing compress"):
        _compress([t], [torch.zeros(16)], archive_dtype, **kw)


@pytest.mark.parametrize("in_dtype,archive_dtype,kw", [
    (torch.float16, torch.bfloat16, {}),
    (torch.float32, torch.float64, {}),
    (torch.float32, torch.bfloat16, dict(sparse=True)),
    (torch.float32, torch.float16, dict(as_float=False)),
])
def test_ops_narrowing_refusal_keeps_priority(in_dtype, archive_dtype, kw):
    t = torch.zeros(16, dtype=in_dtype)
    with pytest.raises(ValueError, match="archive_dtype narrows float32 inputs"):
        _compress([t], [torch.zeros(16)], archive_dtype, **kw)


def test_ops_input_refusal_keeps_its_error():
    # a CPU input fails the input check it always failed, before the residuals are looked at
    with pytest.raises(RuntimeError, match="check failed"):
        _compress([torch.zeros(16)], [Untouchable()])


def _bad_feedback_cases():
    n = 1000
    ins = [FakeCuda(n, ptr=FAKE), FakeCuda(n, ptr=2 * FAKE)]
    ok = lambda: [FakeCuda(n, ptr=3 * FAKE), FakeCuda(n, ptr=4 * FAKE)]  # noqa: E731
    cases = {
        "not a list": (ins, FakeCuda(n, ptr=3 * FAKE)),
        "too short": (ins, ok()[:1]),
        "too long": (ins, ok() + [FakeCuda(n, ptr=5 * FAKE)]),
        "float16": (ins, [FakeCuda(n, torch.float16, ptr=3 * FAKE), ok()[1]]),
        "float64": (ins, [ok()[0], FakeCuda(n, torch.float64, ptr=4 * FAKE)]),
        "cpu": (ins, [torch.zeros(n), ok()[1]]),
        "other device": (ins, [FakeCuda(n, ptr=3 * FAKE, index=1), ok()[1]]),
        "numel": (ins, [FakeCuda(n - 1, ptr=3 * FAKE), ok()[1]]),
        "not contiguous": (ins, [FakeCuda(n, ptr=3 * FAKE, contiguous=False), ok()[1]]),
        "alignment": (ins, [FakeCuda(n, ptr=3 * FAKE + 4), ok()[1]]),
        "alignment 2": (ins, [ok()[0], FakeCuda(n, ptr=4 * FAKE + 8)]),
        "overlaps its input": (ins, [FakeCuda(n, ptr=FAKE), ok()[1]]),
        "overlaps the other input": (ins, [FakeCuda(n, ptr=2 * FAKE + 16), ok()[1]]),
        "ends inside an input": (ins, [FakeCuda(n, ptr=2 * FAKE - 4 * n + 16), ok()[1]]),
        "overlaps another residual": (ins, [FakeCuda(n, ptr=3 * FAKE), FakeCuda(n, ptr=3 * FAKE + 4 * n - 16)]),
        "the same residual twice": (ins, [FakeCuda(n, ptr=3 * FAKE), FakeCuda(n, ptr=3 * FAKE)]),
    }
    return cases


@pytest.mark.parametrize("case", list(_bad_feedback_cases()))
def test_ops_bad_error_feedback_is_refused_before_the_device(case):
    ins, errs = _bad_feedback_cases()[case]
    with pytest.raises(ValueError, match="error_feedback"):
        _compress(ins, errs)
    with pytest.raises(ValueError, match="error_feedback"):
        _compress(ins, errs, archive_dtype=torch.float16)


def test_ops_inputs_may_overlap_each_other_and_empty_members_are_free():
    # two inputs at one address, and empty members at address 0 or misaligned, pass every check
    ins = [FakeCuda(100, ptr=FAKE), FakeCuda(100, ptr=FAKE), FakeCuda(0, ptr=0)]
    errs = [FakeCuda(100, ptr=2 * FAKE), FakeCuda(100, ptr=3 * FAKE), FakeCuda(0, ptr=FAKE + 4)]
    with pytest.raises(Reached):
        _compress(ins, errs)
    with pytest.raises(Reached):
        _compress(ins, errs, archive_dtype=torch.float16)


# ---- the collectives -------------------------------------------------------------------------------------------------

def _collectives():
    import dietgpu_b200 as dg

    return [dg.reduce_scatter_compressed, dg.all_gather_compressed]


@pytest.mark.parametrize("which", [0, 1])
def test_collectives_error_feedback_needs_wire_dtype(which, no_communication):
    f = _collectives()[which]
    with pytest.raises(ValueError, match="error_feedback needs wire_dtype"):
        f(FakeCuda(64), error_feedback=FakeCuda(64, ptr=2 * FAKE))


def _bad_collective_feedback():
    return {
        "float16": FakeCuda(64, torch.float16, ptr=2 * FAKE),
        "cpu": torch.zeros(64),
        "other device": FakeCuda(64, ptr=2 * FAKE, index=1),
        "shape": FakeCuda(64, ptr=2 * FAKE, shape=(8, 8)),
        "numel": FakeCuda(63, ptr=2 * FAKE),
        "not contiguous": FakeCuda(64, ptr=2 * FAKE, contiguous=False),
        "alignment": FakeCuda(64, ptr=2 * FAKE + 12),
        "overlaps t": FakeCuda(64, ptr=FAKE + 128),
        "is t": FakeCuda(64, ptr=FAKE),
        "not a tensor": [0.0] * 64,
    }


@pytest.mark.parametrize("which", [0, 1])
@pytest.mark.parametrize("case", list(_bad_collective_feedback()))
def test_collectives_refuse_bad_error_feedback_before_communicating(which, case, no_communication):
    f = _collectives()[which]
    e = _bad_collective_feedback()[case]
    for wire in (torch.float16, torch.bfloat16):
        with pytest.raises(ValueError, match="error_feedback"):
            f(FakeCuda(64), wire_dtype=wire, error_feedback=e)


@pytest.mark.parametrize("which", [0, 1])
def test_collectives_existing_refusals_keep_their_messages(which, no_communication):
    f = _collectives()[which]
    e = FakeCuda(64, ptr=2 * FAKE)
    with pytest.raises(ValueError, match="sparse=True cannot be combined with wire_dtype"):
        f(FakeCuda(64), wire_dtype=torch.bfloat16, sparse=True, error_feedback=e)
    with pytest.raises(ValueError, match="contiguous CUDA tensor expected"):
        f(torch.zeros(64), wire_dtype=torch.bfloat16, error_feedback=e)
    with pytest.raises(ValueError, match="wire_dtype is None, or float16 / bfloat16 for a float32 tensor"):
        f(FakeCuda(64, torch.float16), wire_dtype=torch.bfloat16, error_feedback=e)
    with pytest.raises(ValueError, match="wire_dtype is None, or float16 / bfloat16 for a float32 tensor"):
        f(FakeCuda(64), wire_dtype=torch.float32, error_feedback=e)


def test_reduce_scatter_existing_refusals_keep_their_messages(no_communication):
    import dietgpu_b200 as dg

    e = FakeCuda(64, ptr=2 * FAKE)
    t = FakeCuda(64)
    with pytest.raises(ValueError, match="pass average=True or a scale, not both"):
        dg.reduce_scatter_compressed(t, wire_dtype=torch.bfloat16, average=True, scale=0.5, error_feedback=e)
    with pytest.raises(ValueError, match="found_inf needs scale_tensor"):
        dg.reduce_scatter_compressed(t, wire_dtype=torch.bfloat16, found_inf=FakeCuda(1), error_feedback=e)
    with pytest.raises(ValueError, match="out_dtype"):
        dg.reduce_scatter_compressed(t, wire_dtype=torch.bfloat16, out_dtype=torch.float16, error_feedback=e)
    with pytest.raises(ValueError, match="reduce_dtype"):
        dg.reduce_scatter_compressed(t, wire_dtype=torch.bfloat16, reduce_dtype=torch.float16, error_feedback=e)


def test_all_gather_peer_refusal_keeps_its_message(no_communication):
    import dietgpu_b200 as dg

    with pytest.raises(ValueError, match="wire_dtype is not supported with the peer-memory transports"):
        dg.all_gather_compressed(FakeCuda(64), peer=Untouchable(), wire_dtype=torch.bfloat16,
                                 error_feedback=FakeCuda(64, ptr=2 * FAKE))


def test_all_reduce_has_no_error_feedback():
    import dietgpu_b200 as dg

    params = inspect.signature(dg.all_reduce_compressed).parameters
    assert "error_feedback" not in params and "wire_dtype" not in params
