"""CPU tests of the fp8 wire: the argument checks of dgb_float_cast_fp8 and of the fp8 decode-and-sum pairs, which
refuse before any CUDA call; the Python refusals of ops.cast_fp8, compress_data / decompress_data_reduce with an fp8
archive_dtype and the collectives' fp8 wire_dtype / wire_scale, before any device work or communication; and the
numpy restatement of the cast (tests/fp8_reference.py) against torch's CPU clamp-cast on the edge corpus."""
import numpy as np
import pytest
import torch

from dietgpu_b200 import capi
from fp8_reference import E4M3, E5M2, MAX, NAN_BYTE, cast, edge_corpus
from multirank import Untouchable, no_communication  # noqa: F401  (no_communication is a fixture)

FAKE = 1 << 20  # never dereferenced: every call below fails (or returns) before it touches memory
FP8 = {capi.FLOAT8_E4M3: torch.float8_e4m3fn, capi.FLOAT8_E5M2: torch.float8_e5m2}
CAST_PAIRS = {(3, 10), (3, 11), (2, 10), (2, 11)}
# the device-scale decode-and-sum pairs: the existing ten and the two fp8 ones
REDUCE_PAIRS = {(1, 1), (2, 2), (3, 3), (1, 3), (2, 3), (5, 1), (6, 2), (8, 3), (5, 3), (6, 3), (10, 3), (11, 3)}


def _cast(in_ft=3, ft=10, n=1, ins=None, sizes=None, scale=None, outs=None, hist=None):
    L = capi.lib()
    return L.dgb_float_cast_fp8(in_ft, ft, n, None if ins is False else capi.ptr_array(ins or [FAKE] * max(1, n)),
                                capi.u32_array(sizes or [100] * max(1, n)), scale,
                                None if outs is False else capi.ptr_array(outs or [FAKE] * max(1, n)), hist, None)


def test_cast_symbol_is_exported_and_declared():
    assert "dgb_float_cast_fp8" in capi.SYMBOLS
    assert hasattr(capi.lib(), "dgb_float_cast_fp8")
    assert (capi.FLOAT8_E4M3, capi.FLOAT8_E5M2) == (10, 11)


@pytest.mark.parametrize("in_ft", range(16))
def test_cast_type_pairs(in_ft):
    for ft in range(16):
        # n = 0: an allowed pair returns at once, any other pair is refused first
        rc = _cast(in_ft, ft, n=0, ins=False, outs=False)
        assert rc == (capi.OK if (in_ft, ft) in CAST_PAIRS else capi.ERR_INVALID_ARG), (in_ft, ft, rc)
        if (in_ft, ft) not in CAST_PAIRS:
            assert _cast(in_ft, ft) == capi.ERR_INVALID_ARG


@pytest.mark.parametrize("in_ft,wb", [(3, 4), (2, 2)])
def test_cast_null_and_misaligned_arguments(in_ft, wb):
    for ft in (10, 11):
        assert _cast(in_ft, ft, ins=False) == capi.ERR_INVALID_ARG
        assert _cast(in_ft, ft, outs=False) == capi.ERR_INVALID_ARG
        assert _cast(in_ft, ft, ins=[0]) == capi.ERR_INVALID_ARG
        assert _cast(in_ft, ft, outs=[0]) == capi.ERR_INVALID_ARG
        for off in range(1, wb):
            assert _cast(in_ft, ft, ins=[FAKE + off]) == capi.ERR_INVALID_ARG, off
        for off in (1, 2, 3):
            assert _cast(in_ft, ft, scale=FAKE + off) == capi.ERR_INVALID_ARG, off
            assert _cast(in_ft, ft, hist=FAKE + off) == capi.ERR_INVALID_ARG, off
        # a bad member anywhere in the batch refuses the whole call (before any CUDA call)
        assert _cast(in_ft, ft, n=3, ins=[FAKE, FAKE, 0]) == capi.ERR_INVALID_ARG


def _dev(ft, out_ft, norm=False, groups=1, temp=None, temp_bytes=0):
    L = capi.lib()
    args = (temp, temp_bytes, ft, out_ft, 10, groups, 1, capi.ptr_array([FAKE]), capi.ptr_array([FAKE]),
            capi.u32_array([100]), 0, FAKE, None)
    if norm:
        return L.dgb_float_decompress_reduce_scaled_dev_norm(*args, FAKE, None, None)
    return L.dgb_float_decompress_reduce_scaled_dev(*args, None, None)


@pytest.mark.parametrize("ft", range(16))
def test_fp8_reduce_type_pairs(ft):
    for out_ft in range(16):
        for norm in (False, True):
            rc = _dev(ft, out_ft, norm)
            want = capi.ERR_TEMP_TOO_SMALL if (ft, out_ft) in REDUCE_PAIRS else capi.ERR_INVALID_ARG
            assert rc == want, (ft, out_ft, norm, rc)


def test_other_float_entries_refuse_fp8():
    L = capi.lib()
    p, u = capi.ptr_array([FAKE]), capi.u32_array([100])
    for ft in (10, 11):
        assert L.dgb_float_max_compressed_size(ft, 100) == 0
        assert L.dgb_float_compress_temp_bytes(ft, 1, 100) == 0
        assert L.dgb_float_compress_pointer(None, 0, ft, 10, 0, 1, p, u, p, FAKE, None) == capi.ERR_INVALID_ARG
        assert L.dgb_float_decompress_pointer(None, 0, ft, 10, 0, 1, p, p, u, None, None, None, None) == \
            capi.ERR_INVALID_ARG
        assert L.dgb_float_decompress_split_size(None, 0, ft, 10, 0, 1, p, FAKE, u, None, None, None, None) == \
            capi.ERR_INVALID_ARG
        for in_ft in range(16):
            assert L.dgb_float_compress_to(None, 0, in_ft, ft, 10, 0, 1, p, u, p, FAKE, None) == capi.ERR_INVALID_ARG
            assert L.dgb_float_compress_to(None, 0, ft, in_ft, 10, 0, 1, p, u, p, FAKE, None) == capi.ERR_INVALID_ARG
            assert L.dgb_float_compress_to_ef(None, 0, 3, ft, 10, 0, 1, p, u, p, p, FAKE, None) == capi.ERR_INVALID_ARG
        for out_ft in range(16):
            assert L.dgb_float_decompress_reduce_to(None, 0, ft, out_ft, 10, 1, 1, p, p, u, 0, None, None) == \
                capi.ERR_INVALID_ARG
            assert L.dgb_float_decompress_reduce_sparse(None, 0, ft, out_ft, 10, 1, 1, p, p, u, 0, None, None) == \
                capi.ERR_INVALID_ARG
            assert L.dgb_float_decompress_reduce_scaled(None, 0, ft, out_ft, 10, 1, 1, p, p, u, 0, 1.0, None, None) \
                == capi.ERR_INVALID_ARG
        assert L.dgb_float_decompress_reduce(None, 0, ft, 10, 1, 1, p, p, u, 0, None, None) == capi.ERR_INVALID_ARG
        assert L.dgb_float_decompress_reduce_narrow(None, 0, ft, 10, 1, 1, p, p, p, u, 0, None, FAKE, None, None,
                                                    None) == capi.ERR_INVALID_ARG
        assert L.dgb_float_decompress_reduce_narrow_norm(None, 0, ft, 10, 1, 1, p, p, p, u, 0, FAKE, None, FAKE, None,
                                                         None) == capi.ERR_INVALID_ARG
        assert L.dgb_float_sq_norm(None, 0, ft, 1, p, u, FAKE, None) == capi.ERR_INVALID_ARG
        assert L.dgb_archives_pull(ft, 1, p, p, u, None, None) == capi.ERR_INVALID_ARG


def test_fp8_scratch_sizes():
    L = capi.lib()
    for ft in (10, 11):
        assert L.dgb_float_decompress_temp_bytes(ft, 8, 0) == L.dgb_float_decompress_temp_bytes(capi.FLOAT32, 8, 0) > 0
        sizes = capi.u32_array([100, 9000])
        assert L.dgb_float_decompress_reduce_norm_temp_bytes(ft, 2, 3, sizes) == \
            L.dgb_float_decompress_reduce_norm_temp_bytes(capi.FLOAT32, 2, 3, sizes) > 0
    for ft in (7, 9, 12, 15):
        assert L.dgb_float_decompress_temp_bytes(ft, 8, 0) == 0


# ---- the cast's numpy restatement against torch's CPU clamp-cast -------------------------------------------------

@pytest.mark.parametrize("kind,dtype", [(E4M3, torch.float8_e4m3fn), (E5M2, torch.float8_e5m2)])
@pytest.mark.parametrize("s", [1.0, 0.3, 2.0 ** -7, 3.0e4, 1e-30])
def test_reference_cast_matches_torch_clamp_cast(kind, dtype, s):
    rng = np.random.default_rng(11)
    x = np.concatenate([edge_corpus(kind, s),
                        (rng.standard_normal(50000) * 10.0 ** rng.uniform(-12, 8, 50000)).astype(np.float32)])
    got = cast(x, s, kind)
    p = torch.from_numpy(x) * torch.tensor(s, dtype=torch.float32)
    want = p.clamp(-MAX[kind], MAX[kind]).to(dtype).view(torch.uint8).numpy()
    finite = ~torch.isnan(p).numpy()
    assert finite.sum() > 0.99 * x.size
    bad = np.nonzero((got != want) & finite)[0]
    assert bad.size == 0, (x[bad[:8]], got[bad[:8]], want[bad[:8]])
    assert np.all(got[~finite] == NAN_BYTE)
    # the corpus reaches saturation, both zeros, ties rounded down and up, and the subnormals
    assert {0x00, 0x80, 0x01, 0x81}.issubset(set(got.tolist()))
    top = int(torch.tensor(MAX[kind]).to(dtype).view(torch.uint8))
    assert top in got and (top | 0x80) in got


def test_reference_cast_of_bf16_words():
    w = np.arange(1 << 16, dtype=np.uint16)
    x = (w.astype(np.uint32) << 16).view(np.float32)
    for kind in (E4M3, E5M2):
        assert np.array_equal(cast(w, 0.75, kind), cast(x, 0.75, kind))


# ---- Python refusals --------------------------------------------------------------------------------------------

class FakeCuda:
    """The metadata of a CUDA tensor: enough for every check; any other use fails the test."""

    def __init__(self, numel, dtype=torch.float32, ptr=FAKE, contiguous=True, index=0):
        self.dtype, self.is_cuda, self.device = dtype, True, torch.device("cuda", index)
        self.shape = torch.Size((numel,))
        self._numel, self._ptr, self._contiguous = numel, ptr, contiguous

    def numel(self):
        return self._numel

    def data_ptr(self):
        return self._ptr

    def element_size(self):
        return torch.empty(0, dtype=self.dtype).element_size()

    def is_contiguous(self):
        return self._contiguous

    def reshape(self, *a):
        return self

    def __getattr__(self, name):
        raise AssertionError(f"{name} of a tensor used before the call was refused")


@pytest.fixture
def no_device_work(monkeypatch):
    """Every path below must refuse before it allocates or calls the library."""
    from dietgpu_b200 import ops

    def boom(*a, **k):
        raise AssertionError("device work before the refusal")

    monkeypatch.setattr(torch, "empty", boom)
    monkeypatch.setattr(ops, "_cast_fp8_ptrs", boom)
    return monkeypatch


def test_cast_fp8_refusals(no_device_work):
    from dietgpu_b200 import ops

    x = FakeCuda(64)
    with pytest.raises(ValueError, match="fp8 dtype"):
        ops.cast_fp8([x], torch.float16)
    with pytest.raises(ValueError, match="fp8 dtype"):
        ops.cast_fp8([x], torch.uint8)
    with pytest.raises(ValueError, match="non-empty list"):
        ops.cast_fp8([], torch.float8_e4m3fn)
    for bad in (FakeCuda(64, torch.float16), FakeCuda(64, torch.float64), FakeCuda(64, contiguous=False),
                torch.zeros(0)):
        with pytest.raises(ValueError, match="float32 or bfloat16 CUDA"):
            ops.cast_fp8([bad], torch.float8_e5m2)
    with pytest.raises(ValueError, match="one dtype"):
        ops.cast_fp8([x, FakeCuda(64, torch.bfloat16)], torch.float8_e5m2)
    for bad_scale in (FakeCuda(2), FakeCuda(1, torch.float16), FakeCuda(1, index=1), 2.0):
        with pytest.raises(ValueError, match="scale_tensor"):
            ops.cast_fp8([x], torch.float8_e4m3fn, bad_scale)


def test_compress_data_fp8_refusals(no_device_work):
    from dietgpu_b200 import ops

    x = FakeCuda(64)
    for kw in (dict(sparse=True), dict(error_feedback=[FakeCuda(64)])):
        with pytest.raises(ValueError, match="fp8 archive_dtype"):
            ops.compress_data(True, [x], archive_dtype=torch.float8_e4m3fn, **kw)
    with pytest.raises(ValueError, match="fp8 archive_dtype"):
        ops.compress_data(False, [x], archive_dtype=torch.float8_e4m3fn)
    with pytest.raises(ValueError, match="float32 or bfloat16 CUDA"):
        ops.compress_data(True, [FakeCuda(64, torch.float16)], archive_dtype=torch.float8_e5m2)
    with pytest.raises(ValueError, match="scale_tensor is the scale of an fp8 compress"):
        ops.compress_data(True, [x], archive_dtype=torch.bfloat16, scale_tensor=FakeCuda(1))
    with pytest.raises(ValueError, match="scale_tensor is the scale of an fp8 compress"):
        ops.compress_data(True, [x], scale_tensor=FakeCuda(1))
    # the existing narrowing refusal keeps its text
    with pytest.raises(ValueError, match="archive_dtype narrows float32 inputs"):
        ops.compress_data(True, [x], archive_dtype=torch.float64)


def test_decompress_data_reduce_fp8_refusals(no_device_work):
    from dietgpu_b200 import ops

    no_device_work.setattr(ops, "_check_flag_tensor", lambda *a: None)  # the fake scale passes as a device tensor

    a, o, s = Untouchable(), FakeCuda(64), FakeCuda(1)
    for kw in (dict(), dict(scale=0.5), dict(scale_tensor=s, sparse=True), dict(scale_tensor=s, acc=[o]),
               dict(scale_tensor=s, reduce_dtype=torch.float16)):
        with pytest.raises(ValueError):
            ops.decompress_data_reduce([[a]], [o], archive_dtype=torch.float8_e4m3fn, **kw)
    with pytest.raises(ValueError, match="float32 outputs"):
        ops.decompress_data_reduce([[a]], [FakeCuda(64, torch.bfloat16)], archive_dtype=torch.float8_e5m2,
                                   scale_tensor=s)


def _collectives():
    import dietgpu_b200 as dg

    return [dg.reduce_scatter_compressed, dg.all_gather_compressed]


@pytest.mark.parametrize("which", [0, 1])
def test_collectives_fp8_refusals(which, no_communication, no_device_work):
    f = _collectives()[which]
    t, s = FakeCuda(64), FakeCuda(1, ptr=2 * FAKE)
    for wire in (None, torch.float16, torch.bfloat16):
        with pytest.raises(ValueError, match="wire_scale is the scale of an fp8 wire"):
            f(t, wire_dtype=wire, wire_scale=s)
    for fp8 in (torch.float8_e4m3fn, torch.float8_e5m2):
        with pytest.raises(ValueError, match="wire_dtype is None, or float16 / bfloat16 for a float32 tensor"):
            f(FakeCuda(64, torch.float16), wire_dtype=fp8)
        with pytest.raises(ValueError, match="error_feedback is not supported with an fp8 wire"):
            f(t, wire_dtype=fp8, error_feedback=FakeCuda(64, ptr=3 * FAKE))
        with pytest.raises(ValueError, match="wire_scale"):
            f(t, wire_dtype=fp8, wire_scale=FakeCuda(2))
        with pytest.raises(ValueError, match="sparse=True cannot be combined with wire_dtype"):
            f(t, wire_dtype=fp8, sparse=True)
        if which == 0:
            for kw in (dict(reduce_dtype=torch.bfloat16), dict(out_dtype=torch.bfloat16), dict(out_dtype=fp8)):
                with pytest.raises(ValueError, match="an fp8 wire sums in float32"):
                    f(t, wire_dtype=fp8, **kw)
        else:
            with pytest.raises(ValueError, match="not supported with the peer-memory transports"):
                f(t, wire_dtype=fp8, peer=object())


def test_all_reduce_has_no_wire():
    import dietgpu_b200 as dg

    with pytest.raises(TypeError):
        dg.all_reduce_compressed(FakeCuda(64), wire_dtype=torch.float8_e4m3fn)
    with pytest.raises(TypeError):
        dg.all_to_all_compressed([FakeCuda(64)], wire_dtype=torch.float8_e4m3fn)
