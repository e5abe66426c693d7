"""torch.ops.dietgpu.* (the C++ operators) and dietgpu_b200.ops (their Python mirror), pinned to the oracle.

Every test runs once per layer ("torch": torch_library.load(), "mirror": dietgpu_b200.ops) at the
reference's fixed 10 prob bits.  Archives land in sentinel-filled rows with spare rows and columns, decoded
outputs in sentinel-filled buffers with guard space, and after each call every byte the operator was not
entitled to write must still hold the sentinel.  Covered:
  - every operator against the oracle, with and without checksums: mixed-dtype byte batches, float members at
    unaligned element offsets, split-size batches of many tiny members, the simple forms, decode of the
    reference's own archives, capacities one element short and larger than needed;
  - the scratch count each call returns: that much caller scratch must be enough to allocate nothing;
  - inputs the layers must refuse before they reach memory the caller did not hand over: byte batches of
    mixed dtypes (rows sized in bytes), split sizes past the tensor they index, float outputs of different
    dtypes, and input the C ABI rejects (misaligned archives and rows, checksum verification while capturing),
    which must raise RuntimeError rather than end the process;
  - compress_data, decompress_data and decompress_data_split_size captured together into one CUDA graph and
    replayed on new data, at 6 members and at 130 (member tables above 64 take the copy-kernel path).
"""
import os

import numpy as np
import pytest
import torch

from codec_helpers import GUARD, KINDS, SENTINEL, assert_guard_intact, guarded_out, oracle_archive, placed_inputs
from conftest import exp_bytes, normal_words
from oracle import oracle as O

gpu = pytest.mark.gpu

PB = 10  # the operators' fixed precision (DietGpu.cpp:114)
SIZE_SENTINEL = 0x5A5A5A5A
STATUS_SENTINEL = 0xEE
WORD = {"f16": np.uint16, "bf16": np.uint16, "f32": np.uint32}
GOLD_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_golden.npz")


@pytest.fixture(params=["torch", "mirror"])
def L(request):
    if request.param == "torch":
        from dietgpu_b200 import torch_library

        return torch_library.load()
    from dietgpu_b200 import ops

    return ops


def _dtype(kind):
    return torch.uint8 if kind == "bytes" else KINDS[kind][1]


def _raw(t):
    """The bytes of a contiguous tensor."""
    return t.contiguous().view(torch.uint8)


def framed(numel, dtype, offset, guard):
    """(buffer, view, (lo, hi)) like codec_helpers.guarded_out, with `guard` bytes of sentinel on either side."""
    es = torch.empty(0, dtype=dtype).element_size()
    guard = -(-guard // 16) * 16
    buf = torch.full((2 * guard + (8 + numel) * es,), SENTINEL, dtype=torch.uint8, device="cuda")
    start = guard // es + offset
    return buf, buf.view(dtype)[start:start + numel], (start * es, (start + numel) * es)


def assert_archive(kind, got, want, what):
    if kind == "bytes":
        O.assert_same_ans(got, want, what)
    else:
        O.assert_same_float(got, want, KINDS[kind][0], what)


def check_matrix(kind, comp, sizes, wants, what):
    """Rows [0, n) of `comp` hold archives equal to the oracle's `wants`; every byte of a row from its archive's
    size on, and every row past n, still holds the sentinel.  Returns the host sizes."""
    n = len(wants)
    hs = sizes[:n].cpu().tolist()
    host = comp.cpu().numpy()
    for i, want in enumerate(wants):
        assert hs[i] == want.size, f"{what}: member {i}: size {hs[i]} != oracle {want.size}"
        assert_archive(kind, host[i, :hs[i]], want, f"{what}: member {i}")
        stray = np.flatnonzero(host[i, hs[i]:] != SENTINEL)
        assert stray.size == 0, f"{what}: member {i}: {stray.size} byte(s) written past the archive (first at +{stray[0]})"
    assert (host[n:] == SENTINEL).all(), f"{what}: rows past the batch were written"
    return hs


def decode_into_guards(L, as_float, rows, expect, checksum, caps=None, what="decompress_data"):
    """decompress_data into guard-banded views at element offsets 0..7 of `caps[i]` elements (default: the
    expected length) of each expected tensor's dtype.  A member with room for its data must decode bit-exactly
    and write nothing past it; a member without room must get status 0, the required size, and no write."""
    n = len(rows)
    caps = [e.numel() for e in expect] if caps is None else caps
    outs = [guarded_out(c, e.dtype, (5 * i + 3) % 8) for i, (c, e) in enumerate(zip(caps, expect))]
    status = torch.full((n,), STATUS_SENTINEL, dtype=torch.uint8, device="cuda")
    osz = torch.full((n,), SIZE_SENTINEL, dtype=torch.int32, device="cuda")
    used = L.decompress_data(as_float, rows, [o[1] for o in outs], checksum, None, status, osz)
    st, sz = status.cpu().tolist(), osz.cpu().tolist()
    for i, ((buf, view, (lo, _)), e, c) in enumerate(zip(outs, expect, caps)):
        need = e.numel() if as_float else e.numel() * e.element_size()  # words or bytes
        assert sz[i] == need, f"{what}: member {i}: reported size {sz[i]} != {need}"
        if c < e.numel():
            assert st[i] == 0, f"{what}: member {i} decoded into a capacity of {c} < {e.numel()} elements"
            assert_guard_intact(buf, lo, lo, f"{what}: member {i} (too small)")
        else:
            assert st[i] == 1, f"{what}: member {i}: status {st[i]}"
            assert torch.equal(_raw(view[:e.numel()]), _raw(e)), f"{what}: member {i} decodes differently"
            assert_guard_intact(buf, lo, lo + e.numel() * e.element_size(), f"{what}: member {i}")
    return used


# ---- inputs ---------------------------------------------------------------------------------------------------

BYTE_SIZES = (0, 1, 3, 4095, 4096, 4097, 65537)
BYTE_DTYPES = (torch.uint8, torch.int16, torch.float32, torch.int64)


def mixed_byte_batch(seed):
    """Members of every byte dtype at (about) each size of BYTE_SIZES bytes: (raw uint8 arrays, device tensors)."""
    raws, ts = [], []
    for d, dt in enumerate(BYTE_DTYPES):
        es = torch.empty(0, dtype=dt).element_size()
        for j, s in enumerate(BYTE_SIZES):
            raw = exp_bytes(-(-s // es) * es, 0.05 + 0.15 * j, seed + 10 * d + j)
            raws.append(raw)
            ts.append(dev_bytes_as(raw, dt))
    return raws, ts


def host_data(kind, n, seed):
    return exp_bytes(n, 0.1, seed) if kind == "bytes" else normal_words(n, kind, seed)


def dev_bytes_as(raw, dtype):
    """Device copy of the uint8 array `raw`, viewed as `dtype` (also for empty members)."""
    t = torch.empty(raw.size, dtype=torch.uint8, device="cuda")
    t.copy_(torch.from_numpy(raw))
    return t.view(dtype)


def dev_tensor(kind, a):
    """Device tensor of dtype _dtype(kind) holding the uint8 array / float words `a`."""
    return placed_inputs([a], kind, None)[0]


# ---- sizes: byte batches of mixed dtypes (no GPU needed) -----------------------------------------------------------

def test_byte_rows_are_sized_by_the_largest_member_in_bytes(L):
    # the reference multiplies the largest element count by the FIRST member's element size: a 100-byte
    # member ahead of a 4 MiB float32 member got rows of max_any_compressed_size(1 MiB)
    for ts in ([torch.empty(100, dtype=torch.uint8), torch.empty(1 << 20, dtype=torch.float32)],
               [torch.empty(3, dtype=torch.int16), torch.empty(5, dtype=torch.int64), torch.empty(9000, dtype=torch.uint8)],
               [torch.empty(4096, dtype=torch.float32)]):
        want = max(L.max_any_compressed_size(t.numel() * t.element_size()) for t in ts)
        assert tuple(L.max_any_compressed_output_size(ts)) == (len(ts), want), [(t.dtype, t.numel()) for t in ts]


# ---- parity with the oracle, every operator ---------------------------------------------------------------------

@gpu
@pytest.mark.parametrize("checksum", [False, True])
def test_compress_bytes_of_mixed_dtypes(L, checksum):
    raws, ts = mixed_byte_batch(11)
    n = len(ts)
    _, cols = L.max_any_compressed_output_size(ts)
    assert cols == max(L.max_any_compressed_size(r.size) for r in raws)
    # more rows and wider rows than needed; sizes longer than the batch
    comp = torch.full((n + 3, cols + 48), SENTINEL, dtype=torch.uint8, device="cuda")
    sizes = torch.full((n + 5,), SIZE_SENTINEL, dtype=torch.int32, device="cuda")
    before = [_raw(t).clone() for t in ts]
    rc, rs, used = L.compress_data(False, ts, checksum, None, comp, sizes)
    assert rc.data_ptr() == comp.data_ptr() and rs.data_ptr() == sizes.data_ptr() and used > 0
    hs = check_matrix("bytes", comp, sizes, [oracle_archive("bytes", r, PB, checksum) for r in raws], "compress_data")
    assert sizes[n:].cpu().tolist() == [SIZE_SENTINEL] * 5, "entries of out_compressed_bytes past n were written"
    for i, (t, b) in enumerate(zip(ts, before)):
        assert torch.equal(_raw(t), b), f"member {i}: compress changed its input"
    decode_into_guards(L, False, [comp[i, :hs[i]] for i in range(n)], ts, checksum)


@gpu
@pytest.mark.parametrize("checksum", [False, True])
@pytest.mark.parametrize("kind", ["f16", "bf16", "f32"])
def test_compress_floats_at_unaligned_offsets(L, kind, checksum):
    words = [normal_words(s, kind, 20 + i) for i, s in enumerate((1, 7, 4097, 70001) * 2)]
    ts = placed_inputs(words, kind, range(8))  # element offsets 0..7: not 16 B aligned
    n = len(ts)
    _, cols = L.max_float_compressed_output_size(ts)
    assert cols == L.max_float_compressed_size(ts[0], 70001)
    comp = torch.full((n + 2, cols + 32), SENTINEL, dtype=torch.uint8, device="cuda")
    sizes = torch.full((n + 3,), SIZE_SENTINEL, dtype=torch.int32, device="cuda")
    L.compress_data(True, ts, checksum, None, comp, sizes)
    hs = check_matrix(kind, comp, sizes, [oracle_archive(kind, w, PB, checksum) for w in words], "compress_data")
    assert sizes[n:].cpu().tolist() == [SIZE_SENTINEL] * 3
    decode_into_guards(L, True, [comp[i, :hs[i]] for i in range(n)], ts, checksum)


SPLITS = {"bytes": [4096, 4, 8, 12, 4100, 65536, 20, 4097],  # interior multiples of 4, the last one odd
          "float": [1, 3, 5, 7, 9, 1, 9, 4097, 3, 70001, 5]}  # odd word counts, tiny members back to back


@gpu
@pytest.mark.parametrize("checksum", [False, True])
@pytest.mark.parametrize("kind", ["bytes", "f16", "bf16", "f32"])
def test_split_size_round_trip(L, kind, checksum):
    as_float = kind != "bytes"
    splits = SPLITS["float" if as_float else "bytes"]
    n, total = len(splits), sum(splits)
    data = host_data(kind, total, 31)
    # t_in is a view at an offset: 4 B for bytes, 3 words for floats
    t_in = placed_inputs([data], kind, [4 if kind == "bytes" else 3])[0]
    split_t = torch.tensor(splits, dtype=torch.int32)
    cols = (L.max_float_compressed_size(t_in, max(splits)) if as_float else L.max_any_compressed_size(max(splits)))
    comp = torch.full((n + 2, cols + 32), SENTINEL, dtype=torch.uint8, device="cuda")
    sizes = torch.full((n + 2,), SIZE_SENTINEL, dtype=torch.int32, device="cuda")
    rows, rs, _ = L.compress_data_split_size(as_float, t_in, split_t, checksum, None, comp, sizes)
    offs = np.cumsum([0] + splits)
    wants = [oracle_archive(kind, data[offs[i]:offs[i + 1]], PB, checksum) for i in range(n)]
    hs = check_matrix(kind, comp, sizes, wants, "compress_data_split_size")
    assert rs.data_ptr() == sizes.data_ptr() and len(rows) == n
    for i, r in enumerate(rows):
        assert r.numel() == hs[i] and r.data_ptr() == comp[i].data_ptr(), f"member {i}: returned row"
    # decode every member back to back into one sentinel-framed buffer
    buf, t_out, (lo, hi) = guarded_out(total, t_in.dtype, 5)
    status = torch.full((n,), STATUS_SENTINEL, dtype=torch.uint8, device="cuda")
    osz = torch.full((n,), SIZE_SENTINEL, dtype=torch.int32, device="cuda")
    L.decompress_data_split_size(as_float, rows, t_out, split_t, checksum, None, status, osz)
    assert status.cpu().tolist() == [1] * n and osz.cpu().tolist() == splits
    assert torch.equal(_raw(t_out), _raw(t_in)), "split-size decode differs from the input"
    assert_guard_intact(buf, lo, hi, "decompress_data_split_size")


@gpu
@pytest.mark.parametrize("checksum", [False, True])
@pytest.mark.parametrize("kind", ["bytes", "f16", "bf16", "f32"])
def test_simple_round_trip(L, kind, checksum):
    as_float = kind != "bytes"
    if as_float:
        words = [normal_words(s, kind, 40 + i) for i, s in enumerate((4097, 1, 70001))]
        ts, raws = [dev_tensor(kind, w) for w in words], words
    else:
        raws = [exp_bytes(s, 0.07, 40 + i) for i, s in enumerate((4097, 2000, 12000))]
        ts = [dev_bytes_as(r, dt) for r, dt in zip(raws, (torch.uint8, torch.int16, torch.float32))]
    comps = L.compress_data_simple(as_float, ts, checksum)
    assert len(comps) == len(ts)
    for i, (c, r) in enumerate(zip(comps, raws)):
        want = oracle_archive(kind, r, PB, checksum)
        assert c.dtype == torch.uint8 and c.numel() == want.size, f"member {i}: size"
        assert_archive(kind, c.cpu().numpy(), want, f"compress_data_simple member {i}")  # incl. the checksum flag
    outs = L.decompress_data_simple(as_float, comps, checksum)
    for i, (o, t) in enumerate(zip(outs, ts)):
        # dtype and length come from the headers: the float type, or bytes
        assert o.dtype == (t.dtype if as_float else torch.uint8), f"member {i}: dtype {o.dtype}"
        assert torch.equal(_raw(o), _raw(t)), f"decompress_data_simple member {i}"


@gpu
def test_simple_refuses_mixed_float_types(L):
    a = dev_tensor("f16", normal_words(100, "f16", 1))
    b = dev_tensor("bf16", normal_words(100, "bf16", 2))
    with pytest.raises(RuntimeError):
        L.compress_data_simple(True, [a, b])
    archives = [L.compress_data_simple(True, [t])[0] for t in (a, b)]
    with pytest.raises(RuntimeError):
        L.decompress_data_simple(True, archives)


@gpu
@pytest.mark.parametrize("checksum", [False, True])
@pytest.mark.parametrize("kind", ["bytes", "f16", "bf16", "f32"])
def test_decompress_capacities(L, kind, checksum):
    """The oracle's archives into outputs of exact capacity, one element short, and 100 elements more."""
    if kind == "bytes":
        data = [exp_bytes(s, 0.1, 50 + i) for i, s in enumerate((4097, 1, 65537, 4096))]
        expect = [torch.from_numpy(d).cuda() for d in data]
        expect[3] = expect[3].view(torch.int32)  # capacity in bytes, whatever the output's dtype
    else:
        data = [normal_words(s, kind, 50 + i) for i, s in enumerate((4097, 7, 70001, 1))]
        expect = [dev_tensor(kind, d) for d in data]
    rows = [dev_tensor("bytes", oracle_archive(kind, d, PB, checksum)) for d in data]
    caps = [expect[0].numel(), expect[1].numel() - 1, expect[2].numel() + 100, expect[3].numel()]
    decode_into_guards(L, kind != "bytes", rows, expect, checksum, caps)


@gpu
def test_decodes_the_references_archives(L):
    """Archives the unmodified reference wrote on an H100 (tests/golden/ref_golden.npz), decoded through the
    API the reference's own users call."""
    gold = np.load(GOLD_PATH)
    names = sorted({k.rsplit("/", 1)[0] for k in gold.files if k.startswith("ans/")})
    assert len(names) >= 6
    expect = [torch.from_numpy(np.ascontiguousarray(gold[f"{b}/in"])).cuda() for b in names]
    rows = [dev_tensor("bytes", gold[f"{b}/pb10"]) for b in names]
    decode_into_guards(L, False, rows, expect, True, what="reference ans archives")
    for kind in ("f16", "bf16", "f32"):
        names = sorted({k.rsplit("/", 1)[0] for k in gold.files if k.startswith(f"float/{kind}/")})
        assert len(names) >= 3
        expect = [dev_tensor(kind, gold[f"{b}/in"]) for b in names]
        rows = [dev_tensor("bytes", gold[f"{b}/pb10"]) for b in names]
        decode_into_guards(L, True, rows, expect, True, what=f"reference {kind} archives")


@gpu
@pytest.mark.parametrize("kind", ["bytes", "bf16"])
def test_returned_scratch_count_suffices(L, kind):
    """temp_mem of exactly the returned byte count is enough: with every output supplied the call takes nothing
    from the caching allocator.  An unaligned or one-byte-short temp_mem still gives correct results."""
    as_float = kind != "bytes"
    data = [host_data(kind, s, 60 + i) for i, s in enumerate((4097, 70001, 33))]
    ts = [dev_tensor(kind, d) for d in data]
    n = len(ts)
    wants = [oracle_archive(kind, d, PB, False) for d in data]
    _, cols = L.max_float_compressed_output_size(ts) if as_float else L.max_any_compressed_output_size(ts)
    _, _, used = L.compress_data(as_float, ts)
    assert used > 0
    comp = torch.full((n, cols), SENTINEL, dtype=torch.uint8, device="cuda")
    sizes = torch.empty(n, dtype=torch.int32, device="cuda")
    outs = [torch.empty_like(t) for t in ts]
    status = torch.empty(n, dtype=torch.uint8, device="cuda")
    osz = torch.empty(n, dtype=torch.int32, device="cuda")

    def temps(nbytes):
        big = torch.empty(nbytes + 512, dtype=torch.uint8, device="cuda")
        return {"exact": torch.empty(nbytes, dtype=torch.uint8, device="cuda"), "unaligned": big[1:1 + nbytes],
                "one byte short": torch.empty(nbytes - 1, dtype=torch.uint8, device="cuda")}

    for name, temp in temps(used).items():
        comp.fill_(SENTINEL)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        L.compress_data(as_float, ts, False, temp, comp, sizes)
        torch.cuda.synchronize()
        if name == "exact":
            assert torch.cuda.max_memory_allocated() == base, "compress_data allocated despite enough temp_mem"
        hs = check_matrix(kind, comp, sizes, wants, f"compress_data, {name} temp_mem")
    rows = [comp[i, :hs[i]] for i in range(n)]
    used_d = L.decompress_data(as_float, rows, outs)
    assert used_d > 0
    for name, temp in temps(used_d).items():
        for o in outs:
            o.view(torch.uint8).fill_(SENTINEL)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        L.decompress_data(as_float, rows, outs, False, temp, status, osz)
        torch.cuda.synchronize()
        if name == "exact":
            assert torch.cuda.max_memory_allocated() == base, "decompress_data allocated despite enough temp_mem"
        assert status.cpu().tolist() == [1] * n, name
        for i, (o, t) in enumerate(zip(outs, ts)):
            assert torch.equal(_raw(o), _raw(t)), f"decompress_data, {name} temp_mem: member {i}"


# ---- inputs that would reach memory the caller did not hand over ---------------------------------------------------
# Each sentinel region is sized from the CORRECT bound, so a layer without the check writes only into memory
# the test owns.

@gpu
def test_mixed_dtype_byte_batch_fits_its_rows(L):
    raws = [exp_bytes(100, 0.1, 70), np.random.default_rng(71).integers(0, 256, 4 << 20, dtype=np.uint8)]
    ts = [dev_bytes_as(raws[0], torch.uint8), dev_bytes_as(raws[1], torch.float32)]
    n = len(ts)
    correct = max(L.max_any_compressed_size(r.size) for r in raws)
    _, cols = L.max_any_compressed_output_size(ts)
    flat = torch.full(((n + 3) * correct,), SENTINEL, dtype=torch.uint8, device="cuda")
    comp = flat[:n * cols].view(n, cols)
    sizes = torch.empty(n, dtype=torch.int32, device="cuda")
    L.compress_data(False, ts, False, None, comp, sizes)
    hs = sizes.cpu().tolist()
    host = flat.cpu().numpy()
    written = np.zeros(host.size, dtype=bool)
    for i in range(n):
        written[i * cols:i * cols + min(hs[i], cols)] = True
    stray = np.flatnonzero((host != SENTINEL) & ~written)
    assert stray.size == 0, (f"rows of {cols} B for archives of {hs} B: {stray.size} byte(s) written past an "
                             f"archive's row (first at flat offset {stray[0]})")
    for i, r in enumerate(raws):
        want = oracle_archive("bytes", r, PB)
        assert hs[i] == want.size
        O.assert_same_ans(host[i * cols:i * cols + hs[i]], want, f"member {i}")


@gpu
@pytest.mark.parametrize("kind", ["bytes", "f16", "bf16", "f32"])
def test_split_sizes_past_t_in_raise(L, kind):
    as_float = kind != "bytes"
    length = 8192
    # t_in is a prefix of a larger buffer: a layer that reads past it stays inside the test's allocation
    base = dev_tensor(kind, host_data(kind, length + 4096, 80))
    t_in = base[:length]
    splits = torch.tensor([4096, length - 4096 + 100], dtype=torch.int32)  # units: words for floats, bytes otherwise
    with pytest.raises(RuntimeError, match="split sizes"):
        L.compress_data_split_size(as_float, t_in, splits)
    ok = torch.tensor([4096, length - 4096], dtype=torch.int32)
    rows, _, _ = L.compress_data_split_size(as_float, t_in, ok)  # the exact sum is fine
    assert len(rows) == 2


@gpu
@pytest.mark.parametrize("kind", ["bytes", "f16", "bf16", "f32"])
def test_split_sizes_past_t_out_raise(L, kind):
    as_float = kind != "bytes"
    data = [host_data(kind, s, 81 + i) for i, s in enumerate((4096, 4000))]
    rows = [dev_tensor("bytes", oracle_archive(kind, d, PB)) for d in data]
    splits = torch.tensor([d.size for d in data], dtype=torch.int32)
    excess = 100
    es = torch.empty(0, dtype=_dtype(kind)).element_size()
    buf, t_out, (lo, _) = framed(int(splits.sum()) - excess, _dtype(kind), 3, guard=excess * es + GUARD)
    with pytest.raises(RuntimeError, match="split sizes"):
        L.decompress_data_split_size(as_float, rows, t_out, splits)
    torch.cuda.synchronize()
    assert_guard_intact(buf, lo, lo, "refused split-size decode")


@gpu
def test_float_outputs_of_different_dtypes_raise(L):
    N = 4097
    data = [normal_words(N, "f32", 90 + i) for i in range(2)]
    rows = [dev_tensor("bytes", oracle_archive("f32", d, PB)) for d in data]
    out0 = torch.empty(N, dtype=torch.float32, device="cuda")
    # a bf16 output of N elements holds 2N bytes: decoded as f32 words, N floats would write 2N bytes past it
    # (4 B aligned, so that f32 words may be written there at all)
    buf, out1, (lo, _) = framed(N, torch.bfloat16, 2, guard=2 * N + GUARD)
    with pytest.raises(RuntimeError, match="same dtype"):
        L.decompress_data(True, rows, [out0, out1])
    torch.cuda.synchronize()
    assert_guard_intact(buf, lo, lo, "bf16 output of an f32 batch")


@gpu
def test_split_output_of_another_float_type_is_not_written(L):
    """A split-size t_out sets the float type the archives are decoded as.  The decoder checks each archive's
    header against it, so f32 archives into a bf16 t_out fail per member and write nothing (raising instead
    would need the headers on the host: a synchronising read that no CUDA graph could capture)."""
    N = 4097
    data = [normal_words(N, "f32", 92 + i) for i in range(2)]
    rows = [dev_tensor("bytes", oracle_archive("f32", d, PB)) for d in data]
    splits = torch.tensor([N, N], dtype=torch.int32)
    buf, t_out, (lo, _) = framed(2 * N, torch.bfloat16, 1, guard=4 * N + GUARD)
    status = torch.full((2,), STATUS_SENTINEL, dtype=torch.uint8, device="cuda")
    osz = torch.full((2,), SIZE_SENTINEL, dtype=torch.int32, device="cuda")
    L.decompress_data_split_size(True, rows, t_out, splits, False, None, status, osz)
    assert status.cpu().tolist() == [0, 0] and osz.cpu().tolist() == [0, 0]
    assert_guard_intact(buf, lo, lo, "f32 archives into a bf16 t_out")


# ---- a batch whose buffers stay put, for capture -------------------------------------------------------------------

class Batch:
    """n members in one flat input (member starts 16 elements apart at least), their archive matrix, pointer-form
    outputs in a flat buffer of the same layout, a split-size output, status and size tensors and scratch."""

    def __init__(self, L, kind, n):
        self.L, self.kind, self.as_float = L, kind, kind != "bytes"
        self.lengths = [1 + (i * 2477) % 9000 for i in range(n)]
        self.starts = np.cumsum([0] + [-(-x // 16) * 16 for x in self.lengths])
        dt = _dtype(kind)
        self.flat_in = torch.zeros(int(self.starts[-1]), dtype=dt, device="cuda")
        self.flat_out = torch.zeros_like(self.flat_in)
        self.ts = [self.flat_in[self.starts[i]:self.starts[i] + x] for i, x in enumerate(self.lengths)]
        self.outs = [self.flat_out[self.starts[i]:self.starts[i] + x] for i, x in enumerate(self.lengths)]
        _, cols = L.max_float_compressed_output_size(self.ts) if self.as_float else L.max_any_compressed_output_size(self.ts)
        self.comp = torch.zeros((n, cols), dtype=torch.uint8, device="cuda")
        self.rows = [self.comp[i] for i in range(n)]  # whole rows: the decoder reads each archive's size from its header
        self.sizes = torch.zeros(n, dtype=torch.int32, device="cuda")
        self.t_out = torch.zeros(sum(self.lengths), dtype=dt, device="cuda")
        self.splits = torch.tensor(self.lengths, dtype=torch.int32)
        self.status = [torch.zeros(n, dtype=torch.uint8, device="cuda") for _ in range(2)]
        self.osz = [torch.zeros(n, dtype=torch.int32, device="cuda") for _ in range(2)]
        self.temp = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")

    def fill(self, seed):
        self.data = [host_data(self.kind, x, seed * 1000 + i) for i, x in enumerate(self.lengths)]
        host = np.zeros(self.flat_in.numel(), dtype=np.uint8 if self.kind == "bytes" else WORD[self.kind])
        for i, d in enumerate(self.data):
            host[self.starts[i]:self.starts[i] + d.size] = d
        self.flat_in.copy_(dev_tensor(self.kind, host))

    def clear(self):
        for t in (self.comp, self.sizes, self.flat_out, self.t_out, *self.status, *self.osz):
            t.view(torch.uint8).fill_(0)

    def compress(self, checksum=True):
        self.checksum = checksum
        self.L.compress_data(self.as_float, self.ts, checksum, self.temp, self.comp, self.sizes)

    def decompress(self, checksum=False):
        self.L.decompress_data(self.as_float, self.rows, self.outs, checksum, self.temp, self.status[0], self.osz[0])

    def decompress_split(self):
        self.L.decompress_data_split_size(self.as_float, self.rows, self.t_out, self.splits, False, self.temp,
                                          self.status[1], self.osz[1])

    def check(self, what, split=True):
        torch.cuda.synchronize()
        n = len(self.lengths)
        hs = self.sizes.cpu().tolist()
        host = self.comp.cpu().numpy()
        for i, d in enumerate(self.data):
            want = oracle_archive(self.kind, d, PB, self.checksum)
            assert hs[i] == want.size, f"{what}: member {i}: size {hs[i]} != oracle {want.size}"
            assert_archive(self.kind, host[i, :hs[i]], want, f"{what}: member {i}")
        units = self.lengths  # words for floats, bytes otherwise
        for k in range(2 if split else 1):
            assert self.status[k].cpu().tolist() == [1] * n, f"{what}: status of decode {k}"
            assert self.osz[k].cpu().tolist() == units, f"{what}: sizes of decode {k}"
        assert torch.equal(_raw(self.flat_out), _raw(self.flat_in)), f"{what}: decompress_data"
        if split:
            assert torch.equal(_raw(self.t_out), _raw(torch.cat(self.ts))), f"{what}: decompress_data_split_size"


@gpu
@pytest.mark.parametrize("n", [6, 130])
@pytest.mark.parametrize("kind", ["bytes", "bf16"])
def test_operators_captured_into_one_graph(L, kind, n):
    b = Batch(L, kind, n)
    b.fill(1)
    b.compress()
    b.decompress()
    b.decompress_split()
    b.check("ordinary calls")
    b.clear()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        b.compress()
        b.decompress()
        b.decompress_split()
    for seed in (2, 3):  # new data in the same buffers; each replay must code it
        b.fill(seed)
        b.clear()
        g.replay()
        b.check(f"replay on data {seed}")


# ---- input the C ABI rejects: RuntimeError, and the process goes on ---------------------------------------------
# The layers check these before the C ABI sees them.  Until they did, the C++ operators reached the compat
# header's detail::check, which calls std::abort() on every code but OK and CHECKSUM: do not run these
# against a build without the checks.

@gpu
@pytest.mark.parametrize("kind", ["bytes", "bf16"])
def test_abi_refusal_misaligned_archives(L, kind):
    as_float = kind != "bytes"
    b = Batch(L, kind, 3)
    b.fill(4)
    b.compress(False)
    hs = b.sizes.cpu().tolist()
    shifted = [b.comp[0, 8:8 + hs[0]]]  # 8 B past a 16 B boundary
    # a row of a matrix whose width is not a multiple of 16
    odd = torch.zeros((2, b.comp.size(1) + 8), dtype=torch.uint8, device="cuda")
    odd[1, :hs[0]] = b.comp[0, :hs[0]]
    for bad in (shifted, [odd[1]]):
        with pytest.raises(RuntimeError, match="16 B aligned"):
            L.decompress_data(as_float, bad, [b.outs[0]])
        with pytest.raises(RuntimeError, match="16 B aligned"):
            L.decompress_data_split_size(as_float, bad, b.outs[0], b.splits[:1].clone())
        with pytest.raises(RuntimeError, match="16 B aligned"):
            L.decompress_data_simple(as_float, bad)
    b.decompress()
    b.check("after the refusals", split=False)


@gpu
@pytest.mark.parametrize("kind", ["bytes", "bf16"])
def test_abi_refusal_misaligned_output_rows(L, kind):
    as_float = kind != "bytes"
    b = Batch(L, kind, 3)
    b.fill(5)
    cols = b.comp.size(1)
    wide = torch.zeros((3, cols + 8), dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError, match="16 B aligned"):
        L.compress_data(as_float, b.ts, False, None, wide)
    splits = torch.tensor([16, 32, 7], dtype=torch.int32)  # valid splits (interior multiples of 4)
    with pytest.raises(RuntimeError, match="16 B aligned"):
        L.compress_data_split_size(as_float, b.flat_in, splits, False, None, wide)
    b.compress()
    b.decompress()
    b.check("after the refusals", split=False)


@gpu
@pytest.mark.parametrize("kind", ["bytes", "bf16"])
def test_abi_refusal_checksum_decode_inside_a_capture(L, kind):
    b = Batch(L, kind, 6)
    b.fill(6)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        b.compress()
        with pytest.raises(RuntimeError, match="cannot be captured"):
            b.decompress(checksum=True)
        b.decompress()
    # the capture stayed valid: its replay codes new data
    b.fill(7)
    b.clear()
    g.replay()
    b.check("replay", split=False)
    # and a verified decode outside a capture still works
    b.fill(8)
    b.clear()
    b.compress()
    b.decompress(checksum=True)
    b.check("ordinary verified call", split=False)
