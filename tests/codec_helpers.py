"""Round-trip helpers shared by the GPU test modules.

Every round trip compresses a batch through the C ABI, compares every member with the CPU oracle and
decodes it again, and checks that nothing was written where it should not have been:
  - archives go into rows of `cols + GUARD` bytes prefilled with SENTINEL; after the call every byte of a
    row from the archive's reported size onwards must still hold the sentinel;
  - each decoded output is a view at an element offset of 0..7 inside a sentinel-filled buffer with GUARD
    bytes on either side; every byte outside the view must still hold the sentinel;
  - compress must leave its inputs unchanged.
The oracle's archive of a member depends only on (kind, prob bits, checksum flag, member data), never on
kernel options, so it is computed once per session and reused by every variant.
"""
from __future__ import annotations

import contextlib
import hashlib

import numpy as np
import pytest
import torch

from oracle import oracle as O

KINDS = {"f16": (O.F16, torch.float16, np.uint16), "bf16": (O.BF16, torch.bfloat16, np.uint16),
         "f32": (O.F32, torch.float32, np.uint32)}
SENTINEL = 0xA5
GUARD = 64


def dg():
    import dietgpu_b200

    return dietgpu_b200


def to_dev_bytes(a):
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a if a.flags.writeable else a.copy()).cuda()


def words_to_tensor(w, kind):
    _, tdt, _ = KINDS[kind]
    t = torch.from_numpy(w.view(np.int16 if w.dtype == np.uint16 else np.int32).copy())
    return t.view(tdt).cuda()


@contextlib.contextmanager
def codec_options(**opts):
    """Sets the given dgb_set_option values for the body and restores every option afterwards."""
    from dietgpu_b200 import capi

    saved = {k: capi.get_option(k) for k in capi.OPTION_NAMES}
    try:
        for k, v in opts.items():
            capi.set_option(k, v)
        yield
    finally:
        for k, v in saved.items():
            capi.set_option(k, v)


@pytest.fixture
def options():
    """options(name=value, ...) sets codec options for the rest of the test; every option is restored when the
    test ends, whatever it changed.  A module uses it by importing it from here."""
    with contextlib.ExitStack() as stack:
        yield lambda **kw: stack.enter_context(codec_options(**kw))


# ---- oracle archives, cached per (kind, prob bits, checksum, member) ----------

_ORACLE_CACHE = {}
_CACHE_MAX_BYTES = 16 << 20  # members above this are recomputed (the >2^24-symbol members)


def oracle_archive(kind, data, pb, checksum=False):
    """kind: 'bytes' or a key of KINDS; data: uint8 array (bytes) or float words."""
    data = np.ascontiguousarray(data)
    key = None
    if data.nbytes <= _CACHE_MAX_BYTES:
        key = (kind, pb, bool(checksum), data.dtype.str, data.size,
               hashlib.blake2b(data.tobytes(), digest_size=16).digest())
        hit = _ORACLE_CACHE.get(key)
        if hit is not None:
            return hit
    if kind == "bytes":
        arch = O.ans_encode(data, pb, checksum)
    else:
        arch = O.float_compress(KINDS[kind][0], data, pb, checksum)
    arch.setflags(write=False)
    if key is not None:
        _ORACLE_CACHE[key] = arch
    return arch


# ---- guard-banded buffers ------------------------------------------------------

def guarded_out(numel, dtype, offset):
    """(buffer, view): a view of `numel` elements at element `offset` (0..7) inside a sentinel-filled
    uint8 buffer with at least GUARD bytes on either side."""
    es = torch.empty(0, dtype=dtype).element_size()
    nbytes = 2 * GUARD + 8 * es + numel * es
    buf = torch.full((nbytes,), SENTINEL, dtype=torch.uint8, device="cuda")
    start = GUARD // es + offset
    return buf, buf.view(dtype)[start:start + numel], (start * es, (start + numel) * es)


def assert_guard_intact(buf, lo, hi, what):
    """Every byte of `buf` outside [lo, hi) still holds the sentinel."""
    head, tail = buf[:lo], buf[hi:]
    bad_head = int((head != SENTINEL).sum())
    bad_tail = int((tail != SENTINEL).sum())
    assert bad_head == 0 and bad_tail == 0, \
        f"{what}: {bad_head} byte(s) written before the output view, {bad_tail} after it"


def placed_inputs(arrays, kind, offsets):
    """Device tensors holding `arrays`, each starting `offsets[i]` elements into its own allocation."""
    ts = []
    for i, a in enumerate(arrays):
        off = 0 if offsets is None else int(offsets[i])
        full = np.concatenate([np.zeros(off, a.dtype), a])
        t = to_dev_bytes(full) if kind == "bytes" else words_to_tensor(full, kind)
        ts.append(t[off:])
    return ts


def _int_view(t):
    if t.dtype == torch.uint8:
        return t
    return t.view(torch.int32 if t.element_size() == 4 else torch.int16)


def guarded_compress(as_float, ts, checksum, pb):
    """compress_data into a sentinel-prefilled [n, cols + GUARD] matrix; checks that the inputs are
    unchanged and that no row has a byte written at or beyond the archive's reported size.
    Returns (matrix, host sizes)."""
    from dietgpu_b200 import ops

    n = len(ts)
    _, cols = ops.max_float_compressed_output_size(ts) if as_float else ops.max_any_compressed_output_size(ts)
    assert cols % 16 == 0
    comp = torch.full((n, cols + GUARD), SENTINEL, dtype=torch.uint8, device="cuda")
    before = [_int_view(t).clone() for t in ts]
    _, sizes, _ = ops.compress_data(as_float, ts, checksum, None, comp, None, prob_bits=pb)
    hs = sizes.cpu().tolist()
    for i, (t, b) in enumerate(zip(ts, before)):
        assert torch.equal(_int_view(t), b), f"member {i}: compress changed its input"
    col = torch.arange(cols + GUARD, device="cuda")
    beyond = col[None, :] >= sizes[:, None].long()
    stray = (comp != SENTINEL) & beyond
    if bool(stray.any()):
        rows = torch.nonzero(stray.any(1)).flatten().cpu().tolist()
        first = [int(torch.nonzero(stray[r]).flatten()[0]) for r in rows[:4]]
        raise AssertionError(f"compress wrote beyond the archive size in rows {rows[:8]} "
                             f"(sizes {[hs[r] for r in rows[:4]]}, first stray columns {first})")
    return comp, hs


def guarded_decode(as_float, rows, lengths, dtype, pb, checksum, expect, what, out_offsets=None):
    """Decodes `rows` into guard-banded views and checks status, sizes, guards and the decoded data
    against `expect` (device tensors)."""
    n = len(rows)
    bufs, outs, spans = [], [], []
    for i in range(n):
        off = (5 * i + 3) % 8 if out_offsets is None else int(out_offsets[i])
        b, v, span = guarded_out(lengths[i], dtype, off)
        bufs.append(b)
        outs.append(v)
        spans.append(span)
    status = torch.zeros(n, dtype=torch.uint8, device="cuda")
    osz = torch.zeros(n, dtype=torch.int32, device="cuda")
    dg().decompress_data(as_float, rows, outs, checksum, None, status, osz, prob_bits=pb)
    assert status.cpu().tolist() == [1] * n, f"{what}: status {status.cpu().tolist()}"
    assert osz.cpu().tolist() == list(lengths), f"{what}: decoded sizes"
    for i in range(n):
        assert torch.equal(_int_view(outs[i]), _int_view(expect[i])), f"{what}: member {i} decodes differently"
        assert_guard_intact(bufs[i], spans[i][0], spans[i][1], f"{what}: member {i}")


def _compare(kind, got, want, exact, what):
    if exact:
        assert np.array_equal(got, want), f"{what}: archive bytes differ from the oracle's"
    elif kind == "bytes":
        O.assert_same_ans(got, want, what)
    else:
        O.assert_same_float(got, want, KINDS[kind][0], what)


def roundtrip(kind, arrays, pb=10, checksum=False, in_offsets=None, out_offsets=None, exact=False,
              decode_oracle=False):
    """Compress `arrays` (uint8 arrays for kind 'bytes', else float words) as one batch, compare every
    member with the oracle (byte for byte when `exact`), decode the archives (and, with `decode_oracle`,
    the oracle's archives too) into guard-banded outputs.  Returns the archives (host uint8 arrays)."""
    as_float = kind != "bytes"
    ts = placed_inputs(arrays, kind, in_offsets)
    comp, hs = guarded_compress(as_float, ts, checksum, pb)
    host = comp[:, :max(hs) if hs else 0].cpu().numpy()
    for i, a in enumerate(arrays):
        want = oracle_archive(kind, a, pb, checksum)
        assert hs[i] == want.size, f"member {i}: size {hs[i]} != oracle {want.size}"
        assert hs[i] % 16 == 0  # ans/ANSTest.cu:131-135
        _compare(kind, host[i, :hs[i]], want, exact, f"member {i}")
    dtype = ts[0].dtype
    lengths = [a.size for a in arrays]
    guarded_decode(as_float, [comp[i, :hs[i]] for i in range(len(ts))], lengths, dtype, pb, checksum, ts,
                   "decode")
    if decode_oracle:
        rows = [to_dev_bytes(oracle_archive(kind, a, pb, checksum)) for a in arrays]
        guarded_decode(as_float, rows, lengths, dtype, pb, checksum, ts, "decode of the oracle's archives")
    return [host[i, :hs[i]] for i in range(len(arrays))]


def ans_roundtrip(arrays, pb, checksum=False, **kw):
    return roundtrip("bytes", arrays, pb, checksum, **kw)


def float_roundtrip(kind, word_arrays, pb=10, checksum=False, offsets=None, **kw):
    """`offsets`: element offsets of the inputs (not 16 B aligned when nonzero)."""
    return roundtrip(kind, word_arrays, pb, checksum, in_offsets=offsets, **kw)


# ---- the bits the reference leaves undefined -------------------------------------
#
# The reference sets its header flags by read-modify-write over uninitialised memory and never writes the
# fields below, so an archive it wrote into a reused buffer carries whatever was there; the pdf of an empty
# member is whatever its scratch held.  Every reader must ignore them; `scribble` writes garbage into exactly
# these places and nowhere else.

_ANS_MAGIC, _FLOAT_MAGIC = 0xD00D0001, 0xF00F0001


def _u32(a, off):
    return int(a[off:off + 4].view(np.uint32)[0])


def _ans_regions(a, base):
    """(name, start, stop, bitmask) of the undefined bits of the ANS archive at byte `base` of `a`."""
    opts = _u32(a, base + 16)
    regs = [("ans options bits 5-31", base + 16, base + 20, 0xE0, 0xFF, 0xFF, 0xFF)]
    if not opts & 0x10:
        regs.append(("ans checksum (flag clear)", base + 20, base + 24))
    regs.append(("ans unused0/1", base + 24, base + 32))
    if _u32(a, base + 8) == 0:
        # an empty member's pdf: the reference copies a table its statistics pass never wrote for it
        regs.append(("pdf of an empty archive", base + 32, base + 544))
    nb = _u32(a, base + 4)
    bw_at = base + 544 + 128 * nb
    if nb & 1:
        regs.append(("block table pad entry", bw_at + 8 * nb, bw_at + 8 * nb + 8))
    data = bw_at + 8 * (nb + (nb & 1))
    bw = a[bw_at:bw_at + 8 * nb].view(np.uint32).reshape(nb, 2).astype(np.int64)
    words, off = bw[:, 0] & 0xFFFF, bw[:, 1]
    for k in np.flatnonzero(words % 8):
        regs.append(("stream padding", data + 2 * int(off[k] + words[k]), data + 2 * int(off[k] + (words[k] + 7) // 8 * 8)))
    return regs


def undefined_regions(archive):
    """The places of a byte or fp16 / bf16 / fp32 archive that the reference leaves undefined, as
    (name, start, stop) byte ranges or (name, start, stop, m0, m1, m2, m3) for a word of which only the bits
    set in the byte masks m0..m3 are undefined.  Derived from the defined fields only."""
    a = np.ascontiguousarray(archive).view(np.uint8).reshape(-1)
    magic = _u32(a, 0)
    if magic == _ANS_MAGIC:
        return _ans_regions(a, 0)
    assert magic == _FLOAT_MAGIC, f"not an ANS or float archive (magic {magic:#x})"
    opts, n = _u32(a, 8), _u32(a, 4)
    ft = opts & 0xF
    assert ft in (O.F16, O.BF16, O.F32), f"float type {ft} has no reference counterpart"
    regs = [("float options bits 5-31", 8, 12, 0xE0, 0xFF, 0xFF, 0xFF)]
    if not opts & 0x10:
        regs.append(("float checksum (flag clear)", 12, 16))
    nc = O.float_noncomp_bytes(ft, n)
    if ft == O.F32:
        p1 = 16 + 2 * ((n + 7) // 8 * 8)
        regs += [("plane padding", 16 + 2 * n, p1), ("plane padding", p1 + n, 16 + nc)]
    else:
        regs.append(("plane padding", 16 + n, 16 + nc))
    return regs + _ans_regions(a, 16 + nc)


def undefined_mask(archive):
    """uint8 array as long as the archive: per byte, the bits `scribble` may change."""
    a = np.ascontiguousarray(archive).view(np.uint8).reshape(-1)
    m = np.zeros(a.size, np.uint8)
    for r in undefined_regions(a):
        m[r[1]:r[2]] = r[3:] if len(r) > 3 else 0xFF
    return m


def _defined_fields(a):
    """Every defined field of a byte or float archive, as comparable values."""
    f = {}
    base = 0
    if _u32(a, 0) == _FLOAT_MAGIC:
        n, opts = _u32(a, 4), _u32(a, 8)
        ft = opts & 0xF
        f.update(fmagic=_FLOAT_MAGIC, fsize=n, fopts=opts & 0x1F, fchecksum=_u32(a, 12) if opts & 0x10 else None)
        if ft == O.F32:
            p1 = 16 + 2 * ((n + 7) // 8 * 8)
            f["planes"] = (a[16:16 + 2 * n].tobytes(), a[p1:p1 + n].tobytes())
        else:
            f["planes"] = (a[16:16 + n].tobytes(),)
        base = 16 + O.float_noncomp_bytes(ft, n)
    p = O.parse_ans(a[base:])
    for k in ("magic", "num_blocks", "uncompressed", "total_words", "prob_bits", "use_checksum", "size"):
        f[k] = p[k]
    f["checksum"] = p["checksum"] if p["use_checksum"] else None
    f["pdf"] = p["pdf"].tobytes() if p["uncompressed"] else None
    f["states"], f["block_words"] = p["states"].tobytes(), p["block_words"].tobytes()
    f["streams"] = [s.tobytes() for s in p["streams"]]
    return f


def scribble(archive, rng):
    """A copy of a byte or fp16 / bf16 / fp32 archive with random values in every undefined place (the
    options' undefined bits always change), checked to leave every defined field as it was."""
    a = np.ascontiguousarray(archive).view(np.uint8).reshape(-1)
    mask = undefined_mask(a)
    out = (a & ~mask) | (rng.integers(0, 256, a.size, dtype=np.uint8) & mask)
    # the options' bits 5-31 (of the float header and of the ANS header) always get a nonzero garbage value
    for r in undefined_regions(a):
        if "options" in r[0]:
            w = out[r[1]:r[2]].view(np.uint32)
            w[0] = (_u32(a, r[1]) & 0x1F) | (int(rng.integers(1, 1 << 27)) << 5)
    assert _defined_fields(out) == _defined_fields(a), "scribble changed a defined field"
    return out


# ---- statistics helpers --------------------------------------------------------

def coded_bytes(t, kind):
    """The byte of each element that the float codec entropy-codes (float/GpuFloatUtils.cuh), as uint8."""
    if kind == "bytes":
        return t
    if kind == "f32":
        w = t.view(torch.int32)
        return ((w >> 23) & 0xff).to(torch.uint8)
    w = t.view(torch.int16).to(torch.int32) & 0xffff
    return ((w >> 8) if kind == "f16" else ((w >> 7) & 0xff)).to(torch.uint8)


def exact_histogram(t, kind):
    """Exact histogram of the coded bytes (torch.bincount counts in int64, on the device; chunked so the
    temporaries stay small for members of a billion elements)."""
    flat = t.flatten()
    h = torch.zeros(256, dtype=torch.int64, device=t.device)
    for a in range(0, flat.numel(), 1 << 28):
        h += torch.bincount(coded_bytes(flat[a:a + (1 << 28)], kind), minlength=256)
    return h.cpu().numpy()


def stored_pdf(arch, kind):
    """The pdf stored in an archive's ANS header (uint16[256])."""
    a = np.ascontiguousarray(arch).view(np.uint8).reshape(-1)
    if kind != "bytes":
        n = int(a[4:8].view(np.uint32)[0])
        a = a[16 + O.float_noncomp_bytes(KINDS[kind][0], n):]
    return a[32:544].view(np.uint16)


def assert_pdf_matches(arch, t, kind, pb, what):
    """Stored pdf == O.normalize(exact histogram, n, pb)."""
    h = exact_histogram(t, kind)
    assert int(h.sum()) == t.numel()
    want = O.normalize(h.astype(np.uint32), t.numel(), pb)
    got = stored_pdf(arch, kind)
    assert np.array_equal(got.astype(np.uint32), want), f"{what}: pdf differs from normalize(bincount)"
