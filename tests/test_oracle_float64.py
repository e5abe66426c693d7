"""The float64 restatement (tests/f64_oracle.py, float type 4) against an independent scalar statement of the
wire format, its stored archives (tests/golden/f64_golden.npz) and the library's size bound.  Needs no GPU."""
import os

import numpy as np
import pytest

import f64_oracle as F
from oracle import oracle as O

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "f64_golden.npz")


def _r(n, k):
    return -(-n // k) * k


def scalar_archive(w, pb, checksum):
    """Float type 4 word by word with Python integers: header | u32 | u16 | u8 plane | ANS of the coded bytes."""
    n = len(w)
    u32, u16, u8 = bytearray(4 * _r(n, 4)), bytearray(2 * _r(n, 8)), bytearray(_r(n, 16))
    coded, cks = bytearray(n), 0
    for i, x in enumerate(int(x) for x in w):
        v = ((x << 1) | (x >> 63)) & (2 ** 64 - 1)
        u32[4 * i:4 * i + 4] = (v & 0xFFFFFFFF).to_bytes(4, "little")
        u16[2 * i:2 * i + 2] = ((v >> 32) & 0xFFFF).to_bytes(2, "little")
        u8[i] = (v >> 48) & 0xFF
        coded[i] = v >> 56
    if checksum:
        raw = b"".join(int(x).to_bytes(8, "little") for x in w)[:n]
        for b in raw:
            cks ^= b
    hdr = b"".join(x.to_bytes(4, "little") for x in ((0xF00F << 16) | 1, n, 4 | (int(checksum) << 4), cks))
    body = np.frombuffer(bytes(hdr + u32 + u16 + u8), np.uint8)
    return np.concatenate([body, O.ans_encode(np.frombuffer(bytes(coded), np.uint8), pb)])


def _words(n, seed):
    return np.random.default_rng(seed).standard_normal(n).view(np.uint64)


@pytest.mark.parametrize("n", [0, 1, 3, 4, 5, 15, 16, 17, 4095, 4096, 4097, 20001])
@pytest.mark.parametrize("pb", [9, 10, 11])
def test_archive_equals_scalar_statement(n, pb):
    w = _words(n, 10 + n)
    for checksum in (False, True):
        got = F.compress(w, pb, checksum)
        assert np.array_equal(got, scalar_archive(w, pb, checksum)), (n, pb, checksum)
        assert got.size == 16 + F.noncomp_bytes(n) + O.ans_info(F.ans_part(got))["size"]
    # the coded byte is exponent bits 10..3, i.e. fp32's coded byte of the word's high half
    hi = (w >> np.uint64(32)).astype(np.uint32)
    assert np.array_equal((w >> np.uint64(55)).astype(np.uint8), ((hi >> 23) & 0xFF).astype(np.uint8))


def test_full_range_round_trip_is_bit_exact():
    rng = np.random.default_rng(3)
    w = np.concatenate([
        rng.integers(0, 2 ** 64, 50000, dtype=np.uint64),                         # NaN payloads, +-Inf, all
        np.array([0, 1 << 63, 0x7FF0000000000000, 0xFFF0000000000000, 0x7FF8000000000123,
                  0xFFF4000000000001, 1, 0x000FFFFFFFFFFFFF, 0x800FFFFFFFFFFFFF], np.uint64),
        rng.integers(0, 2 ** 52, 3000, dtype=np.uint64),                          # subnormals
    ])
    for pb in (9, 10, 11):
        a = F.compress(w, pb, True)
        hd = F.info(a)
        assert (hd["float_type"], hd["size"], hd["has_checksum"]) == (4, w.size, True)
        rc, out = F.decompress(a, pb, verify_checksum=True)
        assert rc == O.OK and out.dtype == np.uint64 and np.array_equal(out, w)
    bad = F.compress(w, 10, True)
    bad[16] ^= 1  # a stored-plane bit of word 0
    assert F.decompress(bad, 10, verify_checksum=True)[0] == O.ERR_CHECKSUM


def test_stored_archives_are_reproduced():
    g = np.load(GOLD)
    names = sorted({k.split("/")[1] for k in g.files})
    assert len(names) >= 5
    for name in names:
        w = g[f"f64/{name}/in"]
        for pb in (9, 10, 11):
            want = g[f"f64/{name}/pb{pb}"]
            assert np.array_equal(F.compress(w, pb, True), want), (name, pb)
            rc, out = F.decompress(want, pb, verify_checksum=True)
            assert rc == O.OK and np.array_equal(out, w)


def test_normal_ratio_beats_the_byte_codec():
    w = _words(1 << 20, 99)
    a = F.compress(w, 10)
    b = O.ans_encode(w.view(np.uint8), 10)
    assert a.size / w.nbytes <= 0.90, a.size / w.nbytes
    assert a.size < b.size


def _largest_nonzero(bound):
    lo, hi = 1, 1 << 32
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if bound(mid):
            lo = mid
        else:
            hi = mid
    return lo


def test_max_compressed_size_matches_the_library():
    from dietgpu_b200 import capi

    L = capi.lib()
    top = _largest_nonzero(lambda n: F.max_compressed_size(n) != 0)
    assert 500_000_000 < top < 530_000_000
    for n in [0, 1, 2, 3, 4, 5, 8, 15, 16, 17, 4095, 4096, 4097, 1 << 20, 123456789, top - 1, top, top + 1,
              top + 4096, 0xFFFFFFFF]:
        assert L.dgb_float_max_compressed_size(capi.FLOAT64, n) == F.max_compressed_size(n), n
    assert F.max_compressed_size(top + 1) == 0
    # the other float types keep their values
    for ft in (O.F16, O.BF16, O.F32):
        for n in (0, 1, 4097, 1 << 24):
            assert L.dgb_float_max_compressed_size(ft, n) == O.float_max_compressed_size(ft, n)
