"""CPU restatement of the float64 archive (float type 4) -- TEST INFRASTRUCTURE ONLY.

The reference has no float64 codec, so this format is the library's own extension.  The float layer is stated
here in numpy; the entropy-coded part is the C oracle's byte rANS archive (oracle/dietgpu_oracle.c through
oracle.oracle), which the reference's known-answer tests and stored archives pin.

    archive = 16 B float header | u32 plane | u16 plane | u8 plane | ANS archive of the n coded bytes
    v = rotl64(w, 1): coded byte = v >> 56 (exponent bits 10..3), u32 = v & 0xffffffff,
                      u16 = (v >> 32) & 0xffff, u8 = (v >> 48) & 0xff
Each plane starts 16 B aligned (4 roundUp(n, 4), 2 roundUp(n, 8), roundUp(n, 16) bytes) and is zero padded.
The header holds the magic / version, n (words), the type 4 in the low bits of the options word with the
checksum flag in bit 4, and the checksum: the XOR of the first n BYTES of the input (the reference's float
rule, so the first n / 8 words).
"""
from __future__ import annotations

import numpy as np

from oracle import oracle as O

F64 = 4
FLOAT_MAGIC_VERSION = (0xF00F << 16) | 1
_ONE, _W63, _32, _48, _56 = (np.uint64(k) for k in (1, 63, 32, 48, 56))


def _r(n: int, k: int) -> int:
    return -(-n // k) * k


def noncomp_bytes(n: int) -> int:
    return 4 * _r(n, 4) + 2 * _r(n, 8) + _r(n, 16)


def max_compressed_size(n: int) -> int:
    """16 + the ANS bound + the planes; 0 when that does not fit 32 bits (dgb_float_max_compressed_size)."""
    total = 16 + O.ans_max_compressed_size(n) + noncomp_bytes(n)
    return total if total <= 0xFFFFFFFF else 0


def _words(w) -> np.ndarray:
    return np.ascontiguousarray(w).view(np.uint64).reshape(-1)


def compress(words, pb: int = 10, use_checksum: bool = False) -> np.ndarray:
    w = _words(words)
    n = w.size
    v = (w << _ONE) | (w >> _W63)
    u32 = np.zeros(_r(n, 4), np.uint32)
    u32[:n] = v.astype(np.uint32)
    u16 = np.zeros(_r(n, 8), np.uint16)
    u16[:n] = (v >> _32).astype(np.uint16)
    u8 = np.zeros(_r(n, 16), np.uint8)
    u8[:n] = (v >> _48).astype(np.uint8)
    coded = (v >> _56).astype(np.uint8)
    cks = O.checksum(w.view(np.uint8), n) if (use_checksum and n) else 0
    hdr = np.array([FLOAT_MAGIC_VERSION, n, F64 | (int(use_checksum) << 4), cks], np.uint32)
    return np.concatenate([hdr.view(np.uint8), u32.view(np.uint8), u16.view(np.uint8), u8, O.ans_encode(coded, pb)])


def info(arch) -> dict:
    h = np.ascontiguousarray(arch).view(np.uint8).reshape(-1)[:16].view(np.uint32)
    ok = int(h[0]) == FLOAT_MAGIC_VERSION
    return dict(ok=ok, size=int(h[1]), float_type=int(h[2]) & 0xF, has_checksum=bool(int(h[2]) & 0x10),
                checksum=int(h[3]))


def decompress(arch, pb: int = 10, verify_checksum: bool = False):
    """(rc, words) with rc an oracle.oracle error code (OK, ERR_BAD_MAGIC, ERR_BAD_FLOAT_TYPE, ERR_CHECKSUM, ...)."""
    a = np.ascontiguousarray(arch).view(np.uint8).reshape(-1)
    hd = info(a)
    if not hd["ok"]:
        return O.ERR_BAD_MAGIC, None
    if hd["float_type"] != F64:
        return O.ERR_BAD_FLOAT_TYPE, None
    n = hd["size"]
    p16, p8 = 16 + 4 * _r(n, 4), 16 + 4 * _r(n, 4) + 2 * _r(n, 8)
    rc, coded, got = O.ans_decode(a[16 + noncomp_bytes(n):], pb)
    if rc != O.OK or got != n:
        return (rc if rc != O.OK else O.ERR_CORRUPT), None
    v = (coded.astype(np.uint64) << _56) | (a[p8:p8 + n].astype(np.uint64) << _48) \
        | (a[p16:p16 + 2 * n].view(np.uint16).astype(np.uint64) << _32) | a[16:16 + 4 * n].view(np.uint32).astype(np.uint64)
    w = (v >> _ONE) | (v << _W63)
    if verify_checksum and hd["has_checksum"] and O.checksum(w.view(np.uint8), n) != hd["checksum"]:
        return O.ERR_CHECKSUM, w
    return O.OK, w


def ans_part(arch) -> np.ndarray:
    a = np.ascontiguousarray(arch).view(np.uint8).reshape(-1)
    return a[16 + noncomp_bytes(info(a)["size"]):]


def assert_same(mine, ref, what: str = "") -> None:
    """Header and stored planes byte-equal, ANS part semantically equal (stream order may differ)."""
    m, r = np.ascontiguousarray(mine).view(np.uint8).reshape(-1), np.ascontiguousarray(ref).view(np.uint8).reshape(-1)
    assert m.size == r.size, f"{what}: size {m.size} != {r.size}"
    nc = 16 + noncomp_bytes(info(r)["size"])
    assert np.array_equal(m[:nc], r[:nc]), f"{what}: float header / stored planes"
    O.assert_same_ans(m[nc:], r[nc:], what)
