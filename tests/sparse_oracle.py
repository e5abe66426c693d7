"""CPU restatement of the sparse fp16 / bf16 archives (float types 5 and 6) -- TEST INFRASTRUCTURE ONLY.

The reference has no sparse float codec, so this format is the library's own extension.  The float layer is
stated here in numpy; the entropy-coded part is the C oracle's byte rANS archive (oracle/dietgpu_oracle.c through
oracle.oracle), which the reference's known-answer tests and stored archives pin.

A word's coded symbol and stored byte are the dense type's: fp16 coded = w >> 8, stored = w & 0xff; bf16
coded = (w >> 7) & 0xff, stored = rotl16(w, 1) & 0xff.  U = the coded symbols of the words that are neither +0
(0x0000) nor -0 (0x8000).  When at least two symbols are outside U, E+ is the smallest and E- the second
smallest: every +0 word is coded as E+, every -0 word as E-, and neither stores a byte.  Otherwise nothing is
elided (eliding only one kind of zero could make E+ the natural symbol of a -0 word still coded as itself).

    header  32 B   u32 magic/version, n, type | checksum flag << 4, checksum,
                   S (words that store a byte), esc = E+ | E- << 8 | 1 << 16 (0 when nothing is elided), 0, 0
    table   4 roundUp(nb, 4) B   u32 per 4 KiB block: stored bytes of all earlier blocks (nb = ceil(n / 4096))
    plane   roundUp(S, 16) B     the stored bytes of the kept words, in element order
    ANS     the byte archive of the n symbols after the E+ / E- substitution
Every section starts 16 B aligned and is zero padded.  The checksum is the float rule: XOR of the first n BYTES.
"""
from __future__ import annotations

import numpy as np

from oracle import oracle as O

F16S, BF16S = 5, 6
FLOAT_MAGIC_VERSION = (0xF00F << 16) | 1


def _r(n: int, k: int) -> int:
    return -(-n // k) * k


def _words(w) -> np.ndarray:
    return np.ascontiguousarray(w).view(np.uint16).reshape(-1)


def coded_stored(w: np.ndarray, ft: int):
    """(natural coded symbol, stored byte) of every word, as uint8 arrays."""
    w = w.astype(np.uint32)
    if ft == F16S:
        return (w >> 8).astype(np.uint8), (w & 0xFF).astype(np.uint8)
    assert ft == BF16S, ft
    return ((w >> 7) & 0xFF).astype(np.uint8), (((w << 1) | (w >> 15)) & 0xFF).astype(np.uint8)


def escapes(words, ft: int):
    """(E+, E-), or None when fewer than two symbols are free."""
    w = _words(words)
    coded, _ = coded_stored(w, ft)
    used = np.zeros(256, bool)
    used[coded[(w & 0x7FFF) != 0]] = True
    free = np.flatnonzero(~used)
    return (int(free[0]), int(free[1])) if free.size >= 2 else None


def table_bytes(n: int) -> int:
    return 4 * _r(-(-n // 4096), 4)


def max_compressed_size(n: int) -> int:
    """dgb_float_max_compressed_size(5 | 6, n): 0 when the bound does not fit 32 bits, or when the ANS part's bound
    exceeds INT32_MAX (where the reference refuses a byte archive, ans/GpuANSEncode.cu:13-25)."""
    ans = O.ans_max_compressed_size(n)
    if ans == 0 or ans > 0x7FFFFFFF:
        return 0
    total = 32 + table_bytes(n) + _r(n, 16) + ans
    return total if total <= 0xFFFFFFFF else 0


def compress(words, ft: int, pb: int = 10, use_checksum: bool = False) -> np.ndarray:
    w = _words(words)
    n = w.size
    coded, stored = coded_stored(w, ft)
    esc = escapes(w, ft)
    sym = coded.copy()
    keep = np.ones(n, bool)
    escw = 0
    if esc is not None:
        ep, em = esc
        sym[w == 0] = ep
        sym[w == 0x8000] = em
        keep = (w & 0x7FFF) != 0
        escw = ep | (em << 8) | (1 << 16)
    nb = -(-n // 4096)
    per_block = np.add.reduceat(keep.astype(np.int64), np.arange(0, n, 4096)) if n else np.zeros(0, np.int64)
    table = np.zeros(table_bytes(n) // 4, np.uint32)
    table[:nb] = np.concatenate([[0], np.cumsum(per_block)[:-1]]) if nb else []
    S = int(keep.sum())
    plane = np.zeros(_r(S, 16), np.uint8)
    plane[:S] = stored[keep]
    cks = O.checksum(w.view(np.uint8), n) if (use_checksum and n) else 0
    hdr = np.array([FLOAT_MAGIC_VERSION, n, ft | (int(use_checksum) << 4), cks, S, escw, 0, 0], np.uint32)
    return np.concatenate([hdr.view(np.uint8), table.view(np.uint8), plane, O.ans_encode(sym, pb)])


def info(arch) -> dict:
    h = np.ascontiguousarray(arch).view(np.uint8).reshape(-1)[:32].view(np.uint32)
    ok = int(h[0]) == FLOAT_MAGIC_VERSION
    return dict(ok=ok, size=int(h[1]), float_type=int(h[2]) & 0xF, has_checksum=bool(int(h[2]) & 0x10),
                checksum=int(h[3]), stored=int(h[4]), esc=int(h[5]))


def extra_bytes(arch) -> int:
    """Bytes in front of the ANS archive: header, table and stored bytes."""
    hd = info(arch)
    return 32 + table_bytes(hd["size"]) + _r(hd["stored"], 16)


def ans_part(arch) -> np.ndarray:
    a = np.ascontiguousarray(arch).view(np.uint8).reshape(-1)
    return a[extra_bytes(a):]


def decompress(arch, ft: int, pb: int = 10, verify_checksum: bool = False):
    """(rc, words) with rc an oracle.oracle error code (OK, ERR_BAD_MAGIC, ERR_BAD_FLOAT_TYPE, ERR_CHECKSUM, ...)."""
    a = np.ascontiguousarray(arch).view(np.uint8).reshape(-1)
    hd = info(a)
    if not hd["ok"]:
        return O.ERR_BAD_MAGIC, None
    if hd["float_type"] != ft:
        return O.ERR_BAD_FLOAT_TYPE, None
    n, S, esc = hd["size"], hd["stored"], hd["esc"]
    if S > n or not (esc == 0 or (esc >> 16 == 1 and (esc & 0xFF) < ((esc >> 8) & 0xFF))):
        return O.ERR_CORRUPT, None
    rc, sym, got = O.ans_decode(a[extra_bytes(a):], pb)
    if rc != O.OK or got != n:
        return (rc if rc != O.OK else O.ERR_CORRUPT), None
    keep = np.ones(n, bool)
    if esc:
        keep = (sym != (esc & 0xFF)) & (sym != ((esc >> 8) & 0xFF))
    if int(keep.sum()) != S:
        return O.ERR_CORRUPT, None
    base = 32 + table_bytes(n)
    v = sym.astype(np.uint32) << 8
    v[keep] |= a[base:base + S].astype(np.uint32)
    w = v if ft == F16S else ((v >> 1) | ((v & 1) << 15)) & 0xFFFF
    w = w.astype(np.uint16)
    if esc:
        w[sym == (esc & 0xFF)] = 0
        w[sym == ((esc >> 8) & 0xFF)] = 0x8000
    if verify_checksum and hd["has_checksum"] and O.checksum(w.view(np.uint8), n) != hd["checksum"]:
        return O.ERR_CHECKSUM, w
    return O.OK, w


def assert_same(mine, ref, what: str = "") -> None:
    """Header, table and stored bytes byte-equal, ANS part semantically equal (stream order may differ)."""
    m, r = np.ascontiguousarray(mine).view(np.uint8).reshape(-1), np.ascontiguousarray(ref).view(np.uint8).reshape(-1)
    assert m.size == r.size, f"{what}: size {m.size} != {r.size}"
    nc = extra_bytes(r)
    assert np.array_equal(m[:32], r[:32]), f"{what}: header {m[:32].view(np.uint32)} != {r[:32].view(np.uint32)}"
    assert np.array_equal(m[32:nc], r[32:nc]), f"{what}: block table / stored bytes"
    O.assert_same_ans(m[nc:], r[nc:], what)
