"""CPU restatement of the sparse fp32 archive (float type 8) -- TEST INFRASTRUCTURE ONLY.

The reference has no sparse float codec, so this format is the library's own extension.  The float layer is stated
here in numpy; the entropy-coded part is the C oracle's byte rANS archive (oracle/dietgpu_oracle.c through
oracle.oracle), which the reference's known-answer tests and stored archives pin.

A word's coded symbol and stored bits are dense fp32's: r = rotl32(w, 1), coded = r >> 24 (the exponent byte),
u16 = r & 0xffff, u8 = (r >> 16) & 0xff.  +0 (0x00000000) and -0 (0x80000000) both have coded symbol 0.  U = the
coded symbols of the words that are neither +0 nor -0.  When at least two symbols are outside U, E+ is the smallest
and E- the second smallest: every +0 word is coded as E+, every -0 word as E-, and neither stores anything.
Otherwise nothing is elided (both or neither, as for types 5 and 6).

    header  32 B   u32 magic/version, n, 8 | checksum flag << 4, checksum,
                   S (kept words), esc = E+ | E- << 8 | 1 << 16 (0 when nothing is elided), 0, 0
    table   4 roundUp(nb, 4) B   u32 per 4096-word block: kept words of all earlier blocks (nb = ceil(n / 4096))
    u16     2 roundUp(S, 8) B    low 16 bits of r for the kept words, in element order
    u8      roundUp(S, 16) B     bits 16..23 of r for the kept words, in element order
    ANS     the byte archive of the n symbols after the E+ / E- substitution
Every section starts 16 B aligned and is zero padded.  The checksum is the float rule: XOR of the first n BYTES.
"""
from __future__ import annotations

import numpy as np

from oracle import oracle as O

F32S = 8
FLOAT_MAGIC_VERSION = (0xF00F << 16) | 1
NEG0 = 0x80000000


def _r(n: int, k: int) -> int:
    return -(-n // k) * k


def _words(w) -> np.ndarray:
    return np.ascontiguousarray(w).view(np.uint32).reshape(-1)


def rot(w: np.ndarray) -> np.ndarray:
    w = w.astype(np.uint32)
    return ((w << np.uint32(1)) | (w >> np.uint32(31))).astype(np.uint32)


def coded(w: np.ndarray) -> np.ndarray:
    return (rot(w) >> np.uint32(24)).astype(np.uint8)


def escapes(words):
    """(E+, E-), or None when fewer than two symbols are free."""
    w = _words(words)
    used = np.zeros(256, bool)
    used[coded(w)[(w & 0x7FFFFFFF) != 0]] = True
    free = np.flatnonzero(~used)
    return (int(free[0]), int(free[1])) if free.size >= 2 else None


def table_bytes(n: int) -> int:
    return 4 * _r(-(-n // 4096), 4)


def stored_bytes(S: int) -> int:
    return 2 * _r(S, 8) + _r(S, 16)


def max_compressed_size(n: int) -> int:
    """dgb_float_max_compressed_size(8, n): 0 when the bound does not fit 32 bits, or when the ANS part's bound
    exceeds INT32_MAX (where the reference refuses a byte archive, ans/GpuANSEncode.cu:13-25)."""
    ans = O.ans_max_compressed_size(n)
    if ans == 0 or ans > 0x7FFFFFFF:
        return 0
    total = 32 + table_bytes(n) + stored_bytes(n) + ans
    return total if total <= 0xFFFFFFFF else 0


def symbols(w: np.ndarray):
    """(coded symbols after the substitution, kept mask, escape word)."""
    sym = coded(w)
    esc = escapes(w)
    keep = np.ones(w.size, bool)
    escw = 0
    if esc is not None:
        ep, em = esc
        sym[w == 0] = ep
        sym[w == NEG0] = em
        keep = (w & 0x7FFFFFFF) != 0
        escw = ep | (em << 8) | (1 << 16)
    return sym, keep, escw


def compress(words, pb: int = 10, use_checksum: bool = False) -> np.ndarray:
    w = _words(words)
    n = w.size
    sym, keep, escw = symbols(w)
    nb = -(-n // 4096)
    per_block = np.add.reduceat(keep.astype(np.int64), np.arange(0, n, 4096)) if n else np.zeros(0, np.int64)
    table = np.zeros(table_bytes(n) // 4, np.uint32)
    table[:nb] = np.concatenate([[0], np.cumsum(per_block)[:-1]]) if nb else []
    S = int(keep.sum())
    r = rot(w[keep])
    u16 = np.zeros(_r(S, 8), np.uint16)
    u16[:S] = r & 0xFFFF
    u8 = np.zeros(_r(S, 16), np.uint8)
    u8[:S] = (r >> 16) & 0xFF
    cks = O.checksum(w.view(np.uint8), n) if (use_checksum and n) else 0
    hdr = np.array([FLOAT_MAGIC_VERSION, n, F32S | (int(use_checksum) << 4), cks, S, escw, 0, 0], np.uint32)
    return np.concatenate([hdr.view(np.uint8), table.view(np.uint8), u16.view(np.uint8), u8, O.ans_encode(sym, pb)])


def info(arch) -> dict:
    h = np.ascontiguousarray(arch).view(np.uint8).reshape(-1)[:32].view(np.uint32)
    ok = int(h[0]) == FLOAT_MAGIC_VERSION
    return dict(ok=ok, size=int(h[1]), float_type=int(h[2]) & 0xF, has_checksum=bool(int(h[2]) & 0x10),
                checksum=int(h[3]), stored=int(h[4]), esc=int(h[5]))


def extra_bytes(arch) -> int:
    """Bytes in front of the ANS archive: header, table and the two stored planes."""
    hd = info(arch)
    return 32 + table_bytes(hd["size"]) + stored_bytes(hd["stored"])


def ans_part(arch) -> np.ndarray:
    a = np.ascontiguousarray(arch).view(np.uint8).reshape(-1)
    return a[extra_bytes(a):]


def decompress(arch, pb: int = 10, verify_checksum: bool = False):
    """(rc, words) with rc an oracle.oracle error code (OK, ERR_BAD_MAGIC, ERR_BAD_FLOAT_TYPE, ERR_CHECKSUM, ...)."""
    a = np.ascontiguousarray(arch).view(np.uint8).reshape(-1)
    hd = info(a)
    if not hd["ok"]:
        return O.ERR_BAD_MAGIC, None
    if hd["float_type"] != F32S:
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
    p16 = 32 + table_bytes(n)
    p8 = p16 + 2 * _r(S, 8)
    v = sym.astype(np.uint32) << np.uint32(24)
    v[keep] |= a[p16:p16 + 2 * S].view(np.uint16).astype(np.uint32) | (a[p8:p8 + S].astype(np.uint32) << np.uint32(16))
    w = ((v >> np.uint32(1)) | (v << np.uint32(31))).astype(np.uint32)
    if esc:
        w[sym == (esc & 0xFF)] = 0
        w[sym == ((esc >> 8) & 0xFF)] = NEG0
    if verify_checksum and hd["has_checksum"] and O.checksum(w.view(np.uint8), n) != hd["checksum"]:
        return O.ERR_CHECKSUM, w
    return O.OK, w


def assert_same(mine, ref, what: str = "") -> None:
    """Header, table and stored planes byte-equal, ANS part semantically equal (stream order may differ)."""
    m, r = np.ascontiguousarray(mine).view(np.uint8).reshape(-1), np.ascontiguousarray(ref).view(np.uint8).reshape(-1)
    assert m.size == r.size, f"{what}: size {m.size} != {r.size}"
    nc = extra_bytes(r)
    assert np.array_equal(m[:32], r[:32]), f"{what}: header {m[:32].view(np.uint32)} != {r[:32].view(np.uint32)}"
    tb = 32 + table_bytes(info(r)["size"])
    assert np.array_equal(m[32:tb], r[32:tb]), f"{what}: block table"
    if not np.array_equal(m[tb:nc], r[tb:nc]):
        bad = np.flatnonzero(m[tb:nc] != r[tb:nc])
        raise AssertionError(f"{what}: stored planes differ at {bad.size} bytes, first at plane byte {bad[:8].tolist()}")
    O.assert_same_ans(m[nc:], r[nc:], what)
