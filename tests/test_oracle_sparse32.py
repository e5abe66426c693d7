"""The sparse fp32 restatement (tests/sparse32_oracle.py, float type 8) against an independent word-by-word statement
of the wire format, its stored archives (tests/golden/sparse32_golden.npz), the escape rule's edges, the library's size
bound and the archive ratios DESIGN.md quotes.  Needs no GPU."""
import os

import numpy as np
import pytest
import torch

import sparse32_oracle as S
from oracle import oracle as O

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sparse32_golden.npz")
NEG0 = S.NEG0


def _r(n, k):
    return -(-n // k) * k


def f32_words(x):
    return np.ascontiguousarray(np.asarray(x, np.float32)).view(np.uint32).copy()


def relu_words(n, seed):
    g = torch.Generator().manual_seed(seed)
    return f32_words(torch.randn(n, generator=g).clamp_min(0).numpy())


def masked_words(n, seed, keep=0.1):
    """x * mask for N(0,1) x and a Bernoulli(keep) mask: +0 where x >= 0 is masked, -0 where x < 0 is."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, generator=g)
    return f32_words((x * (torch.rand(n, generator=g) < keep).float()).numpy())


def pruned_words(x, frac=0.9):
    """x with the `frac` smallest magnitudes set to +0."""
    x = np.array(x, np.float32)
    x[np.argsort(np.abs(x), kind="stable")[:int(frac * x.size)]] = 0
    return f32_words(x)


def word_with_symbol(s):
    """A word whose coded symbol (exponent byte) is s and that is neither +0 nor -0."""
    return (s << 23) | 1


def all_but(free, zeros=200):
    """One word of every symbol except `free`, then +0 and -0 words."""
    w = [word_with_symbol(s) for s in range(256) if s not in free]
    return np.array(w + [0] * zeros + [NEG0] * zeros, np.uint32)


def segment_boundary_member(seed=21, tail=1234):
    """Blocks whose kept counts are 1 (mod 16), so the block boundaries in the planes (table[k]) run through every
    residue mod 16 of the u8 plane and mod 8 of the u16 plane, twice; some blocks keep 1 or 17 words only, so two or
    more neighbouring segments share one 16 B vector of each plane.  +0 and -0 both occur, in runs and scattered."""
    rng = np.random.default_rng(seed)
    blocks = []
    kept_counts = [1, 17, 4081, 2049, 1, 33, 4065, 3217, 17, 1, 1025, 4081, 49, 2913, 1, 4081,
                   17, 4081, 1, 1, 3105, 65, 4081, 2241, 17, 1, 4001, 81, 1, 4081, 17, 1649, 1, 4081]
    for j, c in enumerate(kept_counts):
        x = (rng.standard_normal(4096) + 3.0).astype(np.float32)  # no zeros
        w = f32_words(x)
        zeros = rng.permutation(4096)[:4096 - c] if j % 3 else np.arange(4096 - c)  # scattered or one run
        w[zeros] = np.where(rng.random(zeros.size) < 0.3, NEG0, 0).astype(np.uint32)
        blocks.append(w)
    w = f32_words(rng.standard_normal(tail))
    w[rng.random(tail) < 0.5] = 0
    blocks.append(w)
    return np.concatenate(blocks)


def edge_corpus():
    """Members that exercise the escape rule and the block / 16 B bookkeeping."""
    rng = np.random.default_rng(58)
    c = [relu_words(n, 300 + n) for n in (0, 1, 31, 4095, 4096, 4097, 300000)]
    # zero runs across block and 16 B boundaries; a block of only zeros next to blocks without any
    w = f32_words(rng.standard_normal(20000) + 8.0)
    w[4090:4110] = 0
    w[3:11] = NEG0
    w[8192:12288] = 0
    w[16380:16390] = NEG0
    c.append(w)
    c.append(masked_words(70001, 7))                                       # ~90 % +-0
    nan_inf = [0x7F800000, 0xFF800000, 0x7FC00000, 0x7F800001, 0xFFC00001]
    c.append(np.array((nan_inf + [0, NEG0, 0x3F800000, 0x00000001, 0x807FFFFF]) * 1500, np.uint32))  # NaN/Inf/denormals
    c.append(np.zeros(9000, np.uint32))                                    # all +0
    c.append(np.full(9000, NEG0, np.uint32))                               # all -0
    c.append(f32_words(rng.standard_normal(5000) + 4.0))                   # no zeros
    c.append(rng.integers(0, 1 << 32, 70001, dtype=np.uint32))             # full range: nothing free, nothing elided
    c.append(all_but((17, 200)))                                           # exactly two free symbols
    c.append(all_but((99,)))                                               # exactly one free symbol
    sub = np.arange(1, 0x800, 7, dtype=np.uint32)                          # denormals use symbol 0
    c.append(np.concatenate([sub, sub | NEG0, np.zeros(300, np.uint32), np.full(300, NEG0, np.uint32)]))
    c.append(np.concatenate([f32_words(rng.uniform(1, 2, 3000)), np.zeros(100, np.uint32),
                             np.full(50, NEG0, np.uint32)]))                # E+ = 0, the zeros' natural symbol
    c.append(np.concatenate([f32_words(rng.uniform(1, 2, 3000)), np.full(700, NEG0, np.uint32)]))  # -0 only
    c.append(np.concatenate([np.zeros(5000, np.uint32), f32_words(rng.uniform(1, 2, 3000))]))     # +0 only
    c.append(segment_boundary_member())
    return c


def scalar_archive(w, pb, checksum):
    """Type 8 word by word with Python integers."""
    n = len(w)
    ws = [int(x) for x in w]
    rots = [((x << 1) | (x >> 31)) & 0xFFFFFFFF for x in ws]
    coded = [r >> 24 for r in rots]
    used = sorted({c for x, c in zip(ws, coded) if x not in (0, NEG0)})
    free = [s for s in range(256) if s not in used]
    elide = len(free) >= 2
    sym, u16, u8, kept = [], bytearray(), bytearray(), []
    for x, c, r in zip(ws, coded, rots):
        if elide and x == 0:
            sym.append(free[0])
        elif elide and x == NEG0:
            sym.append(free[1])
        else:
            sym.append(c)
            u16 += (r & 0xFFFF).to_bytes(2, "little")
            u8.append((r >> 16) & 0xFF)
        kept.append(0 if elide and x in (0, NEG0) else 1)
    nb = -(-n // 4096)
    table, run = [], 0
    for k in range(nb):
        table.append(run)
        run += sum(kept[4096 * k:4096 * (k + 1)])
    table += [0] * (_r(nb, 4) - nb)
    cks = 0
    if checksum:
        for b in b"".join(x.to_bytes(4, "little") for x in ws)[:n]:
            cks ^= b
    S_ = len(u8)
    esc = free[0] | (free[1] << 8) | (1 << 16) if elide else 0
    hdr = [(0xF00F << 16) | 1, n, 8 | (int(checksum) << 4), cks, S_, esc, 0, 0]
    body = (b"".join(x.to_bytes(4, "little") for x in hdr + table) + bytes(u16) + bytes(2 * _r(S_, 8) - 2 * S_)
            + bytes(u8) + bytes(_r(S_, 16) - S_))
    return np.concatenate([np.frombuffer(body, np.uint8), O.ans_encode(np.array(sym, np.uint8), pb)])


@pytest.mark.parametrize("n", [0, 1, 7, 8, 9, 15, 16, 17, 4095, 4096, 4097, 9000])
def test_archive_equals_scalar_statement(n):
    for k, w in enumerate((relu_words(n, n), masked_words(n, n + 1))):
        for pb, checksum in ((9, False), (10, True), (11, False)):
            got = S.compress(w, pb, checksum)
            assert np.array_equal(got, scalar_archive(w, pb, checksum)), (n, k, pb, checksum)
            assert got.size == S.extra_bytes(got) + O.ans_info(S.ans_part(got))["size"]


def test_full_range_round_trip_is_bit_exact():
    rng = np.random.default_rng(8)
    w = np.concatenate([rng.integers(0, 1 << 32, 50000, dtype=np.uint32), np.zeros(3000, np.uint32),
                        np.full(3000, NEG0, np.uint32)])
    for pb in (9, 10, 11):
        a = S.compress(w, pb, True)
        hd = S.info(a)
        assert (hd["float_type"], hd["size"], hd["has_checksum"], hd["esc"]) == (8, w.size, True, 0)
        rc, out = S.decompress(a, pb, verify_checksum=True)
        assert rc == O.OK and np.array_equal(out, w)
    bad = S.compress(w).copy()
    bad[8] = 3  # dense fp32's type
    assert S.decompress(bad)[0] == O.ERR_BAD_FLOAT_TYPE


def test_escape_rule_edges():
    for i, w in enumerate(edge_corpus()):
        a = S.compress(w, 10, True)
        rc, out = S.decompress(a, 10, verify_checksum=True)
        assert rc == O.OK and np.array_equal(out, w), i
    # 0 free symbols: nothing elided
    w = np.random.default_rng(3).integers(0, 1 << 32, 70001, dtype=np.uint32)
    w[::5] = 0
    assert S.escapes(w) is None and S.info(S.compress(w))["esc"] == 0
    assert S.info(S.compress(w))["stored"] == w.size
    # 1 free symbol: nothing elided
    w = all_but((99,))
    hd = S.info(S.compress(w))
    assert (hd["esc"], hd["stored"]) == (0, w.size)
    # 2 free symbols: they are E+ and E-
    w = all_but((17, 200))
    assert S.info(S.compress(w))["esc"] == 17 | 200 << 8 | 1 << 16
    assert S.info(S.compress(w))["stored"] == 254
    # 256 free symbols (only zeros): symbols 0 and 1, nothing stored
    for w in (np.zeros(9000, np.uint32), np.full(9000, NEG0, np.uint32)):
        hd = S.info(S.compress(w))
        assert (hd["esc"], hd["stored"]) == (0 | 1 << 8 | 1 << 16, 0)
    # no zeros: the escapes are still chosen, every word stores its bits
    w = f32_words(np.random.default_rng(1).standard_normal(5000) + 4.0)
    hd = S.info(S.compress(w))
    assert hd["esc"] >> 16 == 1 and hd["stored"] == w.size
    # E+ = 0: the common case without denormals
    w = np.concatenate([f32_words(np.random.default_rng(2).uniform(1, 2, 3000)), np.zeros(10, np.uint32),
                        np.full(10, NEG0, np.uint32)])
    assert S.escapes(w)[0] == 0
    assert np.array_equal(S.decompress(S.compress(w))[1], w)
    # denormals use symbol 0, so E+ is another symbol
    sub = np.arange(1, 0x80, dtype=np.uint32)
    w = np.concatenate([sub, sub | NEG0, np.zeros(30, np.uint32), np.full(30, NEG0, np.uint32)])
    assert 0 not in S.escapes(w)
    assert np.array_equal(S.decompress(S.compress(w))[1], w)
    # -0 only and +0 only
    base = f32_words(np.random.default_rng(4).uniform(1, 2, 3000))
    for z in (np.full(500, NEG0, np.uint32), np.zeros(500, np.uint32)):
        w = np.concatenate([base, z])
        hd = S.info(S.compress(w))
        assert hd["stored"] == base.size and hd["esc"] >> 16 == 1
        assert np.array_equal(S.decompress(S.compress(w))[1], w)


def test_segment_boundary_member_covers_every_residue():
    w = segment_boundary_member()
    a = S.compress(w)
    nb = -(-w.size // 4096)
    table = a[32:32 + 4 * nb].view(np.uint32)
    assert set((table % 16).tolist()) == set(range(16))
    assert set((table % 8).tolist()) == set(range(8))
    assert np.array_equal(S.decompress(a)[1], w)


def test_stored_archives_are_reproduced():
    g = np.load(GOLD)
    names = sorted({k.rsplit("/", 1)[0] for k in g.files})
    assert len(names) >= 8
    for name in names:
        w = g[f"{name}/in"]
        for pb in (9, 10, 11):
            want = g[f"{name}/pb{pb}"]
            assert np.array_equal(S.compress(w, pb, True), want), (name, pb)
            rc, out = S.decompress(want, pb, verify_checksum=True)
            assert rc == O.OK and np.array_equal(out, w)
    kinds = {(S.info(g[f"{n}/pb10"])["esc"] != 0, S.info(g[f"{n}/pb10"])["size"] == 0) for n in names}
    assert {(True, False), (False, False), (True, True)} <= kinds


def _ratio_inputs():
    x = np.random.default_rng(1234).standard_normal(1 << 20).astype(np.float32)
    return {"relu": f32_words(np.maximum(x, 0)), "pruned90": pruned_words(x), "normal": f32_words(x)}


@pytest.mark.parametrize("name,dense,sparse", [("relu", 0.828, 0.454), ("pruned90", 0.775, 0.100),
                                               ("normal", 0.837, 0.837)])
def test_archive_ratios(name, dense, sparse):
    w = _ratio_inputs()[name]
    a = S.compress(w, 10)
    d = O.float_compress(O.F32, w, 10)
    assert round(a.size / w.nbytes, 3) == sparse, a.size / w.nbytes
    assert round(d.size / w.nbytes, 3) == dense, d.size / w.nbytes
    if name == "normal":  # no zeros: 16 B of header and 4 B per block more than dense
        assert a.size - d.size == 16 + S.table_bytes(w.size)


def _largest_nonzero(bound):
    lo, hi = 1, 1 << 32
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if bound(mid) else (lo, mid)
    return lo


def test_max_compressed_size_matches_the_library():
    from dietgpu_b200 import capi

    L = capi.lib()
    top = _largest_nonzero(lambda n: S.max_compressed_size(n) != 0)
    assert top == _largest_nonzero(lambda n: L.dgb_float_max_compressed_size(capi.FLOAT32_SPARSE, n) != 0)
    for n in [0, 1, 2, 7, 8, 9, 15, 16, 17, 4095, 4096, 4097, 16385, 1 << 20, 123456789, top - 1, top, top + 1,
              top + 4096, 0xFFFFFFFF]:
        assert L.dgb_float_max_compressed_size(capi.FLOAT32_SPARSE, n) == S.max_compressed_size(n), n
    assert S.max_compressed_size(top + 1) == 0
    assert S.max_compressed_size(top) == 32 + S.table_bytes(top) + S.stored_bytes(top) + O.ans_max_compressed_size(top)
    # 7 stays an unknown type; the other types keep their values
    assert L.dgb_float_max_compressed_size(7, 100) == 0
    for ft in (O.F16, O.BF16, O.F32):
        for n in (0, 1, 4097, 1 << 24):
            assert L.dgb_float_max_compressed_size(ft, n) == O.float_max_compressed_size(ft, n)


def test_sparse_keyword_with_float32():
    from dietgpu_b200 import capi, ops

    t32, t16 = torch.zeros(4), torch.zeros(4, dtype=torch.float16)
    with pytest.raises(ValueError):
        ops.compress_data(False, [t32], sparse=True)
    with pytest.raises(ValueError):
        ops.max_float_compressed_output_size([torch.zeros(4, dtype=torch.float64)], sparse=True)
    with pytest.raises(ValueError):
        ops.max_float_compressed_size(torch.zeros(4, dtype=torch.float64), 10, sparse=True)
    with pytest.raises(ValueError):
        ops.decompress_data_simple(False, [torch.zeros(64, dtype=torch.uint8)], sparse=True)
    # the single-size bound keeps its 16-bit-only sparse contract; the batch bound covers float32
    with pytest.raises(ValueError):
        ops.max_float_compressed_size(t32, 5000, sparse=True)
    L = capi.lib()
    assert ops.max_float_compressed_output_size([torch.zeros(5000)], sparse=True)[1] == \
        L.dgb_float_max_compressed_size(8, 5000)
    assert ops.max_float_compressed_output_size([torch.zeros(9)], sparse=True)[1] == \
        L.dgb_float_max_compressed_size(capi.FLOAT32_SPARSE, 9)
    assert ops.max_float_compressed_size(t16, 5000, sparse=True) == \
        L.dgb_float_max_compressed_size(capi.FLOAT16_SPARSE, 5000)
