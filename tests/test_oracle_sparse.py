"""The sparse fp16 / bf16 restatement (tests/sparse_oracle.py, float types 5 and 6) against an independent
word-by-word statement of the wire format, its stored archives (tests/golden/sparse_golden.npz), the escape rule's
edges and the library's size bound.  Needs no GPU."""
import os

import numpy as np
import pytest
import torch

import sparse_oracle as S
from oracle import oracle as O

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sparse_golden.npz")
TYPES = {S.F16S: torch.float16, S.BF16S: torch.bfloat16}


def _r(n, k):
    return -(-n // k) * k


def words_of(x, ft):
    """uint16 words of a float tensor / array converted to the type's dtype."""
    return torch.as_tensor(x, dtype=torch.float32).to(TYPES[ft]).view(torch.int16).numpy().view(np.uint16).copy()


def relu_words(n, ft, seed):
    g = torch.Generator().manual_seed(seed)
    return words_of(torch.randn(n, generator=g).clamp_min(0), ft)


def masked_words(n, ft, seed, keep=0.1):
    """x * mask for N(0,1) x and a Bernoulli(keep) mask: +0 where x >= 0 is masked, -0 where x < 0 is."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, generator=g).to(TYPES[ft])
    return (x * (torch.rand(n, generator=g) < keep).to(TYPES[ft])).view(torch.int16).numpy().view(np.uint16).copy()


def word_with_symbol(s, ft):
    """A word whose coded symbol is s and that is neither +0 nor -0."""
    return (s << 8) | 1 if ft == S.F16S else (s << 7) | 1


def all_but(free, ft, zeros=200):
    """One word of every symbol except `free`, then +0 and -0 words."""
    w = [word_with_symbol(s, ft) for s in range(256) if s not in free]
    return np.array(w + [0] * zeros + [0x8000] * zeros, np.uint16)


def edge_corpus(ft):
    """Members that exercise the escape rule and the block / 16 B bookkeeping."""
    rng = np.random.default_rng(50 + ft)
    c = [relu_words(n, ft, 300 + n) for n in (0, 1, 31, 4095, 4096, 4097, 300000)]
    # zero runs across block and 16 B boundaries; a block of only zeros next to a block without any
    w = words_of(rng.standard_normal(20000) + 8.0, ft)
    w[4090:4110] = 0
    w[3:11] = 0x8000
    w[8192:12288] = 0
    w[16380:16390] = 0x8000
    c.append(w)
    c.append(masked_words(70001, ft, 7))                                 # ~90 % +-0
    nan_inf = [0x7C00, 0xFC00, 0x7E00, 0x7C01] if ft == S.F16S else [0x7F80, 0xFF80, 0x7FC0, 0x7F81]
    c.append(np.array((nan_inf + [0, 0x8000, 0x3C00]) * 1500, np.uint16))  # NaN / Inf among zeros
    c.append(np.zeros(9000, np.uint16))                                  # all +0
    c.append(np.full(9000, 0x8000, np.uint16))                           # all -0
    c.append(words_of(rng.standard_normal(5000) + 4.0, ft))              # no zeros
    c.append(rng.integers(0, 1 << 16, 70001, dtype=np.uint16))           # full range: nothing free, nothing elided
    c.append(all_but((17, 200), ft))                                     # exactly two free symbols
    c.append(all_but((99,), ft))                                         # exactly one free symbol
    sub = np.arange(1, 0x100, dtype=np.uint16) if ft == S.F16S else np.arange(1, 0x80, dtype=np.uint16)
    c.append(np.concatenate([sub, sub | 0x8000, np.zeros(300, np.uint16), np.full(300, 0x8000, np.uint16)]))
    c.append(np.concatenate([words_of(rng.uniform(1, 2, 3000), ft), np.zeros(100, np.uint16),
                             np.full(50, 0x8000, np.uint16)]))          # E+ = 0, a zero's natural symbol
    return c


def scalar_archive(w, ft, pb, checksum):
    """Types 5 / 6 word by word with Python integers."""
    n = len(w)
    ws = [int(x) for x in w]
    coded = [(x >> 8) if ft == S.F16S else (x >> 7) & 0xFF for x in ws]
    stored = [(x & 0xFF) if ft == S.F16S else ((x << 1) | (x >> 15)) & 0xFF for x in ws]
    used = sorted({c for x, c in zip(ws, coded) if x not in (0, 0x8000)})
    free = [s for s in range(256) if s not in used]
    elide = len(free) >= 2
    sym, plane, kept = [], bytearray(), []
    for x, c, b in zip(ws, coded, stored):
        if elide and x == 0:
            sym.append(free[0])
        elif elide and x == 0x8000:
            sym.append(free[1])
        else:
            sym.append(c)
            plane.append(b)
        kept.append(0 if elide and x in (0, 0x8000) else 1)
    nb = -(-n // 4096)
    table, run = [], 0
    for k in range(nb):
        table.append(run)
        run += sum(kept[4096 * k:4096 * (k + 1)])
    table += [0] * (_r(nb, 4) - nb)
    cks = 0
    if checksum:
        for b in b"".join(x.to_bytes(2, "little") for x in ws)[:n]:
            cks ^= b
    esc = free[0] | (free[1] << 8) | (1 << 16) if elide else 0
    hdr = [(0xF00F << 16) | 1, n, ft | (int(checksum) << 4), cks, len(plane), esc, 0, 0]
    body = b"".join(x.to_bytes(4, "little") for x in hdr + table) + bytes(plane) + bytes(_r(len(plane), 16) - len(plane))
    return np.concatenate([np.frombuffer(body, np.uint8), O.ans_encode(np.array(sym, np.uint8), pb)])


@pytest.mark.parametrize("ft", [S.F16S, S.BF16S])
@pytest.mark.parametrize("n", [0, 1, 15, 16, 17, 4095, 4096, 4097, 9000])
def test_archive_equals_scalar_statement(ft, n):
    for k, w in enumerate((relu_words(n, ft, n), masked_words(n, ft, n + 1))):
        for pb, checksum in ((9, False), (10, True), (11, False)):
            got = S.compress(w, ft, pb, checksum)
            assert np.array_equal(got, scalar_archive(w, ft, pb, checksum)), (ft, n, k, pb, checksum)
            assert got.size == S.extra_bytes(got) + O.ans_info(S.ans_part(got))["size"]


@pytest.mark.parametrize("ft", [S.F16S, S.BF16S])
def test_full_range_round_trip_is_bit_exact(ft):
    rng = np.random.default_rng(ft)
    w = np.concatenate([rng.integers(0, 1 << 16, 50000, dtype=np.uint16), np.zeros(3000, np.uint16),
                        np.full(3000, 0x8000, np.uint16)])
    for pb in (9, 10, 11):
        a = S.compress(w, ft, pb, True)
        hd = S.info(a)
        assert (hd["float_type"], hd["size"], hd["has_checksum"], hd["esc"]) == (ft, w.size, True, 0)
        rc, out = S.decompress(a, ft, pb, verify_checksum=True)
        assert rc == O.OK and np.array_equal(out, w)
    assert S.decompress(S.compress(w, ft), F := (S.BF16S if ft == S.F16S else S.F16S))[0] == O.ERR_BAD_FLOAT_TYPE


@pytest.mark.parametrize("ft", [S.F16S, S.BF16S])
def test_escape_rule_edges(ft):
    neg = 0x80 if ft == S.F16S else 0
    cases = edge_corpus(ft)
    for i, w in enumerate(cases):
        a = S.compress(w, ft, 10, True)
        rc, out = S.decompress(a, ft, 10, verify_checksum=True)
        assert rc == O.OK and np.array_equal(out, w), i
    # all +0 / all -0: symbols 0 and 1 are the escapes, nothing is stored
    for w in (np.zeros(9000, np.uint16), np.full(9000, 0x8000, np.uint16)):
        hd = S.info(S.compress(w, ft))
        assert (hd["esc"], hd["stored"]) == (0 | 1 << 8 | 1 << 16, 0)
    # no zeros: the escapes are still chosen, every word stores its byte
    w = words_of(np.random.default_rng(1).standard_normal(5000) + 4.0, ft)
    hd = S.info(S.compress(w, ft))
    assert hd["esc"] >> 16 == 1 and hd["stored"] == w.size
    # exactly two free symbols: they are E+ and E-; exactly one: nothing is elided
    w = all_but((17, 200), ft)
    assert S.info(S.compress(w, ft))["esc"] == 17 | 200 << 8 | 1 << 16
    assert S.info(S.compress(w, ft))["stored"] == 254
    w = all_but((99,), ft)
    hd = S.info(S.compress(w, ft))
    assert (hd["esc"], hd["stored"]) == (0, w.size)
    # subnormals share the natural symbol of +-0, so E+ / E- are other symbols
    sub = np.arange(1, 0x80, dtype=np.uint16)
    w = np.concatenate([sub, sub | 0x8000, np.zeros(30, np.uint16), np.full(30, 0x8000, np.uint16)])
    ep, em = S.escapes(w, ft)
    assert 0 not in (ep, em) and neg not in (ep, em)
    a = S.compress(w, ft)
    assert np.array_equal(S.decompress(a, ft)[1], w)
    # E+ equal to a zero's natural symbol
    w = np.concatenate([words_of(np.random.default_rng(2).uniform(1, 2, 3000), ft), np.zeros(10, np.uint16),
                        np.full(10, 0x8000, np.uint16)])
    assert S.escapes(w, ft)[0] == 0
    assert np.array_equal(S.decompress(S.compress(w, ft), ft)[1], w)


def test_stored_archives_are_reproduced():
    g = np.load(GOLD)
    names = sorted({k.rsplit("/", 1)[0] for k in g.files})
    assert len(names) >= 10
    for name in names:
        ft = int(name.split("/")[1])
        w = g[f"{name}/in"]
        for pb in (9, 10, 11):
            want = g[f"{name}/pb{pb}"]
            assert np.array_equal(S.compress(w, ft, pb, True), want), (name, pb)
            rc, out = S.decompress(want, ft, pb, verify_checksum=True)
            assert rc == O.OK and np.array_equal(out, w)
    kinds = {(int(n.split("/")[1]), S.info(g[f"{n}/pb10"])["esc"] != 0, S.info(g[f"{n}/pb10"])["size"] == 0)
             for n in names}
    for ft in (S.F16S, S.BF16S):
        assert {(ft, True, False), (ft, False, False), (ft, True, True)} <= kinds


@pytest.mark.parametrize("ft,limit", [(S.F16S, 0.50), (S.BF16S, 0.45)])
def test_relu_ratio(ft, limit):
    w = relu_words(1 << 20, ft, 4)
    a = S.compress(w, ft, 10)
    assert a.size / w.nbytes <= limit, a.size / w.nbytes
    assert a.size < O.float_compress(O.F16 if ft == S.F16S else O.BF16, w, 10).size


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
    assert top == _largest_nonzero(lambda n: L.dgb_float_max_compressed_size(capi.FLOAT16_SPARSE, n) != 0)
    for ft in (capi.FLOAT16_SPARSE, capi.BFLOAT16_SPARSE):
        for n in [0, 1, 2, 15, 16, 17, 4095, 4096, 4097, 16385, 1 << 20, 123456789, top - 1, top, top + 1,
                  top + 4096, 0xFFFFFFFF]:
            assert L.dgb_float_max_compressed_size(ft, n) == S.max_compressed_size(n), (ft, n)
    assert S.max_compressed_size(top + 1) == 0
    # the other float types keep their values
    for ft in (O.F16, O.BF16, O.F32):
        for n in (0, 1, 4097, 1 << 24):
            assert L.dgb_float_max_compressed_size(ft, n) == O.float_max_compressed_size(ft, n)


def test_sparse_keyword_refusals():
    from dietgpu_b200 import ops

    t32, t16 = torch.zeros(4), torch.zeros(4, dtype=torch.float16)
    with pytest.raises(ValueError):
        ops.compress_data(False, [t16], sparse=True)
    with pytest.raises(ValueError):
        ops.max_float_compressed_size(t32, 10, sparse=True)
    with pytest.raises(ValueError):
        ops.max_float_compressed_output_size([torch.zeros(4, dtype=torch.float64)], sparse=True)
    with pytest.raises(ValueError):
        ops.decompress_data_simple(False, [torch.zeros(64, dtype=torch.uint8)], sparse=True)
    from dietgpu_b200 import capi

    assert ops.max_float_compressed_size(t16, 5000, sparse=True) == \
        capi.lib().dgb_float_max_compressed_size(capi.FLOAT16_SPARSE, 5000)
    assert ops.max_float_compressed_output_size([torch.zeros(9, dtype=torch.bfloat16)], sparse=True)[1] == \
        capi.lib().dgb_float_max_compressed_size(capi.BFLOAT16_SPARSE, 9)
