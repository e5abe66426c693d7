"""include/dietgpu_b200_device.cuh (warp / CTA level device API, SURVEY.md 8f-4; reference README.md:105).

Two vehicles, both built by build():
- tests/cpp/device_api_example.cu: example user kernels. A kernel that compresses the tile it holds in
  shared memory must write archives byte-identical to the CPU oracle's at probBits 9, 10 and 11, decodable
  by the library's own decoder (and by the reference where it was built); the device-level decoder must
  read library-written archives and refuse ones of another probBits.
- tests/cpp/device_api_probe.cu: one small kernel per entry point, so that each is pinned on its own:
  normalisation and the encoder table against O.normalize and the documented fields, the encoder's
  division-free arithmetic against integer division, each coded block against the oracle's single-block
  archive in both memory spaces, the decode LUT at 32, 96, 256 and 1024 threads, and the documented false
  returns of the LUT builder and the block decoder.
Every device output lands in a sentinel-filled buffer whose bytes past the data are read back.
"""
import ctypes as C
import functools
import os

import numpy as np
import pytest
import torch

from conftest import exp_bytes, zipf_bytes
from oracle import oracle as O
from test_gpu_normalization import crafted_histograms

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
PBS = (9, 10, 11)
S8, S16, S32 = 0xA5, 0xA5A5, 0xA5A5A5A5
TILE = 32768  # the example's largest tile: 8 warps x 4 KiB


def _load(name):
    path = os.path.join(HERE, "cpp", name)
    if not os.path.exists(path):
        pytest.fail(f"{path} missing: python -c 'import __graft_entry__ as g; g.build()'")
    return C.CDLL(path)


@functools.lru_cache(None)
def _lib():
    L = _load("libdevice_api_example.so")
    u32, vp = C.c_uint32, C.c_void_p
    L.example_tile_compress.restype = C.c_int
    L.example_tile_compress.argtypes = [vp, u32, u32, vp, u32, vp, C.c_int, vp]
    L.example_tile_decompress.restype = C.c_int
    L.example_tile_decompress.argtypes = [vp, u32, u32, vp, u32, vp, C.c_int, vp]
    return L


@functools.lru_cache(None)
def _probe():
    L = _load("libdevice_api_probe.so")
    u32, i32, vp = C.c_uint32, C.c_int, C.c_void_p
    for f, args in (("probe_normalise", [vp, vp, u32, u32, i32, vp, vp, vp, vp, vp]),
                    ("probe_encode_entry", [vp, vp, vp, u32, vp, vp]),
                    ("probe_block_encode", [i32, i32, u32, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
                    ("probe_block_decode", [i32, i32, u32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
                    ("probe_decode_lut", [i32, i32, u32, u32, vp, vp, vp, vp])):
        getattr(L, f).restype = i32
        getattr(L, f).argtypes = args
    for f, args in (("probe_archive_overhead", [u32]), ("probe_max_block_words", [i32]),
                    ("probe_out_guard", []), ("probe_lut_guard", [])):
        getattr(L, f).restype = u32
        getattr(L, f).argtypes = args
    return L


def _st():
    return torch.cuda.current_stream().cuda_stream


_SIGNED = {np.dtype(np.uint8): np.uint8, np.dtype(np.uint16): np.int16, np.dtype(np.uint32): np.int32,
           np.dtype(np.int32): np.int32}


def _dev(a):
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(_SIGNED[a.dtype]).copy()).cuda()


def _full(n, dtype, value):
    return _dev(np.full(n, value, dtype))


def _host(t, dtype):
    torch.cuda.synchronize()
    return t.cpu().numpy().view(dtype)


def _exclusive_cumsum(pdf):
    return (np.cumsum(pdf, dtype=np.int64) - pdf).astype(np.uint32)


def expected_entry(pdf, cdf, pb):
    """EncodeEntry {magic, pack} as the header documents it."""
    K = 1 << pb
    shift, magic, term = 0, 0, cdf
    if pdf > 1:
        shift = (pdf - 1).bit_length() - 1
        magic = -(-(1 << (32 + shift)) // pdf)
    elif pdf == 1:
        magic, term = 0xFFFFFFFF, cdf + K - 1
    return magic, (shift | ((K - pdf) << 5) | (term << 20)) & 0xFFFFFFFF


def expected_lut(pdf, pb):
    pdf = np.asarray(pdf, np.int64)
    sym = np.repeat(np.arange(256, dtype=np.int64), pdf)
    j = np.arange(1 << pb, dtype=np.int64) - np.repeat(np.cumsum(pdf) - pdf, pdf)
    return ((np.repeat(pdf, pdf) << 20) | (j << 8) | sym).astype(np.uint32)


# ---- example user kernels: whole tiles --------------------------------------------------------------

def _tile_compress(data, tile, pb):
    """The example's archives (one row per tile, sentinel past each archive checked), with the oracle's."""
    import dietgpu_b200 as dg

    L = _lib()
    total = data.size
    tiles = (total + tile - 1) // tile
    stride = dg.max_any_compressed_size(tile)
    d_in = torch.from_numpy(data).cuda()
    d_out = torch.full((tiles, stride), S8, dtype=torch.uint8, device="cuda")
    d_sz = torch.zeros(tiles + 1, dtype=torch.int32, device="cuda")
    assert L.example_tile_compress(d_in.data_ptr(), total, tile, d_out.data_ptr(), stride, d_sz.data_ptr(), pb,
                                   _st()) == 0
    torch.cuda.synchronize()
    assert np.array_equal(d_in.cpu().numpy(), data), "the example changed its input"
    sizes = d_sz.cpu().tolist()
    assert sizes[tiles] == 0, "size written past the last tile"
    rows = []
    for i in range(tiles):
        want = O.ans_encode(data[i * tile:(i + 1) * tile], pb)
        got = d_out[i].cpu().numpy()
        assert sizes[i] == want.size, f"pb {pb} tile {i}: size"
        assert np.array_equal(got[:sizes[i]], want), f"pb {pb} tile {i}: archive differs from the oracle"
        assert np.all(got[sizes[i]:] == S8), f"pb {pb} tile {i}: bytes written past the archive"
        rows.append(d_out[i, :sizes[i]])
    return d_out, stride, rows


def _tile_decompress(comp, stride, tiles, tile, pb):
    """tileDecompress<pb> of `tiles` rows: (ok per tile, output incl. one guard tile)."""
    L = _lib()
    d_back = torch.full(((tiles + 1) * tile,), S8, dtype=torch.uint8, device="cuda")
    d_ok = torch.full((tiles + 1,), 7, dtype=torch.int32, device="cuda")
    assert L.example_tile_decompress(comp.data_ptr(), stride, tiles, d_back.data_ptr(), tile, d_ok.data_ptr(), pb,
                                     _st()) == 0
    torch.cuda.synchronize()
    ok = d_ok.cpu().tolist()
    assert ok[tiles] == 7, "ok flag written past the last tile"
    return ok[:tiles], d_back.cpu().numpy()


def _reference_decodes(rows, data, tile, pb):
    from oracle import ref_lib

    outs = [torch.full((min(tile, data.size - i * tile),), S8, dtype=torch.uint8, device="cuda")
            for i in range(len(rows))]
    status = torch.zeros(len(rows), dtype=torch.uint8, device="cuda")
    sizes = torch.zeros(len(rows), dtype=torch.int32, device="cuda")
    assert ref_lib.RefCodec(64 << 20).ans_decode(rows, outs, status, sizes, pb=pb) == 0
    torch.cuda.synchronize()
    assert status.cpu().tolist() == [1] * len(rows), f"pb {pb}: the reference refused the example's archives"
    assert sizes.cpu().tolist() == [o.numel() for o in outs]
    assert np.array_equal(torch.cat(outs).cpu().numpy(), data), f"pb {pb}: reference decode"


def tile_roundtrip(data, tile, pb):
    """Example archives == oracle; decoded by the library and by tileDecompress."""
    import dietgpu_b200 as dg

    total = data.size
    tiles = (total + tile - 1) // tile
    comp, stride, rows = _tile_compress(data, tile, pb)
    outs = [torch.full((min(tile, total - i * tile),), S8, dtype=torch.uint8, device="cuda") for i in range(tiles)]
    dg.decompress_data(False, rows, outs, prob_bits=pb)
    assert np.array_equal(torch.cat(outs).cpu().numpy(), data), f"pb {pb}: library decode"
    ok, back = _tile_decompress(comp, stride, tiles, tile, pb)
    assert ok == [1] * tiles, f"pb {pb}: tileDecompress refused"
    assert np.array_equal(back[:total], data), f"pb {pb}: tileDecompress output"
    assert np.all(back[total:] == S8), f"pb {pb}: tileDecompress wrote past the data"
    return rows


@pytest.mark.parametrize("tile,total", [(32768, 32768 * 5 + 1234), (4096, 4096 * 3), (10000, 70001), (32768, 17)])
def test_user_kernel_archives_equal_oracle(tile, total):
    data = np.concatenate([zipf_bytes(total // 2, 1.1, 3), exp_bytes(total - total // 2, 30.0, 4)])
    for pb in PBS:
        tile_roundtrip(data, tile, pb)


def worst_case_block():
    """4096 bytes over symbols 1..255, 16 or 17 of each: next to 7 blocks of symbol 0 every one has pdf 1."""
    return np.random.default_rng(31).permutation(np.tile(np.arange(1, 256, dtype=np.uint8), 17)[:4096])


def _tile_cases():
    cases = {}
    for k in range(1, 9):  # 1 to 8 blocks: a ragged last block, and whole blocks at odd counts
        cases[f"blocks{k}_ragged"] = zipf_bytes(4096 * k - 97 * k, 1.2, 40 + k)
        if k & 1:
            cases[f"blocks{k}_whole"] = exp_bytes(4096 * k, 12.0, 50 + k)
    cases["worst_block"] = np.concatenate([np.zeros(4096 * 3, np.uint8), worst_case_block(),
                                           np.zeros(4096 * 4, np.uint8)])
    cases["one_symbol"] = np.full(4096 * 5 + 3, 200, np.uint8)
    cases["one_symbol_255_one_byte"] = np.full(1, 255, np.uint8)
    return cases


@pytest.mark.parametrize("name", sorted(_tile_cases()))
@pytest.mark.parametrize("pb", PBS)
def test_user_kernel_tile_edges(pb, name):
    data = _tile_cases()[name]
    rows = tile_roundtrip(data, TILE, pb)
    if name == "worst_block":
        p = O.parse_ans(rows[0].cpu().numpy())
        assert int(p["block_words"][3, 0]) & 0xFFFF == 256 * pb, "the pdf-1 block must cost probBits per byte"
        assert int(p["block_words"][3, 0]) & 0xFFFF <= _probe().probe_max_block_words(pb)


@pytest.mark.parametrize("pb", PBS)
def test_reference_decodes_user_kernel_archives(pb):
    from oracle import ref_lib

    if not ref_lib.available():
        pytest.skip("the reference was not built here (oracle/_ref)")
    cases = _tile_cases()
    for data in (np.concatenate([zipf_bytes(50000, 1.1, 3), exp_bytes(50001, 30.0, 4)]), cases["worst_block"],
                 cases["one_symbol"], cases["blocks3_ragged"]):
        _, _, rows = _tile_compress(data, TILE, pb)
        _reference_decodes(rows, data, TILE, pb)


def test_example_launchers_refuse_other_probbits():
    L = _lib()
    for pb in (0, 8, 12, 16):
        # refused before anything is launched, so null pointers are never read
        assert L.example_tile_compress(None, 4096, 4096, None, 8192, None, pb, _st()) != 0
        assert L.example_tile_decompress(None, 8192, 1, None, 4096, None, pb, _st()) != 0


def test_device_decoder_reads_library_archives():
    import dietgpu_b200 as dg

    parts = [zipf_bytes(TILE, 1.3, i) for i in range(4)] + [exp_bytes(9000, 10.0, 9), np.full(4097, 3, np.uint8)]
    ts = [torch.from_numpy(p).cuda() for p in parts]
    for pb in PBS:
        comp, sizes, _ = dg.compress_data(False, ts, prob_bits=pb)
        ok, back = _tile_decompress(comp, comp.size(1), len(parts), TILE, pb)
        assert ok == [1] * len(parts), f"pb {pb}: tileDecompress refused a library archive"
        for i, p in enumerate(parts):
            assert np.array_equal(back[i * TILE:i * TILE + p.size], p), f"pb {pb} member {i}"
            assert np.all(back[i * TILE + p.size:(i + 1) * TILE] == S8), f"pb {pb} member {i}: written past its size"
        # tileDecompress<PB> of an archive of another probBits: its pdf does not sum to 2^PB, every tile is
        # refused and nothing is written
        for other in PBS:
            if other != pb:
                ok, back = _tile_decompress(comp, comp.size(1), len(parts), TILE, other)
                assert ok == [0] * len(parts), f"pb {pb} archive accepted by tileDecompress<{other}>"
                assert np.all(back == S8), f"pb {pb} archive in tileDecompress<{other}>: output written"


# ---- probe: normalisation and the encoder table -----------------------------------------------------

@pytest.mark.parametrize("pb", PBS)
def test_normalise_and_encode_table_match_oracle(pb):
    P = _probe()
    hs = [np.asarray(h, np.uint32) for h in crafted_histograms(pb)]
    nh, per = len(hs), 7  # seven histograms back to back in each CTA
    totals = np.array([int(h.sum()) for h in hs], np.uint32)
    d_counts, d_totals = _dev(np.concatenate(hs)), _dev(totals)
    g = 256  # one histogram's worth of guard after each output
    d_pdf, d_cdf = _full(nh * 256 + g, np.uint32, S32), _full(nh * 256 + g, np.uint32, S32)
    d_pdf16, d_tab = _full(nh * 256 + g, np.uint16, S16), _full(2 * (nh * 256 + g), np.uint32, S32)
    assert P.probe_normalise(d_counts.data_ptr(), d_totals.data_ptr(), nh, per, pb, d_pdf.data_ptr(),
                             d_cdf.data_ptr(), d_pdf16.data_ptr(), d_tab.data_ptr(), _st()) == 0
    pdf, cdf = _host(d_pdf, np.uint32), _host(d_cdf, np.uint32)
    pdf16, tab = _host(d_pdf16, np.uint16), _host(d_tab, np.uint32).reshape(-1, 2)
    for out, s in ((pdf, S32), (cdf, S32), (pdf16, S16), (tab, S32)):
        assert np.all(out[nh * 256:] == s), f"pb {pb}: written past the last histogram"
    for i, h in enumerate(hs):
        want = O.normalize(h, int(totals[i]), pb)
        r = slice(i * 256, (i + 1) * 256)
        assert np.array_equal(pdf[r], want), f"pb {pb} histogram {i}: blockNormalizedPdf"
        assert np.array_equal(pdf16[r].astype(np.uint32), want), f"pb {pb} histogram {i}: blockBuildEncodeTable pdf"
        wcdf = _exclusive_cumsum(want)
        assert np.array_equal(cdf[r], wcdf), f"pb {pb} histogram {i}: cdf"
        wtab = np.array([expected_entry(int(p), int(c), pb) for p, c in zip(want, wcdf)], np.uint32)
        assert np.array_equal(tab[r], wtab), f"pb {pb} histogram {i}: encode table"


def _encode_entries(pdf, cdf, pb):
    P = _probe()
    n = len(pdf)
    d_out = _full(2 * n + 64, np.uint32, S32)
    assert P.probe_encode_entry(_dev(np.asarray(pdf, np.uint32)).data_ptr(), _dev(np.asarray(cdf, np.uint32)).data_ptr(),
                                _dev(np.full(n, pb, np.int32)).data_ptr(), n, d_out.data_ptr(), _st()) == 0
    out = _host(d_out, np.uint32)
    assert np.all(out[2 * n:] == S32)
    return out[:2 * n].reshape(n, 2)


@pytest.mark.parametrize("pb", PBS)
def test_encoder_arithmetic_is_exact(pb):
    """For every pdf, makeEncodeEntry's {magic, pack} drives warpEncodeBlock's threshold and state update:
    thr = kmp * -(2^(31-pb)) + 2^31 must be pdf << (31 - pb), and for every state the coder can hold
    before the update, [min(2^15, thr >> 16), thr), the division-free update must equal
    (x // pdf) * 2^pb + x % pdf + cdf."""
    K = 1 << pb
    pdfs = np.arange(1, K + 1, dtype=np.int64)
    cdfs = (pdfs * 7919) % (K - pdfs + 1)  # any cdf with cdf + pdf <= 2^pb
    ent = _encode_entries(pdfs, cdfs, pb).astype(np.int64)
    rng = np.random.default_rng(pb)
    M = 1 << 12
    for pdf, cdf, (magic, pack) in zip(pdfs.tolist(), cdfs.tolist(), ent.tolist()):
        assert (magic, pack) == expected_entry(pdf, cdf, pb), f"pb {pb} pdf {pdf}: entry"
        shift, kmp, term = pack & 31, (pack >> 5) & 0xFFF, pack >> 20
        thr = (kmp * ((-(1 << (31 - pb))) & 0xFFFFFFFF) + (1 << 31)) & 0xFFFFFFFF
        assert thr == pdf << (31 - pb), f"pb {pb} pdf {pdf}: emit threshold"
        lo, hi = min(1 << 15, thr >> 16), thr
        k_lo, k_hi = -(-lo // pdf), (hi - 1) // pdf
        ks = np.concatenate([np.arange(k_lo, min(k_lo + M, k_hi + 1)), np.arange(max(k_hi - M, k_lo), k_hi + 2)])
        x = np.concatenate([ks * pdf - 1, ks * pdf, rng.integers(lo, hi, M), [lo, hi - 1]]).astype(np.uint64)
        x = np.unique(x[(x >= lo) & (x < hi)])
        div = ((x * np.uint64(magic)) >> np.uint64(32)) >> np.uint64(shift)
        got = (div * np.uint64(kmp) + x + np.uint64(term)) & np.uint64(0xFFFFFFFF)
        want = (x // np.uint64(pdf)) * np.uint64(K) + x % np.uint64(pdf) + np.uint64(cdf)
        bad = np.nonzero(got != want)[0]
        assert bad.size == 0, f"pb {pb} pdf {pdf}: state {int(x[bad[0]])} -> {int(got[bad[0]])} != {int(want[bad[0]])}"
        assert int(want.max()) < 1 << 31


# ---- probe: block coder against the oracle's single-block archives ----------------------------------

BLOCK_LENGTHS = list(range(1, 97)) + [127, 128, 129, 511, 512, 513, 4063, 4064, 4065, 4095, 4096]


@functools.lru_cache(None)
def block_cases(pb):
    """[(name, block bytes, oracle archive of the member whose first block it is)]."""
    rng = np.random.default_rng(500 + pb)
    out = []

    def add(name, block, member=None, hist=None):
        member = block if member is None else member
        out.append((name, block, O.ans_encode(member, pb, hist=hist)))

    for n in BLOCK_LENGTHS:
        add(f"len{n}", zipf_bytes(n, 1.1, n) if n % 2 else exp_bytes(n, 8.0, n))
    for s in (0, 255, 77):
        for n in (1, 33, 4096):
            add(f"one_symbol_{s}_{n}", np.full(n, s, np.uint8))
    for n in (2, 1000, 4096):
        add(f"two_symbols_{n}", rng.choice(np.array([3, 250], np.uint8), n, p=[0.9, 0.1]))
    add("uniform256", rng.permutation(np.repeat(np.arange(256, dtype=np.uint8), 16)))
    for n in (777, 4096):
        add(f"ids_ge_200_{n}", rng.integers(200, 256, n).astype(np.uint8))
    # coded under a superset histogram: every symbol present in the pdf, only two in the block
    two = rng.choice(np.array([9, 10], np.uint8), 3000)
    add("two_symbols_superset_hist", two, hist=O.histogram(two) + 1)
    # the first block of a member whose other 7 blocks are symbol 0: all 4096 bytes have pdf 1
    worst = worst_case_block()
    add("worst_case", worst, member=np.concatenate([worst, np.zeros(7 * 4096, np.uint8)]))
    return out


def _oracle_block(arch):
    p = O.parse_ans(arch)
    bw = int(p["block_words"][0, 0])
    return dict(pdf=p["pdf"], states=p["states"][0], words=p["streams"][0], n=bw >> 16, nw=bw & 0xFFFF)


def probe_encode(pb, smem, blocks, pdfs):
    """warpEncodeBlock of each block: (word counts, states [nb, 32], [words of each block], [tail of each])."""
    P = _probe()
    nb = len(blocks)
    ns = np.array([b.size for b in blocks], np.uint32)
    in_off = np.concatenate([[0], np.cumsum(ns)[:-1]]).astype(np.uint32)
    w_off = np.concatenate([[0], np.cumsum(ns + 8)[:-1]]).astype(np.uint32)
    w_total = int((ns + 8).sum())
    data = np.concatenate(blocks)
    d_in = _dev(data)
    d_words = _full(w_total + 64, np.uint16, S16)
    d_nw = _full(nb + 8, np.uint32, S32)
    d_states = _full(32 * (nb + 1), np.uint32, S32)
    assert P.probe_block_encode(pb, int(smem), nb, d_in.data_ptr(), _dev(in_off).data_ptr(), _dev(ns).data_ptr(),
                                _dev(np.concatenate(pdfs).astype(np.uint16)).data_ptr(), d_words.data_ptr(),
                                _dev(w_off).data_ptr(), d_nw.data_ptr(), d_states.data_ptr(), _st()) == 0
    words, nw, states = _host(d_words, np.uint16), _host(d_nw, np.uint32), _host(d_states, np.uint32)
    assert np.array_equal(_host(d_in, np.uint8), data), "warpEncodeBlock changed its input"
    assert np.all(words[w_total:] == S16) and np.all(nw[nb:] == S32) and np.all(states[32 * nb:] == S32), \
        "written past the last block"
    got = [words[o:o + n + 8] for o, n in zip(w_off.tolist(), ns.tolist())]
    return nw[:nb], states[:32 * nb].reshape(nb, 32), got


def probe_decode(pb, smem, blocks, pdfs, states, streams, offsets=None, counts=None):
    """warpDecodeBlock of each block: (ok [nb, 32], [decoded bytes + guard of each block]).
    streams[b] is placed whole; the decoder gets streams[b][offsets[b]:] and counts[b] words."""
    P = _probe()
    G = P.probe_out_guard()
    nb = len(blocks)
    ns = np.array([b.size for b in blocks], np.uint32)
    lens = np.array([s.size for s in streams], np.int64)
    s_base = np.concatenate([[0], np.cumsum(lens + 8)[:-1]]).astype(np.int64)  # 8 spare words between streams
    offsets = np.zeros(nb, np.int64) if offsets is None else np.asarray(offsets, np.int64)
    counts = lens if counts is None else np.asarray(counts, np.int64)
    assert np.all(offsets + counts <= lens + 8)
    flat = np.zeros(int((lens + 8).sum()) + 8, np.uint16)
    for b, s in zip(s_base.tolist(), streams):
        flat[b:b + s.size] = s
    o_off = np.concatenate([[0], np.cumsum(ns + G)[:-1]]).astype(np.uint32)
    o_total = int((ns + G).sum())
    d_out = _full(o_total + 64, np.uint8, S8)
    d_ok = _full(32 * (nb + 1), np.uint32, S32)
    assert P.probe_block_decode(pb, int(smem), nb, _dev(np.concatenate(pdfs).astype(np.uint16)).data_ptr(),
                                _dev(np.concatenate(states).astype(np.uint32)).data_ptr(), _dev(flat).data_ptr(),
                                _dev((s_base + offsets).astype(np.uint32)).data_ptr(),
                                _dev(counts.astype(np.uint32)).data_ptr(), _dev(ns).data_ptr(), d_out.data_ptr(),
                                _dev(o_off).data_ptr(), d_ok.data_ptr(), _st()) == 0
    out, ok = _host(d_out, np.uint8), _host(d_ok, np.uint32)
    assert np.all(out[o_total:] == S8) and np.all(ok[32 * nb:] == S32), "written past the last block"
    return ok[:32 * nb].reshape(nb, 32), [out[o:o + n + G] for o, n in zip(o_off.tolist(), ns.tolist())]


@pytest.mark.parametrize("smem", [True, False], ids=["shared", "global"])
@pytest.mark.parametrize("pb", PBS)
def test_blocks_match_oracle(pb, smem):
    cases = block_cases(pb)
    ref = [_oracle_block(a) for _, _, a in cases]
    blocks = [b for _, b, _ in cases]
    for (name, b, _), r in zip(cases, ref):
        assert r["n"] == b.size, name
    mbw = _probe().probe_max_block_words(pb)
    nw, states, words = probe_encode(pb, smem, blocks, [r["pdf"] for r in ref])
    for i, ((name, b, _), r) in enumerate(zip(cases, ref)):
        what = f"pb {pb} {'shared' if smem else 'global'} {name}"
        assert int(nw[i]) == r["nw"], f"{what}: word count {int(nw[i])} != {r['nw']}"
        assert int(nw[i]) <= mbw, f"{what}: more words than maxBlockWords"
        assert np.array_equal(states[i], r["states"]), f"{what}: lane states"
        assert np.array_equal(words[i][:r["nw"]], r["words"]), f"{what}: words"
        assert np.all(words[i][r["nw"]:] == S16), f"{what}: written past the block's words"
        if name == "worst_case":
            assert r["nw"] == 256 * pb and r["nw"] + 8 <= mbw
    ok, outs = probe_decode(pb, smem, blocks, [r["pdf"] for r in ref], [r["states"] for r in ref],
                            [r["words"] for r in ref])
    for i, ((name, b, _), o) in enumerate(zip(cases, outs)):
        what = f"pb {pb} {'shared' if smem else 'global'} {name}"
        assert ok[i].tolist() == [1] * 32, f"{what}: decoder returned {ok[i].tolist()}"
        assert np.array_equal(o[:b.size], b), f"{what}: decoded bytes"
        assert np.all(o[b.size:] == S8), f"{what}: written past n"


@pytest.mark.parametrize("smem", [True, False], ids=["shared", "global"])
@pytest.mark.parametrize("pb", PBS)
def test_block_decoder_rejects_inconsistent_streams(pb, smem):
    """warpDecodeBlock's false: every lane returns it, and nothing is written past n."""
    cases = {name: (b, _oracle_block(a)) for name, b, a in block_cases(pb)}
    sel = []  # (label, block, oracle block, stream placed, decoder's offset into it, word count, lane + 1, accept)
    for name in ("len4096", "len4065", "len513", "ids_ge_200_777", "two_symbols_4096", "worst_case"):
        b, r = cases[name]
        assert r["nw"] > 0, name
        junk = np.concatenate([np.arange(0x1111, 0x1119, dtype=np.uint16), r["words"]])
        sel.append((f"{name} control", b, r, r["words"], 0, r["nw"], None, True))
        # 8 extra leading words: the decoder pops from the end, so the states still come out right and only
        # the word count can tell
        sel.append((f"{name} 8 leading words", b, r, junk, 0, r["nw"] + 8, None, False))
        sel.append((f"{name} numWords - 1", b, r, r["words"], 0, r["nw"] - 1, None, False))
    for name in ("one_symbol_0_4096", "one_symbol_255_33", "one_symbol_77_1"):
        b, r = cases[name]
        assert r["nw"] == 0
        sel.append((f"{name} control", b, r, r["words"], 0, 0, None, True))
        # no words at all: only the final-state check can tell
        for lane in (0, 13, 31):
            sel.append((f"{name} lane {lane} state + 1", b, r, r["words"], 0, 0, lane, False))
    states = []
    for label, b, r, s, off, cnt, lane, _ in sel:
        st = r["states"].copy()
        if lane is not None:
            st[lane] += 1
        states.append(st)
    ok, outs = probe_decode(pb, smem, [x[1] for x in sel], [x[2]["pdf"] for x in sel], states,
                            [x[3] for x in sel], [x[4] for x in sel], [x[5] for x in sel])
    for i, (label, b, r, s, off, cnt, lane, accept) in enumerate(sel):
        what = f"pb {pb} {'shared' if smem else 'global'} {label}"
        assert ok[i].tolist() == [int(accept)] * 32, f"{what}: lanes returned {ok[i].tolist()}"
        assert np.all(outs[i][b.size:] == S8), f"{what}: written past n"
        if accept:
            assert np.array_equal(outs[i][:b.size], b), f"{what}: decoded bytes"


# ---- probe: decode LUT --------------------------------------------------------------------------------

def lut_pdfs(pb):
    """[(label, u16 pdf, valid)]: crafted pdfs that sum to 2^pb and ones that do not."""
    K = 1 << pb
    hs = crafted_histograms(pb)
    good = [(f"crafted {i}", O.normalize(hs[i], int(hs[i].sum()), pb)) for i in range(0, len(hs), 9)]
    for s in (0, 128, 255):
        p = np.zeros(256, np.uint32)
        p[s] = K  # pdf = 2^pb: bit 31 of the LUT entry at pb 11
        good.append((f"single symbol {s}", p))
    good.append(("uniform", np.full(256, K // 256, np.uint32)))
    p = np.zeros(256, np.uint32)
    p[200:] = 1
    p[255] += K - 56
    good.append(("ids >= 200", p))
    base = good[0][1]
    short, over = base.copy(), base.copy()
    short[np.argmax(short)] -= 1
    over[np.argmax(over)] += 1
    h = hs[1]
    bad = [("sum 2^pb - 1", short), ("sum 2^pb + 1", over),
           ("pb - 1 archive", O.normalize(h, int(h.sum()), pb - 1)), ("all zero", np.zeros(256, np.uint32))]
    # interleaved, so that CTAs build valid and refused LUTs back to back
    out = []
    for i, (l, p) in enumerate(good):
        out.append((l, p, True))
        if i < len(bad):
            out.append(bad[i] + (False,))
    return out


@pytest.mark.parametrize("threads", [32, 96, 256, 1024])
@pytest.mark.parametrize("pb", PBS)
def test_decode_lut(pb, threads):
    P = _probe()
    K, per = 1 << pb, 4
    slot = K + P.probe_lut_guard()
    cases = lut_pdfs(pb)
    while len(cases) % per:
        cases.append(cases[0])
    n = len(cases)
    pdf = np.concatenate([p for _, p, _ in cases]).astype(np.uint16)
    d_lut = _full(n * slot + 64, np.uint32, S32)
    d_ret = _full(n * threads + 64, np.uint32, S32)
    assert P.probe_decode_lut(pb, threads, n // per, per, _dev(pdf).data_ptr(), d_lut.data_ptr(), d_ret.data_ptr(),
                              _st()) == 0
    lut, ret = _host(d_lut, np.uint32), _host(d_ret, np.uint32)
    assert np.all(lut[n * slot:] == S32) and np.all(ret[n * threads:] == S32)
    for i, (label, p, valid) in enumerate(cases):
        what = f"pb {pb} THREADS {threads} {label}"
        assert ret[i * threads:(i + 1) * threads].tolist() == [int(valid)] * threads, f"{what}: return values"
        got = lut[i * slot:(i + 1) * slot]
        if valid:
            assert int(p.sum()) == K
            assert np.array_equal(got[:K], expected_lut(p, pb)), f"{what}: LUT"
            assert np.all(got[K:] == S32), f"{what}: written past 2^pb"
        else:
            assert np.all(got == S32), f"{what}: refused LUT written"


def test_probe_refuses_unsupported_arguments():
    P = _probe()
    # refused before anything is launched, so null pointers are never read
    for pb in (8, 12):
        assert P.probe_block_encode(pb, 0, 1, *([None] * 8), _st()) != 0
        assert P.probe_block_decode(pb, 0, 1, *([None] * 9), _st()) != 0
        assert P.probe_decode_lut(pb, 256, 1, 1, None, None, None, _st()) != 0
        assert P.probe_normalise(None, None, 1, 1, pb, None, None, None, None, _st()) != 0
    for threads in (0, 64, 128, 512):
        assert P.probe_decode_lut(10, threads, 1, 1, None, None, None, _st()) != 0
    assert P.probe_decode_lut(10, 256, 1, 5, None, None, None, _st()) != 0


# ---- layout constants -----------------------------------------------------------------------------------

def test_layout_constants():
    P = _probe()
    for nb in list(range(0, 300)) + [4095, 4096, 4097, 65535, 65536, 1 << 20]:
        assert P.probe_archive_overhead(nb) == O.ans_overhead(nb), f"archiveOverhead({nb})"
    for pb in PBS:
        # a block of 4096 pdf-1 symbols costs probBits bits each: 256 * pb words, padded to 8 words
        assert P.probe_max_block_words(pb) == 256 * pb + 8
