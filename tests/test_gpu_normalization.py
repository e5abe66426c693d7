"""Normalisation and statistics against the oracle on crafted histograms, and the precomputed-histogram
encode.

The pdf is defined through fp32 arithmetic (count and total converted to fp32, divided, scaled by 2^pb,
truncated; ans/GpuANSStatistics.cuh:178-341), so the reference here is the oracle's integer / fp32-exact
restatement, O.normalize -- a float64 reference would disagree with the format.  Members are built from
explicit histograms (the symbols repeated, then a seeded permutation) so that each one sits on an edge:
truncation exactly at an integer, one below and one above it; the add quirk onto absent low symbol ids;
the subtract branch with many pdf-1 symbols; totals above 2^24 where the fp32 conversion rounds.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from codec_helpers import (GUARD, SENTINEL, codec_options, guarded_decode, oracle_archive, roundtrip,
                           stored_pdf, to_dev_bytes)
from conftest import exp_bytes, zipf_bytes
from oracle import oracle as O

pytestmark = pytest.mark.gpu


def from_hist(h, seed):
    x = np.repeat(np.arange(256, dtype=np.uint8), np.asarray(h, np.int64))
    return np.random.default_rng(seed).permutation(x)


def crafted_histograms(pb):
    rng = np.random.default_rng(1000 + pb)
    hs = []
    # every symbol once plus one dominant symbol, totals 257 .. 10^6
    for k, total in enumerate(np.unique(np.geomspace(257, 10 ** 6, 24).astype(np.int64))):
        h = np.ones(256, np.int64)
        h[(37 * k) % 256] += total - 256
        hs.append(h)
    # uniform over m symbols
    for m in (1, 2, 3, 5, 7, 255, 256):
        for c in (1, 17, 4000):
            h = np.zeros(256, np.int64)
            h[rng.choice(256, m, replace=False)] = c
            hs.append(h)
    # mass only on ids >= 200: the leftover is added to symbol ids below it, which are all absent
    for _ in range(12):
        h = np.zeros(256, np.int64)
        h[200:] = rng.integers(0, 3000, 56)
        h[200 + rng.integers(0, 56)] += 1
        hs.append(h)
    # truncation edges: count * 2^pb / total an integer j, and one count on either side of it
    K = 1 << pb
    for k in (3, 37, 500):
        total = K * k
        for j in (1, 2, 5, 100):
            if 3 * j * k + 3 > total:
                continue
            h = np.zeros(256, np.int64)
            h[[11, 12, 13]] = [j * k, j * k + 1, max(j * k - 1, 1)]
            rest = total - int(h.sum())
            h[14:] += rng.multinomial(rest, np.full(242, 1 / 242))
            hs.append(h)
    # seeded heavy-tailed random histograms (many pdf-1 symbols at pb 9: the subtract branch)
    for _ in range(160):
        h = np.floor(rng.pareto(rng.uniform(0.6, 2.0), 256) * rng.uniform(1, 400)).astype(np.int64)
        h[rng.random(256) < rng.uniform(0, 0.7)] = 0
        if h.sum() == 0:
            h[rng.integers(0, 256)] = 1
        h = np.minimum(h, 50000)
        if h.sum() > 400000:
            h = np.maximum(h * 400000 // h.sum(), (h > 0).astype(np.int64))
        hs.append(h)
    return hs


@pytest.mark.parametrize("pb", [9, 10, 11])
def test_crafted_histograms_match_oracle(pb):
    hs = crafted_histograms(pb)
    members = [from_hist(h, 7 * i + pb) for i, h in enumerate(hs)]
    archives = roundtrip("bytes", members, pb, checksum=(pb == 11))
    for i, (h, x, arch) in enumerate(zip(hs, members, archives)):
        assert np.array_equal(O.histogram(x), h)
        want = O.normalize(h.astype(np.uint32), x.size, pb)
        assert np.array_equal(stored_pdf(arch, "bytes").astype(np.uint32), want), f"member {i}: pdf"


def big_histograms():
    """Members above 2^24 symbols, where (float)count and (float)total round."""
    out = []
    h = np.ones(256, np.int64)                # total 2^24 + 1, every symbol present
    h[5] = (1 << 24) + 1 - 255
    out.append(h)
    h = np.zeros(256, np.int64)               # total 2^24 + 3, one symbol with count total - 1
    h[0], h[255] = (1 << 24) + 2, 1
    out.append(h)
    h = np.zeros(256, np.int64)               # counts whose fp32 conversion rounds down (2^24 + 1) and up (2^24 + 3)
    h[1], h[2], h[3:6] = (1 << 24) + 1, (1 << 24) + 3, 1
    out.append(h)
    rng = np.random.default_rng(5)            # odd total above 2^24 spread over a heavy-tailed histogram
    h = np.floor(rng.pareto(1.1, 256) * 5000).astype(np.int64) + 1
    h[17] += (1 << 24) + 12345 - int(h.sum())
    out.append(h)
    return out


def test_members_above_2_24_symbols():
    hs = big_histograms()
    members = [from_hist(h, 90 + i) for i, h in enumerate(hs)]
    for pb in (9, 10, 11):
        archives = roundtrip("bytes", members, pb)
        for i, (h, x, arch) in enumerate(zip(hs, members, archives)):
            want = O.normalize(h.astype(np.uint32), x.size, pb)
            assert np.array_equal(stored_pdf(arch, "bytes").astype(np.uint32), want), f"pb {pb} member {i}: pdf"


# ---- precomputed histograms (histogram_dev) ----------------------------------------

def _hist_inputs():
    n = 20000  # equal sizes, multiple of 4: valid for the pointer, stride and split-size forms alike
    rng = np.random.default_rng(8)
    return [exp_bytes(n, 20, 1), zipf_bytes(n, 1.3, 2), np.full(n, 9, np.uint8),
            rng.integers(0, 256, n, dtype=np.uint8), exp_bytes(n, 2, 3)]


def _encode_with_histogram(api, arrays, hist, pb, checksum):
    """Encodes through dgb_ans_encode_{pointer,stride,split_size} with histogram_dev = hist [n][256];
    archives land in sentinel-prefilled rows; returns (matrix, host sizes)."""
    from dietgpu_b200 import capi

    L = capi.lib()
    n, size = len(arrays), arrays[0].size
    cols = L.dgb_ans_max_compressed_size(size)
    assert cols % 16 == 0
    row = cols + GUARD
    comp = torch.full((n, row), SENTINEL, dtype=torch.uint8, device="cuda")
    csz = torch.zeros(n, dtype=torch.int32, device="cuda")
    hdev = torch.from_numpy(np.ascontiguousarray(hist, np.uint32).view(np.int32)).cuda()
    tb = L.dgb_ans_encode_temp_bytes(n, size)
    temp = torch.empty(tb + 256, dtype=torch.uint8, device="cuda")
    tp = temp.data_ptr() + (-temp.data_ptr()) % 256
    st = torch.cuda.current_stream().cuda_stream
    if api == "pointer":
        ins = [(to_dev_bytes(a), a) for a in arrays]
        rc = L.dgb_ans_encode_pointer(tp, tb, pb, int(checksum), n, capi.ptr_array([t.data_ptr() for t, _ in ins]),
                                      capi.u32_array([size] * n), C.c_void_p(hdev.data_ptr()),
                                      capi.ptr_array([comp.data_ptr() + i * row for i in range(n)]),
                                      csz.data_ptr(), st)
    elif api == "stride":
        stride = size + 52
        host = np.zeros(n * stride, np.uint8)
        for i, a in enumerate(arrays):
            host[i * stride:i * stride + size] = a
        buf = to_dev_bytes(host)
        ins = [(buf, host)]
        rc = L.dgb_ans_encode_stride(tp, tb, pb, int(checksum), n, buf.data_ptr(), size, stride,
                                     C.c_void_p(hdev.data_ptr()), comp.data_ptr(), row, csz.data_ptr(), st)
    else:
        host = np.concatenate(arrays)
        flat = to_dev_bytes(host)
        ins = [(flat, host)]
        rc = L.dgb_ans_encode_split_size(tp, tb, pb, int(checksum), n, flat.data_ptr(), capi.u32_array([size] * n),
                                         C.c_void_p(hdev.data_ptr()), comp.data_ptr(), row, csz.data_ptr(), st)
    capi.check(rc, f"encode_{api}")
    hs = csz.cpu().tolist()
    for t, a in ins:
        assert np.array_equal(t.cpu().numpy(), a), "encode changed its input"
    for i, k in enumerate(hs):
        assert bool((comp[i, k:] == SENTINEL).all()), f"member {i}: bytes written beyond the archive size"
    return comp, hs


@pytest.mark.parametrize("opts", [{}, dict(encode_fused=1), dict(encode_canonical=1)],
                         ids=["defaults", "encode_fused", "encode_canonical"])
@pytest.mark.parametrize("api", ["pointer", "stride", "split_size"])
def test_precomputed_histogram(api, opts):
    # with histogram_dev the statistics pass skips the data entirely (checksum off) or only checksums it
    arrays = _hist_inputs()
    exact = np.stack([O.histogram(a) for a in arrays]).astype(np.uint32)
    ts = [to_dev_bytes(a) for a in arrays]
    with codec_options(**opts):
        for pb in (9, 10, 11):
            for checksum in (False, True):
                for label, hist in (("exact", exact), ("superset", exact + 1)):
                    comp, hs = _encode_with_histogram(api, arrays, hist, pb, checksum)
                    what = f"{api} pb {pb} checksum {checksum} {label} histogram"
                    for i, a in enumerate(arrays):
                        got = comp[i, :hs[i]].cpu().numpy()
                        want = O.ans_encode(a, pb, checksum, hist=hist[i])
                        if label == "exact":
                            # the archive equals the one encoded without a histogram
                            assert np.array_equal(want, oracle_archive("bytes", a, pb, checksum))
                        assert hs[i] == want.size, f"{what} member {i}: size"
                        if opts.get("encode_canonical"):
                            assert np.array_equal(got, want), f"{what} member {i}: bytes"
                        else:
                            O.assert_same_ans(got, want, f"{what} member {i}")
                    guarded_decode(False, [comp[i, :hs[i]] for i in range(len(arrays))], [a.size for a in arrays],
                                   torch.uint8, pb, checksum, ts, what)
