"""The sparse fp32 codec (float type 8) on the GPU, pinned to the CPU restatement in tests/sparse32_oracle.py.

  - an edge corpus (sizes 0 .. 300000 at word offsets 0..3, zero runs across block and 16 B boundaries, blocks of only
    zeros next to blocks without any, NaN / Inf / denormals, every edge of the escape rule) at prob bits 9, 10 and 11,
    with and without checksum, through a guard-banded round trip (no byte outside the archive or the output changes);
  - a member whose block boundaries fall on every residue of both stored planes, byte for byte against the
    restatement in the default and the canonical coder: a warp that stored a whole 16 B vector at its segment's end
    would overwrite the neighbouring block's bytes;
  - both table formats, the canonical coder (byte-identical archives), 4- and 8-warp decoders, and the option values
    that select kernels the sparse kinds do not have (they run the defaults); torch.profiler confirms that every
    type-8 instantiation runs and that no other exists;
  - the restatement's archives decoded by the GPU, the pointer / split-size / simple forms, the header query, the
    archive mover, graph capture at 6 and 130 members, wrong-type pairings;
  - 64 x 1 Mi ReLU members (every pdf and archive) and the largest member the format allows;
  - three members through the C++ compatibility header (tests/cpp/sparse32_roundtrip.cu).
"""
import hashlib
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import sparse32_oracle as S
from codec_helpers import GUARD, SENTINEL, assert_guard_intact, codec_options, guarded_out
from multirank import run_ranks
from oracle import oracle as O
from test_oracle_sparse32 import edge_corpus, relu_words, segment_boundary_member

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CORPUS = edge_corpus()
OFFSETS = [i % 4 for i in range(len(CORPUS))]

_ORACLE = {}


def oracle_archive(w, pb, checksum=False):
    """The CPU restatement's archive, cached per (prob bits, checksum flag, member)."""
    w = np.ascontiguousarray(w, np.uint32)
    key = (pb, bool(checksum), w.size, hashlib.blake2b(w.tobytes(), digest_size=16).digest())
    if key not in _ORACLE:
        a = S.compress(w, pb, checksum)
        a.setflags(write=False)
        _ORACLE[key] = a
    return _ORACLE[key]


def _i32(t):
    return t.view(torch.int32)


def _t(w):
    return torch.from_numpy(np.ascontiguousarray(w).view(np.int32).copy()).view(torch.float32).cuda()


def placed_inputs(arrays, offsets):
    """float32 device tensors holding `arrays`, each `offsets[i]` words into its own allocation."""
    ts = []
    for a, off in zip(arrays, offsets):
        full = np.concatenate([np.zeros(off, np.uint32), a]).view(np.int32)
        ts.append(torch.from_numpy(full.copy()).view(torch.float32).cuda()[off:])
    return ts


def guarded_compress(ts, checksum, pb):
    from dietgpu_b200 import ops

    n = len(ts)
    _, cols = ops.max_float_compressed_output_size(ts, sparse=True)
    comp = torch.full((n, cols + GUARD), SENTINEL, dtype=torch.uint8, device="cuda")
    before = [_i32(t).clone() for t in ts]
    _, sizes, _ = ops.compress_data(True, ts, checksum, None, comp, None, prob_bits=pb, sparse=True)
    hs = sizes.cpu().tolist()
    for i, (t, b) in enumerate(zip(ts, before)):
        assert torch.equal(_i32(t), b), f"member {i}: compress changed its input"
    col = torch.arange(cols + GUARD, device="cuda")
    stray = (comp != SENTINEL) & (col[None, :] >= sizes[:, None].long())
    assert not bool(stray.any()), f"compress wrote beyond the archive size in rows {torch.nonzero(stray.any(1)).flatten().tolist()[:8]}"
    return comp, hs


def guarded_decode(rows, lengths, pb, checksum, expect, what):
    from dietgpu_b200 import ops

    n = len(rows)
    bufs, outs, spans = [], [], []
    for i in range(n):
        b, v, span = guarded_out(lengths[i], torch.float32, (5 * i + 3) % 8)
        bufs.append(b)
        outs.append(v)
        spans.append(span)
    status = torch.zeros(n, dtype=torch.uint8, device="cuda")
    osz = torch.zeros(n, dtype=torch.int32, device="cuda")
    ops.decompress_data(True, rows, outs, checksum, None, status, osz, prob_bits=pb, sparse=True)
    assert status.cpu().tolist() == [1] * n, f"{what}: status {status.cpu().tolist()}"
    assert osz.cpu().tolist() == list(lengths), f"{what}: decoded sizes"
    for i in range(n):
        assert torch.equal(_i32(outs[i]), _i32(expect[i])), f"{what}: member {i} decodes differently"
        assert_guard_intact(bufs[i], spans[i][0], spans[i][1], f"{what}: member {i}")


def roundtrip(arrays, pb=10, checksum=False, in_offsets=None, exact=False, decode_oracle=False):
    """Compress as one batch, compare every member with the restatement (byte for byte when `exact`), decode the
    archives (and, with `decode_oracle`, the restatement's) into guard-banded outputs.  Returns the archives."""
    ts = placed_inputs(arrays, in_offsets or [0] * len(arrays))
    comp, hs = guarded_compress(ts, checksum, pb)
    host = comp[:, :max(hs)].cpu().numpy()
    for i, a in enumerate(arrays):
        want = oracle_archive(a, pb, checksum)
        assert hs[i] == want.size and hs[i] % 16 == 0, f"member {i}: size {hs[i]} != oracle {want.size}"
        if exact:
            assert np.array_equal(host[i, :hs[i]], want), f"member {i}: archive bytes differ from the oracle's"
        else:
            S.assert_same(host[i, :hs[i]], want, f"member {i}")
    lengths = [a.size for a in arrays]
    guarded_decode([comp[i, :hs[i]] for i in range(len(ts))], lengths, pb, checksum, ts, "decode")
    if decode_oracle:
        rows = [torch.from_numpy(oracle_archive(a, pb, checksum).copy()).cuda() for a in arrays]
        guarded_decode(rows, lengths, pb, checksum, ts, "decode of the oracle's archives")
    return [host[i, :hs[i]] for i in range(len(arrays))]


@pytest.mark.parametrize("checksum", [False, True])
@pytest.mark.parametrize("pb", [9, 10, 11])
def test_edge_corpus_matches_oracle(pb, checksum):
    roundtrip(CORPUS, pb, checksum, OFFSETS, decode_oracle=(pb == 10))


@pytest.mark.parametrize("offset", [0, 1, 3])
def test_segment_boundaries_default_and_canonical(offset):
    """Every block boundary at every residue of the u8 plane (mod 16) and of the u16 plane (mod 8); neighbouring
    blocks are coded by different warps at the same time, so a store past a segment's end would show here."""
    w = segment_boundary_member()
    arrays = [w, relu_words(70001, 5), w[4096 * 3 + 5:]]
    for rep in range(2):
        got = roundtrip(arrays, 10, False, [offset, (offset + 1) % 4, offset])
        with codec_options(encode_canonical=1):
            canon = roundtrip(arrays, 10, False, [offset, (offset + 1) % 4, offset], exact=True)
        for a, b in zip(got, canon):
            n = S.extra_bytes(b)
            assert np.array_equal(a[:n], b[:n]), "default and canonical coders store different planes"


VARIANTS = [
    ("packed_table", dict(encode_wide_table=0), False),
    ("wide_table", dict(encode_wide_table=1), False),
    ("canonical", dict(encode_canonical=1), True),
    ("decode_warps4", dict(decode_warps=4), False),
    ("decode_warps8", dict(decode_warps=8), False),
    # kernels the sparse kinds do not have: the defaults run
    ("encode_fused", dict(encode_fused=1), False),
    ("decode_fused0", dict(decode_fused=0), False),
    ("stats_stage", dict(stats_stage=1), False),
    ("decode_warps20", dict(decode_warps=20), False),
]


@pytest.mark.parametrize("name,opts,exact", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_variant_matches_oracle(name, opts, exact):
    with codec_options(**opts):
        for pb in (9, 11):
            roundtrip(CORPUS, pb, pb == 11, OFFSETS, exact=exact)


def test_fallback_options_give_the_default_archives():
    arrays = CORPUS[:9]
    with codec_options(encode_canonical=1):
        want = roundtrip(arrays, exact=True)
    for opts in (dict(encode_fused=1), dict(stats_stage=1)):
        with codec_options(encode_canonical=1, **opts):
            got = roundtrip(arrays, exact=True)
        assert all(np.array_equal(a, b) for a, b in zip(got, want)), opts


def test_every_type8_instantiation_runs():
    # in a fresh process: in a long-lived one the GPU's timestamps drift against the host clock that bounds the
    # profiler's window, and every record of a window can fall outside it
    run_ranks(_every_type8_instantiation_runs, 1, backend="gloo")


def _every_type8_instantiation_runs(rank, world, dev):
    from torch.profiler import ProfilerActivity, profile

    from dietgpu_b200 import ops

    small = CORPUS[:8]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for pb in (9, 10, 11):
            for opts in ({}, dict(encode_wide_table=0), dict(encode_wide_table=1), dict(encode_canonical=1),
                         dict(decode_warps=4), dict(encode_fused=1, stats_stage=1, decode_fused=0, decode_warps=20)):
                with codec_options(**opts):
                    roundtrip(small, pb, in_offsets=[1] * len(small))
        comp, sizes, _ = ops.compress_data(True, [_t(CORPUS[5])], sparse=True)
        ops.pull_archives(True, [comp[0]], [torch.empty_like(comp[0])], float_dtype=torch.float32, sparse=True)
        torch.cuda.synchronize()
    names = {re.sub(r"\s", "", e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    want = ["pullArchivesSparse32Kernel", "statsFloatKernel<8>", "encodeKernel<8>"]
    want += [f"encodeKernelFast<{w},8>" for w in ("false", "true")]
    want += [f"decodeFusedKernel<8,{pb},{w}>" for pb in (9, 10, 11) for w in (4, 8)]
    missing = [w for w in want if not any(w in n for n in names)]
    assert not missing, f"not launched: {missing}; kernels seen: {sorted(n[:120] for n in names)}"
    extra = [n for n in names if re.search(r"(encodeFusedKernel|decodeKernel)<8,", n)
             or re.search(r"(statsFloatStagedKernel|planKernel)<8>", n) or re.search(r"decodeFusedKernel<8,\d+,20>", n)]
    assert not extra, extra
    # and the library holds no such instantiation at all
    so = os.path.join(ROOT, "dietgpu_b200", "libdietgpu_b200.so")
    syms = subprocess.run(["cuobjdump", "-symbols", so], capture_output=True, text=True).stdout
    if syms:
        dem = subprocess.run(["c++filt"], input=syms, capture_output=True, text=True).stdout
        bad = re.findall(r"(?:encodeFusedKernel<8,|statsFloatStagedKernel<8>|planKernel<8>|decodeKernel<8,|"
                         r"decodeFusedKernel<8, \d+, 20>)", dem)
        assert not bad, bad


# ---- operator layer ------------------------------------------------------------------------------

@pytest.mark.parametrize("checksum", [False, True])
def test_operators_pointer_split_simple(checksum):
    from dietgpu_b200 import ops

    members = [relu_words(n, 900 + n) for n in (1, 4097, 70001, 12345)]
    ts = [_t(w) for w in members]
    comp, sizes, _ = ops.compress_data(True, ts, checksum, sparse=True)
    hs = sizes.cpu().tolist()
    for i, w in enumerate(members):
        want = oracle_archive(w, 10, checksum)
        assert hs[i] == want.size
        S.assert_same(comp[i, :hs[i]].cpu().numpy(), want, f"member {i}")
    outs = [torch.empty_like(t) for t in ts]
    ops.decompress_data(True, [comp[i, :hs[i]] for i in range(len(ts))], outs, checksum, sparse=True)
    assert all(torch.equal(_i32(a), _i32(b)) for a, b in zip(ts, outs))
    flat = torch.cat(ts)
    split = torch.tensor([t.numel() for t in ts], dtype=torch.int32)
    archs, _, _ = ops.compress_data_split_size(True, flat, split, checksum, sparse=True)
    for i, w in enumerate(members):
        S.assert_same(archs[i].cpu().numpy(), oracle_archive(w, 10, checksum), f"split {i}")
    out = torch.full_like(flat, float("nan"))
    ops.decompress_data_split_size(True, archs, out, split, checksum, sparse=True)
    assert torch.equal(_i32(out), _i32(flat))
    simple = ops.compress_data_simple(True, ts, checksum, sparse=True)
    back = ops.decompress_data_simple(True, simple, checksum, sparse=True)
    assert all(b.dtype == torch.float32 for b in back)
    assert all(torch.equal(_i32(a), _i32(b)) for a, b in zip(ts, back))


def test_info_query_and_archive_mover():
    from dietgpu_b200 import capi, ops

    members = [relu_words(n, 40 + n) for n in (0, 33, 4097, 70001)]
    ts = [_t(w) for w in members]
    comp, sizes, _ = ops.compress_data(True, ts, True, sparse=True)
    hs = sizes.cpu().tolist()
    n = len(ts)
    ptrs = capi.ptr_array([comp[i].data_ptr() for i in range(n)])
    osz, oty, ock = (torch.zeros(n, dtype=torch.int32, device="cuda") for _ in range(3))
    tmp = torch.empty(4096, dtype=torch.uint8, device="cuda")
    capi.check(capi.lib().dgb_float_get_compressed_info(tmp.data_ptr(), 4096, ptrs, 0, n, osz.data_ptr(),
                                                        oty.data_ptr(), ock.data_ptr(),
                                                        torch.cuda.current_stream().cuda_stream), "info")
    assert oty.cpu().tolist() == [8] * n
    assert osz.cpu().tolist() == [t.numel() for t in ts]
    assert ock.cpu().tolist() == [S.info(oracle_archive(w, 10, True))["checksum"] for w in members]
    dst = torch.full_like(comp, 0x5A)
    nb = torch.zeros(n, dtype=torch.int32, device="cuda")
    ops.pull_archives(True, [comp[i] for i in range(n)], [dst[i] for i in range(n)], float_dtype=torch.float32,
                      out_bytes=nb, sparse=True)
    assert nb.cpu().tolist() == hs
    for i, h in enumerate(hs):
        assert torch.equal(dst[i, :h], comp[i, :h])
        assert bool((dst[i, h:] == 0x5A).all())


def test_wrong_type_pairings_fail_per_member():
    from dietgpu_b200 import ops

    words = [relu_words(n, n) for n in (100, 5000)]
    ts = [_t(w) for w in words]
    sparse, ssz, _ = ops.compress_data(True, ts, sparse=True)
    dense, dsz, _ = ops.compress_data(True, ts)
    h16 = [t.to(torch.float16) for t in ts]
    s16, s16z, _ = ops.compress_data(True, h16, sparse=True)
    b16 = [t.to(torch.bfloat16) for t in ts]
    sb16, sb16z, _ = ops.compress_data(True, b16, sparse=True)

    def expect_fail(comp, sz, outs, as_sparse, what):
        rows = [comp[i, :int(sz[i])] for i in range(2)]
        st = torch.full((2,), 0xEE, dtype=torch.uint8, device="cuda")
        ops.decompress_data(True, rows, outs, False, None, st, None, sparse=as_sparse)
        assert st.cpu().tolist() == [0, 0], what
        assert all(bool((o == 7.0).all()) for o in outs), what

    f32 = lambda: [torch.full_like(t, 7.0) for t in ts]  # noqa: E731
    expect_fail(sparse, ssz, f32(), False, "type 8 read as type 3")
    expect_fail(dense, dsz, f32(), True, "type 3 read as type 8")
    expect_fail(s16, s16z, f32(), True, "type 5 read as type 8")
    expect_fail(sb16, sb16z, f32(), True, "type 6 read as type 8")
    expect_fail(sparse, ssz, [torch.full((t.numel(),), 7.0, dtype=torch.float16, device="cuda") for t in ts], True,
                "type 8 read as type 5")
    expect_fail(sparse, ssz, [torch.full((t.numel(),), 7.0, dtype=torch.bfloat16, device="cuda") for t in ts], True,
                "type 8 read as type 6")


@pytest.mark.parametrize("n", [6, 130])
def test_graph_capture_replays_new_data(n):
    from dietgpu_b200 import ops

    lens = [(37 * i + 11) % 9000 + 1 for i in range(n)]
    ins = [torch.empty(k, dtype=torch.float32, device="cuda") for k in lens]
    _, cols = ops.max_float_compressed_output_size(ins, sparse=True)
    comp = torch.zeros((n, cols), dtype=torch.uint8, device="cuda")
    sizes = torch.zeros(n, dtype=torch.int32, device="cuda")
    outs = [torch.empty_like(t) for t in ins]
    rows = [comp[i] for i in range(n)]
    temp = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for t in ins:
            t.normal_().relu_()
        ops.compress_data(True, ins, False, temp, comp, sizes, sparse=True)  # warm-up outside the capture
        ops.decompress_data(True, rows, outs, False, temp, sparse=True)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.compress_data(True, ins, False, temp, comp, sizes, sparse=True)
        ops.decompress_data(True, rows, outs, False, temp, sparse=True)
    for rep in range(2):
        data = [relu_words(k, 7000 * rep + i) for i, k in enumerate(lens)]
        for t, w in zip(ins, data):
            t.copy_(torch.from_numpy(w.view(np.int32)).view(torch.float32))
        g.replay()
        torch.cuda.synchronize()
        hs = sizes.cpu().tolist()
        for i, w in enumerate(data):
            S.assert_same(comp[i, :hs[i]].cpu().numpy(), oracle_archive(w, 10), f"replay {rep} {i}")
            assert torch.equal(_i32(outs[i]), _i32(ins[i]))


def test_64_members_of_1mi_relu():
    from dietgpu_b200 import ops

    n, k = 64, 1 << 20
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn((n, k), generator=g, device="cuda").relu_()
    ts = [x[i] for i in range(n)]
    comp, sizes, _ = ops.compress_data(True, ts, sparse=True)
    hs = sizes.cpu().tolist()
    for i in range(n):
        arch = comp[i, :hs[i]].cpu().numpy()
        w = _i32(ts[i]).cpu().numpy().view(np.uint32)
        sym, _, _ = S.symbols(w)
        want_pdf = O.normalize(np.bincount(sym, minlength=256).astype(np.uint32), k, 10)
        assert np.array_equal(S.ans_part(arch)[32:544].view(np.uint16).astype(np.uint32), want_pdf), f"member {i}: pdf"
        S.assert_same(arch, S.compress(w, 10), f"member {i}")
    out = torch.empty_like(x)
    ops.decompress_data(True, [comp[i, :hs[i]] for i in range(n)], [out[i] for i in range(n)], sparse=True)
    assert torch.equal(_i32(out), _i32(x))
    assert sum(hs) / x.numel() / 4 <= 0.47


def test_largest_member_the_format_allows():
    from dietgpu_b200 import capi, ops

    L = capi.lib()
    lo, hi = 1, 1 << 32
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if L.dgb_float_max_compressed_size(8, mid) else (lo, mid)
    top = lo
    assert S.max_compressed_size(top) == L.dgb_float_max_compressed_size(8, top) != 0
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randint(0x3F000000, 0x40800000, (top,), device="cuda", generator=g, dtype=torch.int32)
    x[::3] = 0
    x[1::7] = -0x80000000
    comp, sizes, _ = ops.compress_data(True, [x.view(torch.float32)], sparse=True)
    size = int(sizes[0]) & 0xFFFFFFFF
    assert 32 < size <= comp.size(1)
    pz, nz = int((x == 0).sum()), int((x == -0x80000000).sum())
    nat = (x >> 23) & 0xFF
    other = torch.bincount(nat, minlength=256).cpu()
    other[0] -= pz + nz
    free = torch.nonzero(other == 0).flatten().tolist()
    ep, em = free[0], free[1]
    S_ = top - pz - nz
    hdr = comp[0, :32].cpu().numpy().view(np.uint32).tolist()
    assert hdr == [(0xF00F << 16) | 1, top, 8, 0, S_, ep | em << 8 | 1 << 16, 0, 0]
    nb = -(-top // 4096)
    kept = ((x & 0x7FFFFFFF) != 0).to(torch.int32)
    kept = torch.nn.functional.pad(kept, (0, nb * 4096 - top)).view(nb, 4096).sum(1)
    want_table = torch.cumsum(kept, 0) - kept
    got_table = comp[0, 32:32 + 4 * nb].view(torch.int32).to(torch.int64)
    assert torch.equal(got_table, want_table)
    ans_at = 32 + S.table_bytes(top) + S.stored_bytes(S_)
    ans = comp[0, ans_at:ans_at + 544].cpu().numpy()
    assert ans[:32].view(np.uint32)[:3].tolist() == [(0xD00D << 16) | 1, nb, top]
    sym = torch.where(x == 0, ep, torch.where(x == -0x80000000, em, nat))
    h = torch.bincount(sym, minlength=256).cpu().numpy()
    assert np.array_equal(ans[32:544].view(np.uint16).astype(np.uint32), O.normalize(h.astype(np.uint32), top, 10))
    del nat, sym, kept
    out = torch.empty_like(x)
    ops.decompress_data(True, [comp[0, :size]], [out.view(torch.float32)], sparse=True)
    assert torch.equal(out, x)
    del comp, out, x
    with pytest.raises(RuntimeError):
        ops.max_float_compressed_output_size([torch.empty(top + 1, dtype=torch.float32, device="meta")], sparse=True)


def test_cpp_compat_sparse32_roundtrip():
    exe = os.path.join(ROOT, "tests", "cpp", "sparse32_roundtrip")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "dietgpu_b200", "csrc"), "-s", "sparse32_test"])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "all passed" in r.stdout
