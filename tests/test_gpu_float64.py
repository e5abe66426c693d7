"""The float64 codec (float type 4) on the GPU, pinned to the CPU restatement in tests/f64_oracle.py.

  - an edge corpus of float64 words at prob bits 9, 10 and 11 under every kernel variant of
    test_gpu_variants.VARIANTS (except the 20-warp decoder, which is byte-only), with the shared
    guard-banded round trip; torch.profiler confirms that every float64 instantiation runs;
  - both operator layers: pointer, split-size and simple forms, capacities one word short, a float64 archive
    decoded into a float32 output, mixed output dtypes, size bounds and the header query;
  - a corrupted stored plane fails checksum verification;
  - CUDA-graph capture at 6 and 130 members, the HostCodec pipeline and the archive mover;
  - 64 x 512 Ki N(0,1) doubles (every pdf and archive), and the largest member the format allows;
  - three members through the C++ compatibility header (tests/cpp/f64_roundtrip.cu).
"""
import hashlib
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import f64_oracle as F
from codec_helpers import GUARD, SENTINEL, assert_guard_intact, codec_options, guarded_out
from multirank import run_ranks
from oracle import oracle as O
from test_gpu_variants import VARIANTS

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = (0, 1, 31, 32, 33, 4095, 4096, 4097, 65537, 300000)


def normal64(n, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, generator=g, dtype=torch.float64) * scale).numpy().view(np.uint64)


def _corpus():
    rng = np.random.default_rng(64)
    c = [normal64(n, 600 + n) for n in SIZES]
    c.append(rng.integers(0, 2 ** 64, 70001, dtype=np.uint64))              # full range: NaN, +-Inf, subnormals
    c.append(np.zeros(5000, np.uint64))                                      # all +0
    c.append(np.full(5000, 1 << 63, np.uint64))                              # all -0
    c.append(np.full(5000, 0x7FF8000000000123, np.uint64))                   # one NaN payload
    c.append(rng.integers(0, 2 ** 64, 40000, dtype=np.uint64) & np.uint64(0x800FFFFFFFFFFFFF))  # subnormals only
    for scale, seed in ((1e-300, 1), (1.0, 2), (1e300, 3)):
        c.append(normal64(30000, seed, scale))
    return c


CORPUS = _corpus()


# ---- the shared guard-banded round trip (tests/codec_helpers.py), for float64 words ---------------------------

_ORACLE = {}


def oracle_archive(w, pb, checksum=False):
    """The CPU restatement's archive, cached per (prob bits, checksum flag, member)."""
    w = np.ascontiguousarray(w, np.uint64)
    key = (pb, bool(checksum), w.size, hashlib.blake2b(w.tobytes(), digest_size=16).digest())
    if key not in _ORACLE:
        a = F.compress(w, pb, checksum)
        a.setflags(write=False)
        _ORACLE[key] = a
    return _ORACLE[key]


def _i64(t):
    return t.view(torch.int64)


def placed_inputs(arrays, offsets):
    """Device float64 tensors holding `arrays`, each starting `offsets[i]` words into its own allocation."""
    ts = []
    for a, off in zip(arrays, offsets):
        full = np.concatenate([np.zeros(off, np.uint64), a]).view(np.int64)
        ts.append(torch.from_numpy(full.copy()).view(torch.float64).cuda()[off:])
    return ts


def guarded_compress(ts, checksum, pb):
    """compress_data into sentinel-prefilled rows; inputs unchanged, nothing written at or past each archive's
    reported size."""
    from dietgpu_b200 import ops

    n = len(ts)
    _, cols = ops.max_float_compressed_output_size(ts)
    comp = torch.full((n, cols + GUARD), SENTINEL, dtype=torch.uint8, device="cuda")
    before = [_i64(t).clone() for t in ts]
    _, sizes, _ = ops.compress_data(True, ts, checksum, None, comp, None, prob_bits=pb)
    hs = sizes.cpu().tolist()
    for i, (t, b) in enumerate(zip(ts, before)):
        assert torch.equal(_i64(t), b), f"member {i}: compress changed its input"
    col = torch.arange(cols + GUARD, device="cuda")
    stray = (comp != SENTINEL) & (col[None, :] >= sizes[:, None].long())
    assert not bool(stray.any()), f"compress wrote beyond the archive size in rows {torch.nonzero(stray.any(1)).flatten().tolist()[:8]}"
    return comp, hs


def guarded_decode(rows, lengths, pb, checksum, expect, what):
    """Decodes into views at word offsets 0..7 inside sentinel-filled buffers and checks status, sizes, data and
    guards."""
    from dietgpu_b200 import ops

    n = len(rows)
    bufs, outs, spans = [], [], []
    for i in range(n):
        b, v, span = guarded_out(lengths[i], torch.float64, (5 * i + 3) % 8)
        bufs.append(b)
        outs.append(v)
        spans.append(span)
    status = torch.zeros(n, dtype=torch.uint8, device="cuda")
    osz = torch.zeros(n, dtype=torch.int32, device="cuda")
    ops.decompress_data(True, rows, outs, checksum, None, status, osz, prob_bits=pb)
    assert status.cpu().tolist() == [1] * n, f"{what}: status {status.cpu().tolist()}"
    assert osz.cpu().tolist() == list(lengths), f"{what}: decoded sizes"
    for i in range(n):
        assert torch.equal(_i64(outs[i]), _i64(expect[i])), f"{what}: member {i} decodes differently"
        assert_guard_intact(bufs[i], spans[i][0], spans[i][1], f"{what}: member {i}")


def roundtrip(arrays, pb=10, checksum=False, in_offsets=None, exact=False, decode_oracle=False):
    """Compress float64 `arrays` as one batch, compare every member with the CPU restatement (byte for byte when
    `exact`), decode the archives (and, with `decode_oracle`, the restatement's) into guard-banded outputs."""
    ts = placed_inputs(arrays, in_offsets or [0] * len(arrays))
    comp, hs = guarded_compress(ts, checksum, pb)
    host = comp[:, :max(hs) if hs else 0].cpu().numpy()
    for i, a in enumerate(arrays):
        want = oracle_archive(a, pb, checksum)
        assert hs[i] == want.size and hs[i] % 16 == 0, f"member {i}: size {hs[i]} != oracle {want.size}"
        if exact:
            assert np.array_equal(host[i, :hs[i]], want), f"member {i}: archive bytes differ from the oracle's"
        else:
            F.assert_same(host[i, :hs[i]], want, f"member {i}")
    lengths = [a.size for a in arrays]
    guarded_decode([comp[i, :hs[i]] for i in range(len(ts))], lengths, pb, checksum, ts, "decode")
    if decode_oracle:
        rows = [torch.from_numpy(oracle_archive(a, pb, checksum).copy()).cuda() for a in arrays]
        guarded_decode(rows, lengths, pb, checksum, ts, "decode of the oracle's archives")


def exact_histogram(t):
    """Exact histogram of the coded bytes (bits 62..55 of each word), on the device, chunked."""
    flat = _i64(t.flatten())
    h = torch.zeros(256, dtype=torch.int64, device=t.device)
    for a in range(0, flat.numel(), 1 << 28):
        h += torch.bincount(((flat[a:a + (1 << 28)] >> 55) & 0xFF).to(torch.uint8), minlength=256)
    return h.cpu().numpy()


def _cells():
    for pb in (9, 10, 11):
        for name, opts, role in VARIANTS:
            if name == "decode_warps20":
                continue  # 20-warp CTAs exist for byte archives only
            yield pytest.param(pb, opts, role, id=f"f64-pb{pb}-{name}")


@pytest.mark.parametrize("pb,opts,role", list(_cells()))
def test_variant_matches_oracle(pb, opts, role):
    in_offsets = [i % 8 for i in range(len(CORPUS))]
    with codec_options(**opts):
        roundtrip(CORPUS, pb, checksum=(pb == 10), in_offsets=in_offsets, exact=(role == "exact"),
                  decode_oracle=(role == "dec"))


def test_every_float64_instantiation_runs():
    # in a fresh process: in a long-lived one the GPU's timestamps drift against the host clock that bounds the
    # profiler's window, and every record of a window can fall outside it
    run_ranks(_every_float64_instantiation_runs, 1, backend="gloo")


def _every_float64_instantiation_runs(rank, world, dev):
    from torch.profiler import ProfilerActivity, profile

    from dietgpu_b200 import ops

    small = CORPUS[:8] + CORPUS[-1:]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for pb in (9, 10, 11):
            for opts in ({}, dict(encode_wide_table=0), dict(encode_canonical=1), dict(decode_warps=4),
                         dict(decode_fused=0), dict(stats_stage=1)):
                with codec_options(**opts):
                    roundtrip(small, pb)
        for ws in (0, 1):
            for st in (0, 1):
                with codec_options(encode_fused=1, fused_stage=st, encode_wide_table=ws):
                    roundtrip(small, 10)
        comp, sizes, _ = ops.compress_data(True, [torch.from_numpy(CORPUS[5].view(np.float64)).cuda()])
        dst = torch.empty_like(comp[0])
        ops.pull_archives(True, [comp[0]], [dst], float_dtype=torch.float64)
        torch.cuda.synchronize()
    names = {re.sub(r"\s", "", e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    want = ["statsFloatKernel<4>", "statsFloatStagedKernel<4>", "encodeKernel<4>", "planKernel<4>",
            "pullArchivesF64Kernel"]
    want += [f"encodeKernelFast<{w},4>" for w in ("false", "true")]
    want += [f"encodeFusedKernel<4,{w},{s}>" for w in ("false", "true") for s in ("false", "true")]
    want += [f"decodeFusedKernel<4,{pb},{w}>" for pb in (9, 10, 11) for w in (4, 8)]
    want += [f"decodeKernel<4,{pb},8,true,false>" for pb in (9, 10, 11)]
    missing = [w for w in want if not any(w in n for n in names)]
    assert not missing, f"not launched: {missing}; kernels seen: {sorted(n[:120] for n in names)}"


# ---- operator layers ---------------------------------------------------------------

@pytest.fixture(params=["torch", "mirror"])
def L(request):
    if request.param == "torch":
        from dietgpu_b200 import torch_library

        return torch_library.load()
    from dietgpu_b200 import ops

    return ops


def _t(w):
    return torch.from_numpy(np.ascontiguousarray(w).view(np.float64).copy()).cuda()


MEMBERS = [normal64(n, 900 + n) for n in (1, 4097, 70001, 12345)]


@pytest.mark.parametrize("checksum", [False, True])
def test_operators_pointer_split_simple(L, checksum):
    ts = [_t(w) for w in MEMBERS]
    comp, sizes, _ = L.compress_data(True, ts, checksum)
    hs = sizes.cpu().tolist()
    for i, w in enumerate(MEMBERS):
        want = oracle_archive(w, 10, checksum)
        assert hs[i] == want.size
        F.assert_same(comp[i, :hs[i]].cpu().numpy(), want, f"member {i}")
    outs = [torch.empty_like(t) for t in ts]
    L.decompress_data(True, [comp[i, :hs[i]] for i in range(len(ts))], outs, checksum)
    assert all(torch.equal(a.view(torch.int64), b.view(torch.int64)) for a, b in zip(ts, outs))
    # split-size forms
    flat = torch.cat(ts)
    split = torch.tensor([t.numel() for t in ts], dtype=torch.int32)
    archs, ssz, _ = L.compress_data_split_size(True, flat, split, checksum)
    for i, w in enumerate(MEMBERS):
        F.assert_same(archs[i].cpu().numpy(), oracle_archive(w, 10, checksum), f"split {i}")
    out = torch.full_like(flat, float("nan"))
    L.decompress_data_split_size(True, archs, out, split, checksum)
    assert torch.equal(out.view(torch.int64), flat.view(torch.int64))
    # simple forms
    simple = L.compress_data_simple(True, ts, checksum)
    back = L.decompress_data_simple(True, simple, checksum)
    assert all(b.dtype == torch.float64 for b in back)
    assert all(torch.equal(a.view(torch.int64), b.view(torch.int64)) for a, b in zip(ts, back))


def test_operators_refusals_and_queries(L):
    ts = [_t(w) for w in MEMBERS[:3]]
    comp, sizes, _ = L.compress_data(True, ts)
    hs = sizes.cpu().tolist()
    rows = [comp[i, :hs[i]] for i in range(3)]
    n = len(ts)
    # capacities one word short: status 0, the required size, nothing written
    outs = [torch.full((t.numel() - 1,), 7.0, dtype=torch.float64, device="cuda") for t in ts]
    st = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
    words = torch.zeros(n, dtype=torch.int32, device="cuda")
    L.decompress_data(True, rows, outs, False, None, st, words)
    assert st.cpu().tolist() == [0] * n and words.cpu().tolist() == [t.numel() for t in ts]
    assert all(bool((o == 7.0).all()) for o in outs)
    # a float64 archive decoded into float32 outputs: status 0, nothing written
    outs = [torch.full((2 * t.numel(),), 7.0, dtype=torch.float32, device="cuda") for t in ts]
    L.decompress_data(True, rows, outs, False, None, st, None)
    assert st.cpu().tolist() == [0] * n and all(bool((o == 7.0).all()) for o in outs)
    # float64 and float32 outputs in one call
    with pytest.raises(RuntimeError):
        L.decompress_data(True, rows[:2], [torch.empty_like(ts[0]), torch.empty(ts[1].numel(), device="cuda")])
    from dietgpu_b200 import capi

    for k in (0, 1, 4097, 1 << 20):
        want = capi.lib().dgb_float_max_compressed_size(capi.FLOAT64, k)
        assert L.max_float_compressed_size(torch.empty(0, dtype=torch.float64), k) == want
    assert L.max_float_compressed_output_size(ts)[1] == max(
        capi.lib().dgb_float_max_compressed_size(capi.FLOAT64, t.numel()) for t in ts)


def test_info_query_reports_type_4():
    from dietgpu_b200 import capi

    ts = [_t(w) for w in MEMBERS]
    from dietgpu_b200 import ops

    comp, sizes, _ = ops.compress_data(True, ts, True)
    n = len(ts)
    ptrs = capi.ptr_array([comp[i].data_ptr() for i in range(n)])
    osz = torch.zeros(n, dtype=torch.int32, device="cuda")
    oty = torch.zeros(n, dtype=torch.int32, device="cuda")
    ock = torch.zeros(n, dtype=torch.int32, device="cuda")
    tmp = torch.empty(4096, dtype=torch.uint8, device="cuda")
    rc = capi.lib().dgb_float_get_compressed_info(tmp.data_ptr(), 4096, ptrs, 0, n, osz.data_ptr(), oty.data_ptr(),
                                                  ock.data_ptr(), torch.cuda.current_stream().cuda_stream)
    capi.check(rc, "info")
    assert oty.cpu().tolist() == [4] * n
    assert osz.cpu().tolist() == [t.numel() for t in ts]
    assert ock.cpu().tolist() == [F.info(oracle_archive(w, 10, True))["checksum"] for w in MEMBERS]


def test_flipped_stored_byte_fails_the_checksum():
    from dietgpu_b200 import ops

    t = _t(MEMBERS[2])
    comp, sizes, _ = ops.compress_data(True, [t], True)
    row = comp[0, :int(sizes[0])].clone()
    row[16] ^= 0x01  # first byte of word 0 in the u32 plane
    with pytest.raises(RuntimeError, match="checksum mismatch"):
        ops.decompress_data(True, [row], [torch.empty_like(t)], True)


@pytest.mark.parametrize("n", [6, 130])
def test_graph_capture_replays_new_data(n):
    from dietgpu_b200 import ops

    lens = [(37 * i + 11) % 9000 + 1 for i in range(n)]
    ins = [torch.empty(k, dtype=torch.float64, device="cuda") for k in lens]
    _, cols = ops.max_float_compressed_output_size(ins)
    comp = torch.zeros((n, cols), dtype=torch.uint8, device="cuda")
    sizes = torch.zeros(n, dtype=torch.int32, device="cuda")
    outs = [torch.empty_like(t) for t in ins]
    rows = [comp[i] for i in range(n)]
    temp = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for t in ins:
            t.normal_()
        ops.compress_data(True, ins, False, temp, comp, sizes)  # warm-up outside the capture
        ops.decompress_data(True, rows, outs, False, temp)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.compress_data(True, ins, False, temp, comp, sizes)
        ops.decompress_data(True, rows, outs, False, temp)
    for rep in range(2):
        data = [normal64(k, 7000 * rep + i) for i, k in enumerate(lens)]
        for t, w in zip(ins, data):
            t.copy_(torch.from_numpy(w.view(np.float64)))
        g.replay()
        torch.cuda.synchronize()
        hs = sizes.cpu().tolist()
        for i, w in enumerate(data):
            F.assert_same(comp[i, :hs[i]].cpu().numpy(), oracle_archive(w, 10), f"replay {rep} {i}")
            assert torch.equal(outs[i].view(torch.int64), ins[i].view(torch.int64))


def test_host_codec_pipeline():
    import dietgpu_b200 as dg

    host_in = [torch.from_numpy(w.view(np.float64).copy()).pin_memory() for w in MEMBERS * 4]
    hc = dg.HostCodec(True, host_in, groups=4, checksum=True)
    comp = torch.zeros((len(host_in), hc.max_archive_bytes()), dtype=torch.uint8).pin_memory()
    hs = hc.compress(host_in, comp)
    for i, t in enumerate(host_in):
        F.assert_same(comp[i, :hs[i]].numpy(), oracle_archive(t.numpy().view(np.uint64), 10, True), f"member {i}")
    outs = [torch.full_like(t, float("nan")).pin_memory() for t in host_in]
    hc.decompress([comp[i, :k] for i, k in enumerate(hs)], outs)
    assert all(torch.equal(a.view(torch.int64), b.view(torch.int64)) for a, b in zip(host_in, outs))


def test_pull_archives_copies_exactly_each_archive():
    from dietgpu_b200 import ops

    ts = [_t(w) for w in MEMBERS]
    comp, sizes, _ = ops.compress_data(True, ts)
    hs = sizes.cpu().tolist()
    dst = torch.full_like(comp, 0x5A)
    nb = torch.zeros(len(ts), dtype=torch.int32, device="cuda")
    ops.pull_archives(True, [comp[i] for i in range(len(ts))], [dst[i] for i in range(len(ts))],
                      float_dtype=torch.float64, out_bytes=nb)
    assert nb.cpu().tolist() == hs
    for i, h in enumerate(hs):
        assert torch.equal(dst[i, :h], comp[i, :h])
        assert bool((dst[i, h:] == 0x5A).all())


def test_64_members_of_512ki_normal_doubles():
    from dietgpu_b200 import ops

    n, k = 64, 512 * 1024
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn((n, k), generator=g, dtype=torch.float64, device="cuda")
    ts = [x[i] for i in range(n)]
    comp, sizes, _ = ops.compress_data(True, ts)
    hs = sizes.cpu().tolist()
    for i in range(n):
        arch = comp[i, :hs[i]].cpu().numpy()
        h = exact_histogram(ts[i])
        want_pdf = O.normalize(h.astype(np.uint32), k, 10)
        assert np.array_equal(F.ans_part(arch)[32:544].view(np.uint16).astype(np.uint32), want_pdf), f"member {i}: pdf"
        F.assert_same(arch, F.compress(ts[i].cpu().numpy().view(np.uint64), 10), f"member {i}")
    out = torch.empty_like(x)
    ops.decompress_data(True, [comp[i, :hs[i]] for i in range(n)], [out[i] for i in range(n)])
    assert torch.equal(out.view(torch.int64), x.view(torch.int64))
    assert sum(hs) / x.numel() / 8 <= 0.90


def test_largest_member_the_format_allows():
    from dietgpu_b200 import capi, ops

    L = capi.lib()
    lo, hi = 1, 1 << 32
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if L.dgb_float_max_compressed_size(capi.FLOAT64, mid) else (lo, mid)
    top = lo
    assert F.max_compressed_size(top) == L.dgb_float_max_compressed_size(capi.FLOAT64, top) != 0
    x = torch.empty(top, dtype=torch.float64, device="cuda")
    x.view(torch.int64).copy_(torch.randint(0x3F00000000000000, 0x4010000000000000, (top,), device="cuda"))
    comp, sizes, _ = ops.compress_data(True, [x])
    size = int(sizes[0]) & 0xFFFFFFFF
    assert 16 < size <= comp.size(1)
    hdr = comp[0, :16].cpu().numpy().view(np.uint32)
    assert hdr.tolist() == [(0xF00F << 16) | 1, top, 4, 0]
    ans = comp[0, 16 + F.noncomp_bytes(top):].narrow(0, 0, 544).cpu().numpy()
    assert ans[:32].view(np.uint32)[:3].tolist() == [(0xD00D << 16) | 1, -(-top // 4096), top]
    h = exact_histogram(x)
    assert np.array_equal(ans[32:544].view(np.uint16).astype(np.uint32), O.normalize(h.astype(np.uint32), top, 10))
    del comp
    with pytest.raises(RuntimeError):
        ops.max_float_compressed_output_size([torch.empty(top + 1, dtype=torch.float64, device="meta")])


def test_cpp_compat_float64_roundtrip():
    exe = os.path.join(ROOT, "tests", "cpp", "f64_roundtrip")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "dietgpu_b200", "csrc"), "-s", "f64_test"])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "all passed" in r.stdout
