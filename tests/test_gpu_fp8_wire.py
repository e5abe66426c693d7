"""The fp8 wire on the GPU: the scaled fp8 cast (ops.cast_fp8, dgb_float_cast_fp8) against torch's CUDA clamp-cast on
every fp32 and bf16 bit pattern, its fused histogram against bincount, fp8 archives (compress_data(archive_dtype=))
against the CPU oracle's byte archives and the unmodified reference's byte decoder, the fp8 decode-and-sum against
torch's fold of q.float() * d, CUDA-graph replays with the scales changed between them, and the kernels one fp8
compress and sum launch."""
import numpy as np
import pytest
import torch

from codec_helpers import codec_options
from fp8_reference import E4M3, E5M2, NAN_BYTE, cast as ref_cast
from multirank import run_ranks
from oracle import oracle as O

pytestmark = pytest.mark.gpu

FP8 = [torch.float8_e4m3fn, torch.float8_e5m2]
MAX = {torch.float8_e4m3fn: 448.0, torch.float8_e5m2: 57344.0}
KIND = {torch.float8_e4m3fn: E4M3, torch.float8_e5m2: E5M2}
IDS = ["e4m3", "e5m2"]


def ops():
    from dietgpu_b200 import ops as o

    return o


def torch_cast(x, s, dt):
    """torch's clamp-cast, the cast's contract for every product that is not NaN."""
    p = x.float() * s
    return p.clamp(-MAX[dt], MAX[dt]).to(dt), torch.isnan(p)


def u8(t):
    return t.view(torch.uint8)


def scale(v):
    return torch.full((1,), v, dtype=torch.float32, device="cuda")


# ---- the cast -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dt", FP8, ids=IDS)
@pytest.mark.parametrize("s", [1.0, 0.3])
def test_cast_every_fp32_pattern(dt, s):
    st = scale(s)
    nans = 0
    for c in range(16):
        base = (c << 28) - ((1 << 32) if c >= 8 else 0)
        x = (torch.arange(0, 1 << 28, dtype=torch.int32, device="cuda") + base).view(torch.float32)
        q = ops().cast_fp8([x], dt, st)[0]
        want, nan = torch_cast(x, st, dt)
        assert bool(((u8(q) == u8(want)) | nan).all()), f"block {c}: bytes differ from torch's clamp-cast"
        assert bool((u8(q)[nan] == NAN_BYTE).all()), f"block {c}: a NaN product is not 0x7F"
        nans += int(nan.sum())
        del x, q, want, nan
    assert nans > 0


@pytest.mark.parametrize("dt", FP8, ids=IDS)
def test_cast_every_bf16_pattern(dt):
    w = torch.arange(0, 1 << 16, dtype=torch.int32, device="cuda").to(torch.int16)
    x = w.view(torch.bfloat16)
    # 1, a non-power of two, scales that saturate most words and that flush most words to +-0
    for s in (1.0, 0.3, 2.0 ** 100, 3.0e38, 2.0 ** -100, 2.0 ** -140):
        q = ops().cast_fp8([x], dt, scale(s))[0]
        want, nan = torch_cast(x, scale(s), dt)
        assert bool(((u8(q) == u8(want)) | nan).all()), s
        assert bool((u8(q)[nan] == NAN_BYTE).all()), s
        assert np.array_equal(u8(q).cpu().numpy(), ref_cast(w.cpu().numpy().view(np.uint16), s, KIND[dt])), s
    # without a scale: s = 1
    q = ops().cast_fp8([x], dt)[0]
    assert torch.equal(u8(q), u8(ops().cast_fp8([x], dt, scale(1.0))[0]))


def _cast_into(ts, dt, s, outs, hist):
    from dietgpu_b200 import capi

    ft = {torch.float8_e4m3fn: capi.FLOAT8_E4M3, torch.float8_e5m2: capi.FLOAT8_E5M2}[dt]
    in_ft = capi.FLOAT32 if ts[0].dtype == torch.float32 else capi.BFLOAT16
    rc = capi.lib().dgb_float_cast_fp8(in_ft, ft, len(ts), capi.ptr_array([t.data_ptr() for t in ts]),
                                       capi.u32_array([t.numel() for t in ts]), s.data_ptr() if s is not None else None,
                                       capi.ptr_array(outs), hist.data_ptr() if hist is not None else None,
                                       torch.cuda.current_stream().cuda_stream)
    capi.check(rc, "cast_fp8")


@pytest.mark.parametrize("dt", FP8, ids=IDS)
@pytest.mark.parametrize("in_dtype", [torch.float32, torch.bfloat16])
def test_cast_histogram_guards_and_alignment(dt, in_dtype):
    g = torch.Generator(device="cuda").manual_seed(5)
    sizes = [0, 1, 3, 7, 8, 9, 15, 17, 4095, 4096, 4097, 65537, 300001, 2 * 2 ** 20 + 5]
    ts, srcs, outs, bufs, spans = [], [], [], [], []
    for i, n in enumerate(sizes):
        src = (torch.randn(n + 16, generator=g, device="cuda") * 100).to(in_dtype)
        src[5::97] = float("nan")
        src[7::89] = float("inf")
        off = i % 7  # unaligned input offsets (in words)
        t = src[off:off + n]
        ts.append(t)
        srcs.append(t.clone())
        buf = torch.full((n + 256,), 0xA5, dtype=torch.uint8, device="cuda")
        o = 128 + (i * 3) % 9  # unaligned outputs too
        bufs.append(buf)
        spans.append((o, o + n))
        outs.append(buf.data_ptr() + o)
    s = scale(0.37)
    hist = torch.full((len(ts) * 256,), -1, dtype=torch.int32, device="cuda")  # overwritten, not accumulated
    _cast_into(ts, dt, s, outs, hist)
    hist2 = hist.clone()
    _cast_into(ts, dt, s, outs, hist)  # a second call gives the same histogram
    assert torch.equal(hist, hist2)
    for i, (t, src, buf, (lo, hi)) in enumerate(zip(ts, srcs, bufs, spans)):
        q = buf[lo:hi]
        want, nan = torch_cast(t, s, dt)
        assert bool(((q == u8(want)) | nan).all()), f"member {i}"
        assert torch.equal(hist[i * 256:(i + 1) * 256], torch.bincount(q.long(), minlength=256).int()), f"member {i}"
        assert bool((buf[:lo] == 0xA5).all()) and bool((buf[hi:] == 0xA5).all()), f"member {i}: guard band"
        assert torch.equal(t.view(torch.int16 if t.element_size() == 2 else torch.int32),
                           src.view(torch.int16 if t.element_size() == 2 else torch.int32)), f"member {i}: input"


# ---- archives --------------------------------------------------------------------------------------------------

def _members(in_dtype, sizes, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for i, n in enumerate(sizes):
        src = torch.randn(n + 8, generator=g, device="cuda").to(in_dtype)
        out.append(src[i % 5:i % 5 + n])
    return out


def _rows(comp, sizes):
    hs = sizes.cpu().tolist()
    return [comp[i, :hs[i]] for i in range(len(hs))]


@pytest.mark.parametrize("dt", FP8, ids=IDS)
@pytest.mark.parametrize("in_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("pb", [9, 10, 11])
def test_archives_equal_the_oracle(dt, in_dtype, pb):
    ts = _members(in_dtype, [0, 1, 33, 4096, 4097, 65537, 2 * 2 ** 20 + 5], 100 + pb)
    before = [t.clone() for t in ts]
    s = scale(64.0 / 3.0)
    q = ops().cast_fp8(ts, dt, s)
    for checksum in (False, True):
        with codec_options(encode_canonical=1):
            comp, sizes, _ = ops().compress_data(True, ts, checksum, prob_bits=pb, archive_dtype=dt, scale_tensor=s)
        for i, row in enumerate(_rows(comp, sizes)):
            want = O.ans_encode(u8(q[i]).cpu().numpy(), pb, checksum)
            O.assert_same_ans(row.cpu().numpy(), want, f"member {i} checksum {checksum}")
        # default mode: the archives decode to q
        comp, sizes, _ = ops().compress_data(True, ts, checksum, prob_bits=pb, archive_dtype=dt, scale_tensor=s)
        outs = [torch.empty_like(u8(x)) for x in q]
        st = torch.zeros(len(ts), dtype=torch.uint8, device="cuda")
        ops().decompress_data(False, _rows(comp, sizes), outs, checksum, None, st, prob_bits=pb)
        assert bool(st.all())
        for i, (o, x) in enumerate(zip(outs, q)):
            assert torch.equal(o, u8(x)), f"member {i}"
    for t, b in zip(ts, before):
        assert torch.equal(t, b)


@pytest.mark.parametrize("batch", [64, 65])
def test_archives_in_large_batches(batch):
    ts = _members(torch.float32, [(i * 977) % 9000 for i in range(batch)], batch)
    q = ops().cast_fp8(ts, torch.float8_e4m3fn, scale(3.0))
    with codec_options(encode_canonical=1):
        comp, sizes, _ = ops().compress_data(True, ts, archive_dtype=torch.float8_e4m3fn, scale_tensor=scale(3.0))
    for i, row in enumerate(_rows(comp, sizes)):
        O.assert_same_ans(row.cpu().numpy(), O.ans_encode(u8(q[i]).cpu().numpy(), 10), f"member {i}")


def test_reference_reads_fp8_archives():
    from oracle import ref_lib

    if not ref_lib.available():
        pytest.skip("the reference was not built (oracle/_ref)")
    from test_gpu_reference_interchange import ref_decode

    for dt in FP8:
        ts = _members(torch.bfloat16, [1, 4097, 300001], 9)
        q = ops().cast_fp8(ts, dt, scale(5.0))
        comp, sizes, _ = ops().compress_data(True, ts, archive_dtype=dt, scale_tensor=scale(5.0))
        outs, st, sz, rc = ref_decode("bytes", _rows(comp, sizes), [t.numel() for t in ts], 10, False)
        assert rc == 0 and st == [1] * len(ts) and sz == [t.numel() for t in ts], (rc, st, sz)
        for o, x in zip(outs, q):
            assert torch.equal(o, u8(x))


# ---- decode-and-sum ------------------------------------------------------------------------------------------

def _fold(qs, d, init=None):
    acc = init.clone() if init is not None else qs[0].float() * d
    for q in (qs if init is not None else qs[1:]):
        acc = acc + q.float() * d
    return acc


def _all_bytes(n, seed):
    """n fp8 bytes covering all 256 codes (NaN codes, +-0, +-max and the subnormals included)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    b = torch.randint(0, 256, (n,), generator=g, device="cuda", dtype=torch.int32).to(torch.uint8)
    k = min(n, 256)
    b[:k] = torch.arange(256, device="cuda").to(torch.uint8)[torch.randperm(256, generator=g, device="cuda")][:k]
    return b


def _block_words(row):
    return (O.parse_ans(row.cpu().numpy())["block_words"][:, 0] & 0xFFFF).astype(np.int64)


@pytest.mark.parametrize("dt", FP8, ids=IDS)
@pytest.mark.parametrize("mode", ["default", "slot8"])
def test_decode_and_sum(dt, mode):
    opts = {} if mode == "default" else dict(decode_slot_words=1)
    sizes = [1, 256, 4097, 70001]
    for width in range(1, 10):
        qs = [[_all_bytes(n, 1000 * width + 10 * g + j) for j in range(width)] for g, n in enumerate(sizes)]
        comp, csz, _ = ops().compress_data(False, [q for grp in qs for q in grp])
        rows = _rows(comp, csz)
        groups = [rows[g * width:(g + 1) * width] for g in range(len(sizes))]
        bws = [_block_words(r) for r in rows]
        # the staged branch (stream in the slot) in default mode, the global-memory one with an 8-word slot
        if mode == "default":
            assert all(int(b.max(initial=0)) <= 256 * 10 + 8 for b in bws)
        else:
            assert any(int(b.max(initial=0)) > 8 for b in bws) and any(int(b.min(initial=1)) <= 8 for b in bws)
        for accumulate in (False, True):
            d = scale(-0.7)
            outs, inits = [], []
            for n in sizes:
                init = torch.randn(n, device="cuda")
                init[::13] = float("nan") if accumulate else 0.0
                inits.append(init)
                outs.append(init.clone())
            flag = torch.zeros(1, device="cuda")
            sq = torch.empty(len(sizes), dtype=torch.float64, device="cuda")
            st = torch.zeros(len(rows), dtype=torch.uint8, device="cuda")
            with codec_options(**opts):
                ops().decompress_data_reduce(groups, outs, accumulate, None, st, archive_dtype=dt, scale_tensor=d,
                                             found_inf=flag, sq_norm=sq)
            assert bool(st.all())
            fp8 = [[q.view(dt) for q in grp] for grp in qs]
            for g in range(len(sizes)):
                want = _fold(fp8[g], d.reshape(()), inits[g] if accumulate else None)
                assert torch.equal(outs[g].view(torch.int32), want.view(torch.int32)), (width, accumulate, g)
            assert float(flag) == 1.0  # the NaN codes are in every group
            assert torch.equal(sq.view(torch.int64), ops().sq_norm(outs).view(torch.int64))
            # finite sums leave the flag alone: e4m3 has no infinities, so drop the NaN codes
            if accumulate:
                continue
            fin = [[torch.where((q & 0x7F) >= (0x7F if dt == torch.float8_e4m3fn else 0x7C), 0, q) for q in grp]
                   for grp in qs]
            comp, csz, _ = ops().compress_data(False, [q for grp in fin for q in grp])
            rows = _rows(comp, csz)
            flag.zero_()
            with codec_options(**opts):
                ops().decompress_data_reduce([rows[g * width:(g + 1) * width] for g in range(len(sizes))], outs,
                                             archive_dtype=dt, scale_tensor=d, found_inf=flag)
            assert float(flag) == 0.0
            for g in range(len(sizes)):
                assert torch.equal(outs[g].view(torch.int32), _fold([q.view(dt) for q in fin[g]], d.reshape(())).view(
                    torch.int32))


def test_invalid_archives_leave_their_group():
    dt = torch.float8_e4m3fn
    sizes = [5000, 5000, 5000]
    qs = [[_all_bytes(n, 7 * g + j) for j in range(3)] for g, n in enumerate(sizes)]
    comp, csz, _ = ops().compress_data(False, [q for grp in qs for q in grp], prob_bits=10)
    rows = [r.clone() for r in _rows(comp, csz)]
    rows[1][0] ^= 1          # group 0: bad magic
    short = _all_bytes(4999, 99)  # group 1: one archive of the wrong size
    c2, s2, _ = ops().compress_data(False, [short])
    rows[4] = _rows(c2, s2)[0].clone()
    groups = [rows[0:3], rows[3:6], rows[6:9]]
    outs = [torch.full((n,), 7.0, device="cuda") for n in sizes]
    st = torch.zeros(9, dtype=torch.uint8, device="cuda")
    sq = torch.full((3,), -1.0, dtype=torch.float64, device="cuda")
    ops().decompress_data_reduce(groups, outs, False, None, st, archive_dtype=dt, scale_tensor=scale(1.0), sq_norm=sq)
    assert st.cpu().tolist() == [1, 0, 1, 1, 0, 1, 1, 1, 1]
    assert bool((outs[0] == 7.0).all()) and bool((outs[1] == 7.0).all())
    assert sq[0].item() == -1.0 and sq[1].item() == -1.0
    assert torch.equal(outs[2].view(torch.int32), _fold([q.view(dt) for q in qs[2]], 1.0).view(torch.int32))
    # another prob_bits is invalid too
    st.zero_()
    ops().decompress_data_reduce(groups[2:], outs[2:], False, None, st[:3], prob_bits=9, archive_dtype=dt,
                                 scale_tensor=scale(1.0))
    assert st[:3].cpu().tolist() == [0, 0, 0]


# ---- CUDA graphs -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dt", FP8, ids=IDS)
def test_graph_replays_read_the_current_scales(dt):
    x = [torch.randn(70001, device="cuda") * 30, torch.randn(4096, device="cuda")]
    s, d = scale(1.0), scale(1.0)
    out = [torch.empty(70001, device="cuda"), torch.empty(4096, device="cuda")]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):  # warm-up outside the capture
        comp, sizes, _ = ops().compress_data(True, x, archive_dtype=dt, scale_tensor=s)
        rows = [comp[i, :comp.size(1)] for i in range(2)]
        ops().decompress_data_reduce([[rows[0]], [rows[1]]], out, archive_dtype=dt, scale_tensor=d)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        comp, sizes, _ = ops().compress_data(True, x, archive_dtype=dt, scale_tensor=s)
        rows = [comp[i, :comp.size(1)] for i in range(2)]
        ops().decompress_data_reduce([[rows[0]], [rows[1]]], out, archive_dtype=dt, scale_tensor=d)
    for sv, dv in ((1.0, 1.0), (0.25, 4.0), (3.0, -1.0 / 3.0), (1e-3, 1e3)):
        s.fill_(sv)
        d.fill_(dv)
        g.replay()
        torch.cuda.synchronize()
        for xi, oi in zip(x, out):
            q, _ = torch_cast(xi, s, dt)
            assert torch.equal(oi.view(torch.int32), (q.float() * d.reshape(())).view(torch.int32)), (sv, dv)


# ---- kernels launched -------------------------------------------------------------------------------------------

def _profile_worker(rank, world, dev):
    import dietgpu_b200 as dg
    from torch.profiler import ProfilerActivity, profile

    x = [torch.randn(300001, device=dev), torch.randn(5000, device=dev)]
    s = torch.full((1,), 8.0, device=dev)
    for _ in range(2):
        comp, sizes, _ = dg.ops.compress_data(True, x, archive_dtype=torch.float8_e4m3fn, scale_tensor=s)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        comp, sizes, _ = dg.ops.compress_data(True, x, archive_dtype=torch.float8_e4m3fn, scale_tensor=s)
        out = [torch.empty_like(t) for t in x]
        dg.ops.decompress_data_reduce([[comp[0]], [comp[1]]], out, archive_dtype=torch.float8_e4m3fn, scale_tensor=s)
        torch.cuda.synchronize()
    names = [e.name for e in p.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    kernels = [n for n in names if "Memset" not in n and "Memcpy" not in n and "memcpy" not in n]
    assert sum("castFp8Kernel" in n for n in kernels) == 1, kernels
    assert any("decodeReduceDevScaleKernel" in n for n in kernels), kernels
    # the statistics pass runs only to publish the given histogram's table; nothing else of the codec or of torch
    assert all(any(k in n for k in ("castFp8Kernel", "stats", "encode", "decodeReduceDevScaleKernel"))
               for n in kernels), kernels
    return 1


def test_profiler_kernel_list():
    run_ranks(_profile_worker, 1, backend="gloo")
