"""Narrowing compress (dgb_float_compress_to / ops.compress_data(archive_dtype=...)) and the collectives' wire_dtype.

float32 inputs are rounded to float16 / bfloat16 inside the compress kernels.  The reference result of every case is
the existing path applied to the cast x.to(T) made by torch ON THE DEVICE (torch's CPU cast gives other NaNs): the
oracle's archive of the cast words and the library's own compress of the cast.  Default archives are compared
field by field (their streams are in completion order), canonical ones byte for byte."""
import inspect
import re

import numpy as np
import pytest
import torch

from codec_helpers import (GUARD, KINDS, SENTINEL, assert_pdf_matches, codec_options, guarded_decode, oracle_archive,
                           placed_inputs)
from multirank import run_ranks
from oracle import oracle as O
from test_gpu_variants import VARIANTS

pytestmark = pytest.mark.gpu

TYPES = {torch.float16: "f16", torch.bfloat16: "bf16"}
SIZES = [0, 1, 31, 33, 4095, 4096, 4097, 8209, 300001]
POOL = 300001


def _u16(t):
    return t.view(torch.int16).cpu().numpy().view(np.uint16)


def _bits(t):
    return t.view(torch.int32 if t.element_size() == 4 else torch.int16)


# ---- value families (float32 bit patterns, seeded) --------------------------------------------------------------

def family(name, n=POOL, seed=0):
    r = np.random.default_rng(seed + sum(map(ord, name)))
    sign = r.integers(0, 2, n, dtype=np.uint32) << 31
    if name.startswith("normal"):
        scale = {"normal_1e-30": 1e-30, "normal_1": 1.0, "normal_1e30": 1e30}[name]
        return (r.standard_normal(n) * scale).astype(np.float32).view(np.uint32)
    if name == "bits":  # every field at random: NaNs, infinities, subnormals included
        return r.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    if name == "ties":  # exact round-half ties, kept lsb even and odd: bf16 ties and fp16 (normal range) ties
        bf = (r.integers(0, 1 << 16, n, dtype=np.uint32) << 16) | 0x8000
        f16 = sign | (r.integers(113, 143, n, dtype=np.uint32) << 23) | (r.integers(0, 1024, n, dtype=np.uint32) << 13) | 0x1000
        return np.where(r.integers(0, 2, n) == 0, bf, f16).astype(np.uint32)
    if name == "carry":  # kept mantissa all ones, discarded part >= half: rounds into the next binade, or to +-Inf
        bf = sign | (r.integers(200, 255, n, dtype=np.uint32) << 23) | 0x7f0000 | r.integers(0x8000, 0x10000, n, dtype=np.uint32)
        f16 = sign | (r.integers(130, 143, n, dtype=np.uint32) << 23) | (0x3ff << 13) | r.integers(0x1000, 0x2000, n, dtype=np.uint32)
        edge = np.array([65504, 65519, 65519.996, 65520, 65520.004, 65536, 1e5, 3.4e38, np.finfo(np.float32).max,
                         3.3895314e38, 3.3895316e38], dtype=np.float32)
        edge = np.concatenate([edge, -edge]).view(np.uint32)
        w = np.where(r.integers(0, 2, n) == 0, bf, f16).astype(np.uint32)
        w[::7] = edge[(np.arange(w[::7].size) % edge.size)]
        return w
    if name == "tiny":  # fp32 subnormals and tiny normals: fp16 zeros / subnormals, bf16 subnormals / smallest normals
        return sign | (r.integers(0, 121, n, dtype=np.uint32) << 23) | r.integers(0, 1 << 23, n, dtype=np.uint32)
    if name == "special":  # NaNs with assorted payloads and signs (low-bit-only payloads too), +-Inf, +-0, normals
        pick = r.integers(0, 6, n)
        nan_hi = 0x7f800000 | r.integers(1, 1 << 23, n, dtype=np.uint32)
        nan_lo = 0x7f800000 | r.integers(1, 1 << 13, n, dtype=np.uint32)  # payload below every kept bit
        inf, zero = np.uint32(0x7f800000), np.uint32(0)
        normal = r.standard_normal(n).astype(np.float32).view(np.uint32)
        w = np.select([pick == 0, pick == 1, pick == 2, pick == 3, pick == 4], [nan_hi, nan_lo, inf, zero, nan_hi | 1],
                      normal)
        return (w.astype(np.uint32) | np.where(pick < 4, sign, 0).astype(np.uint32)).astype(np.uint32)
    raise KeyError(name)


FAMILIES = ["normal_1e-30", "normal_1", "normal_1e30", "bits", "ties", "carry", "tiny", "special"]


# ---- helpers --------------------------------------------------------------------------------------------------

def narrow_guarded(ts, dtype, checksum=False, pb=10):
    """Narrowing compress into sentinel-prefilled rows; checks inputs unchanged and nothing written past a size."""
    from dietgpu_b200 import ops

    n = len(ts)
    mx = max(t.numel() for t in ts)
    cols = ops.max_float_compressed_size(torch.empty(0, dtype=dtype), mx)
    assert cols % 16 == 0
    comp = torch.full((n, cols + GUARD), SENTINEL, dtype=torch.uint8, device="cuda")
    before = [_bits(t).clone() for t in ts]
    _, sizes, _ = ops.compress_data(True, ts, checksum, None, comp, None, prob_bits=pb, archive_dtype=dtype)
    hs = sizes.cpu().tolist()
    for i, (t, b) in enumerate(zip(ts, before)):
        assert torch.equal(_bits(t), b), f"member {i}: compress changed its input"
    col = torch.arange(cols + GUARD, device="cuda")
    stray = (comp != SENTINEL) & (col[None, :] >= sizes[:, None].long())
    assert not bool(stray.any()), f"compress wrote past the archive size in rows {stray.any(1).nonzero().flatten()[:8]}"
    return comp, hs


def check_against_cast(ts, dtype, pb, checksum, oracle=True, what=""):
    """Narrowing compress of ts == the oracle's and the library's archives of x.to(dtype); decodes (checksum
    verified when on) to x.to(dtype) bit for bit.  Returns the archives (device rows)."""
    from dietgpu_b200 import ops

    kind = TYPES[dtype]
    ft = KINDS[kind][0]
    casts = [t.to(dtype) for t in ts]
    comp, hs = narrow_guarded(ts, dtype, checksum, pb)
    lib_comp, lib_sizes, _ = ops.compress_data(True, casts, checksum, prob_bits=pb)
    lib_hs = lib_sizes.cpu().tolist()
    host = comp[:, :max(hs)].cpu().numpy()
    lib_host = lib_comp[:, :max(lib_hs)].cpu().numpy()
    for i, c in enumerate(casts):
        assert hs[i] == lib_hs[i], f"{what} member {i}: size {hs[i]} != compress of the cast {lib_hs[i]}"
        O.assert_same_float(host[i, :hs[i]], lib_host[i, :lib_hs[i]], ft, f"{what} member {i} vs compress of the cast")
        if oracle:
            want = oracle_archive(kind, _u16(c), pb, checksum)
            assert hs[i] == want.size, f"{what} member {i}: size {hs[i]} != oracle {want.size}"
            O.assert_same_float(host[i, :hs[i]], want, ft, f"{what} member {i} vs oracle")
    rows = [comp[i, :hs[i]] for i in range(len(ts))]
    guarded_decode(True, rows, [t.numel() for t in ts], dtype, pb, checksum, casts, what)
    return rows


# ---- edge corpus ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", list(TYPES))
@pytest.mark.parametrize("pb", [9, 10, 11])
@pytest.mark.parametrize("checksum", [False, True])
def test_edge_corpus_equals_the_cast(dtype, pb, checksum):
    for name in FAMILIES:
        pool = family(name)
        arrays = [pool[:n] for n in SIZES for _ in range(4)]
        offsets = [off for _ in SIZES for off in range(4)]  # element offsets 0-3: the vector and the scalar paths
        ts = placed_inputs(arrays, "f32", offsets)
        check_against_cast(ts, dtype, pb, checksum, what=f"{dtype} pb {pb} checksum {checksum} {name}")


# ---- option variants and the instantiations they reach -----------------------------------------------------------

ENC_VARIANTS = [(name, opts, role) for name, opts, role in VARIANTS if role in ("enc", "exact")]


@pytest.mark.parametrize("dtype", list(TYPES))
@pytest.mark.parametrize("name,opts,role", ENC_VARIANTS, ids=[v[0] for v in ENC_VARIANTS])
def test_option_variants(dtype, name, opts, role):
    sizes = [0, 1, 33, 4097, 65537, 300001]
    arrays = [family(f, n, seed=i) for i, (f, n) in enumerate(zip(["normal_1", "special", "ties", "carry", "tiny", "bits"],
                                                                 sizes))]
    ts = placed_inputs(arrays, "f32", [i % 4 for i in range(len(arrays))])
    with codec_options(**opts):
        rows = check_against_cast(ts, dtype, 10, True, what=f"{dtype} {name}")
        if role == "exact":  # canonical: byte-identical to the oracle's archive of the cast
            for i, t in enumerate(ts):
                want = oracle_archive(TYPES[dtype], _u16(t.to(dtype)), 10, True)
                assert np.array_equal(rows[i].cpu().numpy(), want), f"{dtype} canonical member {i}"


def test_profiler_sees_every_new_instantiation():
    # in a fresh process: in a long-lived one the GPU's timestamps drift against the host clock that bounds the
    # profiler's window, and every record of a window can fall outside it
    run_ranks(_profiler_sees_every_new_instantiation, 1, backend="gloo")


def _profiler_sees_every_new_instantiation(rank, world, dev):
    from torch.profiler import ProfilerActivity, profile

    from dietgpu_b200 import ops

    ts = [torch.randn(n, device="cuda") for n in (70001, 4096, 33)]
    runs = [dict(), dict(encode_wide_table=0), dict(encode_wide_table=1), dict(encode_canonical=1),
            dict(encode_fused=1), dict(encode_fused=1, fused_stage=1), dict(stats_stage=1)]
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device="cuda").add_(1)  # the first kernel of a session can be missing from its trace
        for _ in range(3):
            for opts in runs:
                with codec_options(**opts):
                    for dtype in TYPES:
                        ops.compress_data(True, ts, archive_dtype=dtype)
        torch.cuda.synchronize()
    names = {re.sub(r"\s", "", e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    for kind in (65, 66):  # 0x40 | fp16, 0x40 | bf16
        for want in (f"statsFloatKernel<{kind}>", f"encodeKernelFast<false,{kind}>", f"encodeKernelFast<true,{kind}>",
                     f"encodeKernel<{kind}>"):
            assert any(want in k for k in names), (want, sorted(names))
        for never in (f"encodeFusedKernel<{kind}", f"statsFloatStagedKernel<{kind}>"):
            assert not any(never in k for k in names), (never, sorted(names))
    # the fused and staged options fall back to the default kernels: no fused or staged kernel runs at all
    assert not any("encodeFusedKernel" in k or "statsFloatStagedKernel" in k for k in names), sorted(names)


# ---- every float32 bit pattern ---------------------------------------------------------------------------------

def test_every_fp32_bit_pattern_equals_the_device_cast():
    from dietgpu_b200 import ops

    chunk, members = 1 << 28, 4
    per = chunk // members
    for c in range((1 << 32) // chunk):
        v = torch.arange(c * chunk, (c + 1) * chunk, dtype=torch.int64, device="cuda")
        x = torch.where(v >= 1 << 31, v - (1 << 32), v).to(torch.int32).view(torch.float32)
        del v
        ts = [x[i * per:(i + 1) * per] for i in range(members)]
        for dtype in TYPES:
            comp, sizes, _ = ops.compress_data(True, ts, archive_dtype=dtype)
            hs = sizes.cpu().tolist()
            outs = [torch.empty(per, dtype=dtype, device="cuda") for _ in range(members)]
            st = torch.zeros(members, dtype=torch.uint8, device="cuda")
            ops.decompress_data(True, [comp[i, :hs[i]] for i in range(members)], outs, False, None, st)
            assert bool(st.all()), (c, dtype)
            for i in range(members):
                want = ts[i].to(dtype)
                bad = _bits(outs[i]) != _bits(want)
                assert not bool(bad.any()), \
                    f"{dtype}: fp32 pattern {hex(c * chunk + i * per + int(bad.nonzero()[0]))} decodes differently"
            del comp, outs


# ---- batch shapes, exact scratch, graphs, the same-type pairs ----------------------------------------------------

def _raw_compress_to(in_ft, ft, ts, rows, sizes, pb=10, checksum=False):
    """dgb_float_compress_to(in_ft, ft) (dgb_float_compress_pointer(ft) when in_ft is None) with exactly
    dgb_float_compress_temp_bytes(ft, n, max) bytes of scratch."""
    from dietgpu_b200 import capi

    L = capi.lib()
    n = len(ts)
    need = L.dgb_float_compress_temp_bytes(ft, n, max(t.numel() for t in ts))
    temp = torch.empty(need + 256, dtype=torch.uint8, device="cuda")
    ptr = temp.data_ptr() + (-temp.data_ptr()) % 256
    args = (pb, int(checksum), n, capi.ptr_array([t.data_ptr() for t in ts]), capi.u32_array([t.numel() for t in ts]),
            capi.ptr_array([r.data_ptr() for r in rows]), sizes.data_ptr(), torch.cuda.current_stream().cuda_stream)
    rc = L.dgb_float_compress_to(ptr, need, in_ft, ft, *args) if in_ft is not None else \
        L.dgb_float_compress_pointer(ptr, need, ft, *args)
    assert rc == capi.OK
    return temp


@pytest.mark.parametrize("members", [1, 64, 65, 130, 256])
@pytest.mark.parametrize("inline", [1, 0])
def test_batch_shapes_with_exact_scratch(members, inline):
    from dietgpu_b200 import capi, ops

    for dtype, ft in ((torch.float16, capi.FLOAT16), (torch.bfloat16, capi.BFLOAT16)):
        arrays = [family(FAMILIES[i % len(FAMILIES)], (i * 7919) % 20011, seed=i) for i in range(members)]
        ts = placed_inputs(arrays, "f32", [i % 4 for i in range(members)])
        cols = ops.max_float_compressed_size(torch.empty(0, dtype=dtype), max(t.numel() for t in ts))
        comp = torch.full((members, cols), SENTINEL, dtype=torch.uint8, device="cuda")
        sizes = torch.zeros(members, dtype=torch.int32, device="cuda")
        with codec_options(inline_members=inline):
            _raw_compress_to(capi.FLOAT32, ft, ts, [comp[i] for i in range(members)], sizes)
            want_comp, want_sizes, _ = ops.compress_data(True, [t.to(dtype) for t in ts])
        hs, whs = sizes.cpu().tolist(), want_sizes.cpu().tolist()
        assert hs == whs
        host, whost = comp.cpu().numpy(), want_comp.cpu().numpy()
        for i, t in enumerate(ts):
            O.assert_same_float(host[i, :hs[i]], whost[i, :whs[i]], ft, f"{dtype} member {i}")
            O.assert_same_float(host[i, :hs[i]], oracle_archive(TYPES[dtype], _u16(t.to(dtype)), 10), ft,
                                f"{dtype} member {i} vs oracle")
        guarded_decode(True, [comp[i, :hs[i]] for i in range(members)], [t.numel() for t in ts], dtype, 10, False,
                       [t.to(dtype) for t in ts], f"{dtype} {members} members")


@pytest.mark.parametrize("members", [6, 130])
def test_graph_capture_replays_on_new_data(members):
    from dietgpu_b200 import ops

    n = 20011
    for dtype in TYPES:
        src = torch.empty(members, n, dtype=torch.float32, device="cuda")
        ts = [src[i] for i in range(members)]
        cols = ops.max_float_compressed_size(torch.empty(0, dtype=dtype), n)
        comp = torch.zeros(members, cols, dtype=torch.uint8, device="cuda")
        sizes = torch.zeros(members, dtype=torch.int32, device="cuda")
        scratch = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
        s = torch.cuda.Stream()
        src.normal_()
        with torch.cuda.stream(s):
            ops.compress_data(True, ts, False, scratch, comp, sizes, archive_dtype=dtype)  # warm-up outside the capture
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            ops.compress_data(True, ts, False, scratch, comp, sizes, archive_dtype=dtype)
        for seed in (1, 2):
            for i in range(members):
                src[i].copy_(torch.from_numpy(family(FAMILIES[(i + seed) % len(FAMILIES)], n, seed=seed * 1000 + i)
                                              .view(np.float32)))
            comp.zero_()
            g.replay()
            torch.cuda.synchronize()
            hs = sizes.cpu().tolist()
            want_comp, want_sizes, _ = ops.compress_data(True, [t.to(dtype) for t in ts])
            assert hs == want_sizes.cpu().tolist()
            host, whost = comp.cpu().numpy(), want_comp.cpu().numpy()
            for i in range(members):
                O.assert_same_float(host[i, :hs[i]], whost[i, :hs[i]], KINDS[TYPES[dtype]][0], f"replay {seed} member {i}")
            guarded_decode(True, [comp[i, :hs[i]] for i in range(members)], [n] * members, dtype, 10, False,
                           [t.to(dtype) for t in ts], f"replay {seed}")


def test_same_type_pairs_equal_compress_pointer():
    from dietgpu_b200 import capi

    for dtype, ft in ((torch.float16, capi.FLOAT16), (torch.bfloat16, capi.BFLOAT16), (torch.float32, capi.FLOAT32)):
        ts = [torch.randn(n, device="cuda").to(dtype) for n in (1, 4097, 300001)]
        from dietgpu_b200 import ops

        cols = ops.max_float_compressed_size(torch.empty(0, dtype=dtype), 300001)
        for canonical in (1, 0):
            res = []
            with codec_options(encode_canonical=canonical):
                for in_ft in (ft, None):  # dgb_float_compress_to(ft, ft), then dgb_float_compress_pointer
                    comp = torch.zeros(3, cols, dtype=torch.uint8, device="cuda")
                    sizes = torch.zeros(3, dtype=torch.int32, device="cuda")
                    _raw_compress_to(in_ft, ft, ts, [comp[i] for i in range(3)], sizes, checksum=True)
                    res.append((comp.cpu().numpy(), sizes.cpu().tolist()))
            assert res[0][1] == res[1][1]
            for i in range(3):
                a, b = res[0][0][i, :res[0][1][i]], res[1][0][i, :res[1][1][i]]
                if canonical:
                    assert np.array_equal(a, b), (dtype, i)
                else:
                    O.assert_same_float(a, b, ft, f"{dtype} member {i}")


# ---- large members ------------------------------------------------------------------------------------------------

def test_large_members_64x2mi_bf16():
    from dietgpu_b200 import ops

    members, n = 64, 2 << 20
    g = torch.Generator(device="cuda").manual_seed(5)
    src = torch.randn(members, n, device="cuda", generator=g)
    src[:, ::1001] = float("nan")
    ts = [src[i] for i in range(members)]
    comp, sizes, _ = ops.compress_data(True, ts, archive_dtype=torch.bfloat16)
    hs = sizes.cpu().tolist()
    casts = [t.to(torch.bfloat16) for t in ts]
    want_comp, want_sizes, _ = ops.compress_data(True, casts)
    assert hs == want_sizes.cpu().tolist()
    for i in range(members):
        a = comp[i, :hs[i]].cpu().numpy()
        assert_pdf_matches(a, casts[i], "bf16", 10, f"member {i}")
        O.assert_same_float(a, want_comp[i, :hs[i]].cpu().numpy(), O.BF16, f"member {i}")
    guarded_decode(True, [comp[i, :hs[i]] for i in range(members)], [n] * members, torch.bfloat16, 10, False, casts,
                   "64 x 2 Mi")


def test_reference_decodes_narrowing_archives():
    from oracle import ref_lib

    if not ref_lib.available():
        pytest.skip("oracle/_ref was not built (the reference's sources were absent at build time)")
    from dietgpu_b200 import ops

    ts = placed_inputs([family(f, n, seed=3) for f, n in zip(FAMILIES, [1, 33, 4097, 8209, 300001, 65536, 1000, 77])],
                       "f32", [0] * 8)
    for dtype in TYPES:
        comp, sizes, _ = ops.compress_data(True, ts, archive_dtype=dtype)
        hs = sizes.cpu().tolist()
        outs = [torch.empty(t.numel(), dtype=dtype, device="cuda") for t in ts]
        st = torch.zeros(len(ts), dtype=torch.uint8, device="cuda")
        rc = ref_lib.RefCodec(256 << 20).float_decompress(KINDS[TYPES[dtype]][0], [comp[i, :hs[i]] for i in range(len(ts))],
                                                          outs, st)
        torch.cuda.synchronize()
        assert rc == 0 and bool(st.all())
        for t, o in zip(ts, outs):
            assert torch.equal(_bits(o), _bits(t.to(dtype))), dtype


# ---- collectives --------------------------------------------------------------------------------------------------

def test_single_process_collectives_follow_the_formulas():
    import dietgpu_b200 as dg

    t = torch.from_numpy(family("special", 80000, seed=9).view(np.float32)).cuda()
    for w in TYPES:
        assert torch.equal(_bits(dg.all_gather_compressed(t, wire_dtype=w)), _bits(t.to(w)))
        got = dg.reduce_scatter_compressed(t, wire_dtype=w)
        want = t.to(w).float()
        assert got.dtype == torch.float32 and torch.equal(_bits(got), _bits(want))
        assert torch.equal(_bits(dg.reduce_scatter_compressed(t, wire_dtype=w, reduce_dtype=torch.float32)), _bits(want))
    assert "wire_dtype" not in inspect.signature(dg.all_reduce_compressed).parameters


def _refusals(dg, dev):
    f32 = torch.zeros(16, dtype=torch.float32, device=dev)
    bf = torch.zeros(16, dtype=torch.bfloat16, device=dev)
    calls = [
        lambda: dg.all_gather_compressed(bf, wire_dtype=torch.float16),             # a 16-bit t
        lambda: dg.all_gather_compressed(f32, wire_dtype=torch.float32),            # not a 16-bit wire
        lambda: dg.all_gather_compressed(f32, wire_dtype=torch.float64),
        lambda: dg.all_gather_compressed(f32, wire_dtype=torch.bfloat16, peer=object()),  # peer transports
        lambda: dg.reduce_scatter_compressed(bf, wire_dtype=torch.float16),
        lambda: dg.reduce_scatter_compressed(bf, wire_dtype=torch.bfloat16),
        lambda: dg.reduce_scatter_compressed(f32, wire_dtype=torch.float32),
        lambda: dg.reduce_scatter_compressed(f32, wire_dtype=torch.bfloat16, reduce_dtype=torch.bfloat16),
        lambda: dg.reduce_scatter_compressed(f32, wire_dtype=torch.float16, reduce_dtype=torch.float16),
        lambda: dg.reduce_scatter_compressed(f32, reduce_dtype=torch.float16),      # an existing refusal
    ]
    for k, call in enumerate(calls):
        try:
            call()
        except ValueError:
            continue
        return f"refusal {k} did not raise ValueError"
    return "ok"


def test_refusals_single_process():
    import dietgpu_b200 as dg

    assert _refusals(dg, "cuda") == "ok"


def _worker(rank, world, dev):
    import dietgpu_b200 as dg

    def same(a, b):  # NaN compared as "both NaN" (a sum's NaN payload is not part of the formula)
        nan = torch.isnan(a) & torch.isnan(b)
        return a.dtype == b.dtype and a.shape == b.shape and not bool(((_bits(a) != _bits(b)) & ~nan).any())

    for w in TYPES:
        for n in (2 * 40000, 300002):
            ts = []
            for r in range(world):
                g = torch.Generator(device="cpu").manual_seed(900 + r + n)
                x = torch.randn(n, generator=g) * (1 + r)
                x[::97] = float("nan") if r == 1 else 0.0
                x[5::89] = -0.0
                x[7::211] = float("inf") if r == 0 else float("-inf")
                x[9::301] = 70000.0  # above fp16's range: +Inf in fp16, finite in bf16
                ts.append(x.to(dev))
            for members in (1, 6):
                got = dg.all_gather_compressed(ts[rank], members=members, wire_dtype=w)
                assert torch.equal(_bits(got), _bits(torch.cat([t.to(w) for t in ts]))), f"all_gather {w} {n} {members}"
                shard = n // world
                want = ts[0].to(w).float()
                for t in ts[1:]:
                    want = want + t.to(w).float()
                got = dg.reduce_scatter_compressed(ts[rank], members=members, wire_dtype=w)
                assert same(got, want[rank * shard:(rank + 1) * shard]), f"reduce_scatter {w} {n} {members}"
    refused = _refusals(dg, dev)
    assert refused == "ok", refused


def test_two_rank_collectives_with_a_16_bit_wire():
    run_ranks(_worker, 2, timeout=300)
