"""Narrowing compress with error feedback (dgb_float_compress_to_ef / ops.compress_data(error_feedback=)).

For float32 inputs x and residuals e, every case is checked against torch on the device: the archive must be the
narrowing compress of y = x + e (byte for byte with encode_canonical = 1, field for field and decoded word for word
by default), the residuals must be torch.where(w.isfinite(), y - w.float(), 0) with w = y.to(T) bit for bit, and the
inputs must be unchanged."""
import numpy as np
import pytest
import torch

from codec_helpers import KINDS, SENTINEL, codec_options, guarded_decode, placed_inputs
from oracle import oracle as O
from test_gpu_narrow import FAMILIES, TYPES, family

pytestmark = pytest.mark.gpu

SIZES = [0, 1, 2, 3, 4095, 4096, 4097, (2 << 20) + 5]


def _bits(t):
    return t.view(torch.int32 if t.element_size() == 4 else torch.int16)


def torch_step(x, e, dtype):
    """(y, residual) of the contract, computed by torch on the device"""
    y = x + e
    w = y.to(dtype)
    return y, torch.where(w.isfinite(), y - w.float(), 0)


def residual_pool(n, seed):
    """Residuals of the size a previous step leaves (up to half an ulp of the word), with zeros, signed zeros and a
    few large and non-finite values (a caller's buffer may hold anything)."""
    r = np.random.default_rng(seed)
    e = (r.standard_normal(n) * np.exp2(r.integers(-30, 2, n))).astype(np.float32)
    e[::5] = 0.0
    e[1::11] = -0.0
    e[2::97] = 3e4
    e[3::1009] = np.inf
    e[4::1013] = np.nan
    return e.view(np.uint32)


def clone_placed(t):
    """A copy of t at the same address modulo 16 (a plain clone starts 16 B aligned)."""
    off = (t.data_ptr() % 16) // t.element_size()
    buf = torch.empty(t.numel() + off, dtype=t.dtype, device=t.device)
    assert buf.data_ptr() % 16 == 0
    return buf[off:].copy_(t)


def make_case(sizes, offsets, seed=0):
    """Inputs and residual buffers at the same element offsets (so the same address modulo 16)."""
    xs = [family(FAMILIES[(i + seed) % len(FAMILIES)], max(n, 1), seed=seed + i)[:n] for i, n in enumerate(sizes)]
    es = [residual_pool(max(n, 1), seed + 7 * i)[:n] for i, n in enumerate(sizes)]
    return placed_inputs(xs, "f32", offsets), placed_inputs(es, "f32", offsets)


def check_ef(xs, es, dtype, pb=10, checksum=False, canonical=False, what=""):
    """One compress_data(error_feedback=) call against torch's y = x + e and the compress of y; returns the archives
    (device rows) and sizes."""
    from dietgpu_b200 import ops

    ys, want_res = zip(*[torch_step(x, e, dtype) for x, e in zip(xs, es)])
    x_before = [_bits(x).clone() for x in xs]
    n = len(xs)
    cols = ops.max_float_compressed_size(torch.empty(0, dtype=dtype), max(max(x.numel() for x in xs), 1))
    comp = torch.full((n, cols), SENTINEL, dtype=torch.uint8, device="cuda")
    with codec_options(encode_canonical=int(canonical)):
        _, sizes, _ = ops.compress_data(True, xs, checksum, None, comp, None, prob_bits=pb, archive_dtype=dtype,
                                        error_feedback=list(es))
        want_comp, want_sizes, _ = ops.compress_data(True, list(ys), checksum, prob_bits=pb, archive_dtype=dtype)
    hs, whs = sizes.cpu().tolist(), want_sizes.cpu().tolist()
    assert hs == whs, f"{what}: sizes {hs} != the compress of x + e {whs}"
    for i in range(n):
        assert torch.equal(_bits(xs[i]), x_before[i]), f"{what} member {i}: the input changed"
        bad = _bits(es[i]) != _bits(want_res[i])
        assert not bool(bad.any()), f"{what} member {i}: residual differs at {bad.nonzero().flatten()[:8].tolist()}"
        a, b = comp[i, :hs[i]].cpu().numpy(), want_comp[i, :hs[i]].cpu().numpy()
        if canonical:
            assert np.array_equal(a, b), f"{what} member {i}: canonical archive differs from the compress of x + e"
        else:
            O.assert_same_float(a, b, KINDS[TYPES[dtype]][0], f"{what} member {i}")
    rows = [comp[i, :hs[i]] for i in range(n)]
    guarded_decode(True, rows, [x.numel() for x in xs], dtype, pb, checksum, [y.to(dtype) for y in ys], what)
    return rows, hs


@pytest.mark.parametrize("dtype", list(TYPES))
@pytest.mark.parametrize("pb", [9, 10, 11])
@pytest.mark.parametrize("checksum", [False, True])
def test_sizes_and_offsets(dtype, pb, checksum):
    sizes = [n for n in SIZES for _ in range(4)]
    offsets = [off for _ in SIZES for off in range(4)]  # 0, 4, 8 and 12 B past a 16 B boundary
    xs, es = make_case(sizes, offsets, seed=pb)
    for canonical in (False, True):
        es_now = [clone_placed(e) for e in es]
        check_ef(xs, es_now, dtype, pb, checksum, canonical, f"{dtype} pb {pb} checksum {checksum} canonical {canonical}")


@pytest.mark.parametrize("dtype", list(TYPES))
@pytest.mark.parametrize("members,inline", [(64, 1), (64, 0), (65, 1)])
def test_batches_on_both_residual_tables(dtype, members, inline):
    # up to 64 members the residual table travels in the kernel parameters, beyond (or without inline members) in
    # the scratch
    sizes = [(i * 7919) % 20011 for i in range(members)]
    xs, es = make_case(sizes, [i % 4 for i in range(members)], seed=members)
    with codec_options(inline_members=inline):
        for canonical in (False, True):
            check_ef(xs, [clone_placed(e) for e in es], dtype, 10, True, canonical, f"{dtype} {members} inline {inline}")


@pytest.mark.parametrize("opts", [dict(encode_fused=1), dict(stats_stage=1), dict(encode_wide_table=0),
                                  dict(encode_wide_table=1), dict(parts=2), dict(parts=4),
                                  dict(encode_canonical=1, parts=1)], ids=str)
def test_option_variants_give_the_same_archives(opts):
    from dietgpu_b200 import ops

    sizes = [0, 1, 33, 4097, 65537, 300001, 1 << 20]
    xs, es = make_case(sizes, [i % 4 for i in range(len(sizes))], seed=11)
    for dtype in TYPES:
        base_es = [clone_placed(e) for e in es]
        base, base_sizes, _ = ops.compress_data(True, xs, True, archive_dtype=dtype, error_feedback=base_es)
        var_es = [clone_placed(e) for e in es]
        with codec_options(**opts):
            var, var_sizes, _ = ops.compress_data(True, xs, True, archive_dtype=dtype, error_feedback=var_es)
        hs = base_sizes.cpu().tolist()
        assert hs == var_sizes.cpu().tolist(), opts
        for i in range(len(xs)):
            assert torch.equal(_bits(base_es[i]), _bits(var_es[i])), (opts, dtype, i)
            O.assert_same_float(var[i, :hs[i]].cpu().numpy(), base[i, :hs[i]].cpu().numpy(), KINDS[TYPES[dtype]][0],
                                f"{opts} {dtype} member {i}")
        check_ef(xs, [clone_placed(e) for e in es], dtype, 10, True, False, f"{opts} {dtype}")


def _patterns(c, chunk, nonzero):
    v = torch.arange(c * chunk, (c + 1) * chunk, dtype=torch.int64, device="cuda")
    x = torch.where(v >= 1 << 31, v - (1 << 32), v).to(torch.int32).view(torch.float32)
    if not nonzero:
        return x, torch.zeros_like(x)
    # a fixed residual pattern: small values of both signs at assorted scales, and some exact zeros
    h = (v * 0x9E3779B1) & 0xFFFFFFFF
    e = ((h & 0x807FFFFF) | (((h >> 23) % 40 + 90) << 23)).to(torch.int64)
    e = torch.where(e >= 1 << 31, e - (1 << 32), e).to(torch.int32).view(torch.float32)
    return x, torch.where(h % 13 == 0, torch.zeros_like(e), e)


@pytest.mark.parametrize("nonzero", [False, True], ids=["e=0", "e=pattern"])
def test_every_fp32_bit_pattern(nonzero):
    from dietgpu_b200 import ops

    chunk, members = 1 << 28, 4
    per = chunk // members
    for c in range((1 << 32) // chunk):
        x, e0 = _patterns(c, chunk, nonzero)
        for dtype in TYPES:
            y, want_res = torch_step(x, e0, dtype)
            e = e0.clone()
            comp, sizes, _ = ops.compress_data(True, [x[i * per:(i + 1) * per] for i in range(members)],
                                               archive_dtype=dtype,
                                               error_feedback=[e[i * per:(i + 1) * per] for i in range(members)])
            hs = sizes.cpu().tolist()
            out = torch.empty(chunk, dtype=dtype, device="cuda")
            st = torch.zeros(members, dtype=torch.uint8, device="cuda")
            ops.decompress_data(True, [comp[i, :hs[i]] for i in range(members)],
                                [out[i * per:(i + 1) * per] for i in range(members)], False, None, st)
            assert bool(st.all()), (c, dtype)
            bad = _bits(out) != _bits(y.to(dtype))
            assert not bool(bad.any()), f"{dtype}: pattern {hex(c * chunk + int(bad.nonzero()[0]))} decodes differently"
            bad = _bits(e) != _bits(want_res)
            assert not bool(bad.any()), f"{dtype}: pattern {hex(c * chunk + int(bad.nonzero()[0]))}: residual differs"
            del comp, out, y, want_res, e
        del x, e0


@pytest.mark.parametrize("members", [6, 65])
def test_graph_replays_equal_eager_steps(members):
    from dietgpu_b200 import ops

    n, steps = 20011, 4
    for dtype in TYPES:
        src = torch.empty(members, n, dtype=torch.float32, device="cuda")
        err = torch.empty(members, n, dtype=torch.float32, device="cuda")
        ts, es = [src[i] for i in range(members)], [err[i] for i in range(members)]
        cols = ops.max_float_compressed_size(torch.empty(0, dtype=dtype), n)
        comp = torch.zeros(members, cols, dtype=torch.uint8, device="cuda")
        sizes = torch.zeros(members, dtype=torch.int32, device="cuda")
        scratch = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
        for i in range(members):
            src[i].copy_(torch.from_numpy(family(FAMILIES[i % len(FAMILIES)], n, seed=i).view(np.float32)))
        s = torch.cuda.Stream()
        err.zero_()
        with torch.cuda.stream(s):  # warm-up outside the capture
            ops.compress_data(True, ts, True, scratch, comp, sizes, archive_dtype=dtype, error_feedback=es)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            ops.compress_data(True, ts, True, scratch, comp, sizes, archive_dtype=dtype, error_feedback=es)
        e0 = torch.from_numpy(np.stack([residual_pool(n, 50 + i) for i in range(members)]).view(np.float32)).cuda()
        err.copy_(e0)
        eager = e0.clone()
        eager_es = [eager[i] for i in range(members)]
        for k in range(steps):
            comp.zero_()
            g.replay()
            torch.cuda.synchronize()
            want, want_sizes, _ = ops.compress_data(True, ts, True, archive_dtype=dtype, error_feedback=eager_es)
            hs = sizes.cpu().tolist()
            assert hs == want_sizes.cpu().tolist(), (dtype, k)
            assert torch.equal(_bits(err), _bits(eager)), (dtype, k)
            host, whost = comp.cpu().numpy(), want.cpu().numpy()
            for i in range(members):
                O.assert_same_float(host[i, :hs[i]], whost[i, :hs[i]], KINDS[TYPES[dtype]][0], f"replay {k} member {i}")


def test_large_batch_64x2mi():
    # the benchmark's shape: 64 members of 2 Mi words, canonical archives byte for byte
    g = torch.Generator(device="cuda").manual_seed(9)
    x = torch.randn(64, 2 << 20, device="cuda", generator=g)
    e = torch.randn(64, 2 << 20, device="cuda", generator=g) * 2 ** -9
    for dtype in TYPES:
        check_ef([x[i] for i in range(64)], [r.clone() for r in e], dtype, 10, False, True, f"64 x 2 Mi {dtype}")


def test_steps_accumulate_what_rounding_drops():
    # a constant gradient bf16 cannot hold: the mean of the sent words converges to it, within a bf16 ulp / steps
    from dietgpu_b200 import ops

    g = torch.full((4099,), 1 + 2 ** -10, device="cuda")
    for dtype, ulp in ((torch.bfloat16, 2 ** -7), (torch.float16, 2 ** -10)):
        e = torch.zeros_like(g)
        total = torch.zeros_like(g, dtype=torch.float64)
        steps = 256
        for _ in range(steps):
            comp, sizes, _ = ops.compress_data(True, [g], archive_dtype=dtype, error_feedback=[e])
            out = torch.empty(g.numel(), dtype=dtype, device="cuda")
            ops.decompress_data(True, [comp[0, :int(sizes[0])]], [out])
            total += out.double()
        err = (total / steps - (1 + 2 ** -10)).abs().max().item()
        assert err <= ulp / steps, (dtype, err)
        assert float(e.abs().max()) <= ulp / 2
