"""Every GPU reader ignores the bits the reference leaves undefined (codec_helpers.scribble): ANS options bits
5-31, the checksum when its flag is clear, unused0/1, the block table's pad entry, stream padding, the float
header's options bits 5-31 and checksum (flag clear), the padding after each stored plane, and the pdf of an
empty member.  The reference writes its archives over whatever its output buffer (or, for that pdf, its scratch)
held, so a reader that looked at any of these would refuse (or misread) archives it wrote into a reused buffer.

Each reader runs on the edge corpora of test_gpu_variants.py (bytes, fp16, bf16, fp32 at probBits 9-11),
encoded by the library and then scribbled, and must give bit for bit what the same call gives on the
unscribbled archives (outputs, statuses, sizes, found_inf, norms).  Needs no reference build."""
import functools
import zlib

import numpy as np
import pytest
import torch

from codec_helpers import KINDS, codec_options, scribble, to_dev_bytes, words_to_tensor
from conftest import normal_words, zipf_bytes
from test_gpu_variants import corpus

pytestmark = pytest.mark.gpu

PBS = (9, 10, 11)
ALL_KINDS = ("bytes", "f16", "bf16", "f32")
TDT = {"bytes": torch.uint8, "f16": torch.float16, "bf16": torch.bfloat16, "f32": torch.float32}
INT = {torch.uint8: torch.uint8, torch.float16: torch.int16, torch.bfloat16: torch.int16, torch.float32: torch.int32}
S8 = 0xA5

# decoder-only variants of test_gpu_variants.VARIANTS, and the member tables read from scratch
DECODE_VARIANTS = [
    ("defaults", {}),
    ("decode_warps4", dict(decode_warps=4)),
    ("decode_warps8", dict(decode_warps=8)),
    ("decode_warps20", dict(decode_warps=20)),
    ("decode_two_kernel", dict(decode_fused=0)),
    ("decode_slot_min", dict(decode_slot_words=1)),
    ("inline_members0", dict(inline_members=0)),
]


def dg():
    import dietgpu_b200

    return dietgpu_b200


def ints(t):
    return t.view(INT[t.dtype])


def rng_for(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


@functools.lru_cache(None)
def archives(kind, pb, checksum):
    """(inputs, clean device rows, scribbled device rows, host archives) of kind's corpus, encoded by the
    library with the given checksum flag."""
    c = corpus(kind)
    ts = [to_dev_bytes(a) if kind == "bytes" else words_to_tensor(a, kind) for a in c]
    comp, sizes, _ = dg().compress_data(kind != "bytes", ts, checksum, prob_bits=pb)
    hs = sizes.cpu().tolist()
    host = [comp[i, :hs[i]].cpu().numpy() for i in range(len(ts))]
    rng = np.random.default_rng(7919 * pb + 31 * ALL_KINDS.index(kind) + checksum)
    bad = [scribble(a, rng) for a in host]
    return ts, [to_dev_bytes(a) for a in host], [to_dev_bytes(a) for a in bad], host


def decode(kind, rows, ts, pb, checksum, fn=None):
    """(outputs, status, sizes, error) of one decompress_data call into sentinel-filled outputs."""
    outs = [torch.full((t.numel(),), 0x5A, dtype=INT[t.dtype], device="cuda").view(t.dtype) for t in ts]
    st = torch.zeros(len(rows), dtype=torch.uint8, device="cuda")
    sz = torch.zeros(len(rows), dtype=torch.int32, device="cuda")
    err = None
    try:
        (fn or dg().decompress_data)(kind != "bytes", rows, outs, checksum, None, st, sz, prob_bits=pb)
    except RuntimeError as e:
        err = str(e)
    torch.cuda.synchronize()
    return outs, st.cpu().tolist(), sz.cpu().tolist(), err


def assert_same_decode(got, want, what):
    outs1, st1, sz1, err1 = got
    outs0, st0, sz0, err0 = want
    assert (st1, sz1, err1) == (st0, sz0, err0), f"{what}: status / sizes / error differ"
    for i, (a, b) in enumerate(zip(outs1, outs0)):
        assert torch.equal(ints(a), ints(b)), f"{what}: member {i} decodes differently"


def assert_decodes_inputs(res, ts, what):
    outs, st, sz, err = res
    assert err is None and st == [1] * len(ts) and sz == [t.numel() for t in ts], f"{what}: {err} {st}"
    for i, (o, t) in enumerate(zip(outs, ts)):
        assert torch.equal(ints(o), ints(t)), f"{what}: member {i}"


def _decoder_cells():
    for kind in ALL_KINDS:
        for pb in PBS:
            for name, opts in DECODE_VARIANTS:
                if name == "decode_warps20" and kind != "bytes":
                    continue  # 20-warp CTAs exist for byte archives only
                yield pytest.param(kind, pb, opts, id=f"{kind}-pb{pb}-{name}")


@pytest.mark.parametrize("kind,pb,opts", list(_decoder_cells()))
def test_decoders_ignore_undefined_bits(kind, pb, opts):
    with codec_options(**opts):
        for checksum_flag in (False, True):
            ts, clean, bad, _ = archives(kind, pb, checksum_flag)
            # verification on: the flag-set archives carry a defined checksum that must match; with the flag
            # clear the checksum word is garbage and must not be verified
            for verify in (False, True):
                what = f"flag {checksum_flag} verify {verify}"
                want = decode(kind, clean, ts, pb, verify)
                assert_decodes_inputs(want, ts, what)
                assert_same_decode(decode(kind, bad, ts, pb, verify), want, what)


def test_checksum_mismatch_still_detected_under_scribble():
    """Garbage in the undefined set does not switch verification off: a flag-set archive whose checksum word
    is wrong still fails, scribbled or not."""
    ts, _, bad, _ = archives("bytes", 10, True)
    i = max(range(len(ts)), key=lambda k: ts[k].numel())
    wrong = bad[i].clone()
    wrong[20] ^= 0x5A
    outs = [torch.empty_like(ts[i])]
    with pytest.raises(RuntimeError, match="checksum mismatch"):
        dg().decompress_data(False, [wrong], outs, True, prob_bits=10)


@pytest.mark.parametrize("kind", ALL_KINDS)
def test_other_decode_entry_points_ignore_undefined_bits(kind):
    """Split-size decode, torch.ops.dietgpu and HostCodec.decompress: one call each, at probBits 10 (the
    operators' and HostCodec's default) with checksums set and verified."""
    from dietgpu_b200 import torch_library

    as_float = kind != "bytes"
    ts, clean, bad, host = archives(kind, 10, True)
    keep = [i for i, t in enumerate(ts) if t.numel() > 0]  # split sizes are positive
    splits = torch.tensor([ts[i].numel() for i in keep], dtype=torch.int32)
    res = []
    for rows in (clean, bad):
        flat = torch.full((int(splits.sum()),), 0x5A, dtype=INT[ts[0].dtype], device="cuda").view(ts[0].dtype)
        st = torch.zeros(len(keep), dtype=torch.uint8, device="cuda")
        dg().decompress_data_split_size(as_float, [rows[i] for i in keep], flat, splits, True, None, st,
                                        prob_bits=10)
        res.append((ints(flat).cpu(), st.cpu().tolist()))
    assert res[1][1] == res[0][1] == [1] * len(keep)
    assert torch.equal(res[1][0], res[0][0])
    assert torch.equal(res[0][0], torch.cat([ints(ts[i]).cpu() for i in keep]))

    ops = torch_library.load()
    assert_same_decode(decode(kind, bad, ts, 10, True, lambda f, r, o, c, tm, s, z, prob_bits: ops.decompress_data(
        f, r, o, c, tm, s, z)), decode(kind, clean, ts, 10, True), "torch.ops.dietgpu.decompress_data")

    host_in = [ints(t).cpu().view(t.dtype).pin_memory() for t in ts]
    hc = dg().HostCodec(as_float, host_in, groups=3, checksum=True)
    out = []
    for arch in (host, [scribble(a, rng_for("host", kind)) for a in host]):
        rows = torch.zeros((len(arch), hc.max_archive_bytes()), dtype=torch.uint8).pin_memory()
        for i, a in enumerate(arch):
            rows[i, :a.size] = torch.from_numpy(a)
        host_out = [torch.empty_like(t).pin_memory() for t in host_in]
        hc.decompress([rows[i, :a.size] for i, a in enumerate(arch)], host_out)
        out.append(host_out)
    for a, b, t in zip(out[0], out[1], host_in):
        assert torch.equal(ints(b), ints(a)) and torch.equal(ints(a), ints(t))


def info(kind, rows):
    """(sizes, types, checksums) from dgb_ans_get_compressed_info / dgb_float_get_compressed_info."""
    from dietgpu_b200 import capi

    L, n = capi.lib(), len(rows)
    sizes, types, cks = (torch.full((n,), 0x7777, dtype=torch.int32, device="cuda") for _ in range(3))
    temp = torch.empty(8 * n + 256, dtype=torch.uint8, device="cuda")
    ptrs = capi.ptr_array([r.data_ptr() for r in rows])
    st = torch.cuda.current_stream().cuda_stream
    if kind == "bytes":
        rc = L.dgb_ans_get_compressed_info(temp.data_ptr(), temp.numel(), ptrs, 0, n, sizes.data_ptr(),
                                           cks.data_ptr(), st)
    else:
        rc = L.dgb_float_get_compressed_info(temp.data_ptr(), temp.numel(), ptrs, 0, n, sizes.data_ptr(),
                                             types.data_ptr(), cks.data_ptr(), st)
    capi.check(rc, "get_compressed_info")
    return sizes.cpu().tolist(), types.cpu().tolist(), cks.cpu().tolist()


@pytest.mark.parametrize("checksum", [False, True])
@pytest.mark.parametrize("kind", ALL_KINDS)
def test_info_queries_ignore_undefined_bits(kind, checksum):
    for pb in PBS:
        ts, clean, bad, _ = archives(kind, pb, checksum)
        s0, t0, c0 = info(kind, clean)
        s1, t1, c1 = info(kind, bad)
        assert s1 == s0 == [t.numel() for t in ts], f"pb {pb}: sizes"
        if kind != "bytes":
            assert t1 == t0 == [KINDS[kind][0]] * len(ts), f"pb {pb}: float types"
        if checksum:
            assert c1 == c0, f"pb {pb}: checksums"


@pytest.mark.parametrize("kind", ALL_KINDS)
def test_archive_mover_copies_exactly_the_archive(kind):
    """pull_archives reads each archive's length from its defined fields: the scribbled archives are copied
    byte for byte, nothing past them is written, and the reported sizes are the unscribbled ones."""
    for pb in PBS:
        ts, clean, bad, host = archives(kind, pb, pb == 10)
        room = 64
        dst = [torch.full((a.size + room,), S8, dtype=torch.uint8, device="cuda") for a in host]
        ob = torch.zeros(len(bad), dtype=torch.int32, device="cuda")
        dg().ops.pull_archives(kind != "bytes", bad, dst, TDT[kind] if kind != "bytes" else None, ob)
        torch.cuda.synchronize()
        assert ob.cpu().tolist() == [a.size for a in host], f"pb {pb}: reported sizes"
        for i, (d, b) in enumerate(zip(dst, bad)):
            assert torch.equal(d[:b.numel()], b), f"pb {pb} member {i}: copy differs"
            assert bool((d[b.numel():] == S8).all()), f"pb {pb} member {i}: written past the archive"


# ---- decode-and-sum -----------------------------------------------------------------------------------

REDUCE_LENGTHS = (1, 4097, 70001)


def reduce_groups(kind, W, pb, seed):
    """G = 3 groups of W fp16 / bf16 / fp32 archives of REDUCE_LENGTHS[g] words each: (clean rows, scribbled
    rows), both [G][W] device tensors.  Large magnitudes so that some sums overflow fp16."""
    ft = KINDS[kind][0]
    clean, bad = [], []
    rng = rng_for("reduce", kind, W, pb, seed)
    for g, n in enumerate(REDUCE_LENGTHS):
        ws = [normal_words(n, kind, seed + 97 * g + j) for j in range(W)]
        if kind == "f16":
            ws[0][: n // 3] |= np.uint16(0x7000)  # |x| >= 8192: sums of a few reach the fp16 infinity
        ts = [words_to_tensor(w, kind) for w in ws]
        comp, sizes, _ = dg().compress_data(True, ts, (g + W) % 2 == 1, prob_bits=pb)
        hs = sizes.cpu().tolist()
        host = [comp[j, :hs[j]].cpu().numpy() for j in range(W)]
        assert all(int(a[8:12].view(np.uint32)[0]) & 0xF == ft for a in host)
        clean.append([to_dev_bytes(a) for a in host])
        bad.append([to_dev_bytes(scribble(a, rng)) for a in host])
    return clean, bad


def _families(kind):
    """(name, archive kind, output dtype, keyword builder) of every decode-and-sum family for one archive kind."""
    tdt = TDT[kind]
    fam = [("same", tdt, {}),
           ("host_scaled", tdt, dict(scale=0.37)),
           ("dev_scale_found_inf", tdt, dict(scale_tensor=3.0, found_inf=True)),
           ("sq_norm", tdt, dict(scale_tensor=0.5, found_inf=True, sq_norm=True))]
    if kind != "f32":
        fam += [("widening", torch.float32, dict(archive_dtype=tdt)),
                ("widening_dev_scale", torch.float32, dict(archive_dtype=tdt, scale_tensor=2.0, found_inf=True)),
                ("narrowing", tdt, dict(reduce_dtype=torch.float32)),
                ("narrowing_sq_norm", tdt, dict(reduce_dtype=torch.float32, scale_tensor=1.5, found_inf=True,
                                                sq_norm=True))]
    return fam


def run_reduce(groups, out_dtype, kw, pb):
    """One decompress_data_reduce call; returns (outputs, status, found_inf, sq_norm) on the host."""
    G = len(groups)
    outs = [torch.full((n,), 0x3C00 if out_dtype != torch.float32 else 0x3F800000, dtype=INT[out_dtype],
                       device="cuda").view(out_dtype) for n in REDUCE_LENGTHS[:G]]
    st = torch.zeros(G * len(groups[0]), dtype=torch.uint8, device="cuda")
    args = dict(kw)
    fi = sq = None
    if "scale_tensor" in args:
        args["scale_tensor"] = torch.tensor([args["scale_tensor"]], dtype=torch.float32, device="cuda")
    if args.pop("found_inf", False):
        fi = args["found_inf"] = torch.zeros(1, dtype=torch.float32, device="cuda")
    if args.pop("sq_norm", False):
        sq = args["sq_norm"] = torch.full((G,), -1.0, dtype=torch.float64, device="cuda")
    dg().decompress_data_reduce(groups, outs, False, None, st, prob_bits=pb, **args)
    torch.cuda.synchronize()
    # found_inf and the norms as bit patterns: NaN norms compare equal to themselves
    return ([ints(o).cpu() for o in outs], st.cpu().tolist(), None if fi is None else fi.view(torch.int32).item(),
            None if sq is None else sq.view(torch.int64).cpu().tolist())


def _reduce_cells():
    for kind in ("f16", "bf16", "f32"):
        for W, pb in ((1, 9), (2, 10), (5, 11)):
            yield pytest.param(kind, W, pb, {}, id=f"{kind}-W{W}-pb{pb}")
    # the fused decoder's other stream branch (staged copies) for most blocks
    for kind in ("f16", "f32"):
        yield pytest.param(kind, 2, 10, dict(decode_slot_words=8), id=f"{kind}-W2-pb10-slot8")


@pytest.mark.parametrize("kind,W,pb,opts", list(_reduce_cells()))
def test_decode_and_sum_ignores_undefined_bits(kind, W, pb, opts):
    clean, bad = reduce_groups(kind, W, pb, 11 * W + pb)
    with codec_options(**opts):
        for name, out_dtype, kw in _families(kind):
            want = run_reduce(clean, out_dtype, kw, pb)
            got = run_reduce(bad, out_dtype, kw, pb)
            assert want[1] == [1] * (len(clean) * W), f"{name}: clean archives refused: {want[1]}"
            assert got[1] == want[1], f"{name}: statuses {got[1]} != {want[1]}"
            assert got[2] == want[2], f"{name}: found_inf {got[2]} != {want[2]}"
            assert got[3] == want[3], f"{name}: squared norms {got[3]} != {want[3]}"
            for g, (a, b) in enumerate(zip(got[0], want[0])):
                assert torch.equal(a, b), f"{name}: group {g} sums differently"


# ---- the device-API decoder ---------------------------------------------------------------------------

@pytest.mark.parametrize("pb", PBS)
def test_device_api_decoder_ignores_undefined_bits(pb):
    """tileDecompress<PB> of tests/cpp/device_api_example.cu on the example's archives, scribbled."""
    from test_gpu_device_api import TILE, _tile_compress, _tile_decompress

    rng = rng_for("tile", pb)
    # 8-block tiles and a ragged 3-block tail; a constant 5-block tile (empty streams); one byte
    for data in (zipf_bytes(2 * TILE + 2 * 4096 + 5, 1.1, pb), np.full(5 * 4096, 9, np.uint8), zipf_bytes(1, 1.0, 3)):
        comp, stride, rows = _tile_compress(data, TILE, pb)
        tiles = len(rows)
        ok0, back0 = _tile_decompress(comp, stride, tiles, TILE, pb)
        assert ok0 == [1] * tiles and np.array_equal(back0[:data.size], data)
        bad = comp.clone()
        for i, r in enumerate(rows):
            bad[i, :r.numel()] = to_dev_bytes(scribble(r.cpu().numpy(), rng))
        ok1, back1 = _tile_decompress(bad, stride, tiles, TILE, pb)
        assert ok1 == ok0 and np.array_equal(back1, back0)
