"""Archive interchange with the reference itself (facebookresearch/dietgpu compiled unmodified for sm_90a into
oracle/_ref/ by oracle/build_ref.sh), in both directions and at scale, for the byte codec and the fp16 / bf16 /
fp32 float codec:
  * the reference's own undefined set: its archives of the same inputs written over 0x00 and over 0xFF differ
    only where codec_helpers.scribble may write; the 0xFF archives are the "reference archives" below.  The
    pdf of an empty member is undefined too: the reference copies it from a scratch table its statistics pass
    skips for empty members, so it changes with what earlier calls left there (the comparisons ignore it);
  * encode parity past 10 blocks and at probBits 9-11, checksum on and off: sizes, field-wise archives, the
    canonical encoder's archives byte for byte outside the undefined set, and the maximum-size bounds;
  * the reference decodes what every encoder variant of the library writes, the narrowing compress's archives
    and the large members;
  * the library decodes the reference's archives with every decoder variant, checksum verification, the info
    queries, the archive mover and every decode-and-sum family.

Guardrail: the reference encoder codes each 4 KiB block into 5120 B of scratch and does not check it (its
assert is compiled out), so every input handed to it first passes worst_block_bytes() below; the adversarial
worst-case corpora go to the library's encoder only."""
import functools

import numpy as np
import pytest
import torch

from codec_helpers import KINDS, codec_options, coded_bytes, to_dev_bytes, undefined_mask, undefined_regions, \
    words_to_tensor
from oracle import oracle as O
from oracle import ref_lib
from test_gpu_undefined_bits import (ALL_KINDS, DECODE_VARIANTS, INT, PBS, REDUCE_LENGTHS, TDT, _families,
                                     assert_decodes_inputs, decode, info, ints, run_reduce)
from test_gpu_variants import VARIANTS, corpus

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not ref_lib.available(),
                                 reason="the reference library oracle/_ref/libdietgpu_ref.so was not built "
                                        "(build() compiles it where the reference sources are present)")]

REF_BLOCK_SCRATCH = 5120  # bytes of per-block coder scratch in the reference encoder (ans/GpuANSEncode.cuh)
MIB = 1 << 20


def dg():
    import dietgpu_b200

    return dietgpu_b200


def ft_of(kind):
    return 0 if kind == "bytes" else KINDS[kind][0]


def worst_block_bytes(coded, pb):
    """Upper estimate of the largest block stream the ANS coder writes for the symbols `coded` (uint8 tensor):
    per 4 KiB block, the sum over its symbols of pb - log2 pdf(symbol) bits with the pdf O.normalize gives the
    member, plus one 32-bit state word per lane."""
    n = coded.numel()
    if n == 0:
        return 0.0
    hist = torch.bincount(coded.flatten().long(), minlength=256).cpu().numpy()
    pdf = O.normalize(hist.astype(np.uint32), n, pb).astype(np.float64)
    cost = np.where(pdf > 0, pb - np.log2(np.maximum(pdf, 1.0)), 0.0)
    bits = torch.tensor(cost, dtype=torch.float64, device=coded.device)[coded.flatten().long()]
    bits = torch.nn.functional.pad(bits, (0, (-n) % 4096)).view(-1, 4096).sum(1)
    return (float(bits.max()) + 32 * 32) / 8


def assert_ref_can_encode(kind, ts, pb):
    for i, t in enumerate(ts):
        w = worst_block_bytes(coded_bytes(t, kind), pb)
        assert w < REF_BLOCK_SCRATCH, f"member {i}: a block may need {w:.0f} B, past the reference's scratch"


def ref_codec(ts):
    """A RefCodec whose scratch is sized as bench.py sizes it: 2 x input bytes + 256 MiB."""
    return ref_lib.RefCodec(2 * sum(t.numel() * t.element_size() for t in ts) + 256 * MIB)


def ref_max_size(kind, n):
    L = ref_lib.lib()
    return L.ref_ans_max_compressed_size(n) if kind == "bytes" else L.ref_float_max_compressed_size(ft_of(kind), n)


def ref_encode(kind, ts, pb, checksum, fill):
    """The reference's archives of ts, written into rows prefilled with `fill`: (matrix, host sizes)."""
    assert_ref_can_encode(kind, ts, pb)
    n = len(ts)
    comp = torch.full((n, ref_max_size(kind, max(t.numel() for t in ts))), fill, dtype=torch.uint8, device="cuda")
    sizes = torch.zeros(n, dtype=torch.int32, device="cuda")
    ref = ref_codec(ts)
    if kind == "bytes":
        rc = ref.ans_encode(ts, comp, sizes, pb, checksum)
    else:
        rc = ref.float_compress(ft_of(kind), ts, comp, sizes, pb, checksum)
    assert rc == 0
    torch.cuda.synchronize()
    return comp, sizes.cpu().tolist()


def our_encode(kind, ts, pb, checksum, **opts):
    with codec_options(**opts):
        comp, sizes, _ = dg().compress_data(kind != "bytes", ts, checksum, prob_bits=pb)
    torch.cuda.synchronize()
    return comp, sizes.cpu().tolist()


def assert_same(kind, mine, theirs, what):
    if kind == "bytes":
        O.assert_same_ans(mine, theirs, what)
    else:
        O.assert_same_float(mine, theirs, ft_of(kind), what)


def assert_equal_outside_undefined(mine, theirs, what):
    assert mine.size == theirs.size, f"{what}: size"
    diff = (mine ^ theirs) & ~undefined_mask(theirs)
    if diff.any():
        at = int(np.flatnonzero(diff)[0])
        raise AssertionError(f"{what}: {int(np.count_nonzero(diff))} defined byte(s) differ, first at {at}")


def ref_decode(kind, rows, lengths, pb, checksum, aligned16=True):
    """The reference's decode of `rows`: (outputs, status, sizes, return code).  Outputs are views one word into
    their buffers unless aligned16 (then 16 B aligned)."""
    off = 0 if aligned16 else 1
    dt = TDT[kind]
    outs = [torch.full((n + 1,), 0x5A, dtype=INT[dt], device="cuda").view(dt)[off:off + n] for n in lengths]
    st = torch.zeros(len(rows), dtype=torch.uint8, device="cuda")
    sz = torch.zeros(len(rows), dtype=torch.int32, device="cuda")
    ref = ref_codec(outs)
    if kind == "bytes":
        rc = ref.ans_decode(rows, outs, st, sz, pb, checksum)
    else:
        rc = ref.float_decompress(ft_of(kind), rows, outs, st, sz, pb, checksum, aligned16)
    torch.cuda.synchronize()
    return outs, st.cpu().tolist(), sz.cpu().tolist(), rc


def assert_ref_decodes(kind, rows, ts, pb, checksum, what):
    lengths = [t.numel() for t in ts]
    for aligned16 in ((True,) if kind == "bytes" else (True, False)):
        outs, st, sz, rc = ref_decode(kind, rows, lengths, pb, checksum, aligned16)
        w = f"{what} aligned16={aligned16}"
        assert rc == 0 and st == [1] * len(ts) and sz == lengths, f"{w}: rc {rc} status {st} sizes {sz}"
        for i, (o, t) in enumerate(zip(outs, ts)):
            assert torch.equal(ints(o), ints(t)), f"{w}: member {i} decodes differently"


def member(kind, n, seed):
    """n seeded elements on the device: N(0, 1) words, or bytes of a rounded N(0, 24^2) (about 6.6 bits each)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, generator=g, device="cuda")
    if kind == "bytes":
        return (x * 24).round_().clamp_(-128, 127).to(torch.int8).view(torch.uint8)
    return x.to(TDT[kind])


def rows_of(comp, sizes):
    return [comp[i, :s] for i, s in enumerate(sizes)]


# ---- the reference's own undefined set ---------------------------------------------------------------

def ref_corpus(kind):
    """The edge corpus of test_gpu_variants.py without its adversarial worst-case member (a 4 KiB block of
    pdf-1 symbols: 5632 B at probBits 11), as device tensors."""
    c = corpus(kind)
    if kind == "bytes":
        c = c[:-1]
    return [to_dev_bytes(a) if kind == "bytes" else words_to_tensor(a, kind) for a in c]


@functools.lru_cache(None)
def ref_archives(kind, pb, checksum):
    """(inputs, reference archives over 0x00, reference archives over 0xFF) of ref_corpus(kind), host arrays."""
    ts = ref_corpus(kind)
    out = []
    for fill in (0x00, 0xFF):
        comp, sizes = ref_encode(kind, ts, pb, checksum, fill)
        out.append([a[:s].copy() for a, s in zip(comp.cpu().numpy(), sizes)])
    return ts, out[0], out[1]


@pytest.mark.parametrize("kind", ALL_KINDS)
def test_reference_undefined_set(kind):
    """The bytes that change with the reference's output buffer's prior contents all lie in scribble's set, and
    the reference's archives equal the oracle's field by field."""
    seen = {}
    for pb in PBS:
        for checksum in (False, True):
            ts, a00, aff = ref_archives(kind, pb, checksum)
            for i, (x, y, t) in enumerate(zip(a00, aff, ts)):
                what = f"{kind} pb {pb} checksum {checksum} member {i}"
                assert x.size == y.size, what
                d = x ^ y
                outside = d & ~undefined_mask(y)
                assert not outside.any(), \
                    f"{what}: {int(np.count_nonzero(outside))} byte(s) outside the undefined set depend on the buffer"
                for r in undefined_regions(y):
                    seen[r[0]] = seen.get(r[0], 0) + int(np.count_nonzero(d[r[1]:r[2]]))
                w = t.cpu().numpy() if kind == "bytes" else ints(t).cpu().numpy().view(KINDS[kind][2])
                want = O.ans_encode(w, pb, checksum) if kind == "bytes" else O.float_compress(ft_of(kind), w, pb, checksum)
                assert_same(kind, y, want, what)
    print(f"\nreference {kind} archives over 0x00 vs 0xFF, differing bytes per undefined field: "
          + ", ".join(f"{k}: {v}" for k, v in sorted(seen.items())) + "; none elsewhere")


# ---- encode parity past 10 blocks and at every probBits ----------------------------------------------

PARITY_LENGTHS = (0, 1, 4095, 4096, 4097, 1048573)  # 1048573 = 2^20 - 3 is prime
BATCH = 64  # members of 1 MiB elements each


def parity_members(kind):
    return [member(kind, n, 10 + i) for i, n in enumerate(PARITY_LENGTHS)] + \
           [member(kind, MIB, 100 + i) for i in range(BATCH)]


def check_parity(kind, ts, pb, checksum):
    what = f"{kind} pb {pb} checksum {checksum}"
    ref, rs = ref_encode(kind, ts, pb, checksum, 0xFF)
    mine, ms = our_encode(kind, ts, pb, checksum)
    canon, cs = our_encode(kind, ts, pb, checksum, encode_canonical=1)
    assert ms == rs == cs, f"{what}: compressed sizes differ from the reference's"
    ref_h, mine_h, canon_h = (m.cpu().numpy() for m in (ref, mine, canon))
    for i, s in enumerate(rs):
        assert_same(kind, mine_h[i, :s], ref_h[i, :s], f"{what} member {i}")
        # both lay the streams out in block order: byte for byte outside the undefined set
        assert_equal_outside_undefined(canon_h[i, :s], ref_h[i, :s], f"{what} canonical member {i}")
    # the reference decodes ours, we decode the reference's
    assert_ref_decodes(kind, rows_of(mine, ms), ts, pb, checksum, f"{what}: reference decode of ours")
    assert_decodes_inputs(decode(kind, rows_of(ref, rs), ts, pb, checksum), ts, f"{what}: our decode of the reference's")


@pytest.mark.parametrize("checksum", [False, True])
@pytest.mark.parametrize("pb", PBS)
@pytest.mark.parametrize("kind", ALL_KINDS)
def test_encode_parity_with_reference(kind, pb, checksum):
    ts = parity_members(kind)
    check_parity(kind, ts, pb, checksum)


def test_max_sizes_match_reference():
    L, R = dg().capi.lib(), ref_lib.lib()
    for n in PARITY_LENGTHS + (MIB, 300_000_001, 64 * MIB, BATCH * MIB):
        assert L.dgb_ans_max_compressed_size(n) == R.ref_ans_max_compressed_size(n), n
        for ft in (1, 2, 3):
            assert L.dgb_float_max_compressed_size(ft, n) == R.ref_float_max_compressed_size(ft, n), (n, ft)


@pytest.mark.parametrize("kind,n", [("bytes", 300_000_001), ("bf16", 64 * MIB + 3)])
def test_large_member_parity_with_reference(kind, n):
    """A byte member of 73243 blocks (past 65536) and a bf16 member of 64 Mi + 3 words, both directions."""
    if kind == "bytes":
        assert (n + 4095) // 4096 > 65536
    ts = [member(kind, n, 7)]
    check_parity(kind, ts, 10, True)


# ---- the reference decodes every encoder variant's archives -------------------------------------------
# The reference's decode loop (ans/GpuANSDecode.cuh, ansDecodeKernel and the warp block decoders it calls)
# reads each block's stream in place from the archive through its block-table offset; its only shared-memory
# buffer is the 2^probBits lookup table.  Nothing stages a stream into a fixed-size buffer, so the library's
# 5632 B worst-case block (pdf-1 symbols at probBits 11) is safe to hand it, and the variant corpora go to it
# whole.

def _encoder_cells():
    for kind in ALL_KINDS:
        for name, opts, role in VARIANTS:
            if role == "dec":
                continue
            if name.startswith("stats_stage") and kind == "bytes":
                continue
            yield pytest.param(kind, opts, id=f"{kind}-{name}")


@pytest.mark.parametrize("kind,opts", list(_encoder_cells()))
def test_reference_decodes_every_encoder_variant(kind, opts):
    c = corpus(kind)
    ts = [to_dev_bytes(a) if kind == "bytes" else words_to_tensor(a, kind) for a in c]
    for pb in PBS:
        checksum = pb == 10
        comp, sizes = our_encode(kind, ts, pb, checksum, **opts)
        assert_ref_decodes(kind, rows_of(comp, sizes), ts, pb, checksum, f"{kind} pb {pb} {opts}")


@pytest.mark.parametrize("kind", ["f16", "bf16"])
def test_reference_decodes_narrowing_compress(kind):
    c = corpus("f32")
    src = [words_to_tensor(a, "f32") for a in c]
    ts = [t.to(TDT[kind]) for t in src]
    for pb in PBS:
        comp, sizes, _ = dg().compress_data(True, src, pb == 11, prob_bits=pb, archive_dtype=TDT[kind])
        torch.cuda.synchronize()
        assert_ref_decodes(kind, rows_of(comp, sizes.cpu().tolist()), ts, pb, pb == 11, f"narrowing {kind} pb {pb}")


# ---- the library reads the reference's archives -------------------------------------------------------

def _ref_rows(kind, pb, checksum):
    ts, _, aff = ref_archives(kind, pb, checksum)
    return ts, [to_dev_bytes(a) for a in aff], aff


@pytest.mark.parametrize("kind", ALL_KINDS)
def test_library_reads_reference_archives(kind):
    """The 0xFF-prefilled reference archives through every decoder variant (checksums verified where the
    archives carry them, and requested where they do not), the info queries and the archive mover."""
    for pb in PBS:
        for checksum in (False, True):
            ts, rows, host = _ref_rows(kind, pb, checksum)
            for name, opts in DECODE_VARIANTS:
                if name == "decode_warps20" and kind != "bytes":
                    continue
                with codec_options(**opts):
                    for verify in (False, True):
                        assert_decodes_inputs(decode(kind, rows, ts, pb, verify), ts,
                                              f"{name} pb {pb} checksum {checksum} verify {verify}")
            sizes, types, cks = info(kind, rows)
            assert sizes == [t.numel() for t in ts]
            if kind != "bytes":
                assert types == [ft_of(kind)] * len(ts)
            if checksum:
                w = [O.checksum(t.cpu().numpy() if kind == "bytes" else ints(t).cpu().numpy(), t.numel())
                     for t in ts]
                assert [c & 0xFFFFFFFF for c in cks] == w
            dst = [torch.full((a.size + 64,), 0xA5, dtype=torch.uint8, device="cuda") for a in host]
            ob = torch.zeros(len(rows), dtype=torch.int32, device="cuda")
            dg().ops.pull_archives(kind != "bytes", rows, dst, TDT[kind] if kind != "bytes" else None, ob)
            torch.cuda.synchronize()
            assert ob.cpu().tolist() == [a.size for a in host]
            for i, (d, r) in enumerate(zip(dst, rows)):
                assert torch.equal(d[:r.numel()], r) and bool((d[r.numel():] == 0xA5).all()), f"pull member {i}"


@pytest.mark.parametrize("W,pb", [(1, 9), (2, 10), (5, 11)])
@pytest.mark.parametrize("kind", ["f16", "bf16", "f32"])
def test_decode_and_sum_of_reference_archives(kind, W, pb):
    """Groups of reference archives through every decode-and-sum family give bit for bit what the same call
    gives on the library's archives of the same words."""
    ours, theirs = [], []
    for g, n in enumerate(REDUCE_LENGTHS):
        ts = [member(kind, n, 1000 * W + 10 * g + j) for j in range(W)]
        if kind == "f16":
            ts[0][: n // 3] *= 8192  # sums of a few reach the fp16 infinity
        comp, sizes = our_encode(kind, ts, pb, g == 1)
        ours.append(rows_of(comp, sizes))
        comp, sizes = ref_encode(kind, ts, pb, g == 1, 0xFF)
        theirs.append(rows_of(comp, sizes))
    for name, out_dtype, kw in _families(kind):
        want = run_reduce(ours, out_dtype, kw, pb)
        got = run_reduce(theirs, out_dtype, kw, pb)
        assert want[1] == [1] * (len(ours) * W), f"{name}: our archives refused"
        assert got[1:] == want[1:], f"{name}: status / found_inf / squared norms differ"
        for g, (a, b) in enumerate(zip(got[0], want[0])):
            assert torch.equal(a, b), f"{name}: group {g} sums differently"
