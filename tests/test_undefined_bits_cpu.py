"""The bits the reference leaves undefined, pinned to the CPU oracle (no GPU).

The reference writes its header flags by read-modify-write over uninitialised memory and never writes the ANS
header's options bits 5-31, its checksum when the flag is clear, unused0/1, the block table's pad entry, the
padding after each stream, the float header's options bits 5-31 and checksum (flag clear), or the padding after
each stored plane; the pdf of an empty member is whatever its scratch held.  codec_helpers.scribble fills exactly
those with garbage; here the oracle's decoders and info queries must not see the difference, and the field-wise
archive comparisons the parity tests use must still call a scribbled archive equal to its original."""
import numpy as np
import pytest

from codec_helpers import KINDS, scribble, undefined_mask, undefined_regions
from conftest import normal_words, zipf_bytes
from oracle import oracle as O

# block counts 0, 1, even (2, 4) and odd (3, 25); lengths that leave ragged last blocks and plane padding
LENGTHS = (0, 1, 4095, 8192, 4096 * 2 + 17, 4096 * 3 + 1, 100001)


def _blocks(n):
    return (n + 4095) // 4096


assert {_blocks(n) for n in LENGTHS} >= {0, 1, 2, 3, 4, 25}


def _words(kind, n, seed):
    return normal_words(n, kind, seed)


@pytest.mark.parametrize("checksum", [False, True])
@pytest.mark.parametrize("pb", [9, 10, 11])
def test_ans_readers_ignore_undefined_bits(pb, checksum):
    rng = np.random.default_rng(100 * pb + checksum)
    for n in LENGTHS:
        data = zipf_bytes(n, 1.1, n)
        arch = O.ans_encode(data, pb, checksum)
        bad = scribble(arch, rng)
        assert not np.array_equal(bad, arch)
        what = f"pb {pb} checksum {checksum} n {n}"
        want, got = O.ans_info(arch), O.ans_info(bad)
        if not checksum:
            want.pop("checksum"), got.pop("checksum")
        assert got == want, what
        for verify in (False, True):
            rc0, out0, n0 = O.ans_decode(arch, pb, verify_checksum=verify)
            rc1, out1, n1 = O.ans_decode(bad, pb, verify_checksum=verify)
            assert rc0 == O.OK and (rc1, n1) == (rc0, n0) and np.array_equal(out1, out0), what
            assert np.array_equal(out1, data), what
        O.assert_same_ans(bad, arch, what)
        O.assert_same_ans(arch, bad, what)


@pytest.mark.parametrize("checksum", [False, True])
@pytest.mark.parametrize("pb", [9, 10, 11])
@pytest.mark.parametrize("kind", ["f16", "bf16", "f32"])
def test_float_readers_ignore_undefined_bits(kind, pb, checksum):
    ft = KINDS[kind][0]
    rng = np.random.default_rng(1000 * ft + 10 * pb + checksum)
    for n in LENGTHS:
        w = _words(kind, n, n)
        arch = O.float_compress(ft, w, pb, checksum)
        bad = scribble(arch, rng)
        what = f"{kind} pb {pb} checksum {checksum} n {n}"
        want, got = O.float_info(arch), O.float_info(bad)
        if not checksum:
            want.pop("checksum"), got.pop("checksum")
        assert got == want, what
        for verify in (False, True):
            rc0, out0, n0 = O.float_decompress(ft, arch, pb, verify_checksum=verify)
            rc1, out1, n1 = O.float_decompress(ft, bad, pb, verify_checksum=verify)
            assert rc0 == O.OK and (rc1, n1) == (rc0, n0) and np.array_equal(out1, out0), what
            assert np.array_equal(out1, w), what
        O.assert_same_float(bad, arch, ft, what)
        O.assert_same_float(arch, bad, ft, what)


def test_undefined_set_is_the_documented_list():
    """The regions of a checksum-less fp32 archive of 3 blocks (odd: a pad entry) and of a checksummed byte
    archive of 2 blocks, named field by field, and nothing outside them changes."""
    w = _words("f32", 4096 * 2 + 17, 5)
    arch = O.float_compress(O.F32, w, 10, False)
    names = [r[0] for r in undefined_regions(arch)]
    assert names[:5] == ["float options bits 5-31", "float checksum (flag clear)", "plane padding", "plane padding",
                         "ans options bits 5-31"]
    assert names[5:8] == ["ans checksum (flag clear)", "ans unused0/1", "block table pad entry"]
    assert set(names[8:]) <= {"stream padding"}
    m = undefined_mask(arch)
    assert list(m[8:16]) == [0xE0, 0xFF, 0xFF, 0xFF] + [0xFF] * 4
    nc = O.float_noncomp_bytes(O.F32, w.size)
    assert list(m[16 + nc + 16:16 + nc + 20]) == [0xE0, 0xFF, 0xFF, 0xFF]
    bad = scribble(arch, np.random.default_rng(1))
    assert not np.any((bad ^ arch) & ~m)

    b = O.ans_encode(zipf_bytes(8192, 1.1, 2), 11, True)
    names = [r[0] for r in undefined_regions(b)]
    assert names[:2] == ["ans options bits 5-31", "ans unused0/1"]  # checksum defined, no pad entry
    assert set(names[2:]) <= {"stream padding"}

    # an empty member: no blocks, and its pdf is undefined
    e = O.ans_encode(np.zeros(0, np.uint8), 10, False)
    assert [r[0] for r in undefined_regions(e)] == ["ans options bits 5-31", "ans checksum (flag clear)",
                                                    "ans unused0/1", "pdf of an empty archive"]
    assert not np.array_equal(scribble(e, np.random.default_rng(2))[32:544], e[32:544])
