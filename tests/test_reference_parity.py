"""GPU parity against the REFERENCE ITSELF: archives and size bounds that facebookresearch/dietgpu, compiled
unmodified for sm_90a (oracle/build_ref.sh), produced on an H100 for seeded inputs (tests/golden/ref_golden.npz,
written by tests/golden/make_ref_golden.py).  Pins what the reference's own tests leave unpinned (SURVEY 8c):
byte-exact compressed sizes, field-exact archives (masking only the bits the reference leaves undefined), and
decoding of the reference's archives.
These stored archives stop at 40000 bytes / 30001 floats (at most 10 blocks of 4 KiB) and, for floats, at probBits
10, so the file stays small and the checks here need no reference build.  Where build() compiled the reference
(oracle/_ref/), tests/test_gpu_reference_interchange.py runs it live: the reference decoding OUR archives (every
encoder variant, streams in completion order), encode parity at probBits 9-11 past 65536 blocks and on batches of
64 x 1 Mi elements, and our readers on the reference's archives written over a 0xFF-filled buffer."""
import os

import numpy as np
import pytest
import torch

from oracle import oracle as O

pytestmark = pytest.mark.gpu

KINDS = {"f16": (1, torch.float16), "bf16": (2, torch.bfloat16), "f32": (3, torch.float32)}
GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_golden.npz"))


def dg():
    import dietgpu_b200

    return dietgpu_b200


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def cases(prefix):
    return sorted({k.rsplit("/", 1)[0] for k in GOLD.files if k.startswith(prefix)})


def ref_max_size(n, ft=None):
    """The reference's maximum compressed size for n input bytes (ans) or n floats of type ft."""
    row = [r for r in GOLD["max_sizes"].tolist() if r[0] == n]
    assert row, f"no stored bound for {n}"
    return row[0][1] if ft is None else row[0][1 + ft]


def assert_same_ans(mine: np.ndarray, theirs: np.ndarray):
    # the reference leaves the checksum flag / value bits undefined when off: parse_ans only reads
    # defined fields; stream order inside the data section is free (see oracle.assert_same_ans)
    O.assert_same_ans(mine, theirs)


@pytest.mark.parametrize("pb", [9, 10, 11])
def test_ans_matches_reference(pb):
    names = cases("ans/")
    assert len(names) >= 6
    arrays = [GOLD[f"{b}/in"] for b in names]
    theirs = [GOLD[f"{b}/pb{pb}"] for b in names]
    ts = [dev(a) for a in arrays]
    n = len(ts)
    comp, sizes, _ = dg().compress_data(False, ts, True, prob_bits=pb)
    assert comp.size(1) == ref_max_size(max(a.size for a in arrays))
    torch.cuda.synchronize()
    hs = sizes.cpu().tolist()
    assert hs == [t.size for t in theirs], "compressed sizes differ from the reference"
    for i in range(n):
        mine = comp[i, :hs[i]].cpu().numpy()
        assert_same_ans(mine, theirs[i])
        O.assert_same_ans(mine, O.ans_encode(arrays[i], pb, True))
    # ours <- reference archives
    outs = [torch.empty_like(t) for t in ts]
    dg().decompress_data(False, [dev(a) for a in theirs], outs, True, prob_bits=pb)
    for t, o in zip(ts, outs):
        assert torch.equal(t, o)


@pytest.mark.parametrize("kind", ["f16", "bf16", "f32"])
def test_float_matches_reference(kind):
    ft, tdt = KINDS[kind]
    names = cases(f"float/{kind}/")
    assert len(names) >= 3
    words = [GOLD[f"{b}/in"] for b in names]
    theirs = [GOLD[f"{b}/pb10"] for b in names]
    it = torch.int16 if kind != "f32" else torch.int32
    ts = [torch.from_numpy(w.view(np.int16 if kind != "f32" else np.int32).copy()).view(tdt).cuda() for w in words]
    n = len(ts)
    comp, sizes, _ = dg().compress_data(True, ts, True)
    assert comp.size(1) == ref_max_size(max(w.size for w in words), ft)
    torch.cuda.synchronize()
    hs = sizes.cpu().tolist()
    assert hs == [t.size for t in theirs], "float compressed sizes differ from the reference"
    for i, w in enumerate(words):
        mine, ref = comp[i, :hs[i]].cpu().numpy(), theirs[i]
        nc = O.float_noncomp_bytes(ft, w.size)
        # float header: magic, size, type|checksum flag, checksum
        assert np.array_equal(mine[:8], ref[:8])
        assert (mine[8] & 0x1f) == (ref[8] & 0x1f) and np.array_equal(mine[12:16], ref[12:16])
        # stored planes: compare the defined bytes only (padding is undefined in the reference)
        if kind == "f32":
            assert np.array_equal(mine[16:16 + 2 * w.size], ref[16:16 + 2 * w.size])
            o1 = 16 + 2 * ((w.size + 7) // 8 * 8)
            assert np.array_equal(mine[o1:o1 + w.size], ref[o1:o1 + w.size])
        else:
            assert np.array_equal(mine[16:16 + w.size], ref[16:16 + w.size])
        assert_same_ans(mine[16 + nc:], ref[16 + nc:])
    outs = [torch.empty_like(t) for t in ts]
    dg().decompress_data(True, [dev(a) for a in theirs], outs, True)
    for t, o in zip(ts, outs):
        assert torch.equal(t.view(it), o.view(it))


def test_max_sizes_match_reference():
    L = dg().capi.lib()
    table = GOLD["max_sizes"]
    assert table.shape[0] >= 9
    for n, ans, *floats in table.tolist():
        assert L.dgb_ans_max_compressed_size(n) == ans
        for ft, want in zip((1, 2, 3), floats):
            mine = L.dgb_float_max_compressed_size(ft, n)
            if mine == 0:
                # the exact bound does not fit 32 bits: the reference returns the wrapped sum, this ABI
                # reports "too large" (0) instead of a value a caller would under-allocate from
                assert 16 + L.dgb_ans_max_compressed_size(n) + (3 if ft == 3 else 1) * n > 0xffffffff
                continue
            assert mine == want
