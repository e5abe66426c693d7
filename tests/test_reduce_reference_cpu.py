"""Pins tests/reduce_reference.py (the float64 fold the decode-and-sum tests compare with) to torch's CPU adds and
numpy's float32 adds, without a device: every 16-bit a against the pair_operands b set, fp32 random and edge
pairs, the widened sums, and multi-step folds with an init."""
import numpy as np
import pytest
import torch

from reduce_reference import assert_same_words, f32_to_bf16_words, fold_ref, pair_operands, same_words

T16 = {"f16": torch.float16, "bf16": torch.bfloat16}


def _t(words, t):
    return torch.from_numpy(np.ascontiguousarray(words).view(np.int16)).view(T16[t])


def _w(x):
    return x.contiguous().view(torch.int16).numpy().view(np.uint16)


def test_pair_operands_cover_every_exponent_and_the_edges():
    for t, mbits in (("f16", 10), ("bf16", 7)):
        b = pair_operands(t)
        assert b.size >= 512
        exp = (b.astype(np.int64) >> mbits) & ((1 << (15 - mbits)) - 1)
        for s in (0, 1):
            sel = (b >> 15) == s
            assert set(exp[sel].tolist()) == set(range(1 << (15 - mbits))), (t, s)
        top = ((1 << (15 - mbits)) - 1) << mbits
        for v in (0, 0x8000, 1, 0x8001, top - 1, 0x8000 | (top - 1), top, 0x8000 | top):
            assert v in b, (t, hex(v))
        nans = b[(exp == (1 << (15 - mbits)) - 1) & ((b & ((1 << mbits) - 1)) != 0)]
        assert np.unique(nans).size >= 2, t


@pytest.mark.parametrize("t", ["f16", "bf16"])
def test_every_16bit_a_against_the_b_set(t):
    a = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    ta = _t(a, t).float()
    b = pair_operands(t)
    for k in range(0, b.size, 64):
        bb = b[k:k + 64]
        aa = np.repeat(a[None, :], bb.size, 0).reshape(-1)
        bw = np.repeat(bb[:, None], a.size, 1).reshape(-1)
        want = _w((ta[None, :] + _t(bb, t).float()[:, None]).to(T16[t]).reshape(-1))
        assert_same_words(fold_ref([aa, bw], t, t), want, t, f"{t} b[{k}:{k + 64}]")
        # widened: the same pairs summed into fp32
        want32 = (ta[None, :] + _t(bb, t).float()[:, None]).reshape(-1).numpy().view(np.uint32)
        assert_same_words(fold_ref([aa, bw], t, "f32"), want32, "f32", f"{t} -> f32 b[{k}:{k + 64}]")


def _f32_edges():
    v = [0, 0x80000000, 1, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x00800000, 0x80800000, 0x7F7FFFFF, 0xFF7FFFFF,
         0x7F800000, 0xFF800000, 0x7FC00123, 0xFFA00001, 0x3F800000, 0xBF800000, 0x3F800001, 0x33800000,
         0x33800001, 0x4B000000, 0x4B000001, 0x7F7FFFFE, 0x73800000]
    return np.array(v, dtype=np.uint32)


def test_f32_random_and_edge_pairs():
    rng = np.random.default_rng(5)
    n = 3 << 20
    a = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    # half of the b operands are a's neighbours in exponent, so cancellations and ties are common
    b = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    near = (a & np.uint32(0xFF800000)) + (rng.integers(-(24 << 23), 24 << 23, n).astype(np.int64)
                                           .astype(np.uint32) & np.uint32(0x7FFFFFFF))
    b[: n // 2] = near[: n // 2] ^ (rng.integers(0, 2, n // 2).astype(np.uint32) << np.uint32(31))
    e = _f32_edges()
    a = np.concatenate([a, np.repeat(e, e.size)])
    b = np.concatenate([b, np.tile(e, e.size)])
    with np.errstate(over="ignore", invalid="ignore"):
        want = (a.view(np.float32) + b.view(np.float32)).view(np.uint32)
    assert_same_words(fold_ref([a, b], "f32", "f32"), want, "f32", "fp32 pairs")


@pytest.mark.parametrize("t", ["f16", "bf16", "f32"])
def test_folds_with_init_match_torch(t):
    """Nine-term folds with an init (16-bit and widened), against torch's left fold on the CPU."""
    rng = np.random.default_rng(9)
    n = 1 << 16
    wt = np.uint32 if t == "f32" else np.uint16
    bits = 32 if t == "f32" else 16
    xs = []
    for j in range(9):
        w = rng.integers(0, 1 << bits, n, dtype=np.uint64).astype(wt)
        if j % 3 == 0:  # values of like magnitude, so the order of the adds shows
            x = torch.from_numpy(rng.standard_normal(n) * (1 << j))
            w = (x.float().view(torch.int32).numpy().view(np.uint32) if t == "f32"
                 else _w(x.to(T16[t])))
        xs.append(w)
    tt = torch.float32 if t == "f32" else T16[t]

    def tv(w):
        return torch.from_numpy(w.view(np.int32 if t == "f32" else np.int16)).view(tt)

    init32 = rng.standard_normal(n).astype(np.float32)
    init32[:4] = [np.nan, -0.0, np.inf, np.float32(1.0 + 2.0 ** -20)]  # last: no 16-bit type holds it
    init32[4] = np.float32(1e-40)  # fp32 subnormal
    outs = ["f32"] if t == "f32" else [t, "f32"]
    for out in outs:
        acc = tv(xs[0]) if out == t else tv(xs[0]).float()
        for w in xs[1:]:
            acc = acc + (tv(w) if out == t else tv(w).float())
        want = acc.contiguous().view(torch.int32 if out == "f32" else torch.int16).numpy()
        assert_same_words(fold_ref(xs, t, out), want, out, f"{t} -> {out} fold")
        init = init32.view(np.uint32) if out == "f32" else _w(torch.from_numpy(init32).to(tt))
        acc = torch.from_numpy(init.view(np.int32 if out == "f32" else np.int16)).view(torch.float32 if out == "f32" else tt)
        for w in xs:
            acc = acc + (tv(w) if out == t else tv(w).float())
        want = acc.contiguous().view(torch.int32 if out == "f32" else torch.int16).numpy()
        assert_same_words(fold_ref(xs, t, out, init=init), want, out, f"{t} -> {out} fold with init")


def test_bf16_rounding_and_nan_compare():
    x = np.array([1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, 3.3895314e38, -3.3895314e38, np.nan, -0.0], np.float32)
    got = f32_to_bf16_words(x)
    want = _w(torch.from_numpy(x).to(torch.bfloat16))
    assert got[:4].tolist() == want[:4].tolist() and got[5] == 0x8000
    assert (got[4] & 0x7F80) == 0x7F80 and (got[4] & 0x7F) != 0
    assert same_words(np.array([0x7FC1], np.uint16), np.array([0xFF81], np.uint16), "bf16").all()
    assert not same_words(np.array([0x0000], np.uint16), np.array([0x8000], np.uint16), "bf16").any()
    with pytest.raises(AssertionError):
        assert_same_words(np.array([0], np.uint32), np.array([0x80000000], np.uint32), "f32", "-0")
