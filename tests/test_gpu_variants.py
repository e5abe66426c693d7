"""Kernel-variant matrix: one small edge corpus per data kind, at prob bits 9, 10 and 11, run once under
every option set that selects a different kernel instantiation or code path.  Each cell compares every
member's archive with the CPU oracle (byte for byte for the canonical encoder), decodes it bit-exactly
into guard-banded outputs, checks that compress left its inputs alone and wrote nothing past an
archive's size, and -- for decoder-only variants -- decodes the oracle's own archives too.

Which instantiation each variant is there to reach (KIND = bytes, f16, bf16, f32; PB = 9, 10, 11):
  defaults            statsBytesKernel / statsFloatKernel<FT>, encodeKernelFast<false, bytes|f16>,
                      encodeKernelFast<true, bf16|f32>, decodeFusedKernel<KIND, PB, 8>
  decode_warps 4/8/20 decodeFusedKernel<KIND, PB, 4 | 8 | 20 (bytes only)>
  decode_fused=0      planKernel<KIND>, decodeKernel<KIND, PB, 8, true, false>
  decode_slot_words   the fused decoder's direct-from-global stream path for (nearly) every block
  table_wide/packed   encodeKernelFast<true | false, KIND> for the kinds whose default is the other one
  encode_canonical    encodeKernel<KIND> (archives byte-identical to the oracle's)
  fused_s*_w*         encodeFusedKernel<KIND, WIDE, STAGED> for all four (WIDE, STAGED)
  stats_stage_kb*     statsFloatStagedKernel<FT> (float kinds only; bytes ignore the option)
  hist_slab_1k        1 KiB statistics slabs: many slabs per member, ragged heads at unaligned starts
  hist_ctas_1/64      the statistics grid's slab loop with one CTA per member and with more CTAs than slabs
  parts*              2, 4 and 8 sub-batches with unequal first / last parts, both directions
  k2_ctas_1           one coder CTA per SM
  enc_slot_min        the fast encoder's smallest staging slot (most blocks spill)
  inline_members=0    member tables read from scratch instead of the kernel parameters
"""
import numpy as np
import pytest
import torch

from codec_helpers import codec_options, roundtrip
from conftest import normal_words, zipf_bytes

pytestmark = pytest.mark.gpu

SIZES = (0, 1, 31, 32, 33, 4095, 4096, 4097, 65537, 300000)
FLOAT_KINDS = ("f16", "bf16", "f32")
NAN = {"f16": 0x7E01, "bf16": 0x7FC1, "f32": 0x7FC00123}
SUBNORMAL_MASK = {"f16": 0x83FF, "bf16": 0x807F, "f32": 0x807FFFFF}
WORD = {"f16": np.uint16, "bf16": np.uint16, "f32": np.uint32}


def _bytes_corpus():
    rng = np.random.default_rng(2024)
    c = [zipf_bytes(n, 1.1, 300 + n) for n in SIZES]
    c.append(np.full(10000, 7, np.uint8))                                   # one symbol: pdf == 2^pb
    c.append(rng.choice(np.array([3, 200], np.uint8), 9000))                # two symbols
    c.append(rng.integers(0, 256, 70001, dtype=np.uint8))                   # uniform: spills the default slot
    dom = np.full(200000, 0x41, np.uint8)                                   # dominant symbol + pdf-1 stragglers
    dom[rng.choice(dom.size, 120, replace=False)] = rng.integers(0, 256, 120, dtype=np.uint8)
    c.append(dom)
    # constant except one 4 KiB block made of the rarest symbols only: every symbol of that block has pdf 1,
    # so it costs pb bits -- at pb 11 the block's stream is the 5632 B worst case
    rare = np.full(64 * 4096, 0x10, np.uint8)
    blk = rng.integers(0, 255, 4096).astype(np.uint8)
    rare[5 * 4096:6 * 4096] = np.where(blk >= 0x10, blk + 1, blk)
    c.append(rare)
    return c


def _float_corpus(kind):
    rng = np.random.default_rng(77)
    wt = WORD[kind]
    bits = 8 * np.dtype(wt).itemsize
    c = [normal_words(n, kind, 500 + n) for n in SIZES]
    c.append(rng.integers(0, 2 ** bits, 70001, dtype=np.uint64).astype(wt))     # full range: NaN, +-Inf, subnormals
    c.append(np.zeros(5000, wt))                                                 # all +0
    c.append(np.full(5000, 1 << (bits - 1), wt))                                 # all -0
    c.append(np.full(5000, NAN[kind], wt))                                       # one NaN payload
    c.append(rng.integers(0, 2 ** bits, 40000, dtype=np.uint64).astype(wt) & wt(SUBNORMAL_MASK[kind]))  # subnormal
    for scale, seed in ((1e-30, 1), (1.0, 2), (1e30, 3)):
        g = torch.Generator().manual_seed(seed)
        x = torch.randn(30000, generator=g, dtype=torch.float64) * scale
        if kind == "f32":
            c.append(x.to(torch.float32).view(torch.int32).numpy().view(np.uint32))
        else:
            dt = torch.float16 if kind == "f16" else torch.bfloat16
            c.append(x.to(dt).view(torch.int16).numpy().view(np.uint16))
    return c


_CORPUS = {}


def corpus(kind):
    if kind not in _CORPUS:
        _CORPUS[kind] = _bytes_corpus() if kind == "bytes" else _float_corpus(kind)
    return _CORPUS[kind]


# (name, options, role): role "dec" = decoder-only variant (also decodes the oracle's archives),
# "exact" = canonical encoder (byte equality), "enc" = anything else
VARIANTS = [
    ("defaults", {}, "enc"),
    ("decode_warps4", dict(decode_warps=4), "dec"),
    ("decode_warps8", dict(decode_warps=8), "dec"),
    ("decode_warps20", dict(decode_warps=20), "dec"),
    ("decode_two_kernel", dict(decode_fused=0), "dec"),
    ("decode_slot_min", dict(decode_slot_words=1), "dec"),
    ("table_wide", dict(encode_wide_table=1), "enc"),
    ("table_packed", dict(encode_wide_table=0), "enc"),
    ("canonical", dict(encode_canonical=1), "exact"),
    ("fused_s0_w0", dict(encode_fused=1, fused_stage=0, encode_wide_table=0), "enc"),
    ("fused_s0_w1", dict(encode_fused=1, fused_stage=0, encode_wide_table=1), "enc"),
    ("fused_s1_w0", dict(encode_fused=1, fused_stage=1, encode_wide_table=0), "enc"),
    ("fused_s1_w1", dict(encode_fused=1, fused_stage=1, encode_wide_table=1), "enc"),
    ("stats_stage_kb1", dict(stats_stage=1, stats_stage_kb=1), "enc"),
    ("stats_stage_kb32", dict(stats_stage=1, stats_stage_kb=32), "enc"),
    ("hist_slab_1k", dict(hist_slab_kb=1), "enc"),
    ("hist_ctas_1", dict(hist_ctas_per_sm=1), "enc"),
    ("hist_ctas_64", dict(hist_ctas_per_sm=64), "enc"),
    ("parts2", dict(parts=2, decode_fused=0), "enc"),
    ("parts4_first10_last200", dict(parts=4, first_part_pct=10, last_part_pct=200, decode_fused=0), "enc"),
    ("parts4_first200_last10", dict(parts=4, first_part_pct=200, last_part_pct=10, decode_fused=0), "enc"),
    ("parts8_first200_last200", dict(parts=8, first_part_pct=200, last_part_pct=200, decode_fused=0), "enc"),
    ("k2_ctas_1", dict(encode_k2_ctas=1), "enc"),
    ("enc_slot_min", dict(encode_slot_words=1), "enc"),
    ("inline_members0", dict(inline_members=0), "enc"),
]


def _cells():
    for kind in ("bytes",) + FLOAT_KINDS:
        for pb in (9, 10, 11):
            for name, opts, role in VARIANTS:
                if name == "decode_warps20" and kind != "bytes":
                    continue  # 20-warp CTAs exist for byte archives only (float kinds fall back to 8)
                if name.startswith("stats_stage") and kind == "bytes":
                    continue  # the staged statistics kernel is a float-kind kernel
                yield pytest.param(kind, pb, opts, role, id=f"{kind}-pb{pb}-{name}")


@pytest.mark.parametrize("kind,pb,opts,role", list(_cells()))
def test_variant_matches_oracle(kind, pb, opts, role):
    c = corpus(kind)
    in_offsets = [i % 8 for i in range(len(c))]  # unaligned starts (element offsets 0..7)
    with codec_options(**opts):
        roundtrip(kind, c, pb, checksum=(pb == 10), in_offsets=in_offsets, exact=(role == "exact"),
                  decode_oracle=(role == "dec"))
