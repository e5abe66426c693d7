"""Decode-and-sum (ops.decompress_data_reduce) against decoding the same archives separately, on one GPU.

    python tools/reduce_bench.py [--iters 30] [--json out.json] [--reduce-dtype float32] [--sparse]

For each shape (G groups x W archives x N words of N(0,1) data, seeded) three ways are timed on the same archives,
alternating within the run:
  (1) decompress_data_reduce: one call, every group summed;
  (2) decompress_data of the G * W archives into separate outputs;
  (3) (2) followed by the W - 1 torch adds per group (what a caller does without (1)).
Reported: event time per call, the decoder's kernel time with option timing=1 (slot "decode"), and for (1) and (2)
algorithmic bytes over kernel time as a share of the H100 SXM data sheet's 3.35 TB/s HBM3 bandwidth (archives read
once + outputs written once: G * N words for (1), G * W * N for (2)).  (1)'s result is checked bit for bit against
(3)'s.  The card name and power limit are read in the same run; DIETGPU_B200_LIB selects an experiment build of
the library (make -C dietgpu_b200/csrc variant NAME=p2 DEFS=-DDGB_REDUCE_PASS_ARCHIVES=2).

--sparse: sparse against dense decode-and-sum (bench_sparse) at zero fractions 0 %, ReLU (about 50 %), 90 % and 99 %.
--scale: the scaled decode-and-sum against the unscaled one and against scaling the inputs with torch (bench_scale).
--scale-tensor: the device-scale decode-and-sum with its non-finite flag against the host-scaled one and against
an unscaled sum followed by torch.amp's unscale-and-check (bench_scale_tensor).
--out-dtype: the narrowing decode-and-sum (fp32 sums rounded once to the 16-bit archive dtype) against the widening
one followed by torch's .to() and against the same-type 16-bit sum (bench_out_dtype).
--sq-norm: the device-scale decode-and-sum with its fused squared norm against the same call followed by
ops.sq_norm of the outputs and by torch's fp64 squared norm of the outputs (bench_sq_norm).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from dietgpu_b200 import capi, ops  # noqa: E402

PEAK_GBS = 3350.0  # H100 SXM data sheet, HBM3
SHAPES = [  # (dtype, groups, archives per group, words)
    (torch.bfloat16, 8, 8, 2 << 20),
    (torch.bfloat16, 8, 7, 4 << 20),  # what one rank of an 8-GPU reduce-scatter of 256 Mi words receives
    (torch.float32, 16, 4, 1 << 20),
    (torch.float16, 64, 2, 512 << 10),
]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit unknown"
    return f"{name} ({q})"


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e3  # us


def kernel_us(fn, iters):
    capi.set_option("timing", 1)
    try:
        capi.kernel_times()
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
        ms, _ = capi.kernel_times()["decode"]
    finally:
        capi.set_option("timing", 0)
    return ms / iters * 1e3


def bench(dtype, groups, width, n, iters):
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [torch.randn(n, generator=g, device="cuda").to(dtype) for _ in range(groups * width)]
    comp, sizes, _ = ops.compress_data(True, xs)
    hs = sizes.cpu().tolist()
    arch = [comp[i, :hs[i]] for i in range(len(xs))]
    del xs
    groups_in = [arch[k * width:(k + 1) * width] for k in range(groups)]
    temp = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    red = [torch.empty(n, dtype=dtype, device="cuda") for _ in range(groups)]
    sep = [torch.empty(n, dtype=dtype, device="cuda") for _ in range(groups * width)]
    fold = [torch.empty(n, dtype=dtype, device="cuda") for _ in range(groups)]

    def one():
        ops.decompress_data_reduce(groups_in, red, False, temp)

    def two():
        ops.decompress_data(True, arch, sep, False, temp)

    def three():
        two()
        for k in range(groups):
            torch.add(sep[k * width], sep[k * width + 1], out=fold[k]) if width > 1 else fold[k].copy_(sep[k * width])
            for j in range(2, width):
                fold[k].add_(sep[k * width + j])

    for f in (one, two, three):  # warm-up
        f()
    torch.cuda.synchronize()
    for k in range(groups):
        assert torch.equal(red[k].view(torch.int16 if dtype != torch.float32 else torch.int32),
                           fold[k].view(torch.int16 if dtype != torch.float32 else torch.int32)), k
    t = {"1": [], "2": [], "3": []}
    for _ in range(3):  # alternate
        t["1"].append(timed(one, iters))
        t["2"].append(timed(two, iters))
        t["3"].append(timed(three, iters))
    k1, k2 = kernel_us(one, iters), kernel_us(two, iters)
    es = torch.empty(0, dtype=dtype).element_size()
    abytes = sum(hs)
    bw1 = (abytes + groups * n * es) / (k1 * 1e-6) / 1e9
    bw2 = (abytes + groups * width * n * es) / (k2 * 1e-6) / 1e9
    r = {"shape": f"{str(dtype).split('.')[-1]} {groups}x{width}x{n}", "archive_MB": abytes / 1e6,
         "call_us": {k: min(v) for k, v in t.items()}, "call_us_max": {k: max(v) for k, v in t.items()},
         "kernel_us": {"1": k1, "2": k2}, "hbm_share": {"1": bw1 / PEAK_GBS, "2": bw2 / PEAK_GBS}}
    r["1_over_3"] = r["call_us"]["1"] / r["call_us"]["3"]
    r["1_over_2"] = r["call_us"]["1"] / r["call_us"]["2"]
    return r


SHAPES32 = [s for s in SHAPES if s[0] != torch.float32]


def bench32(dtype, groups, width, n, iters):
    """--reduce-dtype float32: 16-bit archives summed into fp32 outputs, three ways on the same archives:
    (1) decompress_data_reduce(archive_dtype=dtype) into fp32; (2) decompress_data into 16-bit temporaries, then
    acc.copy_(tmp_0) and acc.add_(tmp_j) in fp32 (torch's widening adds); (3) the same-type decode-and-sum into 16-bit
    outputs, for reference.  Algorithmic bytes per element and accumulated archive (r = archive bytes / input
    bytes): (1) 2r + 8 (archive, fp32 read, fp32 write); (2) 2r + 2 + 6 + 4 (archive, 16-bit write; 16-bit and fp32
    read; fp32 write)."""
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [torch.randn(n, generator=g, device="cuda").to(dtype) for _ in range(groups * width)]
    comp, sizes, _ = ops.compress_data(True, xs)
    hs = sizes.cpu().tolist()
    arch = [comp[i, :hs[i]] for i in range(len(xs))]
    del xs
    groups_in = [arch[k * width:(k + 1) * width] for k in range(groups)]
    temp = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    red = [torch.empty(n, dtype=torch.float32, device="cuda") for _ in range(groups)]
    sep = [torch.empty(n, dtype=dtype, device="cuda") for _ in range(groups * width)]
    acc = [torch.empty(n, dtype=torch.float32, device="cuda") for _ in range(groups)]
    red16 = [torch.empty(n, dtype=dtype, device="cuda") for _ in range(groups)]

    def one():
        ops.decompress_data_reduce(groups_in, red, False, temp, archive_dtype=dtype)

    def decode():
        ops.decompress_data(True, arch, sep, False, temp)

    def two():
        decode()
        for k in range(groups):
            acc[k].copy_(sep[k * width])
            for j in range(1, width):
                acc[k].add_(sep[k * width + j])

    def three():
        ops.decompress_data_reduce(groups_in, red16, False, temp)

    for f in (one, two, three):  # warm-up
        f()
    torch.cuda.synchronize()
    for k in range(groups):
        assert torch.equal(red[k].view(torch.int32), acc[k].view(torch.int32)), k
    t = {"1": [], "2": [], "3": []}
    for _ in range(3):  # alternate
        t["1"].append(timed(one, iters))
        t["2"].append(timed(two, iters))
        t["3"].append(timed(three, iters))
    k1, k2, k3 = kernel_us(one, iters), kernel_us(decode, iters), kernel_us(three, iters)
    ratio = sum(hs) / (groups * width * n * 2)
    r = {"shape": f"{str(dtype).split('.')[-1]}->float32 {groups}x{width}x{n}", "archive_MB": sum(hs) / 1e6,
         "ratio": ratio, "bytes_per_elem_archive": {"1": 2 * ratio + 8, "2": 2 * ratio + 12},
         "call_us": {k: min(v) for k, v in t.items()}, "call_us_max": {k: max(v) for k, v in t.items()},
         "kernel_us": {"1": k1, "2_decode": k2, "3": k3}}
    r["1_over_2"] = r["call_us"]["1"] / r["call_us"]["2"]
    r["1_over_3"] = r["call_us"]["1"] / r["call_us"]["3"]
    r["kernel_1_over_3"] = k1 / k3
    return r


SPARSE_SHAPES = [s for s in SHAPES if s[1:] != (8, 7, 4 << 20)]
ZEROS = ["0", "relu", "0.9", "0.99"]


def sparse_data(dtype, n, zeros, g):
    x = torch.randn(n, generator=g, device="cuda")
    if zeros == "relu":
        x = x.clamp_min(0)
    elif zeros != "0":
        x[torch.rand(n, generator=g, device="cuda") < float(zeros)] = 0
    return x.to(dtype)


def bench_sparse(dtype, groups, width, n, iters, zeros, out_dtype):
    """The same words as sparse and as dense archives: (1) decompress_data_reduce(sparse=True), (2) the dense call.
    Reported: call and kernel time of both, and the bytes on the wire (the summed archive sizes)."""
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [sparse_data(dtype, n, zeros, g) for _ in range(groups * width)]
    arch = {}
    for sp in (True, False):
        comp, sizes, _ = ops.compress_data(True, xs, sparse=sp)
        hs = sizes.cpu().tolist()
        arch[sp] = ([comp[i, :hs[i]].clone() for i in range(len(xs))], sum(hs))
        del comp
    del xs
    temp = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    outs = {sp: [torch.empty(n, dtype=out_dtype, device="cuda") for _ in range(groups)] for sp in (True, False)}
    calls = {}
    for sp in (True, False):
        gi = [arch[sp][0][k * width:(k + 1) * width] for k in range(groups)]
        calls[sp] = (lambda gi=gi, sp=sp: ops.decompress_data_reduce(gi, outs[sp], False, temp, archive_dtype=dtype,
                                                                      sparse=sp))
        calls[sp]()
    torch.cuda.synchronize()
    it = torch.int32 if out_dtype == torch.float32 else torch.int16
    for k in range(groups):
        assert torch.equal(outs[True][k].view(it), outs[False][k].view(it)), k
    t = {True: [], False: []}
    for _ in range(3):  # alternate
        for sp in (True, False):
            t[sp].append(timed(calls[sp], iters))
    kt = {sp: kernel_us(calls[sp], iters) for sp in (True, False)}
    raw = groups * width * n * torch.empty(0, dtype=dtype).element_size()
    r = {"shape": f"{str(dtype).split('.')[-1]}->{str(out_dtype).split('.')[-1]} {groups}x{width}x{n}",
         "zeros": zeros, "wire_MB": {"sparse": arch[True][1] / 1e6, "dense": arch[False][1] / 1e6},
         "wire_ratio": {"sparse": arch[True][1] / raw, "dense": arch[False][1] / raw},
         "call_us": {"sparse": min(t[True]), "dense": min(t[False])},
         "call_us_max": {"sparse": max(t[True]), "dense": max(t[False])},
         "kernel_us": {"sparse": kt[True], "dense": kt[False]}}
    r["kernel_sparse_over_dense"] = kt[True] / kt[False]
    return r


SCALE_SHAPES = [  # (dtype, groups, width, words, out dtype, sparse ReLU data)
    (torch.bfloat16, 8, 8, 2 << 20, torch.bfloat16, False),
    (torch.float32, 16, 4, 1 << 20, torch.float32, False),
    (torch.float16, 64, 2, 512 << 10, torch.float16, False),
    (torch.bfloat16, 8, 8, 2 << 20, torch.float32, False),
    (torch.bfloat16, 8, 8, 2 << 20, torch.bfloat16, True),
]


def bench_scale(dtype, groups, width, n, iters, out_dtype, sparse):
    """--scale, s = fp32(1 / W) on the same inputs, alternated:
    (1) the scaled decode-and-sum of the archives; (2) the unscaled one (same archives, same kernel shape);
    (3) the caller's way without (1): term(t) = (t.float() * s32).to(out dtype) with torch, compress, unscaled sum
    (bit-identical to (1), checked).  Reported: call time of (1) and (2), of compress + (1) ("1c"), of (3) and of its
    torch multiply alone ("3_mul"); kernel time (timing=1) of (1) and (2)."""
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [sparse_data(dtype, n, "relu" if sparse else "0", g) for _ in range(groups * width)]
    s32 = torch.tensor(1.0 / width, dtype=torch.float32, device="cuda")
    s = float(s32)
    temp = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    comp, sizes, _ = ops.compress_data(True, xs, sparse=sparse)
    hs = sizes.cpu().tolist()
    gi = [[comp[k * width + j, :hs[k * width + j]] for j in range(width)] for k in range(groups)]
    outs = {k: [torch.empty(n, dtype=out_dtype, device="cuda") for _ in range(groups)] for k in ("1", "2", "3")}
    terms = [torch.empty(n, dtype=out_dtype, device="cuda") for _ in range(groups * width)]

    def one():
        ops.decompress_data_reduce(gi, outs["1"], False, temp, archive_dtype=dtype, sparse=sparse, scale=s)

    def two():
        ops.decompress_data_reduce(gi, outs["2"], False, temp, archive_dtype=dtype, sparse=sparse)

    def one_c():
        c, sz, _ = ops.compress_data(True, xs, sparse=sparse)
        ops.decompress_data_reduce([[c[k * width + j] for j in range(width)] for k in range(groups)], outs["1"], False,
                                   temp, archive_dtype=dtype, sparse=sparse, scale=s)

    def mul():
        # one torch kernel per input: a 16-bit x times the float32 0-dim tensor stays 16-bit and is computed in fp32,
        # which is the same-type term; the widening term needs the fp32 product itself
        for x, t in zip(xs, terms):
            torch.mul(x.float() if out_dtype != dtype else x, s32, out=t)

    def three():
        mul()
        c, sz, _ = ops.compress_data(True, terms, sparse=sparse)
        ops.decompress_data_reduce([[c[k * width + j] for j in range(width)] for k in range(groups)], outs["3"], False,
                                   temp, sparse=sparse)

    fns = {"1": one, "2": two, "1c": one_c, "3": three, "3_mul": mul}
    for f in fns.values():  # warm-up
        f()
    torch.cuda.synchronize()
    it = torch.int32 if out_dtype == torch.float32 else torch.int16
    for k in range(groups):
        same = (outs["1"][k].view(it) == outs["3"][k].view(it)) | (outs["1"][k].isnan() & outs["3"][k].isnan())
        assert bool(same.all()), k
    t = {k: [] for k in fns}
    for _ in range(3):  # alternate
        for k, f in fns.items():
            t[k].append(timed(f, iters))
    kt = {"1": kernel_us(one, iters), "2": kernel_us(two, iters)}
    r = {"shape": f"{'sparse relu ' if sparse else ''}{str(dtype).split('.')[-1]}->{str(out_dtype).split('.')[-1]} "
                  f"{groups}x{width}x{n}", "scale": s,
         "call_us": {k: min(v) for k, v in t.items()}, "call_us_max": {k: max(v) for k, v in t.items()},
         "kernel_us": kt}
    r["kernel_scaled_over_plain"] = kt["1"] / kt["2"]
    r["1c_over_3"] = r["call_us"]["1c"] / r["call_us"]["3"]
    return r


def bench_scale_tensor(dtype, groups, width, n, iters, out_dtype, sparse):
    """--scale-tensor, s = fp32(1 / W) held in a one-element CUDA tensor, on the same archives, alternated:
    (1) the device-scale decode-and-sum with found_inf; (2) the host-scaled one with s = float(s32) (bit-identical to
    (1), checked); (3) what a GradScaler user does today: the unscaled sum, then
    torch._amp_foreach_non_finite_check_and_unscale_(outs, found, s32) (bf16 outputs, which it does not take: a
    torch multiply and isfinite check per output), which multiplies after the sum and so rounds
    differently (timed only).  Reported: call time of all three; kernel time (timing=1) of (1), (2) and of (3)'s
    decode-and-sum."""
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [sparse_data(dtype, n, "relu" if sparse else "0", g) for _ in range(groups * width)]
    s32 = torch.tensor([1.0 / width], dtype=torch.float32, device="cuda")
    s = float(s32)
    temp = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    comp, sizes, _ = ops.compress_data(True, xs, sparse=sparse)
    hs = sizes.cpu().tolist()
    gi = [[comp[k * width + j, :hs[k * width + j]] for j in range(width)] for k in range(groups)]
    del xs
    outs = {k: [torch.empty(n, dtype=out_dtype, device="cuda") for _ in range(groups)] for k in ("1", "2", "3")}
    found = {k: torch.zeros(1, dtype=torch.float32, device="cuda") for k in ("1", "3")}

    def one():
        ops.decompress_data_reduce(gi, outs["1"], False, temp, archive_dtype=dtype, sparse=sparse, scale_tensor=s32,
                                   found_inf=found["1"])

    def two():
        ops.decompress_data_reduce(gi, outs["2"], False, temp, archive_dtype=dtype, sparse=sparse, scale=s)

    def three_sum():
        ops.decompress_data_reduce(gi, outs["3"], False, temp, archive_dtype=dtype, sparse=sparse)

    def three():
        three_sum()
        if out_dtype != torch.bfloat16:
            torch._amp_foreach_non_finite_check_and_unscale_(outs["3"], found["3"], s32)
        else:  # torch.amp's fused unscale has no bf16 kernel: the same multiply and check, per output
            for o in outs["3"]:
                o.mul_(s32)
                torch.maximum(found["3"], (~o.isfinite()).any().float(), out=found["3"])

    fns = {"1": one, "2": two, "3": three}
    for f in fns.values():  # warm-up
        f()
    torch.cuda.synchronize()
    it = torch.int32 if out_dtype == torch.float32 else torch.int16
    for k in range(groups):
        assert torch.equal(outs["1"][k].view(it), outs["2"][k].view(it)), k
    assert float(found["1"].item()) == 0.0 and float(found["3"].item()) == 0.0
    t = {k: [] for k in fns}
    for _ in range(3):  # alternate
        for k, f in fns.items():
            t[k].append(timed(f, iters))
    kt = {"1": kernel_us(one, iters), "2": kernel_us(two, iters), "3_sum": kernel_us(three_sum, iters)}
    r = {"shape": f"{'sparse relu ' if sparse else ''}{str(dtype).split('.')[-1]}->{str(out_dtype).split('.')[-1]} "
                  f"{groups}x{width}x{n}", "scale": s,
         "call_us": {k: min(v) for k, v in t.items()}, "call_us_max": {k: max(v) for k, v in t.items()},
         "kernel_us": kt}
    r["kernel_dev_over_host"] = kt["1"] / kt["2"]
    r["call_dev_over_host"] = r["call_us"]["1"] / r["call_us"]["2"]
    r["call_dev_over_amp"] = r["call_us"]["1"] / r["call_us"]["3"]
    return r


OUT_DTYPE_SHAPES = [  # (dtype, groups, width, words, sparse ReLU data)
    (torch.bfloat16, 8, 8, 2 << 20, False),
    (torch.float16, 64, 2, 512 << 10, False),
    (torch.bfloat16, 8, 8, 2 << 20, True),
]


def bench_out_dtype(dtype, groups, width, n, iters, sparse):
    """--out-dtype, on the same archives, alternated: (1) the narrowing decode-and-sum
    (reduce_dtype=torch.float32, 16-bit outputs, a caller-owned fp32 accumulator); (2) the widening one into fp32
    outputs followed by torch's .to(dtype) (bit-identical to (1), checked); (3) the same-type 16-bit sum.  Reported:
    call time of all three and of (2)'s sum alone ("2_sum"); kernel time (timing=1) of (1), (2)'s sum and (3); the
    modelled HBM bytes per output element of (1) and (2) (the archives are read in both)."""
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [sparse_data(dtype, n, "relu" if sparse else "0", g) for _ in range(groups * width)]
    temp = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    comp, sizes, _ = ops.compress_data(True, xs, sparse=sparse)
    hs = sizes.cpu().tolist()
    gi = [[comp[k * width + j, :hs[k * width + j]] for j in range(width)] for k in range(groups)]
    del xs
    outs = {k: [torch.empty(n, dtype=dtype, device="cuda") for _ in range(groups)] for k in ("1", "2", "3")}
    acc = [torch.empty(n, dtype=torch.float32, device="cuda") for _ in range(groups)]
    wide = [torch.empty(n, dtype=torch.float32, device="cuda") for _ in range(groups)]

    def one():
        ops.decompress_data_reduce(gi, outs["1"], False, temp, archive_dtype=dtype, sparse=sparse,
                                   reduce_dtype=torch.float32, acc=acc)

    def two_sum():
        ops.decompress_data_reduce(gi, wide, False, temp, archive_dtype=dtype, sparse=sparse)

    def two():
        two_sum()
        for w, o in zip(wide, outs["2"]):
            o.copy_(w)

    def three():
        ops.decompress_data_reduce(gi, outs["3"], False, temp, archive_dtype=dtype, sparse=sparse)

    fns = {"1": one, "2": two, "2_sum": two_sum, "3": three}
    for f in fns.values():  # warm-up
        f()
    torch.cuda.synchronize()
    same = all(bool(((a.view(torch.int16) == b.view(torch.int16)) | (a.isnan() & b.isnan())).all())
               for a, b in zip(outs["1"], outs["2"]))
    t = {k: [] for k in fns}
    for _ in range(3):  # alternate
        for k, f in fns.items():
            t[k].append(timed(f, iters))
    kt = {"1": kernel_us(one, iters), "2_sum": kernel_us(two_sum, iters), "3": kernel_us(three, iters)}
    # the bytes per output element that differ (the archives and the fp32 running sums of every archive but the
    # last are the same in both): (1) stores 2 B; (2) stores 4 B, then its cast reads 4 B and writes 2 B
    r = {"shape": f"{'sparse relu ' if sparse else ''}{str(dtype).split('.')[-1]} {groups}x{width}x{n}",
         "bit_equal_1_2": same, "call_us": {k: min(v) for k, v in t.items()},
         "call_us_max": {k: max(v) for k, v in t.items()}, "kernel_us": kt,
         "model_final_bytes_per_elem": {"1": 2, "2": 10}}
    r["call_1_over_2"] = r["call_us"]["1"] / r["call_us"]["2"]
    r["kernel_1_over_2_sum"] = kt["1"] / kt["2_sum"]
    return r


SQ_NORM_SHAPES = SCALE_SHAPES + [  # (dtype, groups, width, words, out dtype, sparse ReLU data, narrowing)
    (torch.bfloat16, 8, 8, 2 << 20, torch.bfloat16, False, True),
]


def bench_sq_norm(dtype, groups, width, n, iters, out_dtype, sparse, narrow=False):
    """--sq-norm, on the same archives, alternated, every call with scale_tensor and found_inf: (1) the decode-and-sum
    with sq_norm; (2) the same call without it, then ops.sq_norm of the outputs; (3) the same call without it, then
    torch's fp64 squared norm of the outputs (one .double().square().sum() per group).  Reported: call time of all
    three (lowest of three alternated runs); kernel time (timing=1) of (1), of the sum without the norm ("sum") and
    of the standalone norm alone ("norm"); the fused norm's extra kernel time ("1" - "sum") against "norm"; and the
    standalone norm's bytes read over its kernel time as a share of the H100 SXM data sheet's 3.35 TB/s."""
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [sparse_data(dtype, n, "relu" if sparse else "0", g) for _ in range(groups * width)]
    temp = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    comp, sizes, _ = ops.compress_data(True, xs, sparse=sparse)
    hs = sizes.cpu().tolist()
    gi = [[comp[k * width + j, :hs[k * width + j]] for j in range(width)] for k in range(groups)]
    del xs
    outs = [torch.empty(n, dtype=out_dtype, device="cuda") for _ in range(groups)]
    kw = dict(archive_dtype=dtype, sparse=sparse, scale_tensor=torch.full((1,), 0.125, device="cuda"),
              found_inf=torch.zeros(1, device="cuda"))
    if narrow:
        kw.update(reduce_dtype=torch.float32, acc=[torch.empty(n, dtype=torch.float32, device="cuda")
                                                   for _ in range(groups)])
    norms = {k: torch.empty(groups, dtype=torch.float64, device="cuda") for k in ("1", "2", "3")}

    def one():
        ops.decompress_data_reduce(gi, outs, False, temp, sq_norm=norms["1"], **kw)

    def the_sum():
        ops.decompress_data_reduce(gi, outs, False, temp, **kw)

    def norm():
        ops.sq_norm(outs, out=norms["2"], temp_mem=temp)

    def two():
        the_sum()
        norm()

    def three():
        the_sum()
        for k, o in enumerate(outs):
            norms["3"][k].copy_(o.double().square().sum())

    fns = {"1": one, "2": two, "3": three}
    for f in list(fns.values()) + [the_sum, norm]:  # warm-up
        f()
    torch.cuda.synchronize()
    one()
    two()
    same = bool(((norms["1"] == norms["2"]) | (norms["1"].isnan() & norms["2"].isnan())).all())
    rel_torch = float(((norms["1"] - norms["3"]).abs() / norms["3"]).max())
    t = {k: [] for k in fns}
    for _ in range(3):  # alternate
        for k, f in fns.items():
            t[k].append(timed(f, iters))
    kt = {"1": kernel_us(one, iters), "sum": kernel_us(the_sum, iters), "norm": kernel_us(norm, iters)}
    es = torch.empty(0, dtype=out_dtype).element_size()
    r = {"shape": f"{'sparse relu ' if sparse else ''}{'narrowing ' if narrow else ''}"
                  f"{str(dtype).split('.')[-1]}->{str(out_dtype).split('.')[-1]} {groups}x{width}x{n}",
         "bit_equal_1_2": same, "max_rel_diff_1_3": rel_torch, "call_us": {k: min(v) for k, v in t.items()},
         "call_us_max": {k: max(v) for k, v in t.items()}, "kernel_us": kt,
         "fused_extra_us": kt["1"] - kt["sum"],
         "norm_share_of_3350GBs": groups * n * es / (kt["norm"] * 1e-6) / 1e9 / PEAK_GBS}
    r["fused_extra_below_norm"] = r["fused_extra_us"] < kt["norm"]
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--json", default=None)
    ap.add_argument("--reduce-dtype", choices=["same", "float32"], default="same",
                    help="float32: sum the 16-bit shapes' archives into fp32 outputs (bench32)")
    ap.add_argument("--sparse", action="store_true", help="sparse against dense archives (bench_sparse)")
    ap.add_argument("--scale", action="store_true", help="scaled against unscaled sums and torch's scaling (bench_scale)")
    ap.add_argument("--scale-tensor", action="store_true",
                    help="device-scale sums with the non-finite flag against host-scaled sums and torch.amp's "
                         "unscale (bench_scale_tensor)")
    ap.add_argument("--out-dtype", action="store_true",
                    help="narrowing sums against widening sums + .to() and same-type sums (bench_out_dtype)")
    ap.add_argument("--sq-norm", action="store_true",
                    help="device-scale sums with the fused squared norm against the sum + ops.sq_norm and the sum + "
                         "torch's norm (bench_sq_norm)")
    args = ap.parse_args()
    info = {"card": card(), "lib": capi.LIB_PATH, "results": []}
    print(info["card"], flush=True)
    if args.sq_norm:
        for shape in SQ_NORM_SHAPES:
            r = bench_sq_norm(*shape[:4], args.iters, *shape[4:])
            info["results"].append(r)
            print(json.dumps(r), flush=True)
        shapes = []
    elif args.out_dtype:
        for shape in OUT_DTYPE_SHAPES:
            r = bench_out_dtype(*shape[:4], args.iters, shape[4])
            info["results"].append(r)
            print(json.dumps(r), flush=True)
        shapes = []
    elif args.scale_tensor:
        for shape in SCALE_SHAPES:
            r = bench_scale_tensor(*shape[:4], args.iters, *shape[4:])
            info["results"].append(r)
            print(json.dumps(r), flush=True)
        shapes = []
    elif args.scale:
        for shape in SCALE_SHAPES:
            r = bench_scale(*shape[:4], args.iters, *shape[4:])
            info["results"].append(r)
            print(json.dumps(r), flush=True)
        shapes = []
    elif args.sparse:
        for dtype, groups, width, n in SPARSE_SHAPES:
            if args.reduce_dtype == "float32" and dtype == torch.float32:
                continue
            out_dtype = torch.float32 if args.reduce_dtype == "float32" else dtype
            for zeros in ZEROS:
                r = bench_sparse(dtype, groups, width, n, args.iters, zeros, out_dtype)
                info["results"].append(r)
                print(json.dumps(r), flush=True)
        shapes = []
    else:
        shapes = SHAPES32 if args.reduce_dtype == "float32" else SHAPES
    for shape in shapes:
        r = (bench32 if args.reduce_dtype == "float32" else bench)(*shape, args.iters)
        info["results"].append(r)
        print(json.dumps(r), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
