"""Narrowing compress (compress_data(archive_dtype=T) on float32 inputs) against casting first, on one GPU.

    python tools/narrow_bench.py [--iters 20] [--rounds 3] [--json out.json]

For each shape (M members x N float32 words of seeded N(0,1) data) and archive type T (bfloat16, float16), three
arms are timed on the same inputs, alternating within the run, and the lowest of `rounds` rounds is reported:
  (1) narrow:  compress_data(True, xs, archive_dtype=T), float32 in, T archives out, no temporary;
  (2) cast:    [x.to(T) for x in xs] followed by compress_data(True, casts), what a caller does without (1);
  (3) fp32:    compress_data(True, xs), the float32 archives, for context.
Reported per arm: call time (CUDA events around `iters` calls), the codec's kernel times with option timing=1 (slots
"stats" and "encode") and, for (2), the cast kernels' time (events around the casts alone); algorithmic bytes
(every pass's input read once plus the archives written: 4 + 4 B per word for (1), 4 + 2 (cast) + 2 + 2 for (2),
4 + 4 for (3), plus the archive bytes) and their rate over the call time as a share of the H100 SXM data sheet's
3.35 TB/s HBM3 bandwidth; and the peak device memory a call allocates beyond its preallocated outputs and scratch
((2) holds the 2 B-per-word cast).  (1)'s archive sizes are checked against (2)'s.  The card name and power limit
are read in the same run.
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
SHAPES = [(64, 2 << 20), (256, 512 << 10), (8, 16 << 20)]  # (members, float32 words per member)
TYPES = {"bfloat16": torch.bfloat16, "float16": torch.float16}


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
        t = capi.kernel_times()
    finally:
        capi.set_option("timing", 0)
    return {k: t[k][0] / iters * 1e3 for k in ("stats", "encode")}


def extra_bytes(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def bench(members, n, dtype, iters, rounds):
    g = torch.Generator(device="cuda").manual_seed(1)
    src = torch.randn(members, n, generator=g, device="cuda")
    xs = [src[i] for i in range(members)]
    temp = torch.empty(capi.lib().dgb_float_compress_temp_bytes(capi.FLOAT32, members, n) + 256, dtype=torch.uint8,
                       device="cuda")
    rows = {}
    for arm, adt in (("narrow", dtype), ("cast", dtype), ("fp32", torch.float32)):
        cols = ops.max_float_compressed_size(torch.empty(0, dtype=adt), n)
        rows[arm] = (torch.empty(members, cols, dtype=torch.uint8, device="cuda"),
                     torch.empty(members, dtype=torch.int32, device="cuda"))

    def narrow():
        ops.compress_data(True, xs, False, temp, *rows["narrow"], archive_dtype=dtype)

    def cast_only():
        return [x.to(dtype) for x in xs]

    def cast():
        ops.compress_data(True, cast_only(), False, temp, *rows["cast"])

    def fp32():
        ops.compress_data(True, xs, False, temp, *rows["fp32"])

    arms = {"narrow": narrow, "cast": cast, "fp32": fp32}
    for fn in arms.values():  # warm-up, and the sizes check
        fn()
    torch.cuda.synchronize()
    assert rows["narrow"][1].tolist() == rows["cast"][1].tolist(), "narrowing archives differ in size from the cast's"
    best = {k: float("inf") for k in list(arms) + ["cast_kernels"]}
    for _ in range(rounds):
        for k, fn in arms.items():
            best[k] = min(best[k], timed(fn, iters))
        best["cast_kernels"] = min(best["cast_kernels"], timed(cast_only, iters))
    words = members * n
    out = []
    for k, fn in arms.items():
        arch = int(rows[k][1].sum())
        per_word = {"narrow": 8, "cast": 10, "fp32": 8}[k]
        alg = per_word * words + arch
        rec = {"arm": k, "dtype": str(dtype).replace("torch.", ""), "members": members, "words": n,
               "call_us": round(best[k], 1), "kernel_us": {s: round(v, 1) for s, v in kernel_us(fn, iters).items()},
               "alg_bytes_per_word": round(alg / words, 3), "alg_GBs": round(alg / best[k] / 1e3, 1),
               "share_of_3.35TBs": round(alg / best[k] / 1e3 / PEAK_GBS, 3),
               "extra_device_bytes": extra_bytes(fn)}
        if k == "cast":
            rec["cast_kernels_us"] = round(best["cast_kernels"], 1)
        out.append(rec)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--dtype", choices=list(TYPES) + ["both"], default="both")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("narrow_bench.py needs a CUDA device")
    head = {"card": card()}
    print(json.dumps(head), flush=True)
    res = [head]
    for name, dtype in TYPES.items():
        if args.dtype not in (name, "both"):
            continue
        for members, n in SHAPES:
            for rec in bench(members, n, dtype, args.iters, args.rounds):
                print(json.dumps(rec), flush=True)
                res.append(rec)
            torch.cuda.empty_cache()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
