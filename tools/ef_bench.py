"""Narrowing compress with error feedback (compress_data(archive_dtype=T, error_feedback=es)) against the same step
made of torch passes around the plain narrowing compress, on one GPU.

    python tools/ef_bench.py [--iters 20] [--rounds 3] [--json out.json]

For M members x N float32 words (seeded N(0,1) gradients, residuals of a previous step) and T in (bfloat16, float16),
three arms are timed on the same inputs, alternating within the run, and the lowest of `rounds` rounds is reported:
  (1) fused:  compress_data(True, xs, archive_dtype=T, error_feedback=es), one call;
  (2) torch:  y = x + e; w = y.to(T); e = torch.where(w.isfinite(), y - w.float(), 0); then compress_data(True, ys,
              archive_dtype=T), the narrowing compress of y;
  (3) plain:  compress_data(True, xs, archive_dtype=T), the narrowing compress without error feedback.
Reported per arm: call time (CUDA events around `iters` calls), the codec's kernel times with option timing=1 (slots
"stats" and "encode"), for (2) the torch passes' time alone, and the byte model per word (not measured):
(1) 8 + 8 + 4 B (statistics and coder each read x and e; the coder writes e'), (2) 12 + 6 + 10 + 4 + 4 B (the add,
the cast, the residual passes, then the compress's two reads of y), (3) 4 + 4 B, each plus the archive bytes, with
their rate over the call time.  Before timing, (1) and (2) run once from the same residuals with encode_canonical=1,
and their archives (byte for byte) and residuals (bit for bit) must be the same.  The card name and power limit are
read in the same run.
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
SHAPES = [(64, 2 << 20)]  # (members, float32 words per member)
TYPES = {"bfloat16": torch.bfloat16, "float16": torch.float16}
MODEL = {"fused": 20, "torch": 36, "plain": 8}  # bytes per word, before the archive


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


def bench(members, n, dtype, iters, rounds):
    g = torch.Generator(device="cuda").manual_seed(1)
    src = torch.randn(members, n, generator=g, device="cuda")
    e_init = torch.randn(members, n, generator=g, device="cuda") * 2 ** -9
    xs = [src[i] for i in range(members)]
    temp = torch.empty(capi.lib().dgb_float_compress_temp_bytes(capi.FLOAT32, members, n) + 256, dtype=torch.uint8,
                       device="cuda")
    cols = ops.max_float_compressed_size(torch.empty(0, dtype=dtype), n)
    rows = {k: (torch.empty(members, cols, dtype=torch.uint8, device="cuda"),
                torch.empty(members, dtype=torch.int32, device="cuda")) for k in MODEL}
    err = {k: e_init.clone() for k in ("fused", "torch")}
    ys = torch.empty_like(src)
    zero = torch.zeros((), device="cuda")

    def fused():
        ops.compress_data(True, xs, False, temp, *rows["fused"], archive_dtype=dtype,
                          error_feedback=[err["fused"][i] for i in range(members)])

    def torch_passes():
        e = err["torch"]
        torch.add(src, e, out=ys)
        w = ys.to(dtype)
        torch.where(w.isfinite(), ys - w.float(), zero, out=e)

    def torch_arm():
        torch_passes()
        ops.compress_data(True, [ys[i] for i in range(members)], False, temp, *rows["torch"], archive_dtype=dtype)

    def plain():
        ops.compress_data(True, xs, False, temp, *rows["plain"], archive_dtype=dtype)

    arms = {"fused": fused, "torch": torch_arm, "plain": plain}
    # the check: one step of (1) and (2) from the same residuals, canonical archives
    capi.set_option("encode_canonical", 1)
    try:
        fused()
        torch_arm()
    finally:
        capi.set_option("encode_canonical", 0)
    torch.cuda.synchronize()
    same_res = torch.equal(err["fused"].view(torch.int32), err["torch"].view(torch.int32))
    hs = rows["fused"][1].tolist()
    same_sizes = hs == rows["torch"][1].tolist()
    same_arch = same_sizes and all(torch.equal(rows["fused"][0][i, :hs[i]], rows["torch"][0][i, :hs[i]])
                                   for i in range(members))
    assert same_res and same_arch, f"fused and torch steps differ: residuals {same_res}, archives {same_arch}"
    for fn in arms.values():  # warm-up of the default (completion-order) path
        fn()
    torch.cuda.synchronize()
    best = {k: float("inf") for k in list(arms) + ["torch_passes"]}
    for _ in range(rounds):
        for k, fn in arms.items():
            best[k] = min(best[k], timed(fn, iters))
        best["torch_passes"] = min(best["torch_passes"], timed(torch_passes, iters))
    words = members * n
    out = []
    for k, fn in arms.items():
        arch = int(rows[k][1].sum())
        alg = MODEL[k] * words + arch
        rec = {"arm": k, "dtype": str(dtype).replace("torch.", ""), "members": members, "words": n,
               "call_us": round(best[k], 1), "kernel_us": {s: round(v, 1) for s, v in kernel_us(fn, iters).items()},
               "model_bytes_per_word": round(alg / words, 3), "model_GBs": round(alg / best[k] / 1e3, 1),
               "share_of_3.35TBs": round(alg / best[k] / 1e3 / PEAK_GBS, 3),
               "canonical_archives_and_residuals_equal": True}
        if k == "torch":
            rec["torch_passes_us"] = round(best["torch_passes"], 1)
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
        sys.exit("ef_bench.py needs a CUDA device")
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
