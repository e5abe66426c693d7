"""fp8 wire measurements (DESIGN.md f-16): CUDA-event times of

  (a) the scaled fp8 cast (ops.cast_fp8) against torch's (x.float() * s).clamp(-M, M).to(fp8), with the cast's share of
      3.35 TB/s (the H100 SXM data sheet's HBM3 bandwidth) for the bytes it must move (read the input, write q);
  (b) the fp8 compress: cast + histogram + byte encode given the histogram (compress_data(archive_dtype=fp8)), cast
      without histogram + byte encode with its own statistics pass, torch's cast + byte compress, and the bf16
      narrowing compress of the same input (compress_data(archive_dtype=bfloat16));
  (c) the fp8 decode-and-sum into fp32 (device scale) against the bf16 widening device-scale sum, on the
      (groups x archives x elements) shapes of tools/reduce_bench.py;
  (d) archive bytes per element of fp8 and bf16 archives for N(0, 1), Student-t(3) and ReLU(N(0, 1)) inputs.

Usage: python tools/fp8_bench.py [--out DIR] [--reps R].  Prints one JSON object and writes it to DIR/fp8_bench.json,
with the card's name and power limit read in the same run.  A GPU is required."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dietgpu_b200 import ops  # noqa: E402

PEAK = 3.35e12
N = 1 << 24  # elements per (a) / (b) input: 64 MiB of fp32
MAX = {torch.float8_e4m3fn: 448.0, torch.float8_e5m2: 57344.0}
SHAPES = [(8, 8, 2 << 20), (16, 4, 1 << 20), (64, 2, 512 << 10)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, reps):
    """Median milliseconds of fn() over reps runs, each bracketed by CUDA events, after three warm-up runs."""
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def data(kind, n, dtype=torch.float32):
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(n, generator=g, device="cuda")
    if kind == "t3":
        c = torch.distributions.Chi2(torch.tensor(3.0, device="cuda")).sample((n,))
        x = x / torch.sqrt(c / 3)
    elif kind == "relu":
        x = x.clamp_min(0)
    return x.to(dtype)


def amax_scale(x, dt):
    return (MAX[dt] / x.abs().float().max()).reshape(1).to(torch.float32)


def bench_cast(reps):
    rows = []
    for dtype in (torch.float32, torch.bfloat16):
        x = data("normal", N, dtype)
        for dt in MAX:
            s = amax_scale(x, dt)
            t_ours = timed(lambda: ops.cast_fp8([x], dt, s), reps)
            t_torch = timed(lambda: (x.float() * s).clamp(-MAX[dt], MAX[dt]).to(dt), reps)
            need = N * (x.element_size() + 1)
            rows.append(dict(input=str(dtype), fp8=str(dt), cast_ms=t_ours, torch_ms=t_torch,
                             cast_share_of_peak=need / (t_ours * 1e-3) / PEAK,
                             torch_share_of_peak=need / (t_torch * 1e-3) / PEAK))
    return rows


def bench_compress(reps):
    rows = []
    for dtype in (torch.float32, torch.bfloat16):
        x = data("normal", N, dtype)
        xs = list(x.split(N // 8))  # 8 members, as the collectives send them
        for dt in MAX:
            s = amax_scale(x, dt)
            fused = timed(lambda: ops.compress_data(True, xs, archive_dtype=dt, scale_tensor=s), reps)

            def no_hist():
                q = ops.cast_fp8(xs, dt, s)
                return ops.compress_data(False, [t.view(torch.uint8) for t in q])

            def torch_cast():
                q = [(t.float() * s).clamp(-MAX[dt], MAX[dt]).to(dt) for t in xs]
                return ops.compress_data(False, [t.view(torch.uint8) for t in q])

            row = dict(input=str(dtype), fp8=str(dt), fused_hist_ms=fused, cast_then_encode_ms=timed(no_hist, reps),
                       torch_cast_then_encode_ms=timed(torch_cast, reps))
            if dtype == torch.float32:
                row["bf16_narrowing_compress_ms"] = timed(
                    lambda: ops.compress_data(True, xs, archive_dtype=torch.bfloat16), reps)
            rows.append(row)
    return rows


def bench_reduce(reps):
    rows = []
    one = torch.ones(1, device="cuda")
    for g, w, n in SHAPES:
        x = data("normal", n)
        members = [(x * (1 + k)).contiguous() for k in range(w)]
        outs = [torch.empty(n, device="cuda") for _ in range(g)]
        row = dict(groups=g, archives=w, elements=n)
        for name, dt in (("e4m3", torch.float8_e4m3fn), ("e5m2", torch.float8_e5m2)):
            s = amax_scale(members[-1], dt)
            comp, sizes, _ = ops.compress_data(True, members, archive_dtype=dt, scale_tensor=s)
            hs = sizes.cpu().tolist()
            arch = [comp[k, :hs[k]] for k in range(w)]
            d = 1.0 / s
            row[f"{name}_sum_ms"] = timed(lambda: ops.decompress_data_reduce([arch] * g, outs, archive_dtype=dt,
                                                                             scale_tensor=d), reps)
        comp, sizes, _ = ops.compress_data(True, [m.to(torch.bfloat16) for m in members])
        hs = sizes.cpu().tolist()
        arch = [comp[k, :hs[k]] for k in range(w)]
        row["bf16_widening_sum_ms"] = timed(lambda: ops.decompress_data_reduce(
            [arch] * g, outs, archive_dtype=torch.bfloat16, scale_tensor=one), reps)
        rows.append(row)
    return rows


def wire_bytes():
    rows = []
    n = 1 << 20
    for kind in ("normal", "t3", "relu"):
        x = data(kind, n)
        row = dict(data=kind)
        comp, sizes, _ = ops.compress_data(True, [x.to(torch.bfloat16)])
        row["bf16_bytes_per_elem"] = int(sizes[0]) / n
        for name, dt in (("e4m3", torch.float8_e4m3fn), ("e5m2", torch.float8_e5m2)):
            comp, sizes, _ = ops.compress_data(True, [x], archive_dtype=dt, scale_tensor=amax_scale(x, dt))
            row[f"{name}_bytes_per_elem"] = int(sizes[0]) / n
        rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fp8_bench needs a CUDA device")
    res = dict(card=card(), reps=a.reps, cast=bench_cast(a.reps), compress=bench_compress(a.reps),
               reduce=bench_reduce(a.reps), wire=wire_bytes())
    js = json.dumps(res, indent=1)
    print(js)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "fp8_bench.json"), "w") as f:
            f.write(js)


if __name__ == "__main__":
    main()
