"""float64 codec against the byte codec on the same N(0,1) float64 tensors, on one GPU.

    python tools/float64_bench.py [--iters 30] [--opts 'encode_wide_table=0' ...]

Shapes: 64 x 512 Ki words (256 MiB, the c3 byte volume) and 1 x 32 Mi words.  For each shape and option set:
  - event-timed encode and decode calls (inputs, archives and scratch preallocated; the two codecs alternate
    within the run), reported as time and as uncompressed GB/s;
  - the compression ratio (archive bytes / input bytes) of both codecs;
  - per-kernel fractions of the H100 SXM data sheet's 3.35 TB/s HBM3 bandwidth with option timing=1: algorithmic
    bytes as in DESIGN.md section 5 with U = 8 n (stats = U, encode = U + C, decode = C + U) over the summed
    event-timed kernel durations.
It prints the card name and power limit first; DIETGPU_B200_LIB selects an experiment build of the library.
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from dietgpu_b200 import capi, ops  # noqa: E402

PEAK_GBS = 3350.0  # H100 SXM data sheet, HBM3


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit unknown"
    return f"{name} ({q})"


class Codec:
    """One codec (float64 or byte) over a fixed batch: every buffer allocated once."""

    def __init__(self, as_float, ts):
        self.as_float = as_float
        self.ins = ts if as_float else [t.view(torch.uint8) for t in ts]
        n = len(ts)
        _, cols = ops.max_float_compressed_output_size(self.ins) if as_float else ops.max_any_compressed_output_size(self.ins)
        self.comp = torch.empty((n, cols), dtype=torch.uint8, device="cuda")
        self.sizes = torch.zeros(n, dtype=torch.int32, device="cuda")
        self.temp = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
        self.outs = [torch.empty_like(t) for t in self.ins]
        self.encode()
        torch.cuda.synchronize()
        hs = self.sizes.cpu().tolist()
        self.rows = [self.comp[i, :hs[i]] for i in range(n)]
        self.archive_bytes = sum(hs)

    def encode(self):
        ops.compress_data(self.as_float, self.ins, False, self.temp, self.comp, self.sizes)

    def decode(self):
        ops.decompress_data(self.as_float, self.rows, self.outs, False, self.temp)

    def check(self):
        self.decode()
        torch.cuda.synchronize()
        return all(torch.equal(a, b) for a, b in zip(self.ins, self.outs)) if not self.as_float else \
            all(torch.equal(a.view(torch.int64), b.view(torch.int64)) for a, b in zip(self.ins, self.outs))


def timed(fn, iters):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3  # us


def kernel_fractions(c, U):
    capi.set_option("timing", 1)
    try:
        capi.kernel_times()
        for _ in range(5):
            c.encode()
            c.decode()
        kt = capi.kernel_times()
    finally:
        capi.set_option("timing", 0)
    C = c.archive_bytes
    alg = {"stats": U, "encode": U + C, "decode": C + U}
    out = {}
    for k, b in alg.items():
        ms, cnt = kt[k]
        if cnt:
            us = ms * 1e3 / 5
            out[k] = (us, b / us / 1e3 / PEAK_GBS)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--opts", nargs="*", default=[""], help="option sets, e.g. 'encode_wide_table=0,encode_slot_words=1536'")
    a = ap.parse_args()
    print("card:", card(), "| library:", capi.LIB_PATH, flush=True)
    g = torch.Generator(device="cuda").manual_seed(1234)
    for shape in ((64, 512 * 1024), (1, 32 * 1024 * 1024)):
        x = torch.randn(shape, generator=g, dtype=torch.float64, device="cuda")
        ts = [x[i] for i in range(shape[0])]
        U = x.numel() * 8
        byte = Codec(False, ts)
        assert byte.check(), "byte codec round trip"
        for v in a.opts:
            saved = {}
            for kv in [s for s in v.split(",") if s]:
                k, val = kv.split("=")
                saved[k] = capi.get_option(k)
                capi.set_option(k, int(val))
            f64 = Codec(True, ts)
            assert f64.check(), "float64 round trip"
            res = {"f64": [[], []], "bytes": [[], []]}
            for _ in range(3):  # alternate the two codecs
                for name, c in (("f64", f64), ("bytes", byte)):
                    res[name][0].append(timed(c.encode, a.iters))
                    res[name][1].append(timed(c.decode, a.iters))
            for name, c in (("f64", f64), ("bytes", byte)):
                te, td = min(res[name][0]), min(res[name][1])
                kf = " ".join(f"{k} {us:.1f}us {fr:.2f}" for k, (us, fr) in kernel_fractions(c, U).items())
                print(f"{shape[0]}x{shape[1]} [{v or 'defaults'}] {name:5s} ratio {c.archive_bytes / U:.4f} | "
                      f"enc {te:.1f}us {U / te / 1e3:.0f} GB/s (runs {' '.join(f'{t:.1f}' for t in res[name][0])}) | "
                      f"dec {td:.1f}us {U / td / 1e3:.0f} GB/s (runs {' '.join(f'{t:.1f}' for t in res[name][1])}) | "
                      f"kernels (us, share of 3.35 TB/s): {kf}", flush=True)
            for k, val in saved.items():
                capi.set_option(k, val)
            del f64
        del byte, x, ts
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
