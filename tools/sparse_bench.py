"""Sparse fp16 / bf16 / fp32 archives (float types 5, 6 and 8) against the dense float codec on the same data, on one
GPU.

    python tools/sparse_bench.py [--iters 30] [--dtype float32]

Shapes: the c4 shape (256 x 512 Ki fp16) and 64 x 2 Mi bf16, both ReLU(N(0,1)); with --dtype float32, 64 x 1 Mi and
256 x 256 Ki fp32 ReLU(N(0,1)) and 64 x 1 Mi fp32 N(0,1) with the 90 % smallest magnitudes of each member set to +0.  For each shape, dense and sparse alternate within
the run:
  - event-timed encode and decode calls (inputs, archives and scratch preallocated), as time and as uncompressed
    GB/s;
  - the compression ratio (archive bytes / input bytes); the sparse archives' sizes are checked member by member
    against the CPU restatement in tests/sparse_oracle.py;
  - per-kernel fractions of the H100 SXM data sheet's 3.35 TB/s HBM3 bandwidth with option timing=1: algorithmic
    bytes as in DESIGN.md section 5 (stats = U, plus the block table for sparse; encode = U + C; decode = C + U)
    over the summed event-timed kernel durations.
It prints the card name and power limit first; DIETGPU_B200_LIB selects an experiment build of the library.
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
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
    """The dense or the sparse float codec over a fixed batch: every buffer allocated once."""

    def __init__(self, sparse, ts):
        self.sparse = sparse
        self.ins = ts
        n = len(ts)
        _, cols = ops.max_float_compressed_output_size(ts, sparse=sparse)
        self.comp = torch.empty((n, cols), dtype=torch.uint8, device="cuda")
        self.sizes = torch.zeros(n, dtype=torch.int32, device="cuda")
        self.temp = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
        self.outs = [torch.empty_like(t) for t in ts]
        self.encode()
        torch.cuda.synchronize()
        self.hs = self.sizes.cpu().tolist()
        self.rows = [self.comp[i, :self.hs[i]] for i in range(n)]
        self.archive_bytes = sum(self.hs)

    def encode(self):
        ops.compress_data(True, self.ins, False, self.temp, self.comp, self.sizes, sparse=self.sparse)

    def decode(self):
        ops.decompress_data(True, self.rows, self.outs, False, self.temp, sparse=self.sparse)

    def check(self):
        self.decode()
        torch.cuda.synchronize()
        iv = torch.int32 if self.ins[0].element_size() == 4 else torch.int16
        return all(torch.equal(a.view(iv), b.view(iv)) for a, b in zip(self.ins, self.outs))


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


def kernel_fractions(c, U, table_bytes):
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
    alg = {"stats": U + (table_bytes if c.sparse else 0), "encode": U + C, "decode": C + U}
    out = {}
    for k, b in alg.items():
        ms, cnt = kt[k]
        if cnt:
            us = ms * 1e3 / 5
            out[k] = (us, b / us / 1e3 / PEAK_GBS)
    return out


def workloads(dtype, g):
    """(label, n x k tensor) pairs"""
    if dtype == "float32":
        for n, k in ((64, 1 << 20), (256, 256 * 1024)):
            yield "relu", torch.randn((n, k), generator=g, device="cuda").relu_()
        x = torch.randn((64, 1 << 20), generator=g, device="cuda")
        kth = x.abs().kthvalue(int(0.9 * x.size(1)), dim=1, keepdim=True).values
        yield "pruned90", x.masked_fill(x.abs() <= kth, 0.0)
        return
    yield "relu", torch.randn((256, 512 * 1024), generator=g, device="cuda").relu_().to(torch.float16)
    yield "relu", torch.randn((64, 2 * 1024 * 1024), generator=g, device="cuda").relu_().to(torch.bfloat16)


def main():
    import sparse32_oracle as S32
    import sparse_oracle as S

    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--dtype", choices=["float16/bfloat16", "float32"], default="float16/bfloat16")
    a = ap.parse_args()
    print("card:", card(), "| library:", capi.LIB_PATH, flush=True)
    g = torch.Generator(device="cuda").manual_seed(1234)
    for label, x in workloads(a.dtype, g):
        n, k = x.shape
        dtype = x.dtype
        ts = [x[i] for i in range(n)]
        U = x.numel() * x.element_size()
        table_bytes = n * S.table_bytes(k)
        codecs = {"dense": Codec(False, ts), "sparse": Codec(True, ts)}
        for name, c in codecs.items():
            assert c.check(), f"{name} round trip"
        if dtype == torch.float32:
            host = x.view(torch.int32).cpu().numpy().view(np.uint32)
            cpu = [S32.compress(host[i], 10).size for i in range(n)]
        else:
            host = x.view(torch.int16).cpu().numpy().view(np.uint16)
            ft = S.F16S if dtype == torch.float16 else S.BF16S
            cpu = [S.compress(host[i], ft, 10).size for i in range(n)]
        assert codecs["sparse"].hs == cpu, "sparse archive sizes differ from the CPU restatement's"
        res = {name: [[], []] for name in codecs}
        for _ in range(3):  # alternate the two codecs
            for name, c in codecs.items():
                res[name][0].append(timed(c.encode, a.iters))
                res[name][1].append(timed(c.decode, a.iters))
        for name, c in codecs.items():
            te, td = min(res[name][0]), min(res[name][1])
            kf = " ".join(f"{kk} {us:.1f}us {fr:.2f}" for kk, (us, fr) in kernel_fractions(c, U, table_bytes).items())
            extra = f" (CPU restatement {sum(cpu) / U:.4f})" if name == "sparse" else ""
            tag = f" {label}" if dtype == torch.float32 else ""  # the fp16 / bf16 lines keep their format
            print(f"{n}x{k} {str(dtype).split('.')[1]}{tag} {name:6s} ratio {c.archive_bytes / U:.4f}{extra} | "
                  f"enc {te:.1f}us {U / te / 1e3:.0f} GB/s (runs {' '.join(f'{t:.1f}' for t in res[name][0])}) | "
                  f"dec {td:.1f}us {U / td / 1e3:.0f} GB/s (runs {' '.join(f'{t:.1f}' for t in res[name][1])}) | "
                  f"kernels (us, share of 3.35 TB/s): {kf}", flush=True)
        del codecs, x, ts
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
