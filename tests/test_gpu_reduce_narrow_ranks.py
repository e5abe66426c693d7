"""The out_dtype of the compressed reduce-scatter and all-reduce on 1-4 ranks, with reduce_dtype=torch.float32 for
16-bit tensors and, in the reduce-scatter, wire_dtype for float32 tensors (gloo ranks sharing cuda:0 on a one-GPU
machine, NCCL with one GPU per rank where there are enough).

rank_data(..., widened=True) makes the float32 sum depend on the rank order, so a result equal to the float32 result
.to(out_dtype) on every rank shows that the fold kept its order through the narrowing kernel, the own chunk's torch
add and the last rank's torch rounding.  The all-reduce's second phase must gather 16-bit archives: the payload of its
all-gather is recorded and compared with the float32 gather's."""
import numpy as np
import pytest
import torch

from multirank import rank_data, run_ranks

pytestmark = pytest.mark.gpu


def _same(a, b, what):
    """Bit equality of two 16-bit tensors, any NaN matching any NaN (the kernel's and torch's roundings may pick
    different NaN payloads)."""
    assert a.dtype == b.dtype and a.shape == b.shape, (what, a.dtype, b.dtype, a.shape, b.shape)
    ok = (a.view(torch.int16) == b.view(torch.int16)) | (a.isnan() & b.isnan())
    assert bool(ok.all()), f"{what}: {int((~ok).sum())} of {a.numel()} elements differ"


class _GatherBytes:
    """Records the uint8 payload bytes every torch.distributed.all_gather_into_tensor call sends."""

    def __init__(self, dist):
        self.dist, self.orig, self.sent = dist, dist.all_gather_into_tensor, []

    def __enter__(self):
        def rec(out, inp, *a, **k):
            if inp.dtype == torch.uint8:
                self.sent.append(inp.numel())
            return self.orig(out, inp, *a, **k)
        self.dist.all_gather_into_tensor = rec
        return self

    def __exit__(self, *exc):
        self.dist.all_gather_into_tensor = self.orig


def _worker(rank, world, dev):
    import torch.distributed as dist

    import dietgpu_b200 as dg

    done = 0
    s = float(np.float32(-0.3) / np.float32(world))
    for dt in (torch.float16, torch.bfloat16):
        n = world * 12289
        for variant in ("plain", "sparse", "average", "scale_tensor", "wire", "wire-average"):
            wire = variant.startswith("wire")
            kw = dict(members=3)
            if wire:
                g = torch.Generator().manual_seed(400 + rank)
                x = (torch.randn(n, generator=g) * (1 + rank)).to(dev)
                x[::97] = 0.0
                x[5] = 65504.0 if dt == torch.float16 else 3e38  # 16-bit words whose float32 sum overflows fp16
                kw["wire_dtype"] = dt
            else:
                x = rank_data(dt, n, world, 500 + done, widened=True)[rank].to(dev)
                kw["reduce_dtype"] = torch.float32
            if variant == "sparse":
                kw["sparse"] = True
            if variant.endswith("average"):
                kw["average"] = True
            tag = f"{dt} {variant} world {world}"
            if variant == "scale_tensor":
                fi_w, fi_n = torch.zeros(1, device=dev), torch.zeros(1, device=dev)
                want = dg.reduce_scatter_compressed(x, scale_tensor=torch.tensor([s], device=dev), found_inf=fi_w,
                                                    **kw).to(dt)
                got = dg.reduce_scatter_compressed(x, scale_tensor=torch.tensor([s], device=dev), found_inf=fi_n,
                                                   out_dtype=dt, **kw)
                assert float(fi_n) == float(bool((~torch.isfinite(want)).any())), f"reduce_scatter {tag} flag"
            else:
                want = dg.reduce_scatter_compressed(x, **kw).to(dt)
                got = dg.reduce_scatter_compressed(x, out_dtype=dt, **kw)
            _same(got, want, f"reduce_scatter {tag}")
            done += 1
            for m in (() if wire else (1, 30001)):  # all_reduce_compressed has no wire dtype
                xa = x[:m].contiguous()
                ekw = dict(kw)
                fi_w = fi_n = None
                if variant == "scale_tensor":
                    fi_w, fi_n = torch.zeros(1, device=dev), torch.zeros(1, device=dev)
                    ekw["scale_tensor"] = torch.tensor([s], device=dev)
                with _GatherBytes(dist) as wide:
                    want = dg.all_reduce_compressed(xa, found_inf=fi_w, **ekw)
                with _GatherBytes(dist) as narrow:
                    got = dg.all_reduce_compressed(xa, out_dtype=dt, found_inf=fi_n, **ekw)
                assert want.dtype == torch.float32 and got.dtype == dt, tag
                _same(got, want.to(dt), f"all_reduce {tag} n {m}")
                if fi_n is not None:
                    assert float(fi_n) == float(bool((~torch.isfinite(got)).any())), f"all_reduce {tag} n {m} flag"
                if world > 1 and m > 1:
                    # the second phase gathered 16-bit archives: well under the float32 gather's payload
                    assert sum(narrow.sent) < 0.75 * sum(wide.sent), (tag, narrow.sent, wide.sent)
                done += 1
    return done


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_out_dtype_collectives(world):
    run_ranks(_worker, world, backend="gloo", timeout=600)
