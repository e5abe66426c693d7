"""Host-buffer front end: pinned host tensors in, archives in pinned host memory out, and back.

The reference's operators (dietgpu/DietGpu.cpp:915-937) take device tensors only, so a caller whose
data lives in host memory copies the whole batch up, runs the operator, and copies the result down:
three phases that use the PCIe link in one direction at a time and leave it idle while the kernels
run.  The codec kernels here move >1 TB/s, so for host data the link is the whole cost.  HostCodec
cuts the batch into groups of members (members are independent, SURVEY.md section 8e) and runs
upload / codec call / download of different groups on three CUDA streams: both PCIe directions are
busy at once and the kernels disappear behind the copies.  Archives are byte-for-byte what
compress_data produces for the same members (a member's archive does not depend on its batch).

Everything below is stream plumbing around dietgpu_b200.ops; the codec work is the same C-ABI calls.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch

from . import capi, ops


def _nbytes(t: torch.Tensor) -> int:
    return t.numel() * t.element_size()


def _storage(t: torch.Tensor) -> int:
    """Identity of the allocation a tensor views."""
    return t.untyped_storage().data_ptr()


def _copy_runs(dst: Sequence[torch.Tensor], src: Sequence[torch.Tensor], stream: torch.cuda.Stream) -> None:
    """dst[i] <- src[i] (same byte sizes), one DMA per maximal run of members that are byte-adjacent on
    BOTH sides (e.g. slices of one pinned buffer -> the packed device staging buffer).  A run never spans
    two allocations: separately pinned tensors may happen to sit back to back, and one copy across both is
    invalid."""
    L, st = capi.lib(), stream.cuda_stream
    i, n = 0, len(dst)
    while i < n:
        d0, s0 = dst[i].data_ptr(), src[i].data_ptr()
        ds, ss = _storage(dst[i]), _storage(src[i])
        total = _nbytes(src[i])
        j = i + 1
        while (j < n and dst[j].data_ptr() == d0 + total and src[j].data_ptr() == s0 + total
               and _storage(dst[j]) == ds and _storage(src[j]) == ss):
            total += _nbytes(src[j])
            j += 1
        capi.check(L.dgb_copy_async(d0, s0, total, st), "copy")
        i = j


def _row_room(rows: Sequence[torch.Tensor]) -> int:
    """Bytes that may safely be read from the start of every row (rows are views into larger storages,
    e.g. [i, :size_i] of a pinned [n, cols] matrix): the smallest distance to the end of a row's storage."""
    return min(r.untyped_storage().nbytes() - r.storage_offset() * r.element_size() for r in rows)


def _copy_rows(dst_ptrs: Sequence[int], src_ptrs: Sequence[int], sizes: Sequence[int], dst_cap: int, src_cap: int,
               stream: torch.cuda.Stream, one_allocation: bool = True) -> None:
    """Row i: sizes[i] bytes from src_ptrs[i] to dst_ptrs[i].  When the rows sit at a constant pitch on both
    sides (rows of two [n, cols] matrices; `one_allocation`: all rows of each side lie in one allocation) and
    have similar sizes, one pitched DMA moves the whole group (every row copies max(sizes) bytes: rows have
    dst_cap / src_cap bytes of room); else one copy per row."""
    L, st = capi.lib(), stream.cuda_stream
    n = len(sizes)
    if n == 0:
        return
    w = max(sizes)
    if n > 1 and w > 0 and one_allocation:
        dp, sp = dst_ptrs[1] - dst_ptrs[0], src_ptrs[1] - src_ptrs[0]
        pitched = dp >= w and sp >= w and w <= dst_cap and w <= src_cap and all(
            dst_ptrs[k + 1] - dst_ptrs[k] == dp and src_ptrs[k + 1] - src_ptrs[k] == sp for k in range(n - 1))
        if pitched and w * n <= 1.1 * sum(sizes) + 4096:
            capi.check(L.dgb_copy_rows_async(dst_ptrs[0], dp, src_ptrs[0], sp, w, n, st), "copy rows")
            return
    for d, sp_, k in zip(dst_ptrs, src_ptrs, sizes):
        capi.check(L.dgb_copy_async(d, sp_, k, st), "copy")


class _Pending:
    """Handle of an enqueued HostCodec call; finish() blocks until its host buffers are complete."""

    def __init__(self, fn):
        self._fn = fn
        self._done = False
        self._result = None

    def finish(self):
        if not self._done:
            self._result = self._fn()
            self._done = True
        return self._result


class HostCodec:
    """Reusable context for one batch shape: device staging buffers, streams, pinned size buffers.

    like        : host (or device) tensors giving the member shapes and dtype; uint8 for the byte codec
    groups      : number of member groups the batch is cut into (pipeline depth); clamped to the batch

    compress / decompress are synchronous.  compress_async / decompress_async enqueue the whole call
    and return a handle whose finish() completes it; one compress and one decompress may be in flight
    at the same time (they use separate device buffers), which keeps BOTH directions of the PCIe link
    busy: e.g. upload + coding of batch i+1 overlaps the download of batch i's decoded output.
    """

    def __init__(self, compress_as_float: bool, like: Sequence[torch.Tensor], device=None, groups: int = 8,
                 checksum: bool = False, prob_bits: int = ops.K_DEFAULT_PRECISION):
        if not torch.cuda.is_available():
            raise RuntimeError("dietgpu_b200 has no CPU fallback: HostCodec needs a CUDA device")
        self.as_float, self.checksum, self.prob_bits = bool(compress_as_float), bool(checksum), int(prob_bits)
        self.dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        n = self.n = len(like)
        ops._check(n > 0, "empty batch")
        with torch.cuda.device(self.dev):
            # members packed back to back in one device buffer each way (every float word stays word
            # aligned; the codec accepts any word alignment), so a run of adjacent host members is one DMA
            total = sum(_nbytes(t) for t in like)
            self._flat_in = torch.empty(total + 16, dtype=torch.uint8, device=self.dev)
            self._flat_out = torch.empty(total + 16, dtype=torch.uint8, device=self.dev)
            self.dev_in, self.dev_out, off = [], [], 0
            for t in like:
                nb = _nbytes(t)
                self.dev_in.append(self._flat_in[off:off + nb].view(t.dtype).view(t.shape))
                self.dev_out.append(self._flat_out[off:off + nb].view(t.dtype).view(t.shape))
                off += nb
            _, cols = (ops.max_float_compressed_output_size(self.dev_in) if self.as_float
                       else ops.max_any_compressed_output_size(self.dev_in))
            self.cols = cols
            # separate archive matrices for the two directions: a compress and a decompress may overlap
            self.comp = torch.empty((n, cols), dtype=torch.uint8, device=self.dev)
            self.comp_in = torch.empty((n, cols), dtype=torch.uint8, device=self.dev)
            self.sizes = torch.zeros(n, dtype=torch.int32, device=self.dev)
            self.status = torch.zeros(n, dtype=torch.uint8, device=self.dev)
            self.words = torch.zeros(n, dtype=torch.int32, device=self.dev)
            self.host_sizes = torch.zeros(n, dtype=torch.int32).pin_memory()
            self.host_status = torch.zeros(n, dtype=torch.uint8).pin_memory()
            # up: host->device copies, k: codec calls, dn: device->host payload copies, sz: the small
            # size vectors (their own stream: an archive download must not queue behind the size copy
            # of a LATER group, which waits for that group's upload and kernel)
            self.up, self.k, self.dn, self.sz = (torch.cuda.Stream(self.dev) for _ in range(4))
        g = max(1, min(int(groups), n))
        # contiguous groups with (almost) equal byte counts
        weights = [t.numel() * t.element_size() for t in like]
        total, acc, bounds = sum(weights), 0, [0]
        for i, w in enumerate(weights):
            acc += w
            if len(bounds) < g and acc * g >= total * len(bounds) and i + 1 < n:
                bounds.append(i + 1)
        bounds.append(n)
        self.bounds = [(bounds[j], bounds[j + 1]) for j in range(len(bounds) - 1) if bounds[j + 1] > bounds[j]]
        self.temp: Optional[torch.Tensor] = None
        self._pending_c: Optional[_Pending] = None
        self._pending_d: Optional[_Pending] = None

    def max_archive_bytes(self) -> int:
        """Row size a host archive matrix [n, cols] needs (reference: max_*_compressed_output_size)."""
        return self.cols

    def _temp_for(self, need: int) -> torch.Tensor:
        if self.temp is None or self.temp.numel() < need:
            # growing the scratch while calls are queued on other streams would free memory they use
            torch.cuda.synchronize(self.dev)
            self.temp = torch.empty(need + 256, dtype=torch.uint8, device=self.dev)
        return self.temp

    # ---- compress -------------------------------------------------------------------------------
    def compress_async(self, host_in: Sequence[torch.Tensor], host_comp: torch.Tensor) -> _Pending:
        """Enqueues host_in[i] (pinned) -> archive i in host_comp[i, :size_i] (pinned uint8 [n, >= cols]).
        finish() returns the archive sizes; host_comp is complete when it returns."""
        ops._check(len(host_in) == self.n and host_comp.dim() == 2 and host_comp.size(0) >= self.n)
        ops._check(host_comp.dtype == torch.uint8 and host_comp.size(1) >= self.cols)
        ops._check(self._pending_c is None or self._pending_c._done, "finish() the previous compress first")
        with torch.cuda.device(self.dev):
            cur = torch.cuda.current_stream(self.dev)
            for s in (self.up, self.k, self.dn, self.sz):
                s.wait_stream(cur)
            ev_k, ev_sz = [], []
            for a, b in self.bounds:
                for i in range(a, b):
                    ops._check((host_in[i].numel() == 0 or host_in[i].is_pinned()) and _nbytes(host_in[i]) == _nbytes(self.dev_in[i]),
                               "host inputs must be pinned and match the shapes given to HostCodec")
                _copy_runs(self.dev_in[a:b], host_in[a:b], self.up)
                ev_up = torch.cuda.Event()
                ev_up.record(self.up)
                with torch.cuda.stream(self.k):
                    self.k.wait_event(ev_up)
                    if self.temp is None:  # size the scratch once, on the first group
                        _, _, need = ops.compress_data(self.as_float, self.dev_in[a:b], self.checksum, None,
                                                       self.comp[a:b], self.sizes[a:b], prob_bits=self.prob_bits)
                        self._temp_for(2 * need)
                    else:
                        _, _, need = ops.compress_data(self.as_float, self.dev_in[a:b], self.checksum, self.temp,
                                                       self.comp[a:b], self.sizes[a:b], prob_bits=self.prob_bits)
                        self._temp_for(need)
                    e = torch.cuda.Event()
                    e.record(self.k)
                    ev_k.append(e)
                with torch.cuda.stream(self.sz):
                    self.sz.wait_event(ev_k[-1])
                    self.host_sizes[a:b].copy_(self.sizes[a:b], non_blocking=True)
                    e = torch.cuda.Event()
                    e.record(self.sz)
                    ev_sz.append(e)

        def finish():
            # the exact-size downloads need the sizes on the host: group by group, while later groups
            # are still uploading / encoding
            with torch.cuda.device(self.dev):
                for (a, b), ek, es in zip(self.bounds, ev_k, ev_sz):
                    es.synchronize()
                    self.dn.wait_event(ek)
                    szs = [int(v) for v in self.host_sizes[a:b].tolist()]
                    _copy_rows([host_comp[i].data_ptr() for i in range(a, b)], [self.comp[i].data_ptr() for i in range(a, b)],
                               szs, host_comp.size(1), self.cols, self.dn)
                done = torch.cuda.Event()
                done.record(self.dn)
                done.synchronize()
                torch.cuda.current_stream(self.dev).wait_stream(self.k)
            return [int(v) for v in self.host_sizes.tolist()]

        self._pending_c = _Pending(finish)
        return self._pending_c

    def compress(self, host_in: Sequence[torch.Tensor], host_comp: torch.Tensor) -> List[int]:
        """host_in[i] (pinned) -> archive i in host_comp[i, :size_i] (pinned uint8 [n, >= cols]).
        Returns the archive sizes; host_comp is complete when the call returns."""
        return self.compress_async(host_in, host_comp).finish()

    # ---- decompress -----------------------------------------------------------------------------
    def decompress_async(self, host_rows: Sequence[torch.Tensor], host_out: Sequence[torch.Tensor]) -> _Pending:
        """Enqueues host_rows[i] (pinned uint8 1-D archive i, exact or padded length) -> host_out[i] (pinned).
        finish() raises RuntimeError if a member fails (capacity / header) or, with checksum=True, on a mismatch."""
        ops._check(len(host_rows) == self.n and len(host_out) == self.n)
        ops._check(self._pending_d is None or self._pending_d._done, "finish() the previous decompress first")
        with torch.cuda.device(self.dev):
            cur = torch.cuda.current_stream(self.dev)
            for s in (self.up, self.k, self.dn):
                s.wait_stream(cur)
            for a, b in self.bounds:
                rows, szs = [], []
                for i in range(a, b):
                    sz = host_rows[i].numel()
                    ops._check(host_rows[i].dtype == torch.uint8 and sz <= self.cols and (sz == 0 or host_rows[i].is_pinned()))
                    rows.append(self.comp_in[i, :sz])
                    szs.append(sz)
                # rows of one pinned [n, cols] matrix go up as one pitched DMA per group
                _copy_rows([self.comp_in[i].data_ptr() for i in range(a, b)], [host_rows[i].data_ptr() for i in range(a, b)],
                           szs, self.cols, _row_room(host_rows[a:b]), self.up,
                           len({_storage(r) for r in host_rows[a:b]}) == 1)
                ev_up = torch.cuda.Event()
                ev_up.record(self.up)
                with torch.cuda.stream(self.k):
                    self.k.wait_event(ev_up)
                    need = ops.decompress_data(self.as_float, rows, self.dev_out[a:b], self.checksum, self.temp,
                                               self.status[a:b], self.words[a:b], prob_bits=self.prob_bits)
                    self._temp_for(need)
                    ev_k = torch.cuda.Event()
                    ev_k.record(self.k)
                self.dn.wait_event(ev_k)
                for i in range(a, b):
                    ops._check((host_out[i].numel() == 0 or host_out[i].is_pinned()) and _nbytes(host_out[i]) == _nbytes(self.dev_out[i]))
                _copy_runs(host_out[a:b], self.dev_out[a:b], self.dn)
            with torch.cuda.stream(self.dn):
                self.host_status.copy_(self.status, non_blocking=True)
                done = torch.cuda.Event()
                done.record(self.dn)

        def finish():
            with torch.cuda.device(self.dev):
                done.synchronize()
                torch.cuda.current_stream(self.dev).wait_stream(self.k)
            if not bool(self.host_status.all()):
                bad = [i for i, v in enumerate(self.host_status.tolist()) if not v]
                raise RuntimeError(f"HostCodec.decompress: members {bad[:8]} failed (capacity or header)")

        self._pending_d = _Pending(finish)
        return self._pending_d

    def decompress(self, host_rows: Sequence[torch.Tensor], host_out: Sequence[torch.Tensor]) -> None:
        """host_rows[i]: pinned uint8 1-D archive i (exact or padded length) -> host_out[i] (pinned).
        Raises RuntimeError if a member fails (capacity / header) or, with checksum=True, on a mismatch."""
        self.decompress_async(host_rows, host_out).finish()
