"""Compressed collectives: the use the reference names for this codec ("compress before a collective",
README.md:72, 103-104; SURVEY.md section 8f rank 3) and ships no code for.

    all_gather_compressed(t)       every rank contributes t, every rank receives the concatenation
    all_to_all_compressed(chunks)  rank r sends chunks[d] to rank d and receives one chunk from every rank
    reduce_scatter_compressed(t)   rank r receives the elementwise sum over ranks of chunk r of t
    all_reduce_compressed(t)       every rank receives the elementwise sum over ranks of t

Each rank compresses what it sends, the ranks exchange the variable-size archives, every rank
decompresses what it received.  The wire carries about `ratio` x the raw bytes (0.67 for bf16
activations).  The work is cut into `stages` pieces that move through compress -> exchange ->
decompress as a pipeline: while piece k is on the wire (NCCL, asynchronous), piece k+1 is being
compressed and piece k-1 decompressed, and the one host synchronisation an exchange needs (the archive
sizes) waits behind the next piece's codec launch instead of in front of the wire.

The codec work is the ordinary operator path (dietgpu_b200.ops -> C ABI -> sm_90a kernels) on the
caller's device; there is no CPU fallback for it.  The exchange itself is torch.distributed plumbing:
NCCL moves device buffers directly; on a backend without device collectives (gloo, used by the
single-GPU multi-process tests) the packed archives are staged through host memory.

Two transports:

  * NCCL (default; any backend torch.distributed offers, gloo for the single-GPU tests): archives are
    packed and exchanged by collectives, with a host synchronisation for the sizes in the middle: a
    tool for links much slower than the codec (inter-node), which is where the reference aims it.
  * peer memory (`PeerWorkspace`, one node, NVLink / NVSwitch): every rank encodes into a buffer its peers
    have mapped (torch symmetric memory: CUDA VMM handles exchanged once at set-up); no packing, no size
    exchange (sizes are read from the archive headers on the device), no host synchronisation, CUDA-graph
    capturable.  Three ways to move the bytes, all bit-exact (tests/test_gpu_collectives.py):
      "pull"   one device-side barrier, then the archive mover (dgb_archives_pull: a 64-CTA kernel that copies
               exactly each archive's bytes) reads the peers' archives on a side stream, unit u+1 while the
               decoder works on unit u from local memory;
      "push"   no barrier: as soon as a group of members is coded the mover writes it into every peer's inbox
               and raises a flag there; receivers decode a group when its flag is up;
      "direct" one barrier, then the decode kernel itself reads the peers' archives (its TMA bulk copies and
               cp.async rings take peer addresses like local ones).
    A rank encodes once and every peer fetches, so the codec cost is amortised over world - 1 links: the
    gain over a plain all-gather grows with the world size and the message.  (Not yet measured on H100.)
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist

from . import ops

_ALIGN = 16  # archives are 16 B aligned in the packed buffer (compressed buffers must be, ans/GpuANSEncode.cu:19-21)


def _world(group) -> int:
    return dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1


def _device_collectives(group) -> bool:
    return dist.get_backend(group) == "nccl"


def _round_up(v: int, a: int) -> int:
    return (v + a - 1) // a * a


def pack_offsets(sizes: Sequence[int]) -> Tuple[List[int], int]:
    """Offsets of archives of the given byte sizes in one packed buffer, each 16 B aligned; total bytes."""
    offs, o = [], 0
    for s in sizes:
        offs.append(o)
        o += _round_up(int(s), _ALIGN)
    return offs, o


def _pieces(members: int, stages: int) -> List[Tuple[int, int]]:
    """The non-empty member ranges [a, b) of a cut of `members` into `stages` nearly equal pipeline pieces."""
    cuts = [round(k * members / stages) for k in range(stages + 1)]
    return [(a, b) for a, b in zip(cuts[:-1], cuts[1:]) if b > a]


class _Exchange:
    """One in-flight archive exchange (all-gather of every rank's packed archives)."""

    def __init__(self, rows: Sequence[torch.Tensor], group):
        n = len(rows)
        if n == 0:
            raise ValueError("exchange_archives: empty contribution")
        self.dev = rows[0].device
        for r in rows:
            if r.dtype != torch.uint8 or r.dim() != 1 or r.device != self.dev:
                raise ValueError("exchange_archives: archives must be uint8 1-D tensors on one device")
        self.rows, self.group, self.n = list(rows), group, n
        self.world = _world(group)
        self.work = None
        self.sizes: Optional[List[List[int]]] = None
        if self.world == 1:
            return
        self.on_device = _device_collectives(group)
        cdev = self.dev if self.on_device else torch.device("cpu")
        local_sizes = torch.tensor([r.numel() for r in rows], dtype=torch.int32, device=cdev)
        all_sizes = torch.empty(self.world * n, dtype=torch.int32, device=cdev)
        dist.all_gather_into_tensor(all_sizes, local_sizes, group=group)
        self.sizes = all_sizes.cpu().view(self.world, n).tolist()  # the one host sync of the exchange
        totals = [pack_offsets(s)[1] for s in self.sizes]
        self.width = max(max(totals), _ALIGN)
        rank = dist.get_rank(group)
        send = torch.zeros(self.width, dtype=torch.uint8, device=self.dev)
        offs, _ = pack_offsets(self.sizes[rank])
        for r, o in zip(rows, offs):
            send[o:o + r.numel()].copy_(r)
        if self.on_device:
            self.recv = torch.empty(self.world * self.width, dtype=torch.uint8, device=self.dev)
            self.work = dist.all_gather_into_tensor(self.recv, send, group=group, async_op=True)
        else:
            host = torch.empty(self.world * self.width, dtype=torch.uint8)
            dist.all_gather_into_tensor(host, send.cpu(), group=group)
            self.recv = host.to(self.dev)

    def wait(self) -> List[List[torch.Tensor]]:
        if self.world == 1:
            return [self.rows]
        if self.work is not None:
            self.work.wait()
        out: List[List[torch.Tensor]] = []
        for w in range(self.world):
            offs, _ = pack_offsets(self.sizes[w])
            base = w * self.width
            out.append([self.recv[base + o: base + o + s] for o, s in zip(offs, self.sizes[w])])
        return out


def exchange_archives(rows: Sequence[torch.Tensor], group=None) -> List[List[torch.Tensor]]:
    """All ranks contribute the same NUMBER of archives (uint8 1-D tensors of any sizes, one device).
    Returns, for every rank in rank order, the list of that rank's archives (views into one gathered
    buffer on the same device).  Two collectives: sizes, then the padded payload."""
    return _Exchange(rows, group).wait()


class PeerWorkspace:
    """A byte buffer of `nbytes` per rank that every rank of `group` (one node) has mapped into its own address
    space.  Setting it up is a collective (allocation + handle exchange); keep it and pass it to every
    `*_compressed(..., peer=ws)` call.  The buffer is used in two halves, alternating per call: the
    barrier of call k+1 orders every rank's reads of call k before any rank's writes of call k+2, so
    one device-side barrier per collective is enough."""

    def __init__(self, nbytes: int, group=None, device: Optional[torch.device] = None):
        import torch.distributed._symmetric_memory as symm

        self.group = group if group is not None else dist.group.WORLD
        if dist.get_backend(self.group) != "nccl":
            raise RuntimeError("PeerWorkspace: peer-mapped memory needs one CUDA device per rank (NCCL group)")
        dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.half = _round_up(int(nbytes), 256)
        self.buf = symm.empty(2 * self.half, dtype=torch.uint8, device=dev)
        self.hdl = symm.rendezvous(self.buf, self.group)
        self.rank, self.world = dist.get_rank(self.group), dist.get_world_size(self.group)
        self.calls = 0
        self.timeout_ms = 20000
        self._views = {}
        self._staging = None
        self.side = torch.cuda.Stream(device=dev)  # archive mover: runs beside the decoder

    def begin(self, nbytes: int) -> int:
        """Byte offset of the half this call uses."""
        if nbytes > self.half:
            raise ValueError(f"PeerWorkspace: call needs {nbytes} B per rank, workspace halves hold {self.half} B")
        off = (self.calls & 1) * self.half
        self.calls += 1
        return off

    def view(self, rank: int, offset: int, nbytes: int) -> torch.Tensor:
        """uint8 tensor on THIS rank's device that aliases bytes [offset, offset + nbytes) of `rank`'s buffer."""
        if rank == self.rank:
            return self.buf[offset:offset + nbytes]
        key = (rank, offset, nbytes)
        v = self._views.get(key)
        if v is None:
            if len(self._views) > 512:  # views are cheap to rebuild; do not grow without bound when sizes vary
                self._views.clear()
            v = self._views[key] = self.hdl.get_buffer(rank, (nbytes,), torch.uint8, offset)
        return v

    def staging(self, nbytes: int) -> torch.Tensor:
        """Local (not peer-mapped) buffer the archive mover fills; grown on demand, kept across calls."""
        if self._staging is None or self._staging.numel() < nbytes:
            self._staging = torch.empty(nbytes, dtype=torch.uint8, device=self.buf.device)
        return self._staging[:nbytes]

    def barrier(self) -> None:
        """Device-side barrier of all ranks on the current stream (no host synchronisation)."""
        self.hdl.barrier(channel=0)

    # point-to-point flags on the current stream (channel 0 belongs to barrier()); a lost signal traps the
    # waiting kernel after `timeout_ms` instead of hanging the device
    def signal(self, dst: int, channel: int) -> None:
        self.hdl.put_signal(dst, channel=channel, timeout_ms=self.timeout_ms)

    def wait(self, src: int, channel: int) -> None:
        self.hdl.wait_signal(src, channel=channel, timeout_ms=self.timeout_ms)


def _archive_cols(as_float: bool, dtype: torch.dtype, longest: int) -> int:
    """Row pitch for archives of members of at most `longest` elements (bytes for the byte codec)."""
    b = ops.max_float_compressed_size(torch.empty(0, dtype=dtype), longest) if as_float else ops.max_any_compressed_size(longest)
    return _round_up(int(b), _ALIGN)


def _pull_and_decode(ws: "PeerWorkspace", as_float: bool, dtype: torch.dtype, units, cols: int, checksum: bool,
                     temp_mem: Optional[torch.Tensor], check: bool, direct: bool) -> None:
    """units = [(source rows [k, cols] in peer memory, [k output tensors]), ...].  direct: the decode kernel reads
    the peer rows itself.  Otherwise a two-deep pipeline: the archive mover (dgb_archives_pull, a small grid on
    the workspace's side stream) brings unit u+1 into local staging while the decoder works on unit u."""
    dev = units[0][1][0].device
    statuses = []
    if direct:
        ins = [rows[i] for rows, outs in units for i in range(len(outs))]
        outs = [o for _, os_ in units for o in os_]
        st = torch.zeros(len(ins), dtype=torch.uint8, device=dev)
        ops.decompress_data(as_float, ins, outs, checksum, temp_mem, st)
        statuses.append(st)
    else:
        cur = torch.cuda.current_stream(dev)
        kmax = max(len(outs) for _, outs in units)
        stage = ws.staging(2 * kmax * cols).view(2, kmax, cols)
        start = torch.cuda.Event()
        start.record(cur)
        ws.side.wait_event(start)
        decoded = [None, None]  # event: the decoder is done with staging buffer b
        for u, (rows, outs) in enumerate(units):
            b, k = u & 1, len(outs)
            with torch.cuda.stream(ws.side):
                if decoded[b] is not None:
                    ws.side.wait_event(decoded[b])
                ops.pull_archives(as_float, [rows[i] for i in range(k)], [stage[b, i] for i in range(k)], dtype)
                pulled = torch.cuda.Event()
                pulled.record(ws.side)
            cur.wait_event(pulled)
            st = torch.zeros(k, dtype=torch.uint8, device=dev)
            ops.decompress_data(as_float, [stage[b, i] for i in range(k)], outs, checksum, temp_mem, st)
            statuses.append(st)
            decoded[b] = torch.cuda.Event()
            decoded[b].record(cur)
    if check and not all(bool(st.all()) for st in statuses):
        raise RuntimeError("compressed collective: a peer archive failed to decode")


def _all_gather_push(flat: torch.Tensor, as_float: bool, bounds: List[int], ws: "PeerWorkspace", checksum: bool,
                     temp_mem: Optional[torch.Tensor], check: bool, stages: int) -> torch.Tensor:
    """Push transport: the members are coded in `stages` groups; as soon as a group is coded, the archive mover
    (side stream) WRITES its archives into every peer's inbox -- stores over NVLink are posted, they do not pay the
    round trip a pull does -- and raises a flag there; the receiver decodes a group from its own memory when the
    flag is up.  Coding of group g+1, the pushes of group g and the decoding of what has arrived overlap; there is
    no barrier: the flags of call k+1 order every rank's reads of call k before the writes of call k+2."""
    n, members, world, rank = flat.numel(), len(bounds) - 1, ws.world, ws.rank
    dev = flat.device
    cols = _archive_cols(as_float, flat.dtype, max(bounds[i + 1] - bounds[i] for i in range(members)))
    region = members * cols
    off = ws.begin((world + 1) * region)  # [own archives | inbox of source 0 | ... | inbox of source world-1]
    out = torch.empty(world * n, dtype=flat.dtype, device=dev)
    mine = ws.view(rank, off, region).view(members, cols)
    groups = _pieces(members, max(1, min(int(stages), members, 7)))  # one flag channel per group
    cur = torch.cuda.current_stream(dev)
    peers = [(rank + k) % world for k in range(1, world)]
    sizes = torch.empty(members, dtype=torch.int32, device=dev)
    for g, (a, b) in enumerate(groups):
        ops.compress_data(as_float, [flat[bounds[i]:bounds[i + 1]] for i in range(a, b)], checksum, temp_mem, mine[a:b], sizes[a:b])
        coded = torch.cuda.Event()
        coded.record(cur)
        with torch.cuda.stream(ws.side):
            ws.side.wait_event(coded)
            for p in peers:
                inbox = ws.view(p, off + (1 + rank) * region, region).view(members, cols)
                ops.pull_archives(as_float, [mine[i] for i in range(a, b)], [inbox[i] for i in range(a, b)], flat.dtype)
                ws.signal(p, 1 + g)
    out[rank * n:(rank + 1) * n].copy_(flat)  # own shard: a local copy, no codec
    statuses = []
    for g, (a, b) in enumerate(groups):
        for src in reversed(peers):  # rank - 1 pushed to this rank first
            ws.wait(src, 1 + g)
            rows = ws.view(rank, off + (1 + src) * region, region).view(members, cols)
            st = torch.zeros(b - a, dtype=torch.uint8, device=dev)
            ops.decompress_data(as_float, [rows[i] for i in range(a, b)],
                                [out[src * n + bounds[i]: src * n + bounds[i + 1]] for i in range(a, b)], checksum, temp_mem, st)
            statuses.append(st)
    done = torch.cuda.Event()
    with torch.cuda.stream(ws.side):
        done.record(ws.side)
    cur.wait_event(done)  # the side stream joins (stream capture needs it; the next call's scratch reuse too)
    if check and not all(bool(st.all()) for st in statuses):
        raise RuntimeError("all_gather_compressed: a peer archive failed to decode")
    return out


def _all_gather_peer(flat: torch.Tensor, as_float: bool, bounds: List[int], ws: "PeerWorkspace", checksum: bool,
                     temp_mem: Optional[torch.Tensor], check: bool, direct: bool, stages: int) -> torch.Tensor:
    n, members, world, rank = flat.numel(), len(bounds) - 1, ws.world, ws.rank
    cols = _archive_cols(as_float, flat.dtype, max(bounds[i + 1] - bounds[i] for i in range(members)))
    off = ws.begin(members * cols)
    out = torch.empty(world * n, dtype=flat.dtype, device=flat.device)
    mine = ws.view(rank, off, members * cols).view(members, cols)
    sizes = torch.empty(members, dtype=torch.int32, device=flat.device)
    ops.compress_data(as_float, [flat[bounds[i]:bounds[i + 1]] for i in range(members)], checksum, temp_mem, mine, sizes)
    ws.barrier()  # every rank's archives are complete (and every rank is done with the previous call's other half)
    out[rank * n:(rank + 1) * n].copy_(flat)  # own shard: a local copy, no codec
    pieces = _pieces(members, max(1, min(int(stages), members)))
    units = []
    for k in range(1, world):
        w = (rank + k) % world  # start with a different peer on every rank: spreads the pulls over the links
        rows = ws.view(w, off, members * cols).view(members, cols)
        for a, b in pieces:
            units.append((rows[a:b], [out[w * n + bounds[i]: w * n + bounds[i + 1]] for i in range(a, b)]))
    if units:
        _pull_and_decode(ws, as_float, flat.dtype, units, cols, checksum, temp_mem, check, direct)
    return out


def _split(n: int, parts: int, quantum: int) -> List[int]:
    """Boundaries of `parts` nearly equal pieces of [0, n), interior boundaries multiples of `quantum`."""
    parts = max(1, min(parts, max(1, n // max(quantum, 1))))
    per = (n // parts) // quantum * quantum if parts > 1 else n
    return [i * per for i in range(parts)] + [n]


def _check_wire(t: torch.Tensor, what: str, wire_dtype: Optional[torch.dtype]) -> None:
    """wire_dtype: None, float16 / bfloat16 for a float32 t (narrowing compress on the send side), or an fp8 dtype for
    a float32 or bfloat16 t (the scaled fp8 cast on the send side)."""
    if wire_dtype is None:
        return
    if wire_dtype in ops.FP8_TYPES and t.dtype in (torch.float32, torch.bfloat16):
        return
    if wire_dtype not in (torch.float16, torch.bfloat16) or t.dtype != torch.float32:
        raise ValueError(f"{what}: wire_dtype is None, or float16 / bfloat16 for a float32 tensor, or float8_e4m3fn / "
                         f"float8_e5m2 for a float32 or bfloat16 tensor; not {wire_dtype} for {t.dtype}")


def _check_wire_scale(what: str, wire_scale, wire_dtype: Optional[torch.dtype], dev) -> None:
    """wire_scale: None, or (with an fp8 wire_dtype) a one-element float32 CUDA tensor on dev."""
    if wire_scale is None:
        return
    if wire_dtype not in ops.FP8_TYPES:
        raise ValueError(f"{what}: wire_scale is the scale of an fp8 wire (wire_dtype torch.float8_e4m3fn or "
                         f"torch.float8_e5m2), not of wire_dtype={wire_dtype}")
    ops._check_flag_tensor(f"{what}: wire_scale", wire_scale, dev)


def _check_fp8_wire(what: str, wire_dtype: Optional[torch.dtype], error_feedback) -> None:
    """An fp8 wire takes no error feedback (the residual of a scaled quantiser is not the narrowing compress's)."""
    if wire_dtype in ops.FP8_TYPES and error_feedback is not None:
        raise ValueError(f"{what}: error_feedback is not supported with an fp8 wire_dtype")


def _check_sparse_wire(dtype: torch.dtype, what: str, sparse: bool, wire_dtype: Optional[torch.dtype] = None,
                       peer: Optional[PeerWorkspace] = None) -> None:
    """sparse=True: sparse fp16 / bf16 / fp32 archives on the NCCL / gloo transport, without narrowing."""
    if not sparse:
        return
    if dtype not in _REDUCE_DTYPES:
        raise ValueError(f"{what}: sparse=True needs a float16, bfloat16 or float32 tensor, not {dtype}")
    if wire_dtype is not None:
        raise ValueError(f"{what}: sparse=True cannot be combined with wire_dtype (there is no narrowing compress "
                         "into sparse archives)")
    if peer is not None:
        raise ValueError(f"{what}: sparse=True is not supported with the peer-memory transports")


def _check_feedback(what: str, e: Optional[torch.Tensor], t: torch.Tensor, wire_dtype: Optional[torch.dtype]) -> None:
    """error_feedback: None, or a float32 CUDA tensor shaped like t, laid out like it (contiguous, same address modulo
    16) and not overlapping it, with wire_dtype (it holds the rounding error of the narrowing compress)."""
    if e is None:
        return
    if wire_dtype is None:
        raise ValueError(f"{what}: error_feedback needs wire_dtype (it holds the rounding error of the float32 -> "
                         "wire_dtype compress)")
    if getattr(e, "dtype", None) != torch.float32 or not getattr(e, "is_cuda", False) or e.device != t.device \
            or e.shape != t.shape or not e.is_contiguous():
        raise ValueError(f"{what}: error_feedback must be a contiguous float32 CUDA tensor shaped like t "
                         f"({tuple(t.shape)} on {t.device}); got {getattr(e, 'dtype', type(e))} "
                         f"{tuple(getattr(e, 'shape', ()))} on {getattr(e, 'device', None)}")
    if e.numel() and e.data_ptr() % 16 != t.data_ptr() % 16:
        raise ValueError(f"{what}: error_feedback must start at t's address modulo 16 ({t.data_ptr() % 16} B), "
                         f"not {e.data_ptr() % 16} B")
    if e.numel() and e.data_ptr() < t.data_ptr() + 4 * t.numel() and t.data_ptr() < e.data_ptr() + 4 * e.numel():
        raise ValueError(f"{what}: error_feedback overlaps t")


def _feedback_step(x: torch.Tensor, e: torch.Tensor, wire_dtype: torch.dtype) -> torch.Tensor:
    """The error-feedback step in torch, for the words no compress kernel takes: returns y = x + e and overwrites e
    with the residual torch.where(w.isfinite(), y - w.float(), 0), w = y.to(wire_dtype) (what
    ops.compress_data(error_feedback=) writes)."""
    y = x + e
    w = y.to(wire_dtype)
    e.copy_(torch.where(w.isfinite(), y - w.float(), 0))
    return y


def all_gather_compressed(t: torch.Tensor, group=None, members: int = 8, checksum: bool = False,
                          temp_mem: Optional[torch.Tensor] = None, stages: int = 2,
                          peer: Optional[PeerWorkspace] = None, check: bool = True,
                          peer_mode: str = "auto", wire_dtype: Optional[torch.dtype] = None,
                          sparse: bool = False, error_feedback: Optional[torch.Tensor] = None,
                          wire_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Every rank contributes the CUDA tensor `t` (same shape and dtype on every rank; fp16 / bf16 / fp32 go
    through the float codec, anything else through the byte codec) and receives the concatenation
    [world * t.numel()] in rank order, bit-exact.  `members` = archives per rank (the codec's parallelism
    comes from blocks, so a handful is enough); `stages` = pipeline pieces (see the module docstring).
    With `peer` (a PeerWorkspace of the same group) the archives move through peer-mapped memory instead of a
    collective; `peer_mode` = "auto" (push for two ranks, pull beyond), "pull" (after a barrier the archive mover reads the peers' archives, unit u+1 while
    unit u is decoded; the fastest at 8 GPUs), "push" (the mover writes each coded group into the peers' inboxes
    and flags it; no barrier; the fastest at 2 GPUs) or "direct" (after a barrier the decode kernel reads peer
    memory itself); `stages` = pipeline groups per peer;
    `check=False` then skips the only host synchronisation (the read of the decode status).

    wire_dtype=torch.float16 / torch.bfloat16 with a float32 t (fp32 master weights gathered as 16-bit
    parameters, FSDP's param_dtype): each member is rounded to wire_dtype inside the compress kernels, the 16-bit
    archives go over the wire, and the result has wire_dtype and equals cat([t_r.to(wire_dtype) for every rank r])
    bit for bit.  NCCL / gloo transport only: with `peer` it raises ValueError.

    sparse=True (float16 / bfloat16 / float32 t): the archives are sparse ones (ops.compress_data(sparse=True)),
    which store no bits for +0 and -0 words, so mostly-zero tensors (ReLU activations, pruned weights) take fewer
    bytes on the wire; the result is the same, bit for bit.  NCCL / gloo transport only, and not with wire_dtype:
    either raises ValueError before any communication.

    error_feedback=e (with wire_dtype; a contiguous float32 CUDA tensor shaped like t, at t's address modulo 16):
    the rounding error of the previous call's compress, added back before this one rounds.  The result is exactly
    all_gather_compressed(t + e, wire_dtype=wire_dtype), and e is overwritten with this call's error,
    torch.where(w.isfinite(), y - w.float(), 0) for y = t + e and w = y.to(wire_dtype), inside the compress kernels
    (ops.compress_data(error_feedback=)).  This is the "server error" of the second phase of an fp32 all-reduce
    composed as all_gather_compressed(reduce_scatter_compressed(g, wire_dtype=w, error_feedback=e_w), wire_dtype=w,
    error_feedback=e_s).  Misuse raises ValueError before any communication.

    wire_dtype=torch.float8_e4m3fn / torch.float8_e5m2 with a float32 or bfloat16 t (fp8 parameters gathered for an
    fp8 forward pass): every member is cast with ops.cast_fp8 at the scale wire_scale (a one-element float32 CUDA
    tensor on t's device, the same value on every rank; None means 1) and sent as an fp8 byte archive, and the result
    has wire_dtype and equals cat([ops.cast_fp8([t_r], wire_dtype, wire_scale)[0] for every rank r]) bit for bit.
    NCCL / gloo transport only, and not with error_feedback; wire_scale without an fp8 wire_dtype raises ValueError."""
    _check_sparse_wire(t.dtype, "all_gather_compressed", sparse, wire_dtype, peer)
    if not t.is_cuda or not t.is_contiguous():
        raise ValueError("all_gather_compressed: contiguous CUDA tensor expected (no CPU fallback)")
    _check_wire(t, "all_gather_compressed", wire_dtype)
    if wire_dtype is not None and peer is not None:
        raise ValueError("all_gather_compressed: wire_dtype is not supported with the peer-memory transports")
    _check_wire_scale("all_gather_compressed", wire_scale, wire_dtype, t.device)
    _check_fp8_wire("all_gather_compressed", wire_dtype, error_feedback)
    _check_feedback("all_gather_compressed", error_feedback, t, wire_dtype)
    ef = None if error_feedback is None else error_feedback.reshape(-1)
    fp8 = wire_dtype in ops.FP8_TYPES
    as_float = t.dtype in (torch.float16, torch.bfloat16, torch.float32)
    flat = t.reshape(-1) if as_float else t.reshape(-1).view(torch.uint8)
    n = flat.numel()
    members = max(1, min(int(members), max(1, n // 4096)))
    # equal member lengths (multiples of 8 elements keep every member 16 B aligned); the last takes the rest
    bounds = _split(n, members, 8)
    members = len(bounds) - 1
    if peer is not None:
        # push needs no barrier, which suits a single peer; with more peers the pipelined pull spreads the reads
        # (a heuristic: the transports have not been timed on H100, DESIGN.md section 6)
        if peer_mode == "auto":
            peer_mode = "push" if peer.world <= 2 else "pull"
        if peer_mode not in ("push", "pull", "direct"):
            raise ValueError("all_gather_compressed: peer_mode is 'auto', 'push', 'pull' or 'direct'")
        if peer_mode == "push":
            out = _all_gather_push(flat, as_float, bounds, peer, checksum, temp_mem, check, stages)
        else:
            out = _all_gather_peer(flat, as_float, bounds, peer, checksum, temp_mem, check, peer_mode == "direct", stages)
        return out if as_float else out.view(t.dtype)
    world = _world(group)
    out = torch.empty(world * n, dtype=wire_dtype or flat.dtype, device=t.device)
    pieces = _pieces(members, max(1, min(int(stages), members)))

    def compress(a, b):
        kw = dict(scale_tensor=wire_scale) if fp8 else {}  # fp8: the scaled cast, then byte archives
        comp, sizes, _ = ops.compress_data(as_float, [flat[bounds[i]:bounds[i + 1]] for i in range(a, b)], checksum, temp_mem,
                                           archive_dtype=wire_dtype, sparse=sparse,
                                           error_feedback=None if ef is None else
                                           [ef[bounds[i]:bounds[i + 1]] for i in range(a, b)], **kw)
        return comp, sizes

    def decompress(a, b, gathered):
        ins, outs = [], []
        for w in range(world):
            for j, i in enumerate(range(a, b)):
                ins.append(gathered[w][j])
                o = out[w * n + bounds[i]: w * n + bounds[i + 1]]
                outs.append(o.view(torch.uint8) if fp8 else o)
        # gathered views are 16 B aligned inside the receive buffer; the decoder needs nothing else
        status = torch.zeros(len(ins), dtype=torch.uint8, device=t.device)
        ops.decompress_data(as_float and not fp8, ins, outs, checksum, temp_mem, status, sparse=sparse)
        return status

    statuses = []
    nxt = compress(*pieces[0])
    inflight = None  # (piece, exchange)
    for k, (a, b) in enumerate(pieces):
        comp, sizes = nxt
        if k + 1 < len(pieces):
            nxt = compress(*pieces[k + 1])  # queued before the size sync below: runs while the host waits
        hs = sizes.cpu().tolist()
        ex = _Exchange([comp[j, :hs[j]] for j in range(b - a)], group)  # payload goes out asynchronously (NCCL)
        if inflight is not None:
            (pa, pb), pex = inflight
            statuses.append(decompress(pa, pb, pex.wait()))  # previous piece decodes while this one is on the wire
        inflight = ((a, b), ex)
    (pa, pb), pex = inflight
    statuses.append(decompress(pa, pb, pex.wait()))
    if not all(bool(s.all()) for s in statuses):
        raise RuntimeError("all_gather_compressed: a received archive failed to decode")
    return out if as_float else out.view(t.dtype)


def _all_to_all_peer(flats: List[torch.Tensor], as_float: bool, ws: PeerWorkspace, checksum: bool,
                     temp_mem: Optional[torch.Tensor], check: bool, direct: bool) -> List[torch.Tensor]:
    """Regular all-to-all (chunk (s, d) has the same length on every rank pair): rank r encodes its chunks as one
    batch into its own peer-mapped rows, and after the barrier decodes row [r] of every peer straight out of
    the peer's memory."""
    world, rank, dev = ws.world, ws.rank, flats[0].device
    m = flats[0].numel()
    if any(f.numel() != m for f in flats):
        raise ValueError("all_to_all_compressed(peer=...): equal chunk lengths expected (sizes are not exchanged)")
    cols = _archive_cols(as_float, flats[0].dtype, m)
    off = ws.begin(world * cols)
    mine = ws.view(rank, off, world * cols).view(world, cols)
    sizes = torch.empty(world, dtype=torch.int32, device=dev)
    ops.compress_data(as_float, flats, checksum, temp_mem, mine, sizes)
    ws.barrier()
    outs = [torch.empty(m, dtype=flats[0].dtype, device=dev) for _ in range(world)]
    outs[rank].copy_(flats[rank])
    units = []
    for k in range(1, world):
        src = (rank + k) % world
        units.append((ws.view(src, off + rank * cols, cols).view(1, cols), [outs[src]]))
    if units:
        _pull_and_decode(ws, as_float, flats[0].dtype, units, cols, checksum, temp_mem, check, direct)
    return outs


def _all_to_all_bytes(send: torch.Tensor, send_sizes: List[int], recv_sizes: List[int], group,
                      on_device: bool) -> torch.Tensor:
    """all_to_all_single of a packed uint8 buffer on send's device; staged through host memory where the
    backend has no device collectives."""
    if on_device:
        recv = torch.empty(sum(recv_sizes), dtype=torch.uint8, device=send.device)
        dist.all_to_all_single(recv, send, recv_sizes, send_sizes, group=group)
        return recv
    host = torch.empty(sum(recv_sizes), dtype=torch.uint8)
    dist.all_to_all_single(host, send.cpu(), recv_sizes, send_sizes, group=group)
    return host.to(send.device)


def _send_to_each(per_dest: List[List[torch.Tensor]], group,
                  extra: Optional[List[int]] = None) -> Tuple[List[List[torch.Tensor]], Optional[List[int]]]:
    """Send the archives per_dest[d] (m exact-length uint8 tensors on one device for every d; an empty tensor sends
    nothing) to rank d.  Returns (per_src, extra_in): per_src[s] = the m archives rank s sent here, views into one
    receive buffer on the same device, and extra_in[s] = extra[this rank] of rank s (None without extra).
    Two all_to_all_single calls: the int64 table of archive sizes (and extras), then the archives packed 16 B
    aligned, so each link carries only its own bytes.  The one host synchronisation is the read of the received
    table."""
    m = len(per_dest[0])
    dev = per_dest[0][0].device
    on_device = _device_collectives(group)
    table = [[a.numel() for a in row] + ([] if extra is None else [int(extra[d])]) for d, row in enumerate(per_dest)]
    table_out = torch.tensor(table, dtype=torch.int64).to(dev if on_device else torch.device("cpu"))
    table_in = torch.empty_like(table_out)
    dist.all_to_all_single(table_in, table_out, group=group)
    recv_table = table_in.tolist()
    sent = [a for row in per_dest for a in row]
    offs, total = pack_offsets([a.numel() for a in sent])
    send = torch.zeros(total, dtype=torch.uint8, device=dev)
    for a, o in zip(sent, offs):
        send[o:o + a.numel()].copy_(a)
    recv = _all_to_all_bytes(send, [pack_offsets(row[:m])[1] for row in table],
                             [pack_offsets(row[:m])[1] for row in recv_table], group, on_device)
    lens = [k for row in recv_table for k in row[:m]]
    offs, _ = pack_offsets(lens)
    views = [recv[o:o + k] for o, k in zip(offs, lens)]
    per_src = [views[s * m:(s + 1) * m] for s in range(len(recv_table))]
    return per_src, None if extra is None else [row[m] for row in recv_table]


def all_to_all_compressed(chunks: Sequence[torch.Tensor], group=None, checksum: bool = False,
                          temp_mem: Optional[torch.Tensor] = None, peer: Optional[PeerWorkspace] = None,
                          check: bool = True, peer_mode: str = "pull", sparse: bool = False) -> List[torch.Tensor]:
    """chunks[d] (CUDA, contiguous, same dtype and shape on every rank for a given (source, destination) pair is
    NOT required: sizes travel with the data) goes to rank d; returns [world] tensors, entry s = what rank s
    sent here, bit-exact.  One archive per destination; the payload moves with all_to_all_single and exact
    split sizes, so each link carries only its own compressed chunk.  sparse=True (float16 / bfloat16 / float32
    chunks, NCCL / gloo transport): sparse archives on the wire, as in all_gather_compressed; same result."""
    world = _world(group)
    if len(chunks) != world:
        raise ValueError("all_to_all_compressed: one chunk per rank expected")
    dt, dev = chunks[0].dtype, chunks[0].device
    _check_sparse_wire(dt, "all_to_all_compressed", sparse, peer=peer)
    for c in chunks:
        if not c.is_cuda or not c.is_contiguous() or c.dtype != dt or c.device != dev:
            raise ValueError("all_to_all_compressed: contiguous CUDA tensors of one dtype on one device expected")
    as_float = dt in (torch.float16, torch.bfloat16, torch.float32)
    flats = [c.reshape(-1) if as_float else c.reshape(-1).view(torch.uint8) for c in chunks]
    if peer is not None:
        outs = _all_to_all_peer(flats, as_float, peer, checksum, temp_mem, check, peer_mode == "direct")
        return [x if as_float else x.view(dt) for x in outs]
    comp, sizes, _ = ops.compress_data(as_float, flats, checksum, temp_mem, sparse=sparse)
    if world == 1:
        out = torch.empty_like(flats[0])
        ops.decompress_data(as_float, [comp[0, :int(sizes[0])]], [out], checksum, temp_mem, sparse=sparse)
        return [out.view(chunks[0].shape) if as_float else out.view(dt).view(chunks[0].shape)]
    hs = sizes.cpu().tolist()  # host sync: the packed layout needs the archive sizes
    per_src, elems = _send_to_each([[comp[d, :hs[d]]] for d in range(world)], group, [f.numel() for f in flats])
    ins = [a for (a,) in per_src]
    outs = [torch.empty(k, dtype=flats[0].dtype, device=dev) for k in elems]
    status = torch.zeros(world, dtype=torch.uint8, device=dev)
    ops.decompress_data(as_float, ins, outs, checksum, temp_mem, status, sparse=sparse)
    if not bool(status.all()):
        raise RuntimeError("all_to_all_compressed: a received archive failed to decode")
    return [x if as_float else x.view(dt) for x in outs]


_REDUCE_DTYPES = (torch.float16, torch.bfloat16, torch.float32)


def _check_reducible(t: torch.Tensor, what: str, reduce_dtype: Optional[torch.dtype]) -> torch.dtype:
    """The dtype the sum is taken in: t's, or float32 for a float16 / bfloat16 t with reduce_dtype=float32."""
    if not t.is_cuda or not t.is_contiguous():
        raise ValueError(f"{what}: contiguous CUDA tensor expected (no CPU fallback)")
    if t.dtype not in _REDUCE_DTYPES:
        raise ValueError(f"{what}: float16, bfloat16 or float32 tensor expected, not {t.dtype}")
    if reduce_dtype is None or reduce_dtype == t.dtype:
        return t.dtype
    if reduce_dtype == torch.float32 and t.dtype in (torch.float16, torch.bfloat16):
        return reduce_dtype
    raise ValueError(f"{what}: reduce_dtype is None, t.dtype or float32 for a float16 / bfloat16 tensor, "
                     f"not {reduce_dtype} for {t.dtype}")


def _check_out_dtype(what: str, out_dtype: Optional[torch.dtype], dtype: torch.dtype,
                     reduce_dtype: Optional[torch.dtype], wire_dtype: Optional[torch.dtype]) -> Optional[torch.dtype]:
    """The result's dtype for a tensor of `dtype`: None for the sum's (which _check_reducible checks), or the archives'
    16-bit dtype for a float32 sum, which the decode-and-sum rounds once from its float32 sums
    (ops.decompress_data_reduce(reduce_dtype=torch.float32)).  Reads dtypes only, so it refuses before any other
    check of t."""
    acc_dtype = torch.float32 if torch.float32 in (dtype, reduce_dtype) else dtype
    arch_dtype = wire_dtype or dtype
    if out_dtype is None or out_dtype == acc_dtype:
        return None
    if acc_dtype == torch.float32 and out_dtype == arch_dtype and arch_dtype in (torch.float16, torch.bfloat16):
        return out_dtype
    raise ValueError(f"{what}: out_dtype is None, the sum's dtype {acc_dtype}, or the archives' dtype for a float32 "
                     f"sum of float16 / bfloat16 archives; not {out_dtype} for {arch_dtype} archives summed in "
                     f"{acc_dtype}")


def _check_scale(what: str, scale, average: bool, scale_tensor=None, found_inf=None,
                 dev=None) -> Optional[np.float32]:
    """The float32 pre-multiplier a scale argument stands for (None: a plain sum, or a device scale_tensor); average
    is resolved later, once the world size is known.  scale_tensor and found_inf are checked as
    ops.decompress_data_reduce checks them, on dev (t's device)."""
    if average and scale is not None:
        raise ValueError(f"{what}: pass average=True or a scale, not both")
    if scale_tensor is not None and (scale is not None or average):
        raise ValueError(f"{what}: scale_tensor replaces scale and average=True (divide it by the world size on the "
                         "device)")
    if found_inf is not None and scale_tensor is None:
        raise ValueError(f"{what}: found_inf needs scale_tensor (torch.ones(1) for the unscaled sum)")
    s32 = ops._scale32(scale)
    if scale_tensor is not None:
        ops._check_flag_tensor(f"{what}: scale_tensor", scale_tensor, dev)
    if found_inf is not None:
        ops._check_flag_tensor(f"{what}: found_inf", found_inf, dev)
    return s32


def _check_sq_norm(what: str, sq_norm, scale_tensor, dev) -> None:
    """sq_norm: None, or a one-element float64 CUDA tensor on dev, with scale_tensor (as found_inf needs it)."""
    if sq_norm is None:
        return
    if scale_tensor is None:
        raise ValueError(f"{what}: sq_norm needs scale_tensor (torch.ones(1) for the unscaled sum)")
    ops._check_sq_norm(f"{what}: sq_norm", sq_norm, 1, dev)


def _fold(out: torch.Tensor, values: torch.Tensor) -> None:
    """out (one element) = ((values[0] + values[1]) + values[2]) + ..., fp64 adds on the device in index order
    (torch's sum() does not specify its order)."""
    out.copy_(values[0:1])
    for i in range(1, values.numel()):
        out.add_(values[i:i + 1])


def _shard_sq_norm(out: Optional[torch.Tensor], res: torch.Tensor, bounds: List[int]) -> None:
    """out = the member-order fold of ops.sq_norm of res's pieces [bounds[i], bounds[i + 1]): what the decode-and-sum
    gives when it writes those pieces, for the shards torch finishes."""
    if out is not None:
        _fold(out, ops.sq_norm([res[bounds[i]:bounds[i + 1]] for i in range(len(bounds) - 1)]))


def _term(x: torch.Tensor, acc_dtype: torch.dtype, s32) -> torch.Tensor:
    """What the scaled decode-and-sum adds for the words x: (x.float() * s32).to(acc_dtype), one float32 multiply
    by a float32 tensor and one rounding; x.to(acc_dtype) without a scale.  s32: a float32 number, or a device
    scale_tensor (one element)."""
    if s32 is None:
        return x.to(acc_dtype)
    if isinstance(s32, torch.Tensor):
        return (x.float() * s32.reshape(())).to(acc_dtype)
    return (x.float() * torch.tensor(float(s32), dtype=torch.float32, device=x.device)).to(acc_dtype)


def _flag_non_finite(found_inf: Optional[torch.Tensor], x: torch.Tensor) -> None:
    """found_inf = max(found_inf, 1 if x has an inf or NaN else 0), on the device (no host sync, never cleared)."""
    if found_inf is not None:
        torch.maximum(found_inf, (~x.isfinite()).any().float(), out=found_inf)


def _local_sum(x: torch.Tensor, acc_dtype: torch.dtype, s32, found_inf: Optional[torch.Tensor]) -> torch.Tensor:
    """A reducing collective's result when this rank's words are the only terms (a world of one, or no elements):
    each word's _term in acc_dtype, always a new tensor, with found_inf raised when one is non-finite."""
    res = x.to(acc_dtype, copy=True) if s32 is None else _term(x, acc_dtype, s32)
    _flag_non_finite(found_inf, res)
    return res


def reduce_scatter_compressed(t: torch.Tensor, group=None, members: int = 8,
                              temp_mem: Optional[torch.Tensor] = None, check: bool = True,
                              reduce_dtype: Optional[torch.dtype] = None,
                              wire_dtype: Optional[torch.dtype] = None, sparse: bool = False,
                              scale: Optional[float] = None, average: bool = False,
                              scale_tensor: Optional[torch.Tensor] = None,
                              found_inf: Optional[torch.Tensor] = None,
                              out_dtype: Optional[torch.dtype] = None,
                              sq_norm: Optional[torch.Tensor] = None,
                              error_feedback: Optional[torch.Tensor] = None,
                              wire_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Like dist.reduce_scatter_tensor with a sum: t (contiguous CUDA fp16 / bf16 / fp32, t.numel() divisible by the
    world size, same shape on every rank) is cut into world chunks, and this rank returns the elementwise sum over
    ranks of chunk `rank`.  Rank r sends chunk d to rank d as `members` float archives (the same split on every
    rank), so the wire carries compressed bytes; the receiver decodes and sums them in one kernel
    (ops.decompress_data_reduce) without a decoded temporary per source.  The sum is the left fold over ranks in
    rank order, with torch's adds in t's dtype, for every element on every rank: the result is bit-identical to
    ((t_0 + t_1) + t_2) + ... whatever `members` and the backend.  `check` raises RuntimeError when a received
    archive fails to decode.

    reduce_dtype=torch.float32 with a float16 / bfloat16 t (mixed-precision gradients summed in fp32): the wire
    still carries the 16-bit archives, the result is float32 and equals the fp32 fold
    ((t_0.float() + t_1.float()) + t_2.float()) + ... bit for bit.  None or t.dtype sums in t's dtype; any other
    value raises ValueError.

    wire_dtype=torch.float16 / torch.bfloat16 with a float32 t (fp32 gradients sent as 16 bits, DeepSpeed's
    communication_data_type, Megatron's bf16 gradient communication): every chunk is rounded to wire_dtype inside
    the compress kernels, the 16-bit archives go over the wire and are summed in fp32, and the float32 result is
    ((t_0.to(w).float() + t_1.to(w).float()) + t_2.to(w).float()) + ... bit for bit, on every rank and for every
    `members`.  reduce_dtype must then be None or float32.

    sparse=True: sparse archives on the wire (no stored bits for +0 and -0 words), summed by the sparse
    decode-and-sum (ops.decompress_data_reduce(sparse=True)); the result is the same fold, bit for bit, with
    reduce_dtype too.  Not with wire_dtype: that raises ValueError before any communication.

    scale=s (a real number, rounded once to float32: np.float32(s)) pre-multiplies every rank's term before the sum,
    as NCCL's average and FSDP / DeepSpeed's gradient pre-division do; average=True means s = np.float32(1 / world),
    and passing both raises ValueError before any communication.  The term of rank r is
    term(x) = (x.float() * s32).to(acc) with s32 = torch.tensor(s, dtype=torch.float32) and x = t_r's chunk in the
    archive dtype (the wire dtype's word with wire_dtype), acc the result's dtype, and the result is the rank-order
    fold ((term(x_0) + term(x_1)) + term(x_2)) + ... bit for bit on every rank, with reduce_dtype, wire_dtype and
    sparse too.  The received archives are scaled inside the decode-and-sum kernel
    (ops.decompress_data_reduce(scale=)), so no rank makes a scaled copy of its input.

    scale_tensor (a one-element float32 CUDA tensor on t's device) is the scale kept on the device, e.g. a
    GradScaler's inverse scale divided by the world size: the kernels read it, the host never does, and the result
    is bit-identical to this call with scale=float(scale_tensor).  Not with scale or average=True.  found_inf (with
    scale_tensor; the same kind of tensor) is set to 1.0 when any element of the returned shard is inf or NaN, and
    never cleared (torch.amp's found_inf convention), without a host sync.  These keywords raise ValueError before
    any communication.

    out_dtype: the result's dtype.  None is the sum's dtype.  When the sum is float32 of float16 / bfloat16 archives
    (reduce_dtype=torch.float32 with a 16-bit t, or a float32 t with wire_dtype), out_dtype may be the archives'
    dtype: the sum is still taken in float32 and rounded once per element inside the decode-and-sum kernel, so the
    result is this call without out_dtype followed by .to(out_dtype), bit for bit on every rank, without a float32
    result (found_inf then sees the rounded elements).  Any other value raises ValueError before any
    communication.

    sq_norm (with scale_tensor; a one-element float64 CUDA tensor on t's device) is overwritten with the squared norm
    of the returned shard, for gradient clipping: the fp64 fold, in member order, of the squared norms
    (ops.sq_norm's definition) of the shard's `members` pieces.  The decode-and-sum that writes the final values takes
    them in the same kernel (decompress_data_reduce(sq_norm=)); the last rank and a world of one, which finish the
    shard with torch, apply ops.sq_norm to the same pieces, so the value is the same function of the shard on every
    path.  Misuse raises ValueError before any communication.

    error_feedback=e (with wire_dtype; a contiguous float32 CUDA tensor shaped like t, at t's address modulo 16)
    keeps the rounding error of the float32 -> wire_dtype compress from one step to the next instead of dropping it
    (DeepSpeed's "worker error"): the result is exactly reduce_scatter_compressed(t + e, wire_dtype=wire_dtype, ...)
    with every other keyword unchanged, on every rank, and all of e is overwritten with this step's error,
    torch.where(w.isfinite(), y - w.float(), 0) for y = t + e and w = y.to(wire_dtype).  The chunks sent to other
    ranks get their new error from the compress kernels (ops.compress_data(error_feedback=)); the own chunk, which is
    never compressed, and a world of one or an empty t get it from that torch expression.  The error of a word that
    rounds to inf or NaN is +0: that step carries the non-finite word (found_inf sees it), the next starts clean.
    Misuse raises ValueError before any communication.

    wire_dtype=torch.float8_e4m3fn / torch.float8_e5m2 with a float32 or bfloat16 t (fp8 gradient communication):
    each rank casts every element of t once with ops.cast_fp8 at the scale wire_scale (a one-element float32 CUDA
    tensor on t's device, the same value on every rank, as an fp8 recipe's scales are; None means 1), sends the other
    ranks' chunks as fp8 byte archives and sums with the dequantisation scale d = u / wire_scale (one float32
    division by torch on the device; d = u without wire_scale), where u is 1, np.float32(scale), np.float32(1 / world)
    with average=True, or scale_tensor.  The float32 result is the rank-order fold of q_r.float() * d, q_r the fp8
    cast of t_r's chunk, bit for bit on every rank; found_inf and sq_norm work as above (with scale_tensor).
    reduce_dtype and out_dtype must be None or float32; error_feedback is not supported.  wire_scale without an fp8
    wire_dtype raises ValueError before any communication."""
    s32 = _check_scale("reduce_scatter_compressed", scale, average, scale_tensor, found_inf, t.device)
    _check_sq_norm("reduce_scatter_compressed", sq_norm, scale_tensor, t.device)
    _check_sparse_wire(t.dtype, "reduce_scatter_compressed", sparse, wire_dtype)
    if wire_dtype in ops.FP8_TYPES:
        return _reduce_scatter_fp8(t, group, members, temp_mem, check, reduce_dtype, wire_dtype, s32, average,
                                   scale_tensor, found_inf, out_dtype, sq_norm, error_feedback, wire_scale)
    _check_wire_scale("reduce_scatter_compressed", wire_scale, wire_dtype, t.device)
    narrow_dtype = _check_out_dtype("reduce_scatter_compressed", out_dtype, t.dtype, reduce_dtype, wire_dtype)
    acc_dtype = _check_reducible(t, "reduce_scatter_compressed", reduce_dtype)
    _check_wire(t, "reduce_scatter_compressed", wire_dtype)
    _check_feedback("reduce_scatter_compressed", error_feedback, t, wire_dtype)
    arch_dtype = wire_dtype or t.dtype  # the archives' (and the own chunk's) dtype
    res_dtype = narrow_dtype or acc_dtype
    world = _world(group)
    if average:
        s32 = np.float32(1 / world)
    sd = s32 if scale_tensor is None else scale_tensor  # the terms' scale: a float32, a device tensor or None
    flat = t.reshape(-1)
    n = flat.numel()
    if n % world:
        raise ValueError(f"reduce_scatter_compressed: numel {n} is not divisible by the world size {world}")
    ef = None if error_feedback is None else error_feedback.reshape(-1)
    shard = n // world
    bounds = _split(shard, max(1, int(members)), 8)
    if world == 1 or n == 0:
        if ef is not None:
            flat = _feedback_step(flat, ef, arch_dtype)
        if res_dtype == acc_dtype:
            res = _local_sum(flat[:shard].to(arch_dtype), acc_dtype, sd, found_inf)
        else:
            res = _local_sum(_term(flat[:shard].to(arch_dtype), acc_dtype, sd), res_dtype, None, found_inf)
        _shard_sq_norm(sq_norm, res, bounds)
        return res
    rank, dev = dist.get_rank(group), t.device
    m = len(bounds) - 1
    dests = [d for d in range(world) if d != rank]
    comp, sizes, _ = ops.compress_data(True, [flat[d * shard + bounds[i]: d * shard + bounds[i + 1]]
                                              for d in dests for i in range(m)], False, temp_mem,
                                       archive_dtype=arch_dtype, sparse=sparse,
                                       error_feedback=None if ef is None else
                                       [ef[d * shard + bounds[i]: d * shard + bounds[i + 1]]
                                        for d in dests for i in range(m)])
    hs = sizes.cpu().tolist()  # host sync: the packed layout needs the archive sizes
    per_dest = [[comp.new_empty(0)] * m for _ in range(world)]  # nothing for this rank's own chunk
    for k, d in enumerate(dests):
        per_dest[d] = [comp[k * m + i, :hs[k * m + i]] for i in range(m)]
    archives, _ = _send_to_each(per_dest, group)  # archives[s][i]: member i of the chunk source s sent here
    out = torch.empty(shard, dtype=acc_dtype, device=dev)  # the running sums (all of it, unless narrowing)
    outs = [out[bounds[i]:bounds[i + 1]] for i in range(m)]
    # narrowing: the later sources' call rounds the float32 sums once into res, accumulating from out
    res = out if res_dtype == acc_dtype else torch.empty(shard, dtype=res_dtype, device=dev)
    narrow = {} if res is out else dict(reduce_dtype=torch.float32, acc=outs)
    own = flat[rank * shard:(rank + 1) * shard]
    if ef is not None:
        own = _feedback_step(own, ef[rank * shard:(rank + 1) * shard], arch_dtype)
    own = own.to(arch_dtype)
    if sd is not None:
        own = _term(own, acc_dtype, sd)  # the kernel's term of the own chunk, already in the result's dtype
    statuses = []
    # rank order: sources 0..r-1 decoded and summed, + own chunk (torch's add is the kernel's add; fp32 += fp16 /
    # bf16 is the same fp32 add of the widened word), + r+1..world-1
    if rank == 0:
        out.copy_(own)
    else:
        st = torch.zeros(m * rank, dtype=torch.uint8, device=dev)
        ops.decompress_data_reduce([[archives[s][i] for s in range(rank)] for i in range(m)], outs, False, temp_mem, st,
                                   archive_dtype=arch_dtype, sparse=sparse, scale=s32, scale_tensor=scale_tensor)
        statuses.append(st)
        out.add_(own)
    if rank + 1 < world:
        # the last call writes the final values: the kernel checks them, and takes their squared norms
        st = torch.zeros(m * (world - rank - 1), dtype=torch.uint8, device=dev)
        pieces_sq = None if sq_norm is None else torch.zeros(m, dtype=torch.float64, device=dev)
        ops.decompress_data_reduce([[archives[s][i] for s in range(rank + 1, world)] for i in range(m)],
                                   [res[bounds[i]:bounds[i + 1]] for i in range(m)], True, temp_mem, st,
                                   archive_dtype=arch_dtype, sparse=sparse, scale=s32, scale_tensor=scale_tensor,
                                   found_inf=found_inf, sq_norm=pieces_sq, **narrow)
        statuses.append(st)
        if sq_norm is not None:
            _fold(sq_norm, pieces_sq)
    else:
        # the last rank ends on torch's add of its own chunk (and torch's rounding of it when narrowing)
        if res is not out:
            res.copy_(out)
        _flag_non_finite(found_inf, res)
        _shard_sq_norm(sq_norm, res, bounds)
    if check and not all(bool(st.all()) for st in statuses):
        raise RuntimeError("reduce_scatter_compressed: a received archive failed to decode")
    return res


def _reduce_scatter_fp8(t, group, members, temp_mem, check, reduce_dtype, wire_dtype, s32, average, scale_tensor,
                        found_inf, out_dtype, sq_norm, error_feedback, wire_scale) -> torch.Tensor:
    """reduce_scatter_compressed with an fp8 wire_dtype (its docstring has the contract)."""
    what = "reduce_scatter_compressed"
    _check_reducible(t, what, None)
    _check_wire(t, what, wire_dtype)
    if reduce_dtype not in (None, torch.float32) or out_dtype not in (None, torch.float32):
        raise ValueError(f"{what}: an fp8 wire sums in float32: reduce_dtype and out_dtype are None or float32, not "
                         f"{reduce_dtype} and {out_dtype}")
    _check_fp8_wire(what, wire_dtype, error_feedback)
    _check_wire_scale(what, wire_scale, wire_dtype, t.device)
    world = _world(group)
    dev = t.device
    if average:
        s32 = np.float32(1 / world)
    # the dequantisation scale d = u / wire_scale, a device tensor the decode-and-sum reads
    if scale_tensor is not None:
        u = scale_tensor
    else:
        u = torch.full((1,), 1.0 if s32 is None else float(s32), dtype=torch.float32, device=dev)
    d = u if wire_scale is None else u / wire_scale
    flat = t.reshape(-1)
    n = flat.numel()
    if n % world:
        raise ValueError(f"{what}: numel {n} is not divisible by the world size {world}")
    shard = n // world
    bounds = _split(shard, max(1, int(members)), 8)

    def own_term(rank):
        q = ops.cast_fp8([flat[rank * shard:(rank + 1) * shard]], wire_dtype, wire_scale)[0]
        return q.float() * d.reshape(())

    if world == 1 or n == 0:
        res = own_term(0)
        _flag_non_finite(found_inf, res)
        _shard_sq_norm(sq_norm, res, bounds)
        return res
    rank = dist.get_rank(group)
    m = len(bounds) - 1
    dests = [k for k in range(world) if k != rank]
    comp, sizes, _ = ops.compress_data(True, [flat[k * shard + bounds[i]: k * shard + bounds[i + 1]]
                                              for k in dests for i in range(m)], False, temp_mem,
                                       archive_dtype=wire_dtype, scale_tensor=wire_scale)
    hs = sizes.cpu().tolist()  # host sync: the packed layout needs the archive sizes
    per_dest = [[comp.new_empty(0)] * m for _ in range(world)]  # nothing for this rank's own chunk
    for j, k in enumerate(dests):
        per_dest[k] = [comp[j * m + i, :hs[j * m + i]] for i in range(m)]
    archives, _ = _send_to_each(per_dest, group)
    out = torch.empty(shard, dtype=torch.float32, device=dev)
    outs = [out[bounds[i]:bounds[i + 1]] for i in range(m)]
    own = own_term(rank)  # the kernel's term of the own chunk, from the same cast kernel
    statuses = []
    if rank == 0:
        out.copy_(own)
    else:
        st = torch.zeros(m * rank, dtype=torch.uint8, device=dev)
        ops.decompress_data_reduce([[archives[s][i] for s in range(rank)] for i in range(m)], outs, False, temp_mem, st,
                                   archive_dtype=wire_dtype, scale_tensor=d)
        statuses.append(st)
        out.add_(own)
    if rank + 1 < world:
        st = torch.zeros(m * (world - rank - 1), dtype=torch.uint8, device=dev)
        pieces_sq = None if sq_norm is None else torch.zeros(m, dtype=torch.float64, device=dev)
        ops.decompress_data_reduce([[archives[s][i] for s in range(rank + 1, world)] for i in range(m)], outs, True,
                                   temp_mem, st, archive_dtype=wire_dtype, scale_tensor=d, found_inf=found_inf,
                                   sq_norm=pieces_sq)
        statuses.append(st)
        if sq_norm is not None:
            _fold(sq_norm, pieces_sq)
    else:
        _flag_non_finite(found_inf, out)
        _shard_sq_norm(sq_norm, out, bounds)
    if check and not all(bool(st.all()) for st in statuses):
        raise RuntimeError(f"{what}: a received archive failed to decode")
    return out


def all_reduce_compressed(t: torch.Tensor, group=None, members: int = 8, temp_mem: Optional[torch.Tensor] = None,
                          check: bool = True, reduce_dtype: Optional[torch.dtype] = None,
                          sparse: bool = False, scale: Optional[float] = None,
                          average: bool = False, scale_tensor: Optional[torch.Tensor] = None,
                          found_inf: Optional[torch.Tensor] = None,
                          out_dtype: Optional[torch.dtype] = None,
                          sq_norm: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Elementwise sum over ranks of t (contiguous CUDA fp16 / bf16 / fp32, any numel, same shape on every rank),
    returned on every rank: reduce_scatter_compressed, then all_gather_compressed of the summed shard.  When
    t.numel() is not world x a multiple of 8, t is zero-padded to world x roundUp(ceil(n / world), 8) elements
    for the exchange.  Bit-identical on every rank to the rank-order left fold with torch's adds.
    reduce_dtype=torch.float32 with a float16 / bfloat16 t sums in fp32 as reduce_scatter_compressed does and
    all-gathers the fp32 shards: the float32 result is the fp32 fold on every rank.  sparse=True sends sparse
    archives in both phases (see reduce_scatter_compressed); the result is the same.  scale=s or average=True
    (s = np.float32(1 / world); not both) pre-multiplies every rank's term as in reduce_scatter_compressed: the
    result is the rank-order fold of (t_r.float() * s32).to(acc) on every rank, bit for bit.  scale_tensor and
    found_inf are reduce_scatter_compressed's, except that found_inf covers the whole result on every rank: the
    shards' flags meet in one MAX all-reduce of a one-element tensor.

    out_dtype is reduce_scatter_compressed's: t.dtype for a float16 / bfloat16 t summed with
    reduce_dtype=torch.float32 makes the shards come back rounded once to t.dtype, the second phase all-gathers
    16-bit archives instead of float32 ones, and the result is this call without out_dtype followed by
    .to(out_dtype), bit for bit on every rank.  Any other out_dtype raises ValueError before any communication.

    sq_norm (with scale_tensor; a one-element float64 CUDA tensor on t's device) is overwritten with the squared norm
    of the whole result, identical on every rank: the rank-order fp64 fold of the shards' reduce_scatter_compressed
    sq_norm values, exchanged with one all-gather (padding zeros add +0).  A world of one, or an empty t, takes
    reduce_scatter_compressed's value for t.  Misuse raises ValueError before any communication."""
    s32 = _check_scale("all_reduce_compressed", scale, average, scale_tensor, found_inf, t.device)
    _check_sq_norm("all_reduce_compressed", sq_norm, scale_tensor, t.device)
    _check_sparse_wire(t.dtype, "all_reduce_compressed", sparse)
    narrow_dtype = _check_out_dtype("all_reduce_compressed", out_dtype, t.dtype, reduce_dtype, None)
    acc_dtype = _check_reducible(t, "all_reduce_compressed", reduce_dtype)
    res_dtype = narrow_dtype or acc_dtype
    world = _world(group)
    if average:
        s32 = np.float32(1 / world)
    flat = t.reshape(-1)
    n = flat.numel()
    if world == 1 or n == 0:
        sd = s32 if scale_tensor is None else scale_tensor
        if res_dtype == acc_dtype:
            res = _local_sum(t, acc_dtype, sd, found_inf)
        else:
            res = _local_sum(_term(t, acc_dtype, sd), res_dtype, None, found_inf)
        _shard_sq_norm(sq_norm, res.reshape(-1), _split(n, max(1, int(members)), 8))
        return res
    per = _round_up(-(-n // world), 8)
    src = flat if world * per == n else torch.cat([flat, flat.new_zeros(world * per - n)])
    # (a padding zero's term is non-finite only for an inf or NaN scale, which makes every element's term so too)
    shard_inf = None if found_inf is None else torch.zeros(1, dtype=torch.float32, device=t.device)
    shard_sq = None if sq_norm is None else torch.zeros(1, dtype=torch.float64, device=t.device)
    shard = reduce_scatter_compressed(src, group, members, temp_mem, check, reduce_dtype=acc_dtype, sparse=sparse,
                                      scale=s32, scale_tensor=scale_tensor, found_inf=shard_inf, out_dtype=res_dtype,
                                      sq_norm=shard_sq)
    if sq_norm is not None:
        # every rank folds the same gathered values in rank order (an all-reduce's order is not defined)
        on_device = _device_collectives(group)
        mine = shard_sq if on_device else shard_sq.cpu()
        every = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(every, mine, group=group)
        _fold(sq_norm, torch.cat(every).to(t.device))
    if found_inf is not None:
        on_device = _device_collectives(group)
        flag = shard_inf if on_device else shard_inf.cpu()
        dist.all_reduce(flag, op=dist.ReduceOp.MAX, group=group)
        torch.maximum(found_inf, flag.to(t.device), out=found_inf)
    full = all_gather_compressed(shard, group, members, temp_mem=temp_mem, check=check, sparse=sparse)
    return full[:n].view(t.shape)
