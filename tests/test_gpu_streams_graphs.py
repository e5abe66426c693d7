"""The host launch path around the kernels: CUDA-graph capture, stream ordering, the host-buffer pipeline and
several devices, every member compared with the CPU oracle and every decode bit-exact.

A call must read none of its host arguments or of the library's per-thread staging after it returns, so a graph
that captured it codes its own batch at every replay, whatever the thread did since.  The tests are built so that
a broken implementation shows up as wrong bytes or a raised error and never as a device fault: whenever a replay
could pick up another call's member table, that call used an intruder batch of the same member count and member
sizes with live buffers of its own, no buffer a graph references is freed before its last replay, and a thread
that captured stays alive until then.
"""
import threading
import time

import numpy as np
import pytest
import torch

from codec_helpers import KINDS, SENTINEL, codec_options, oracle_archive, options  # noqa: F401
from conftest import exp_bytes, normal_words, zipf_bytes
from oracle import oracle as O

pytestmark = pytest.mark.gpu

PB = 10
BLOCK = 4096  # one 4 KiB block of coded bytes: 4096 bytes, or 4096 float words


def member_sizes(n, small=False):
    """n member sizes (elements): 0, 1, one full block, and sizes that are not multiples of it."""
    edge = [0, 1, BLOCK, BLOCK + 1, 3 * BLOCK - 5, 777]
    if small:  # c4's shape (256 fp16 members) at a size the oracle checks quickly
        return [edge[i] if i < len(edge) else 2048 + (i % 3) for i in range(n)]
    return [edge[i] if i < len(edge) else 300 + (i * 997) % 7000 for i in range(n)]


def _data(kind, size, seed):
    if kind == "bytes":
        return zipf_bytes(size, 1.0 + (seed % 5) / 4, seed) if seed % 2 else exp_bytes(size, 5 + seed % 30, seed)
    return normal_words(size, kind, seed, relu=seed % 3 == 0)


class Batch:
    """One batch with buffers of its own: inputs and outputs at 16 B aligned offsets of one flat buffer each (the
    gaps of the output buffer hold a sentinel that must survive), an archive matrix, sizes, status, decoded word
    counts, and encoder and decoder scratch."""

    def __init__(self, kind, sizes, device="cuda"):
        from dietgpu_b200 import capi, ops

        self.kind, self.as_float, self.dev = kind, kind != "bytes", torch.device(device)
        self.dtype = torch.uint8 if kind == "bytes" else KINDS[kind][1]
        es = torch.empty(0, dtype=self.dtype).element_size()
        self.lengths = list(sizes)
        self.offs, total = [], 0
        for s in sizes:
            self.offs.append(total)
            total += (s * es + 15) // 16 * 16 + 16
        self.nbytes = total
        self.flat_in = torch.zeros(total, dtype=torch.uint8, device=self.dev)
        self.flat_out = torch.full((total,), SENTINEL, dtype=torch.uint8, device=self.dev)
        self.ins = [self.flat_in[o:o + s * es].view(self.dtype) for o, s in zip(self.offs, sizes)]
        self.outs = [self.flat_out[o:o + s * es].view(self.dtype) for o, s in zip(self.offs, sizes)]
        mask = torch.zeros(total, dtype=torch.bool)
        for o, s in zip(self.offs, sizes):
            mask[o:o + s * es] = True
        self.mask = mask.to(self.dev)
        n = len(sizes)
        _, cols = (ops.max_float_compressed_output_size(self.ins) if self.as_float
                   else ops.max_any_compressed_output_size(self.ins))
        self.comp = torch.zeros((n, cols), dtype=torch.uint8, device=self.dev)
        self.rows = [self.comp[i] for i in range(n)]
        self.sizes = torch.zeros(n, dtype=torch.int32, device=self.dev)
        self.status = torch.zeros(n, dtype=torch.uint8, device=self.dev)
        self.words = torch.zeros(n, dtype=torch.int32, device=self.dev)
        L, mx = capi.lib(), max(sizes)
        if self.as_float:
            ft = ops._FLOAT_TYPES[self.dtype]
            need_c, need_d = L.dgb_float_compress_temp_bytes(ft, n, mx), L.dgb_float_decompress_temp_bytes(ft, n, mx)
        else:
            need_c, need_d = L.dgb_ans_encode_temp_bytes(n, mx), L.dgb_ans_decode_temp_bytes(n)
        self.temp_c = torch.empty(need_c + 256, dtype=torch.uint8, device=self.dev)
        self.temp_d = torch.empty(need_d + 256, dtype=torch.uint8, device=self.dev)
        self.host = None

    def fill(self, seed):
        """New seeded contents; the host copy is what the oracle and the decode checks use."""
        self.host = [_data(self.kind, s, seed * 1000 + i) for i, s in enumerate(self.lengths)]
        flat = np.zeros(self.nbytes, np.uint8)
        for o, a in zip(self.offs, self.host):
            flat[o:o + a.nbytes] = a.view(np.uint8)
        self.flat_in.copy_(torch.from_numpy(flat))
        self.want = self.flat_in.clone()

    def compress(self, checksum=False):
        from dietgpu_b200 import ops

        ops.compress_data(self.as_float, self.ins, checksum, self.temp_c, self.comp, self.sizes, prob_bits=PB)

    def decompress(self, checksum=False):
        from dietgpu_b200 import ops

        ops.decompress_data(self.as_float, self.rows, self.outs, checksum, self.temp_d, self.status, self.words,
                            prob_bits=PB)

    def step(self, checksum=False):
        """compress + decompress (decode checksum verification synchronises, so it is never part of a step)"""
        self.compress(checksum)
        self.decompress()

    def check_archives(self, comp, sizes, checksum, exact, what):
        hs = sizes.cpu().tolist()
        host = comp.cpu().numpy()
        for i, a in enumerate(self.host):
            want = oracle_archive(self.kind, a, PB, checksum)
            assert hs[i] == want.size, f"{what}: member {i}: size {hs[i]} != oracle {want.size}"
            got = host[i, :hs[i]]
            if exact:
                assert np.array_equal(got, want), f"{what}: member {i}: archive bytes differ from the oracle's"
            elif self.kind == "bytes":
                O.assert_same_ans(got, want, f"{what}: member {i}")
            else:
                O.assert_same_float(got, want, KINDS[self.kind][0], f"{what}: member {i}")

    def check_outputs(self, what):
        assert self.status.cpu().tolist() == [1] * len(self.lengths), f"{what}: status"
        assert self.words.cpu().tolist() == self.lengths, f"{what}: decoded sizes"
        assert torch.equal(self.flat_out[self.mask], self.want[self.mask]), f"{what}: decoded data differs"
        assert bool((self.flat_out[~self.mask] == SENTINEL).all()), f"{what}: decode wrote outside its outputs"

    def check(self, checksum=False, exact=False, what=""):
        torch.cuda.synchronize(self.dev)
        self.check_archives(self.comp, self.sizes, checksum, exact, what)
        self.check_outputs(what)

    def clear(self):
        """Stale results must not pass a check: outputs back to the sentinel, archives and counts to zero."""
        self.flat_out.fill_(SENTINEL)
        self.comp.zero_()
        self.sizes.zero_()
        self.status.zero_()
        self.words.zero_()

    def snapshot(self):
        return [t.clone() for t in (self.comp, self.sizes, self.flat_out, self.status, self.words)]

    def unchanged(self, snap):
        return all(torch.equal(a, b) for a, b in zip(snap, self.snapshot()))


# ---- A1: capture matrix ------------------------------------------------------------------------------------------
# (kind, members, options, encode checksum); member tables above 64 members, and under every option but the
# defaults and decode_warps, go through scratch
CELLS = [
    ("bytes", 6, {}, False),
    ("f16", 64, {}, False),
    ("bf16", 65, {}, False),
    ("f32", 130, {}, False),
    ("f16", 256, {}, False),  # c4's shape, small members
    ("bf16", 6, dict(inline_members=0), False),
    ("bytes", 64, dict(inline_members=0), False),
    ("bytes", 65, dict(encode_fused=1), False),
    ("f32", 6, dict(encode_fused=1), False),
    ("bytes", 6, dict(encode_canonical=1), False),
    ("bf16", 65, dict(encode_canonical=1), False),
    ("f16", 6, dict(stats_stage=1), False),
    ("f32", 65, dict(stats_stage=1), False),
    ("bytes", 130, dict(decode_fused=0), False),
    ("bf16", 6, dict(decode_fused=0), False),
    ("f16", 64, dict(parts=4), False),  # float batches of >= 16 members: the capture forks and joins helper streams
    ("f32", 130, dict(parts=4, decode_fused=0), False),
    ("bytes", 65, dict(decode_warps=20), False),
    ("bf16", 130, {}, True),
    ("bytes", 64, {}, True),
]


def _cell_id(c):
    kind, n, opts, cs = c
    return f"{kind}-{n}-" + (",".join(f"{k}={v}" for k, v in opts.items()) or "defaults") + ("-checksum" if cs else "")


@pytest.mark.parametrize("cell", CELLS, ids=[_cell_id(c) for c in CELLS])
def test_captured_calls_replay_their_own_batch(cell):
    kind, n, opts, checksum = cell
    sizes = member_sizes(n, small=n == 256)
    exact = opts.get("encode_canonical", 0) == 1
    x, x2, y = Batch(kind, sizes), Batch(kind, sizes), Batch(kind, sizes)
    graphs = []
    with codec_options(**opts):
        # 1. an ordinary call, then capture X
        x.fill(1)
        x.step(checksum)
        x.check(checksum, exact, "ordinary call")
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            x.step(checksum)
        graphs.append(g)
        # 2. the intruder Y through the same per-thread staging, then its snapshot
        y.fill(2)
        y.step(checksum)
        y.check(checksum, exact, "intruder")
        y_snap = y.snapshot()
        # 3. a second graph for X2
        x2.fill(3)
        g2 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g2):
            x2.step(checksum)
        graphs.append(g2)
    # 4. default options restored: the replays must still run the variant captured above
    for r in range(3):
        x.fill(10 + r)
        x2.fill(20 + r)
        for b, gr, name in ((x, graphs[0], "X"), (x2, graphs[1], "X2")):
            b.clear()
            gr.replay()
            b.check(checksum, exact, f"replay {r} of {name}")
            assert y.unchanged(y_snap), f"replay {r} of {name} changed the intruder's buffers"


@pytest.mark.parametrize("kind", ["bytes", "f16"])
def test_captured_header_query_keeps_its_pointer_array(kind):
    # dgb_*_get_compressed_info with a host array of archive pointers: the captured call must keep the pointers it
    # was given, not re-read the caller's array at replay (here rewritten to point at another batch's archives)
    from dietgpu_b200 import capi

    n = 8
    x, y = Batch(kind, member_sizes(n)), Batch(kind, [s + 3 for s in member_sizes(n)])
    for bt, seed in ((x, 1), (y, 2)):
        bt.fill(seed)
        bt.compress()
    torch.cuda.synchronize()
    L = capi.lib()
    ptrs = capi.ptr_array([r.data_ptr() for r in x.rows])
    temp = torch.empty(8 * n + 256, dtype=torch.uint8, device="cuda")
    got = torch.zeros(n, dtype=torch.int32, device="cuda")
    types = torch.zeros(n, dtype=torch.int32, device="cuda")

    def query():
        st = torch.cuda.current_stream().cuda_stream
        if kind == "bytes":
            rc = L.dgb_ans_get_compressed_info(temp.data_ptr(), temp.numel(), ptrs, 0, n, got.data_ptr(), None, st)
        else:
            rc = L.dgb_float_get_compressed_info(temp.data_ptr(), temp.numel(), ptrs, 0, n, got.data_ptr(),
                                                 types.data_ptr(), None, st)
        capi.check(rc, "get_compressed_info")

    query()
    torch.cuda.synchronize()
    assert got.cpu().tolist() == x.lengths
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        query()
    for i, r in enumerate(y.rows):
        ptrs[i] = r.data_ptr()
    got.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert got.cpu().tolist() == x.lengths, "the replay read the pointer array as it is now, not as it was captured"
    query()
    torch.cuda.synchronize()
    assert got.cpu().tolist() == y.lengths


# ---- A2: a thread whose first library call is captured -----------------------------------------------------------

def test_first_call_of_a_thread_can_be_captured():
    from dietgpu_b200 import capi

    a, b = Batch("bf16", member_sizes(20)), Batch("bytes", member_sizes(130))
    a.fill(1)
    b.fill(2)
    torch.cuda.synchronize()
    captured, errs = [], []
    done, release = threading.Event(), threading.Event()

    def worker():
        try:
            ga, gb = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            with torch.cuda.graph(ga):
                # the thread's first library calls: sub-batch streams and a decoder variant it has not used
                capi.set_thread_option("parts", 4)
                capi.set_thread_option("decode_warps", 4)
                a.step()
            with torch.cuda.graph(gb):
                b.step()
            captured.extend([ga, gb])
        except Exception as e:  # noqa: BLE001
            errs.append(e)
        finally:
            done.set()
            release.wait()  # alive, with its staging and streams, until the replays are over
            capi.clear_thread_options()

    th = threading.Thread(target=worker)
    th.start()
    try:
        assert done.wait(120), "capture thread did not finish"
        assert not errs, errs
        for r in range(2):
            for bt, gr, seed in ((a, captured[0], 30 + r), (b, captured[1], 40 + r)):
                bt.fill(seed)
                bt.clear()
                gr.replay()
                bt.check(what=f"replay {r} of the cold thread's {bt.kind} graph")
    finally:
        release.set()
        th.join()


# ---- A3: checksum verification inside a capture ---------------------------------------------------------------

@pytest.mark.parametrize("kind", ["bytes", "bf16"])
def test_checksum_verification_is_refused_inside_a_capture(kind):
    from dietgpu_b200 import capi

    x = Batch(kind, member_sizes(6))
    x.fill(1)
    x.compress(True)
    x.decompress(True)
    x.check(True, what="ordinary call")
    x.clear()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        x.compress(True)
        with pytest.raises(capi.DietGpuError, match="cannot be captured") as e:
            x.decompress(True)
        x.decompress(False)
    assert e.value.code == capi.ERR_CAPTURING
    # the capture was not invalidated: it ended, and the graph codes new data
    x.fill(2)
    x.clear()
    g.replay()
    x.check(True, what="replay")
    # and an ordinary verified round trip on the same thread still works
    x.fill(3)
    x.clear()
    x.compress(True)
    x.decompress(True)
    x.check(True, what="ordinary call after the refusal")


# ---- A4: every call follows the caller's stream -----------------------------------------------------------------

SLEEP_CYCLES = 100_000_000  # ~50 ms at the H100's 1.98 GHz boost clock (longer at lower clocks)


@pytest.mark.parametrize("side", [True, False], ids=["side_stream", "default_stream"])
def test_sub_batches_follow_the_callers_stream(side):
    cases = [("bf16", member_sizes(20), dict(parts=4)),  # encoder sub-batches
             ("bytes", member_sizes(65), dict(decode_fused=0, parts=4))]  # decoder sub-batches
    for kind, sizes, opts in cases:
        with codec_options(**opts):
            bt = Batch(kind, sizes)
            bt.fill(5)
            bt.step()  # warm: lazy set-up and first launches happen here, not in the timed window
            bt.check(what="warm-up")
            real = bt.want.clone()
            arch, arch_sizes = torch.empty_like(bt.comp), torch.empty_like(bt.sizes)
            bt.flat_in.fill_(0x3C)  # decoy
            bt.clear()
            torch.cuda.synchronize()
            s = torch.cuda.Stream() if side else torch.cuda.default_stream()
            with torch.cuda.stream(s):
                t0 = time.perf_counter()
                torch.cuda._sleep(SLEEP_CYCLES)
                bt.flat_in.copy_(real)
                bt.compress()
                bt.flat_in.fill_(0x5A)
                bt.temp_c.fill_(0xFF)
                arch.copy_(bt.comp)
                arch_sizes.copy_(bt.sizes)
                bt.decompress()
                bt.comp.fill_(0)
                bt.temp_d.fill_(0xFF)
                enqueue = time.perf_counter() - t0
                busy = not s.query()
            torch.cuda.synchronize()
            what = f"{kind} {opts} on the {'side' if side else 'default'} stream"
            assert busy, f"{what}: the stream was idle right after the calls were enqueued"
            assert enqueue < 0.02, f"{what}: enqueueing took {enqueue * 1e3:.1f} ms, a call blocked the host"
            bt.check_archives(arch, arch_sizes, False, False, what)
            bt.want = real
            bt.check_outputs(what)


# ---- A5: HostCodec compress_async / decompress_async in flight together ------------------------------------------

@pytest.mark.parametrize("groups", [1, 3, 8])
@pytest.mark.parametrize("kind", ["bytes", "bf16"])
def test_host_codec_pipeline(kind, groups):
    import dietgpu_b200 as dg

    sizes = [70001, 0, 1, BLOCK, 20000, 3 * BLOCK - 5, 50000, 777, 33333, 9]
    dtype = torch.uint8 if kind == "bytes" else KINDS[kind][1]
    steps = 4
    data = [[_data(kind, s, 100 * step + i) for i, s in enumerate(sizes)] for step in range(steps)]

    def pinned(a):
        t = torch.from_numpy(a.view(np.uint8) if kind == "bytes" else a.view(np.int16)).view(dtype)
        return t.pin_memory()

    # every member in a pinned allocation of its own: allocations that happen to lie back to back must not be
    # merged into one copy
    host_in = [[pinned(a) for a in d] for d in data]
    hc = dg.HostCodec(kind != "bytes", host_in[0], groups=groups, checksum=True)
    # two archive matrices wider than needed: rows at a constant pitch (one pitched copy per group)
    comp = [torch.full((len(sizes), hc.max_archive_bytes() + 48), 0xEE, dtype=torch.uint8).pin_memory()
            for _ in range(2)]
    outs = [[torch.empty_like(t).pin_memory() for t in host_in[0]] for _ in range(2)]

    def check_archives(step, hs):
        for i, a in enumerate(data[step]):
            want = oracle_archive(kind, a, PB, True)
            assert hs[i] == want.size, f"step {step} member {i}: size"
            got = comp[step & 1][i, :hs[i]].numpy()
            if kind == "bytes":
                O.assert_same_ans(got, want, f"step {step} member {i}")
            else:
                O.assert_same_float(got, want, KINDS[kind][0], f"step {step} member {i}")

    pend = hc.compress_async(host_in[0], comp[0])
    with pytest.raises(RuntimeError, match="finish"):
        hc.compress_async(host_in[1], comp[1])
    for step in range(steps):
        hs = pend.finish()
        check_archives(step, hs)
        if step % 2:  # rows in separate pinned allocations: an uneven pitch, one copy per row
            rows = [comp[step & 1][i, :k].clone().pin_memory() for i, k in enumerate(hs)]
        else:
            rows = [comp[step & 1][i, :k] for i, k in enumerate(hs)]
        for o in outs[step & 1]:
            if o.numel():  # (an empty pinned tensor has stride 0 and no byte view)
                o.view(torch.uint8).fill_(SENTINEL)
        pd =hc.decompress_async(rows, outs[step & 1])
        if step + 1 < steps:
            pend = hc.compress_async(host_in[step + 1], comp[(step + 1) & 1])
        pd.finish()
        for i, (a, o) in enumerate(zip(data[step], outs[step & 1])):
            got = o.view(torch.uint8).numpy() if o.numel() else np.zeros(0, np.uint8)
            assert np.array_equal(got, a.view(np.uint8)), f"step {step} member {i} decodes differently"


# ---- A6: two devices from one thread -----------------------------------------------------------------------------

@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible GPUs")
def test_two_devices_from_one_thread(options):
    options(parts=4)
    b1 = Batch("bf16", member_sizes(65), device="cuda:1")
    b0 = Batch("bytes", member_sizes(65), device="cuda:0")
    for r in range(2):
        for bt, other, seed in ((b1, 0, 50 + r), (b0, 1, 60 + r)):
            with torch.cuda.device(other):  # the current device is the other one; the call follows its tensors
                bt.fill(seed)
                bt.clear()
                bt.step()
                bt.check(what=f"round {r} on {bt.dev}")
    with torch.cuda.device(1):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            b1.step()
    for r in range(2):
        b1.fill(70 + r)
        b0.fill(80 + r)
        b1.clear()
        b0.clear()
        with torch.cuda.device(0):
            g.replay()
            b0.step()
        b1.check(what=f"replay {r} on cuda:1")
        b0.check(what=f"call {r} on cuda:0 beside the replay")
