"""LizardB200_compressStream* (DESIGN.md 3.4e) on the H100: every call's *dWritten and bytes equal this library's host
LizardF_compressBegin / Update / flush / compressEnd fed host copies, and the finished frames equal the reference's.

- Levels 10, 13, 17, 19, 20, 21, 24, 30, 39, 40, 41 and 45 (every encoder kernel and its Huffman twin), block size IDs 1-4, and a
  frame of 64 MiB blocks at level 10; the chunk patterns of the CPU suite; guard bytes around dDst.
- Round trips through DecompressionStream and the host LizardF_decompress.
- Refused calls leave *dWritten unwritten, and the stream answers later calls as the host context does.
- Enqueue-only: a whole sequence returns while a spin kernel queued before it still runs; equal launches for equal sizes.
- Graph capture and replay on new contents; a capture that would grow the buffers is refused and changes nothing.
- Two streams interleaved on two CUDA streams with compressFramesAsync and decompressStream calls between them.
- 1 GiB in 64 MiB chunks at level 10, with and without the content checksum."""
import ctypes
import random

import pytest
import torch

import lizard_b200 as lz
from tests import refs

pytestmark = pytest.mark.gpu
SZ = ctypes.c_size_t
GUARD = 64
SENTINEL = -7
FRAME_SIZE_WRONG = (1 << 64) - 14          # End with a wrong contentSize: the only error a call returns after doing work
BLOCK = {1: 1 << 17, 2: 1 << 18, 3: 1 << 20, 4: 1 << 22, 5: 1 << 24, 6: 1 << 26, 7: 1 << 28}


@pytest.fixture(scope="module")
def L():
    return lz.bind_frame_api(lz.lib())


def is_err(r):
    return r > (1 << 64) - 20


class HostC:
    """This library's host API on host copies."""

    def __init__(self, L, data):
        self.L, self.src = L, ctypes.create_string_buffer(bytes(data), max(len(data), 1))
        self.ctx = ctypes.c_void_p()
        L.LizardF_createCompressionContext(ctypes.byref(self.ctx), 100)

    def call(self, c):
        cap = c[1]
        dst = ctypes.create_string_buffer(cap + 64)
        if c[0] == "begin":
            r = self.L.LizardF_compressBegin(self.ctx, dst, cap, ctypes.byref(c[2]))
        elif c[0] == "update":
            r = self.L.LizardF_compressUpdate(self.ctx, dst, cap, ctypes.byref(self.src, c[2]), c[3], None)
        elif c[0] == "flush":
            r = self.L.LizardF_flush(self.ctx, dst, cap, None)
        else:
            r = self.L.LizardF_compressEnd(self.ctx, dst, cap, None)
        return r, (b"" if is_err(r) else dst.raw[:r])

    def close(self):
        self.L.LizardF_freeCompressionContext(self.ctx)


class DevC:
    """The device stream, enqueue-only calls with *dWritten in device memory and guard bytes around each destination."""

    def __init__(self, data, stream=None):
        self.cs = lz.CompressionStream()
        self.src = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda() if len(data) else torch.zeros(1, dtype=torch.uint8,
                                                                                                             device="cuda")
        self.stream = stream

    def call(self, c):
        cap = c[1]
        buf = torch.full((cap + 2 * GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
        written = torch.full((1,), SENTINEL, dtype=torch.int64, device="cuda")
        d = buf.data_ptr() + GUARD
        s = self.stream
        if c[0] == "begin":
            h = self.cs.begin(d, cap, c[2], written, stream=s)
        elif c[0] == "update":
            h = self.cs.update(self.src.data_ptr() + c[2], c[3], d, cap, written, stream=s)
        else:
            h = getattr(self.cs, c[0])(d, cap, written, stream=s)
        torch.cuda.synchronize()
        w = int(written.item())
        host = buf.cpu().numpy().tobytes()
        assert host[:GUARD] == b"\xa5" * GUARD and host[GUARD + cap:] == b"\xa5" * GUARD
        if is_err(h) and not (c[0] == "end" and h == FRAME_SIZE_WRONG):  # refused before any work: nothing written
            assert w == SENTINEL, (c[0], h, w)
            assert host[GUARD:] == b"\xa5" * (cap + GUARD)
            return h, b""
        assert w != SENTINEL, c[0]
        r = w & ((1 << 64) - 1)
        assert h == (r if is_err(r) else 0), (c[0], h, r)
        return r, (b"" if is_err(r) else host[GUARD:GUARD + r])

    def close(self):
        self.cs.close()


def bound(L, n, prefs):
    return L.LizardF_compressBound(n, ctypes.byref(prefs))


def calls_for(L, prefs, sizes, flush_at=()):
    calls, off = [("begin", 15, prefs)], 0
    bs = BLOCK[prefs.frameInfo.blockSizeID]
    for i, n in enumerate(sizes):
        calls.append(("update", bound(L, n, prefs) + (1 if prefs.autoFlush else 0), off, n))
        off += n
        if i in flush_at:
            calls.append(("flush", bs + 8))
    calls.append(("end", bs + 16))
    return calls


def compare(L, data, calls, stream=None):
    """Every call's result and bytes on the device and on the host; returns the concatenated output of the host."""
    h, d = HostC(L, data), DevC(data, stream)
    out = []
    try:
        for k, c in enumerate(calls):
            a, b = h.call(c), d.call(c)
            assert a[0] == b[0] and a[1] == b[1], (k, c[0], c[2:] if c[0] == "update" else c[1], a[0], b[0])
            out.append(a[1])
    finally:
        h.close()
        d.close()
    return b"".join(out)


def ref_frame(calls, data):
    R = refs.ref_parity()
    if R is None:
        return None
    lz.bind_frame_api(R)
    h = HostC(R, data)
    try:
        return b"".join(h.call(c)[1] for c in calls)
    finally:
        h.close()


ALL_LEVELS = (10, 13, 17, 19, 20, 21, 24, 30, 39, 40, 41, 45)


@pytest.mark.parametrize("level", ALL_LEVELS)
@pytest.mark.parametrize("bsid", (1, 2, 3, 4))
def test_levels_and_block_sizes(L, level, bsid):
    bs = BLOCK[bsid]
    data = lz.datagen(2 * bs + bs // 2 + 777, seed=level + bsid)
    rng = random.Random(level * 7 + bsid)
    p = lz.make_prefs(level, block_id=bsid, checksum=(level + bsid) % 2 == 0)
    p.autoFlush = rng.randrange(2)
    sizes = [bs - 1, 1, bs + 1, rng.randrange(0, bs // 2), 13]
    sizes.append(len(data) - sum(sizes))
    calls = calls_for(L, p, sizes, flush_at=(2,))
    frame = compare(L, data, calls)
    ref = ref_frame(calls, data)
    if ref is not None:
        assert frame == ref
    r, back = lz.frame_decompress(L, frame, len(data) + 1)
    assert back == data


@pytest.mark.parametrize("level", (10, 41))
def test_chunk_patterns(L, level):
    data = lz.datagen(3 * (1 << 17) + 5000, seed=level)
    rng = random.Random(level)
    for auto_flush in (0, 1):
        for checksum in (False, True):
            for sizes in ([n for n in range(20)] * 2, [(1 << 17) - 1, 1 << 17, (1 << 17) + 1],
                          [rng.randrange(0, 70000) for _ in range(8)]):
                p = lz.make_prefs(level, checksum=checksum)
                p.autoFlush = auto_flush
                calls = calls_for(L, p, sizes, flush_at=(1, 3))
                frame = compare(L, data, calls)
                ref = ref_frame(calls, data)
                if ref is not None:
                    assert frame == ref


def test_refused_calls_and_what_follows(L):
    data = lz.datagen((1 << 17) + 300, seed=4)
    p = lz.make_prefs(17, content_size=(1 << 17) + 21)
    b10 = bound(L, 10, p)
    calls = [("update", b10, 0, 10), ("flush", 64), ("end", 64), ("begin", 14, p), ("begin", 15, p), ("begin", 15, p),
             ("update", b10 - 1, 0, 10), ("update", b10, 0, 10), ("flush", 10 + 7), ("flush", 18), ("flush", 64),
             ("update", bound(L, 1, p), 10, 1), ("flush", 1 + 7), ("flush", 10),
             ("update", bound(L, 1 << 17, p), 11, 1 << 17), ("end", 64),               # contentSize wrong
             ("begin", 15, lz.make_prefs(12)), ("begin", 15, lz.make_prefs(26)), ("begin", 15, lz.make_prefs(49)),
             ("begin", 15, lz.make_prefs(10, independent=False)), ("update", b10, 0, 10),
             ("begin", 15, lz.make_prefs(10)), ("update", b10, 0, 10), ("end", 64)]
    compare(L, data, calls)


def test_block_size_64mib_frame(L):
    n = (64 << 20) + (5 << 20)
    data = lz.datagen(n, seed=6)
    p = lz.make_prefs(10, block_id=6, checksum=True)
    calls = [("begin", 15, p), ("update", bound(L, 40 << 20, p), 0, 40 << 20), ("update", bound(L, n - (40 << 20), p), 40 << 20,
                                                                                n - (40 << 20)), ("end", (64 << 20) + 16)]
    frame = compare(L, data, calls)
    ref = ref_frame(calls, data)
    if ref is not None:
        assert frame == ref


def test_round_trip_through_device_decompression(L):
    data = lz.datagen(5 << 20, seed=8)
    p = lz.make_prefs(21, checksum=True)
    calls = calls_for(L, p, [1 << 20, 3 << 20, 1 << 20])
    frame = compare(L, data, calls)
    d_frame = torch.frombuffer(bytearray(frame), dtype=torch.uint8).cuda()
    out = torch.empty(len(data) + 64, dtype=torch.uint8, device="cuda")
    with lz.DecompressionStream() as ds:
        hint, used, made = ds.decompress(d_frame, len(frame), out, len(data) + 64)
    assert hint == 0 and used == len(frame) and made == len(data)
    assert out[:made].cpu().numpy().tobytes() == data


def _sequence(cs, src, n_chunks, chunk, d_dst, cap, written, p, stream=None):
    """Begin at d_dst, the chunks' Updates, Flush and End each into cap bytes behind it; results to written[0..n_chunks + 2]"""
    cs.begin(d_dst, 15, p, written[0:1], stream)
    o = 64
    for k in range(n_chunks):
        cs.update(src.data_ptr() + k * chunk, chunk, d_dst + o, cap, written[k + 1:k + 2], stream)
        o += cap
    cs.flush(d_dst + o, cap, written[n_chunks + 1:n_chunks + 2], stream)
    o += cap
    cs.end(d_dst + o, cap, written[n_chunks + 2:n_chunks + 3], stream)


def _assemble(out, written, n_chunks, cap):
    w = written.cpu().tolist()
    buf = out.cpu().numpy().tobytes()
    parts, o = [buf[:w[0]]], 64
    for k in range(n_chunks + 2):
        parts.append(buf[o:o + w[k + 1]])
        o += cap
    return b"".join(parts)


def _host_frame(L, data, p, n_chunks, chunk, cap):
    h = HostC(L, data)
    try:
        calls = [("begin", 15, p)] + [("update", cap, k * chunk, chunk) for k in range(n_chunks)] + [("flush", cap), ("end", cap)]
        return b"".join(h.call(c)[1] for c in calls)
    finally:
        h.close()


def test_enqueue_only_and_launch_counts(L):
    chunk, n_chunks = 1 << 20, 3
    data = lz.datagen(chunk * n_chunks, seed=9)
    p = lz.make_prefs(10, checksum=True)
    cap = bound(L, chunk, p)
    src = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    out = torch.zeros(64 + (n_chunks + 2) * cap, dtype=torch.uint8, device="cuda")
    written = torch.zeros(n_chunks + 3, dtype=torch.int64, device="cuda")
    s = torch.cuda.Stream()
    with lz.CompressionStream() as cs:
        _sequence(cs, src, n_chunks, chunk, out.data_ptr(), cap, written, p, s.cuda_stream)       # warm-up: the buffers grow
        s.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(1 << 30)
        _sequence(cs, src, n_chunks, chunk, out.data_ptr(), cap, written, p, s.cuda_stream)
        assert not s.query()                                              # returned while the spin kernel runs
        s.synchronize()
        assert _assemble(out, written, n_chunks, cap) == _host_frame(L, data, p, n_chunks, chunk, cap)
        # Two Updates of equal sizes and different data: each completes the carried block, compresses 7 more blocks and carries
        # 1000 bytes again, with the checksum.  They issue the same launches.
        bs = 1 << 17
        assert cs.begin(out, 15, p, written[0:1], s.cuda_stream) == 0
        assert cs.update(src, 1000, out, cap, written[1:2], s.cuda_stream) == 0
        counts, srcs = [], []
        for seed in (1, 2):
            srcs.append(torch.frombuffer(bytearray(lz.datagen(8 * bs, seed=seed)), dtype=torch.uint8).cuda())
            n0 = lz.lib().LizardB200_launchCount()
            assert cs.update(srcs[-1], 8 * bs, out.data_ptr() + 64 + seed * cap, cap, written[seed + 1:seed + 2], s.cuda_stream) == 0
            counts.append(lz.lib().LizardB200_launchCount() - n0)
        assert cs.end(out.data_ptr() + 64 + 3 * cap, cap, written[4:5], s.cuda_stream) == 0
        s.synchronize()
        assert counts[0] > 0 and counts[0] == counts[1], counts
        assert written[1].item() == 0 and all(int(w) > 0 for w in written[2:5].tolist())


def test_graph_capture_and_replay(L):
    chunk, n_chunks = 700000, 3
    p = lz.make_prefs(41, checksum=True)
    cap = bound(L, chunk, p)
    src = torch.empty(chunk * n_chunks, dtype=torch.uint8, device="cuda")
    out = torch.zeros(64 + (n_chunks + 2) * cap, dtype=torch.uint8, device="cuda")
    written = torch.zeros(n_chunks + 3, dtype=torch.int64, device="cuda")
    s = torch.cuda.Stream()
    with lz.CompressionStream() as cs:
        src.copy_(torch.frombuffer(bytearray(lz.datagen(chunk * n_chunks, seed=1)), dtype=torch.uint8))
        torch.cuda.synchronize()
        _sequence(cs, src, n_chunks, chunk, out.data_ptr(), cap, written, p, s.cuda_stream)
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            _sequence(cs, src, n_chunks, chunk, out.data_ptr(), cap, written, p, torch.cuda.current_stream().cuda_stream)
        for seed in (2, 3):
            data = lz.datagen(chunk * n_chunks, seed=seed)
            src.copy_(torch.frombuffer(bytearray(data), dtype=torch.uint8))
            torch.cuda.synchronize()
            g.replay()
            torch.cuda.synchronize()
            assert _assemble(out, written, n_chunks, cap) == _host_frame(L, data, p, n_chunks, chunk, cap)


def test_capture_that_must_grow_is_refused(L):
    p = lz.make_prefs(10)
    data = lz.datagen(3 << 20, seed=5)
    src = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    cap = bound(L, 3 << 20, p)
    out = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
    written = torch.full((4,), SENTINEL, dtype=torch.int64, device="cuda")
    s = torch.cuda.Stream()
    with lz.CompressionStream() as cs:
        assert cs.begin(out, 15, p, written[0:1], s.cuda_stream) == 0
        s.synchronize()
        n0 = lz.lib().LizardB200_launchCount()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            r = cs.update(src.data_ptr(), 3 << 20, out.data_ptr() + 64, cap, written[1:2].data_ptr(),
                          torch.cuda.current_stream().cuda_stream)
        assert r == (1 << 64) - 1 and lz.lib().LizardB200_launchCount() == n0
        assert b"grow" in lz.lib().LizardB200_lastError()
        assert int(written[1].item()) == SENTINEL
        # outside the capture the stream goes on as if the refused call had not been made
        r1 = cs.update(src, 3 << 20, out, cap, stream=s.cuda_stream)
        r2 = cs.end(out, cap, stream=s.cuda_stream)
    h = HostC(L, data)
    try:
        assert h.call(("begin", 15, p))[0] == 7
        assert h.call(("update", cap, 0, 3 << 20))[0] == r1
        assert h.call(("end", cap))[0] == r2
    finally:
        h.close()


def test_two_streams_between_other_device_calls(L):
    chunk = 1 << 20
    datas = [lz.datagen(4 * chunk, seed=s) for s in (11, 12)]
    prefs = [lz.make_prefs(10, checksum=True), lz.make_prefs(21)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    srcs = [torch.frombuffer(bytearray(d), dtype=torch.uint8).cuda() for d in datas]
    caps = [bound(L, chunk, p) for p in prefs]
    outs = [torch.zeros(64 + 6 * c, dtype=torch.uint8, device="cuda") for c in caps]
    writs = [torch.zeros(7, dtype=torch.int64, device="cuda") for _ in caps]
    css = [lz.CompressionStream(), lz.CompressionStream()]
    # a frame for the other device calls in between
    other = lz.frame_compress(L, datas[0][:chunk], lz.make_prefs(17))
    d_other = torch.frombuffer(bytearray(other), dtype=torch.uint8).cuda()
    d_other_out = torch.empty(chunk, dtype=torch.uint8, device="cuda")
    try:
        for i in range(2):
            css[i].begin(outs[i], 15, prefs[i], writs[i][0:1], streams[i].cuda_stream)
        for k in range(4):
            for i in range(2):
                css[i].update(srcs[i].data_ptr() + k * chunk, chunk, outs[i].data_ptr() + 64 + k * caps[i], caps[i],
                              writs[i][k + 1:k + 2], streams[i].cuda_stream)
            if k == 1:
                off = torch.tensor([0], dtype=torch.int64, device="cuda")
                size = torch.tensor([chunk], dtype=torch.int64, device="cuda")
                dcap = torch.tensor([len(other) + 64], dtype=torch.int64, device="cuda")
                res = torch.zeros(1, dtype=torch.int64, device="cuda")
                dst = torch.empty(len(other) + 64, dtype=torch.uint8, device="cuda")
                lz.compress_frames_async(srcs[0], off, size, dst, off, dcap, res, lz.make_prefs(17), 8, 1 << 30,
                                         stream=streams[0].cuda_stream)
            if k == 2:
                with lz.DecompressionStream() as ds:
                    ds.decompress(d_other, len(other), d_other_out, chunk, stream=streams[1].cuda_stream)
        for i in range(2):
            css[i].flush(outs[i].data_ptr() + 64 + 4 * caps[i], caps[i], writs[i][5:6], streams[i].cuda_stream)
            css[i].end(outs[i].data_ptr() + 64 + 5 * caps[i], caps[i], writs[i][6:7], streams[i].cuda_stream)
        torch.cuda.synchronize()
        for i in range(2):
            assert _assemble(outs[i], writs[i], 4, caps[i]) == _host_frame(L, datas[i], prefs[i], 4, chunk, caps[i])
        assert d_other_out.cpu().numpy().tobytes() == datas[0][:chunk]
    finally:
        for cs in css:
            cs.close()


@pytest.mark.parametrize("checksum", [False, True])
def test_one_gib_in_64_mib_chunks(L, checksum):
    n, chunk = 1 << 30, 64 << 20
    src = torch.empty(n, dtype=torch.uint8, device="cuda")
    data = lz.datagen(n, seed=1)
    src.copy_(torch.frombuffer(bytearray(data), dtype=torch.uint8))
    p = lz.make_prefs(10, checksum=checksum)
    cap = bound(L, chunk, p)
    out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    h = HostC(L, data)
    try:
        with lz.CompressionStream() as cs:
            assert cs.begin(out, 15, p) == h.call(("begin", 15, p))[0]
            for k in range(n // chunk):
                r = cs.update(src.data_ptr() + k * chunk, chunk, out, cap)
                hr, hb = h.call(("update", cap, k * chunk, chunk))
                assert r == hr and out[:r].cpu().numpy().tobytes() == hb
            r = cs.end(out, cap)
            hr, hb = h.call(("end", cap))
            assert r == hr and out[:r].cpu().numpy().tobytes() == hb
    finally:
        h.close()


def test_end_after_a_refused_begin_on_a_fresh_stream(L):
    """A fresh stream answers as a fresh host context: a refused Begin keeps its preferences, and End then writes the end mark and
    the checksum of nothing."""
    for p in (lz.make_prefs(12, checksum=True), lz.make_prefs(10, independent=False, checksum=True)):
        compare(L, b"x", [("begin", 15, p), ("flush", 16), ("end", 64)])


def test_one_byte_last_block_past_the_bound(L):
    """The one documented difference (include/lizard_b200.h): autoFlush, no checksum, exactly LizardF_compressBound of room, whole
    blocks that are all stored raw and a 1-byte last block.  Both refuse the call with ERROR_dstMaxSize_tooSmall, the device one
    through *dWritten after enqueueing it; the device stream then counts the chunk, the host context does not, so a later End
    with contentSize set answers differently."""
    bs = 1 << 17
    data = random.Random(5).randbytes(bs + 1)                           # incompressible: the full block is stored raw
    p = lz.make_prefs(10, content_size=bs + 1)
    p.autoFlush = 1
    b = bound(L, bs + 1, p)
    h = HostC(L, data)
    src = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    out = torch.zeros(b + 64, dtype=torch.uint8, device="cuda")
    written = torch.full((4,), SENTINEL, dtype=torch.int64, device="cuda")
    too_small = (1 << 64) - 11
    try:
        with lz.CompressionStream() as cs:
            assert h.call(("begin", 15, p))[0] == cs.begin(out, 15, p) == 15
            assert h.call(("update", b, 0, bs + 1))[0] == too_small
            assert cs.update(src, bs + 1, out, b, written[0:1]) == 0
            torch.cuda.synchronize()
            assert int(written[0].item()) & ((1 << 64) - 1) == too_small
            hr, hb = h.call(("update", b + 1, 0, bs + 1))
            assert hr == bs + 14 and cs.update(src, bs + 1, out, b + 1) == hr and out[:hr].cpu().numpy().tobytes() == hb
            assert h.call(("end", 64))[0] == 4
            assert cs.end(out, 64, written[1:2]) == FRAME_SIZE_WRONG
            torch.cuda.synchronize()
            assert int(written[1].item()) & ((1 << 64) - 1) == FRAME_SIZE_WRONG
    finally:
        h.close()
