"""LizardB200_decompressStream (DESIGN.md 3.4d) on the GPU, call for call against the reference's LizardF_decompress and this
library's host LizardF_decompress: return value, consumed, produced and the bytes produced, with guard bytes around the output.

Reference frames at every level 10-49, block size IDs 4-7, checksum and content size on and off, short and stored blocks,
skippable and concatenated frames; whole-stream, fixed and random chunks; ample, one-block, below-one-block and 1-byte
capacities; decode variants 7 and 23; damaged streams, srcPtr_wrong and a linked frame; launches per call independent of the
blocks a chunk holds; two streams on two CUDA streams beside decompressFrames and compress calls; one 1 GiB frame."""
import ctypes
import random
import struct

import pytest

import lizard_b200 as lz
from tests import refs
from tests.test_frame_stream_cpu import RefDecoder, feed, feed_past_errors, is_err, pieces_for, skippable, streamed_frame

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

G = 256                     # guard bytes on each side of the output


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built")
    return lz.bind_frame_api(L)


@pytest.fixture(scope="module")
def ours():
    return lz.bind_frame_api(lz.lib())


class GpuDecoder:
    """A DecompressionStream over a device copy of the data; call() has RefDecoder's signature (the host buffer is ignored)."""

    def __init__(self, data, stream=None):
        self.d_src = torch.frombuffer(bytearray(data) or bytearray(1), dtype=torch.uint8).cuda()
        self.ds = lz.DecompressionStream()
        self.stream = stream

    def call(self, src, off, n, cap):
        out = torch.empty(cap + 2 * G, dtype=torch.uint8, device="cuda")
        out[:G].fill_(0xA5)
        out[G + cap:].fill_(0xA5)
        r, used, made = self.ds.decompress(self.d_src.data_ptr() + off, n, out.data_ptr() + G, cap,
                                           stream=self.stream if self.stream is not None else 0)
        torch.cuda.synchronize()
        assert bool((out[:G] == 0xA5).all()) and bool((out[G + cap:] == 0xA5).all()), "write outside the output"
        return r, used, made, bytes(out[G:G + made].cpu().numpy()) if made else b""

    def close(self):
        self.ds.close()


def run(ref, ours, data, chunks, caps, stream=None):
    ds = [RefDecoder(ref), RefDecoder(ours), GpuDecoder(data, stream)]
    try:
        return feed(ds, data, chunks, caps)
    finally:
        for d in ds:
            d.close()


@pytest.mark.parametrize("level", range(10, 50))
def test_every_level(ref, ours, level):
    data = lz.datagen(300000, seed=level)
    try:
        frame = lz.frame_compress(ref, data, lz.make_prefs(level, checksum=level % 2 == 1, content_size=len(data) if level % 3 else 0))
    except lz.LizardB200Error:
        pytest.skip("the reference refuses level %d" % level)
    for chunk, cap in ((len(frame), 1 << 20), (65536, 131072), (1 << 20, 100000)):
        calls, out = run(ref, ours, frame, lambda k: chunk, lambda k: cap)
        assert out == data and calls[-1][0] == 0
    # chunks that stop at every position of the headers, size words and the suffix
    pieces = pieces_for(level)
    small = streamed_frame(ref, pieces, level, level % 2 == 1, 1800 if level % 3 else 0)
    for chunk in (1, 7, 19):
        calls, out = run(ref, ours, small, lambda k: chunk, lambda k: 1 << 16)
        assert out == b"".join(pieces) and calls[-1][0] == 0


@pytest.mark.parametrize("bsid", [4, 5, 6, 7])
@pytest.mark.parametrize("checksum", [False, True])
def test_block_sizes(ref, ours, bsid, checksum):
    data = lz.datagen(5 << 20, seed=bsid)
    frame = streamed_frame(ref, [data[:3 << 20], data[3 << 20:]], 21, checksum, len(data), block_id=bsid)
    for chunk in (len(frame), 1 << 20, 65536):
        for cap in (64 << 20, 4 << 20, (4 << 20) - 1):
            calls, out = run(ref, ours, frame, lambda k: chunk, lambda k: cap)
            assert out == data and calls[-1][0] == 0


@pytest.mark.parametrize("variant", [7, 23])
def test_feeding_and_capacities(ref, ours, variant):
    L = lz.lib()
    L.LizardB200_setDecodeVariant(variant)
    try:
        rnd = random.Random(variant)
        data = lz.datagen(3 << 20, seed=7)
        pieces = pieces_for(3) + [data]
        frame = streamed_frame(ref, pieces, 41, True)
        frame += struct.pack("<II", 0x184D2A50, 3) + b"abc" + lz.frame_compress(ref, data, lz.make_prefs(10))
        want = b"".join(pieces) + data
        for chunk in (len(frame), 1 << 20, 65536, 64 << 20):
            for cap in (64 << 20, 131072, 131071):
                calls, out = run(ref, ours, frame, lambda k: chunk, lambda k: cap)
                assert out == want
        sizes = [rnd.choice([1, 4, 7, 19, 65536, 1 << 20, 3 << 20]) for _ in range(5000)]
        caps = [rnd.choice([1, 4096, 131071, 131072, 1 << 22]) for _ in range(5000)]
        calls, out = run(ref, ours, frame, lambda k: sizes[k % 5000], lambda k: caps[k % 5000])
        assert out == want
        small = streamed_frame(ref, pieces_for(4), 10, True, 1800)
        for chunk in (1, 7):
            calls, out = run(ref, ours, small, lambda k: chunk, lambda k: 1)
            assert out == b"".join(pieces_for(4))
    finally:
        L.LizardB200_setDecodeVariant(7)


def test_damaged(ref, ours):
    data = lz.datagen(600000, seed=5)
    frame = bytearray(lz.frame_compress(ref, data, lz.make_prefs(41, checksum=True, content_size=len(data))))
    cases = []
    f = bytearray(frame); f[14] ^= 1; cases.append(f)
    f = bytearray(frame); f[18] = 0x7F; cases.append(f)
    f = bytearray(frame); f[60] ^= 0x55; f[61] ^= 0x55; cases.append(f)
    f = bytearray(frame); f[-1] ^= 1; cases.append(f)
    cases.append(frame[:-7])
    f = bytearray(lz.frame_compress(ref, data, lz.make_prefs(41, content_size=len(data))))
    f[6:14] = struct.pack("<Q", len(data) + 1)
    cases.append(f)
    for f in cases:
        for chunk in (4099, 65536, len(f)):
            for cap in (1 << 20, 1000):
                calls, _ = run(ref, ours, bytes(f), lambda k: chunk, lambda k: cap)


@pytest.mark.parametrize("checksum", [False, True])
def test_skippable_first(ref, ours, checksum):
    pieces = pieces_for(21)
    frame = streamed_frame(ref, pieces, 21, checksum)
    big = lz.frame_compress(ref, lz.datagen(1 << 20, seed=2), lz.make_prefs(41, checksum=checksum))
    for stream in (skippable(bytes(range(16))), skippable(b"") + skippable(b"x" * 300) + frame, skippable(bytes(40)) + big):
        for chunk in ((1, 7, 19) if len(stream) < 10000 else (4099, 65536)) + (len(stream),):
            calls, _ = run(ref, ours, stream, lambda k: chunk, lambda k: 1 << 21)
            assert calls[-1][0] == 0


def test_calls_after_a_checksum_error(ref, ours):
    data = lz.datagen(6000, seed=13)
    frame = bytearray(lz.frame_compress(ref, data, lz.make_prefs(21, checksum=True)))
    frame[-1] ^= 1
    frame = bytes(frame) + lz.frame_compress(ref, data, lz.make_prefs(10))
    for chunk in (1, 3, 4099, len(frame)):
        ds = [RefDecoder(ref), RefDecoder(ours), GpuDecoder(frame)]
        calls = feed_past_errors(ds, frame, lambda k: chunk, lambda k: 1 << 20)
        for d in ds:
            d.close()
        assert sum(is_err(r) for r, _, _ in calls) == 4


def test_src_ptr_wrong_and_linked(ref, ours):
    frame = lz.frame_compress(ref, lz.datagen(200000, seed=9), lz.make_prefs(10))
    src = ctypes.create_string_buffer(frame)
    ds = [RefDecoder(ref), GpuDecoder(frame)]
    first = [d.call(src, 0, 100, 0) for d in ds]
    again = [d.call(src, 0, 100, 0) for d in ds]
    for d in ds:
        d.close()
    assert first[0] == first[1] and again[0] == again[1] and again[0][0] == (1 << 64) - 15
    linked = bytearray(streamed_frame(ref, [lz.datagen(1000), lz.datagen(1000, seed=1)], 10))
    linked[4] &= ~0x20
    calls, _ = run(ref, ours, bytes(linked), lambda k: 64, lambda k: 1 << 16)
    assert is_err(calls[-1][0])


def test_launches_do_not_grow_with_blocks(ref):
    L = lz.lib()
    deltas = []
    for pct in (50, 99):                                           # few and many blocks in chunks of the same length
        data = lz.datagen(64 << 20, match_pct=pct, seed=1)
        frame = lz.frame_compress(ref, data[:16 << 20], lz.make_prefs(10, checksum=True))
        d_src = torch.frombuffer(bytearray(frame), dtype=torch.uint8).cuda()
        out = torch.empty(32 << 20, dtype=torch.uint8, device="cuda")
        with lz.DecompressionStream() as s:
            h = s.decompress(d_src.data_ptr(), 7, out.data_ptr(), out.numel(), stream=0)
            assert h[1] == 7
            n = 300000
            before = L.LizardB200_launchCount()
            h = s.decompress(d_src.data_ptr() + 7, n, out.data_ptr(), out.numel(), stream=0)
            deltas.append((L.LizardB200_launchCount() - before, h[2]))
    assert deltas[0][0] == deltas[1][0] and deltas[1][1] > 2 * deltas[0][1], deltas


def test_two_streams_interleaved(ref):
    data = [lz.datagen(6 << 20, seed=s) for s in (1, 2)]
    frames = [lz.frame_compress(ref, d, lz.make_prefs(21, checksum=True)) for d in data]
    srcs = [torch.frombuffer(bytearray(f), dtype=torch.uint8).cuda() for f in frames]
    outs = [torch.zeros(len(d), dtype=torch.uint8, device="cuda") for d in data]
    cs = [torch.cuda.Stream(), torch.cuda.Stream()]
    other = torch.frombuffer(bytearray(frames[0]), dtype=torch.uint8).cuda()
    other_out = torch.zeros(len(data[0]), dtype=torch.uint8, device="cuda")
    blocks = [data[0][i:i + 131072] for i in range(0, 1 << 20, 131072)]
    streams = [lz.DecompressionStream(), lz.DecompressionStream()]
    pos, made = [0, 0], [0, 0]
    while pos[0] < len(frames[0]) or pos[1] < len(frames[1]):
        for i in (0, 1):
            n = min(1 << 20, len(frames[i]) - pos[i])
            if n == 0:
                continue
            r, u, m = streams[i].decompress(srcs[i].data_ptr() + pos[i], n, outs[i].data_ptr() + made[i], len(data[i]) - made[i],
                                            stream=cs[i])
            assert not is_err(r)
            pos[i] += u
            made[i] += m
        res = lz.decompress_frames(other.data_ptr(), [0], [len(frames[0])], other_out.data_ptr(), [0], [len(data[0])])
        assert res == [len(data[0])]
        assert [c for _, c in lz.compress_batch(blocks, 10)] == [c for _, c in lz.compress_batch(blocks, 10)]
    for s in streams:
        s.close()
    torch.cuda.synchronize()
    assert made == [len(d) for d in data]
    assert bytes(outs[0].cpu().numpy()) == data[0] and bytes(outs[1].cpu().numpy()) == data[1]
    assert bytes(other_out.cpu().numpy()) == data[0]


def test_one_gib_frame_in_64_mib_chunks(ours):
    n = 1 << 30
    data = torch.empty(n, dtype=torch.uint8)
    lz.datagen_into(data.data_ptr(), n, 50.0, 3)
    frame = lz.frame_compress(ours, bytes(data.numpy()), lz.make_prefs(10, checksum=True, content_size=n))
    d_src = torch.frombuffer(bytearray(frame), dtype=torch.uint8).cuda()
    out = torch.empty(n, dtype=torch.uint8, device="cuda")
    pos = made = 0
    r = 1
    with lz.DecompressionStream() as s:
        while pos < len(frame):
            r, u, m = s.decompress(d_src[pos:], min(64 << 20, len(frame) - pos), out[made:], n - made)
            assert not is_err(r), lz.frame_error(r)
            pos += u
            made += m
    assert r == 0 and made == n
    assert torch.equal(out.cpu(), data)
