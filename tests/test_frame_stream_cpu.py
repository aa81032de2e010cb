"""LizardB200_decompressStream (DESIGN.md 3.4d) on the CPU: the host build (lizard_b200/libhostshim.so, TEST-ONLY) of the shared
state machine (frame_stream.h: frame_decompress_run) over the stream's backend (StreamIO: rounds of walk + decode, placements
and checksum pieces), with the walk and the one-lane decoder in place of the kernels, against the reference's LizardF_decompress
call for call: return value, consumed, produced and the bytes produced.

- Reference frames at levels 10, 21, 41 and 45, with and without the content checksum and the content size, and streamed frames
  of short blocks and stored blocks.
- Chunks of 1 to 19 bytes, which stop at every position of the headers, size words and suffixes; random chunks; capacities
  that send blocks through the one-block buffer (DS_flushOut), down to 1 byte.
- Skippable and concatenated frames, damaged frames, srcPtr_wrong and a linked frame.
- The walk resumed at every record boundary, and each of its stop reasons.
- The new kernels' registers, stack and local memory (cuobjdump -res-usage)."""
import ctypes
import os
import random
import re
import struct
import subprocess

import pytest

import lizard_b200 as lz
from tests import refs
from tests.test_encode_resources_cpu import _cuobjdump

SZ = ctypes.c_size_t
LEVELS = (10, 21, 41, 45)


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built")
    return lz.bind_frame_api(L)


@pytest.fixture(scope="module")
def shim():
    p = os.path.join(refs.ROOT, "lizard_b200", "libhostshim.so")
    if not os.path.exists(p):
        pytest.skip("libhostshim.so not built")
    L = ctypes.CDLL(p)
    L.lzb_host_stream_new.restype = ctypes.c_void_p
    L.lzb_host_stream_free.argtypes = [ctypes.c_void_p]
    L.lzb_host_stream_call.restype = SZ
    L.lzb_host_stream_call.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(SZ), ctypes.c_void_p, ctypes.POINTER(SZ),
                                       ctypes.POINTER(ctypes.c_ulonglong)]
    L.lzb_host_stream_walk.argtypes = [ctypes.c_char_p, ctypes.c_ulonglong, ctypes.c_uint, ctypes.c_uint, ctypes.c_uint,
                                       ctypes.POINTER(ctypes.c_ulonglong), ctypes.POINTER(ctypes.c_uint),
                                       ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_uint)]
    return L


class RefDecoder:
    def __init__(self, L):
        self.L = L
        self.ctx = ctypes.c_void_p()
        L.LizardF_createDecompressionContext(ctypes.byref(self.ctx), 100)

    def call(self, src, off, n, cap):
        out = ctypes.create_string_buffer(max(cap, 1))
        si, so = SZ(n), SZ(cap)
        r = self.L.LizardF_decompress(self.ctx, out, ctypes.byref(so), ctypes.byref(src, off), ctypes.byref(si), None)
        return r, si.value, so.value, out.raw[:so.value]

    def close(self):
        self.L.LizardF_freeDecompressionContext(self.ctx)


class ShimDecoder:
    def __init__(self, S):
        self.S = S
        self.h = S.lzb_host_stream_new()
        self.rounds = 0

    def call(self, src, off, n, cap):
        out = ctypes.create_string_buffer(max(cap, 1))
        si, so, rounds = SZ(n), SZ(cap), ctypes.c_ulonglong()
        r = self.S.lzb_host_stream_call(self.h, out, ctypes.byref(so), ctypes.byref(src, off), ctypes.byref(si), ctypes.byref(rounds))
        self.rounds += rounds.value
        return r, si.value, so.value, out.raw[:so.value]

    def close(self):
        self.S.lzb_host_stream_free(self.h)


def is_err(r):
    return r > (1 << 64) - 20


def feed(decoders, data, chunks, caps, max_calls=200000):
    """Feed data to every decoder in the same calls: call k offers the next chunks(k) bytes from where the previous call
    stopped, with caps(k) bytes of room.  Every decoder must answer alike; returns the answers and the bytes produced."""
    src = ctypes.create_string_buffer(data, max(len(data), 1))
    pos, k, out, calls = 0, 0, [], []
    while k < max_calls:
        n = min(chunks(k), len(data) - pos)
        cap = caps(k)
        got = [d.call(src, pos, n, cap) for d in decoders]
        for g in got[1:]:
            assert g == got[0], (k, pos, n, cap, got[0][:3], g[:3])
        r, used, made, b = got[0]
        calls.append((r, used, made))
        out.append(b)
        k += 1
        if is_err(r):
            break
        pos += used
        if pos >= len(data) and (r == 0 or (used == 0 and made == 0)):
            break
        if n == 0 and used == 0 and made == 0:
            break
    return calls, b"".join(out)


def streamed_frame(L, pieces, level, checksum=False, content_size=0, block_id=1, flush=True):
    """A frame written by the reference's compressBegin / compressUpdate / flush: each piece ends a short block."""
    p = lz.make_prefs(level, block_id=block_id, checksum=checksum, content_size=content_size)
    ctx = ctypes.c_void_p()
    L.LizardF_createCompressionContext(ctypes.byref(ctx), 100)
    total = sum(len(x) for x in pieces)
    buf = ctypes.create_string_buffer(L.LizardF_compressBound(total, ctypes.byref(p)) * 2 + 64 * len(pieces) + 64)
    at = L.LizardF_compressBegin(ctx, buf, len(buf), ctypes.byref(p))
    assert not L.LizardF_isError(at)
    for x in pieces:
        r = L.LizardF_compressUpdate(ctx, ctypes.byref(buf, at), len(buf) - at, x, len(x), None)
        assert not L.LizardF_isError(r)
        at += r
        if flush:
            r = L.LizardF_flush(ctx, ctypes.byref(buf, at), len(buf) - at, None)
            assert not L.LizardF_isError(r)
            at += r
    r = L.LizardF_compressEnd(ctx, ctypes.byref(buf, at), len(buf) - at, None)
    assert not L.LizardF_isError(r)
    L.LizardF_freeCompressionContext(ctx)
    return buf.raw[:at + r]


def pieces_for(seed):
    rnd = random.Random(seed)
    return [lz.datagen(600, seed=seed), bytes(rnd.getrandbits(8) for _ in range(300)), lz.datagen(900, seed=seed + 1)]


def both(ref, shim):
    return [RefDecoder(ref), ShimDecoder(shim)]


def close(ds):
    for d in ds:
        d.close()


@pytest.mark.parametrize("level", LEVELS)
@pytest.mark.parametrize("checksum", [False, True])
@pytest.mark.parametrize("csize", [False, True])
def test_small_chunks(ref, shim, level, checksum, csize):
    pieces = pieces_for(level)
    total = sum(len(x) for x in pieces)
    frame = streamed_frame(ref, pieces, level, checksum, total if csize else 0)
    for step in range(1, 20):
        for cap in (1 << 20, 97):
            ds = both(ref, shim)
            calls, out = feed(ds, frame, lambda k: step, lambda k: cap)
            close(ds)
            assert calls[-1][0] == 0 and out == b"".join(pieces), (step, cap, calls[-1])


@pytest.mark.parametrize("level", LEVELS)
def test_random_chunks_and_capacities(ref, shim, level):
    rnd = random.Random(level)
    data = lz.datagen(400000, seed=level)
    for checksum in (False, True):
        for csize in (0, len(data)):
            frame = lz.frame_compress(ref, data, lz.make_prefs(level, checksum=checksum, content_size=csize))
            frame = frame + struct.pack("<II", 0x184D2A53, 5) + b"skip!" + frame
            for trial in range(3):
                sizes = [rnd.choice([1, 3, 4, 5, 17, 1000, 70000, 200000]) for _ in range(4000)]
                caps = [rnd.choice([1, 1000, 131072, 131073, 300000, 1 << 21]) for _ in range(4000)]
                ds = both(ref, shim)
                calls, out = feed(ds, frame, lambda k: sizes[k % 4000], lambda k: caps[k % 4000])
                close(ds)
                assert out == data + data and calls[-1][0] == 0


def test_whole_and_capacities(ref, shim):
    data = lz.datagen(3 * 131072 + 5000, seed=3)
    frame = lz.frame_compress(ref, data, lz.make_prefs(21, checksum=True, content_size=len(data)))
    for cap in (1 << 22, 131072, 131071, 4093):
        ds = both(ref, shim)
        calls, out = feed(ds, frame, lambda k: len(frame), lambda k: cap)
        close(ds)
        assert out == data and calls[-1][0] == 0
    # one call of the whole frame runs one round (walk + decode)
    ds = both(ref, shim)
    calls, out = feed(ds, frame, lambda k: len(frame), lambda k: 1 << 22)
    assert len(calls) == 1 and ds[1].rounds == 1
    close(ds)


def test_damaged(ref, shim):
    data = lz.datagen(300000, seed=5)
    frame = bytearray(lz.frame_compress(ref, data, lz.make_prefs(41, checksum=True, content_size=len(data))))
    hdr = 15
    cases = []
    f = bytearray(frame); f[hdr - 1] ^= 1; cases.append(f)                                  # header checksum
    f = bytearray(frame); f[hdr + 3] = 0x7F; cases.append(f)                                # size word beyond the block size
    f = bytearray(frame); f[hdr + 40] ^= 0x55; f[hdr + 41] ^= 0x55; cases.append(f)         # corrupt block
    f = bytearray(frame); f[-1] ^= 1; cases.append(f)                                       # content checksum
    cases.append(frame[:-7])                                                                # truncated
    f = bytearray(lz.frame_compress(ref, data, lz.make_prefs(41, content_size=len(data) + 1)))
    f[6:14] = struct.pack("<Q", len(data) + 1)
    cases.append(f)
    for f in cases:
        for step in (7, 4096, len(f)):
            ds = both(ref, shim)
            feed(ds, bytes(f), lambda k: step, lambda k: 1 << 20)
            close(ds)


def test_src_ptr_wrong_and_linked(ref, shim):
    data = lz.datagen(200000, seed=9)
    frame = lz.frame_compress(ref, data, lz.make_prefs(10))
    src = ctypes.create_string_buffer(frame)
    ds = both(ref, shim)
    first = [d.call(src, 0, 100, 0) for d in ds]
    assert first[0] == first[1] and first[0][1] < 100
    again = [d.call(src, 0, 100, 0) for d in ds]                      # not where the previous call stopped
    assert again[0] == again[1] and again[0][0] == (1 << 64) - 15
    close(ds)
    linked = streamed_frame(ref, [lz.datagen(1000), lz.datagen(1000, seed=1)], 10, flush=True)
    linked = bytearray(linked)
    linked[4] &= ~0x20                                                  # blockMode: linked
    ds = both(ref, shim)
    calls, _ = feed(ds, bytes(linked), lambda k: 64, lambda k: 1 << 16)
    close(ds)
    assert calls[-1][0] in ((1 << 64) - 3, (1 << 64) - 17)


def walk(shim, buf, max_block, max_recs, slots):
    n = 4096
    pos, word, unit = (ctypes.c_ulonglong * n)(), (ctypes.c_uint * n)(), (ctypes.c_int * n)()
    summ = (ctypes.c_uint * 3)()
    shim.lzb_host_stream_walk(buf, len(buf), max_block, max_recs, slots, pos, word, unit, summ)
    return [(pos[i], word[i], unit[i]) for i in range(summ[0])], summ[1], summ[2]


def test_walk(ref, shim):
    pieces = pieces_for(11) + pieces_for(12)
    frame = streamed_frame(ref, pieces, 10, checksum=True)
    body = frame[7:]
    recs, at = [], 0
    while True:                                                          # the records, parsed here
        w = struct.unpack_from("<I", body, at)[0]
        recs.append((at, w))
        if w & 0x7FFFFFFF == 0:
            break
        at += 4 + (w & 0x7FFFFFFF)
    assert len(recs) >= 7
    for i, (start, _) in enumerate(recs):
        chunk = body[start:]
        got, stop, units = walk(shim, chunk, 1 << 17, 4096, 4096)
        assert [(p + start, w) for p, w, _ in got] == recs[i:] and stop == 1
        assert units == sum(1 for _, w in recs[i:] if w & 0x7FFFFFFF and not w >> 31)
        assert [u for _, _, u in got if u >= 0] == list(range(1, units + 1))
        # stops: fewer than 4 bytes, a partial block, the record bound, the slot bound, a size beyond the block size
        if i + 1 < len(recs):
            nxt = recs[i + 1][0] - start
            assert walk(shim, chunk[:nxt + 3], 1 << 17, 4096, 4096)[1] == 0
            assert walk(shim, chunk[:nxt - 1], 1 << 17, 4096, 4096)[1] == 3
            got, stop, _ = walk(shim, chunk, 1 << 17, 1, 4096)
            assert stop == 4 and len(got) == 1
            if not recs[i][1] >> 31:
                got, stop, units = walk(shim, chunk, 1 << 17, 4096, 0)
                assert stop == 5 and units == 0 and got[-1][2] == -1
            small = (recs[i][1] & 0x7FFFFFFF) - 1
            if small > 0:
                assert walk(shim, chunk, small, 4096, 4096)[1] == 2


STREAM_KERNEL_LIMITS = {"lizard_frame_stream_walk_kernel": (40, 0), "lizard_frame_stream_hash_kernel": (48, 0)}


def test_stream_kernel_resources():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not available")
    lib = os.path.join(refs.ROOT, "lizard_b200", "liblizard_b200.so")
    out = subprocess.run([exe, "-res-usage", lib], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout
    found, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name and "REG:" in line:
            for k in STREAM_KERNEL_LIMITS:
                if re.search(r"\d" + k + r"[A-Z]", name):
                    found[k] = {a: int(b) for a, b in re.findall(r"(REG|STACK|LOCAL|SHARED):(\d+)", line)}
            name = None
    assert set(found) == set(STREAM_KERNEL_LIMITS), found
    for k, (reg, stack) in STREAM_KERNEL_LIMITS.items():
        r = found[k]
        assert r["REG"] <= reg and r["STACK"] <= stack and r["LOCAL"] == 0, (k, r)


def feed_past_errors(decoders, data, chunks, caps, after=3):
    """feed(), but the calls go on `after` times past the first error, offered the bytes from where the stream stands: what a
    caller that keeps calling sees must match too."""
    src = ctypes.create_string_buffer(data, max(len(data), 1))
    pos, k, errors, calls = 0, 0, 0, []
    while errors <= after and k < 100000:
        n = min(chunks(k), len(data) - pos)
        got = [d.call(src, pos, n, caps(k)) for d in decoders]
        for g in got[1:]:
            assert g == got[0], (k, pos, n, got[0][:3], g[:3])
        r, used, made, _ = got[0]
        calls.append((r, used, made))
        k += 1
        errors += is_err(r)
        pos += used
        if not is_err(r) and pos >= len(data) and r == 0:
            break
    return calls


def skippable(payload):
    return struct.pack("<II", 0x184D2A5E, len(payload)) + payload


@pytest.mark.parametrize("checksum", [False, True])
def test_skippable_first(ref, shim, checksum):
    pieces = pieces_for(21)
    frame = streamed_frame(ref, pieces, 21, checksum)
    for stream in (skippable(bytes(range(16))), skippable(b"") + skippable(b"x" * 300) + frame, skippable(bytes(40)) + frame):
        for step in list(range(1, 20)) + [len(stream)]:
            ds = both(ref, shim)
            calls, out = feed(ds, stream, lambda k: step, lambda k: 1 << 16)
            close(ds)
            assert calls[-1][0] == 0 and out == (b"".join(pieces) if len(stream) > 300 else b"")


def test_calls_after_a_checksum_error(ref, shim):
    data = lz.datagen(6000, seed=13)
    frame = bytearray(lz.frame_compress(ref, data, lz.make_prefs(21, checksum=True)))
    frame[-1] ^= 1
    frame = bytes(frame) + lz.frame_compress(ref, data[:5000], lz.make_prefs(10))
    for step in (1, 2, 3, 4099, len(frame)):
        ds = both(ref, shim)
        calls = feed_past_errors(ds, frame, lambda k: step, lambda k: 1 << 20)
        close(ds)
        assert sum(is_err(r) for r, _, _ in calls) == 4
