"""LizardF frames in device memory on the GPU: LizardB200_compressFrames / LizardB200_decompressFrames (DESIGN.md 3.4a).

Compress: every frame equals this library's LizardF_compressFrame on host copies (and the pure reference's frame), byte for
byte and in its return value, at every GPU level; block size IDs 1-7, checksum and content size on and off; inputs of 0, 1
and 15 bytes, block size +- 1, several blocks and incompressible ones, mixed in one call at unaligned offsets with guard
bytes; refused levels, linked mode and a capacity one byte short handled like the host call, writing nothing.

Decompress: every result equals this library's LizardF_decompress on a fresh context handed the whole frame and the capacity
in one call (test_frame_device_cpu.ref_one_call), on reference frames at levels 10-49, streamed frames with short blocks,
skippable frames and every class of damage mixed with good frames; good frames' bytes intact, nothing written outside any
frame's range.  Also: a 5000-frame call, two streams, the launch count, and one 1 GiB frame."""
import ctypes

import numpy as np
import pytest

import lizard_b200 as lz
from tests import refs
from tests.corpus import ENCODE_LEVELS, LP_ENCODE_LEVELS
from tests.test_frame_device_cpu import _damaged, _data, _ref_frames, _stream, frame_of, ref_one_call

pytestmark = pytest.mark.gpu
BS = lz.BLOCK_SIZE
GPU_LEVELS = sorted(ENCODE_LEVELS + LP_ENCODE_LEVELS + [18, 19, 39])
GUARD = 0x5C
ERROR_LIMIT = (1 << 64) - 20


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built")
    lz.bind_frame_api(L)
    L.Lizard_XXH32.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint]
    L.Lizard_XXH32.restype = ctypes.c_uint
    return L


@pytest.fixture(scope="module")
def ours():
    return lz.bind_frame_api(lz.lib())


def _torch():
    import torch
    return torch


class Arena:
    """Buffers back to back in one device allocation, each at its own residue mod 16 behind guard bytes."""

    def __init__(self, seed=0):
        self.h = bytearray()
        self.off = []
        self.rng = np.random.default_rng(seed)

    def put(self, body: bytes):
        pad = 16 + int(self.rng.integers(0, 16))
        self.h += bytes([GUARD]) * pad
        self.off.append(len(self.h))
        self.h += body
        return self

    def device(self):
        torch = _torch()
        self.h += bytes([GUARD]) * 64
        return torch.frombuffer(bytearray(self.h), dtype=torch.uint8).to("cuda:0")


def out_arena(caps, seed=1):
    a = Arena(seed)
    for c in caps:
        a.put(bytes([GUARD]) * c)
    return a


def run_compress(units, caps, prefs, stream=0):
    src = Arena(7)
    for u in units:
        src.put(u)
    d_src = src.device()
    dst = out_arena(caps)
    d_dst = dst.device()
    res = lz.compress_frames(d_src.data_ptr(), src.off, [len(u) for u in units], d_dst.data_ptr(), dst.off, caps, prefs, stream)
    return res, bytes(d_dst.cpu().numpy().tobytes()), dst.off


def run_decompress(frames, caps, stream=0):
    src = Arena(9)
    for f in frames:
        src.put(f)
    d_src = src.device()
    dst = out_arena(caps, 3)
    d_dst = dst.device()
    res = lz.decompress_frames(d_src.data_ptr(), src.off, [len(f) for f in frames], d_dst.data_ptr(), dst.off, caps, stream)
    return res, bytes(d_dst.cpu().numpy().tobytes()), dst.off


def expect(cond, *what):
    """assert without pytest's rewriting: the operands are buffers of up to hundreds of MiB"""
    if not cond:
        raise AssertionError(repr(what)[:2000])


def first_diff(a: bytes, b: bytes):
    if len(a) != len(b):
        return ("sizes", len(a), len(b))
    x, y = np.frombuffer(a, dtype=np.uint8), np.frombuffer(b, dtype=np.uint8)
    d = np.nonzero(x != y)[0]
    return ("first difference at", int(d[0])) if d.size else None


def host_compress(L, data, prefs, cap):
    # slack behind the capacity: the host call writes a 1-byte input's frame past it in one case (include/lizard_b200.h)
    dst = ctypes.create_string_buffer(cap + 64)
    r = L.LizardF_compressFrame(dst, cap, data, len(data), ctypes.byref(prefs))
    return r, (dst.raw[:r] if not L.LizardF_isError(r) else b"")


def check_guards(out, off, caps, sizes):
    """Nothing written outside [off, off + cap), and nothing behind the written size."""
    mask = np.zeros(len(out), dtype=bool)
    for o, s in zip(off, sizes):
        mask[o:o + s] = True
    arr = np.frombuffer(out, dtype=np.uint8)
    bad = np.nonzero((arr != GUARD) & ~mask)[0]
    assert bad.size == 0, f"bytes written outside the frames' results at {bad[:8]}"


def _inputs(seed):
    rng = np.random.default_rng(seed)
    noise = rng.integers(0, 256, BS + 100, dtype=np.uint8).tobytes()
    return [b"", b"x", lz.datagen(15, 50, seed), lz.datagen(BS - 1, 50, seed + 1), lz.datagen(BS, 50, seed + 2),
            lz.datagen(BS + 1, 50, seed + 3), _data(4 * BS + 555, seed + 4), noise, lz.datagen(5000, 0, seed)]


# ---- compress -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level", GPU_LEVELS)
def test_compress_equals_host_and_reference(ref, ours, level):
    units = _inputs(level)
    for checksum, csize in ((True, 1), (False, 0)):
        p = lz.make_prefs(level, 1, True, checksum, csize)
        caps = [ours.LizardF_compressFrameBound(len(u), ctypes.byref(p)) + 7 for u in units]
        res, out, off = run_compress(units, caps, p)
        sizes = []
        for u, r, o, c in zip(units, res, off, caps):
            want_r, want = host_compress(ours, u, p, c)
            expect(r == want_r, level, len(u), r, want_r)
            expect(out[o:o + r] == want, level, len(u), first_diff(out[o:o + r], want))
            expect(want == host_compress(ref, u, p, c)[1], "reference", level, len(u))
            sizes.append(r)
        check_guards(out, off, caps, sizes)


@pytest.mark.parametrize("bsid", [1, 2, 3, 4, 5, 6, 7])
def test_compress_block_sizes(ours, bsid):
    units = [lz.datagen(n, 50, n) for n in (0, 1, 15, 200 << 10, (1 << 20) + 3, (4 << 20) + 1)]
    if bsid >= 5:
        units.append(_data((17 << 20) + 99, bsid))
    if bsid >= 6:
        units.append(lz.datagen((65 << 20) + 5, 50, 6))              # blocks of 64 MiB / one block of 256 MiB
    for checksum in (False, True):
        for csize in (0, 1):
            p = lz.make_prefs(10, bsid, True, checksum, csize)
            caps = [ours.LizardF_compressFrameBound(len(u), ctypes.byref(p)) for u in units]
            res, out, off = run_compress(units, caps, p)
            for u, r, o, c in zip(units, res, off, caps):
                want_r, want = host_compress(ours, u, p, c)
                if not ours.LizardF_isError(want_r) and want_r > c:
                    # the host call wrote past its capacity (a 1-byte input with the content size, include/lizard_b200.h)
                    expect(len(u) == 1 and csize and lz.frame_error(r) == "ERROR_dstMaxSize_tooSmall", bsid, len(u), r, want_r, c)
                    continue
                expect(r == want_r, bsid, checksum, csize, len(u), r, want_r, lz.frame_error(r), lz.frame_error(want_r))
                expect(ours.LizardF_isError(r) or out[o:o + r] == want, bsid, checksum, csize, len(u), first_diff(out[o:o + r], want))
            check_guards(out, off, caps, [0 if ours.LizardF_isError(r) else r for r in res])


def test_compress_errors_like_the_host_call(ours):
    units = _inputs(3)
    p = lz.make_prefs(10, 1, True, True, 1)
    bound = [ours.LizardF_compressFrameBound(len(u), ctypes.byref(p)) for u in units]
    caps = [b - 1 if i % 2 else b for i, b in enumerate(bound)]    # every other frame one byte short
    res, out, off = run_compress(units, caps, p)
    sizes = []
    for u, r, o, c in zip(units, res, off, caps):
        want_r, want = host_compress(ours, u, p, c)
        expect(r == want_r and (ours.LizardF_isError(r) or out[o:o + r] == want), len(u), r, want_r)
        sizes.append(0 if ours.LizardF_isError(r) else r)
    assert any(ours.LizardF_isError(r) for r in res) and not all(ours.LizardF_isError(r) for r in res)
    check_guards(out, off, caps, sizes)
    for level in (12, 26, 33, 49):                                   # refused levels
        p = lz.make_prefs(level, 1, True, False, 0)
        caps = [ours.LizardF_compressFrameBound(len(u), ctypes.byref(p)) for u in units]
        res, out, off = run_compress(units, caps, p)
        assert res == [host_compress(ours, u, p, c)[0] for u, c in zip(units, caps)], level
        assert all(lz.frame_error(r) == "ERROR_compressionLevel_invalid" for r in res), level
        check_guards(out, off, caps, [0] * len(units))
    p = lz.make_prefs(10, 1, False, False, 0)                        # linked: refused for inputs of more than one block
    caps = [ours.LizardF_compressFrameBound(len(u), ctypes.byref(p)) for u in units]
    res, out, off = run_compress(units, caps, p)
    sizes = []
    for u, r, o, c in zip(units, res, off, caps):
        want_r, want = host_compress(ours, u, p, c)
        expect(r == want_r and (ours.LizardF_isError(r) or out[o:o + r] == want), len(u), r, want_r)
        sizes.append(0 if ours.LizardF_isError(r) else r)
    assert lz.frame_error(res[-3]) == "ERROR_blockMode_invalid"
    check_guards(out, off, caps, sizes)


# ---- decompress -----------------------------------------------------------------------------------------------------------
def _check_decode(ours, frames, caps, names):
    res, out, off = run_decompress(frames, caps)
    sizes = []
    for name, f, c, r, o in zip(names, frames, caps, res, off):
        want_r, want = ref_one_call(ours, f, c)
        expect(r == want_r, name, c, r, want_r, lz.frame_error(r), lz.frame_error(want_r))
        if r < ERROR_LIMIT:
            expect(out[o:o + r] == want, name, first_diff(out[o:o + r], want))
            sizes.append(r)
        else:
            sizes.append(c)                                          # unspecified bytes inside the frame's own range
    check_guards(out, off, caps, sizes)
    return res


def test_decompress_reference_frames_all_levels(ref, ours):
    frames, caps, names = [], [], []
    sk = (0x184D2A5F).to_bytes(4, "little") + (9).to_bytes(4, "little") + b"123456789"
    for level in range(10, 50):
        data = _data(3 * BS + 1000 + level, level)
        for checksum, csize in ((True, 1), (False, 0)):
            f = frame_of(ref, data, lz.make_prefs(level, 1, True, checksum, csize))
            frames.append(f); caps.append(len(data)); names.append(f"L{level}c{int(checksum)}")
        frames.append(sk); caps.append(16); names.append("skippable")
    for name, f, n in _ref_frames(ref):
        frames.append(f); caps.append(n); names.append(name)
        frames.append(f); caps.append(n + 4096); names.append(name + "+room")
    res = _check_decode(ours, frames, caps, names)
    failed = [(nm, lz.frame_error(r)) for nm, r in zip(names, res) if r >= ERROR_LIMIT]
    assert not failed, failed


def test_decompress_short_blocks(ref, ours):
    data = _data(9 * BS + 4321, 21)
    frames, caps, names = [], [], []
    for af in (0, 1):
        for level in (10, 21, 41, 45):
            p = lz.make_prefs(level, 1, True, bool(af), len(data) if af else 0)
            p.autoFlush = af
            f = _stream(ref, data, p, [1, BS - 1, 3, 2 * BS + 7, 500, 3 * BS, len(data) - 5 * BS - 511], {0, 2, 4})
            for c in (len(data), len(data) + 1, len(data) - 1, len(data) + BS, 2 * BS):
                frames.append(f); caps.append(c); names.append(f"af{af}L{level}cap{c}")
    _check_decode(ours, frames, caps, names)


def test_decompress_damage_mixed_with_good_frames(ref, ours):
    good_data = _data(3 * BS + 17, 4)
    good = frame_of(ref, good_data, lz.make_prefs(41, 1, True, True, 1))
    frames, caps, names = [], [], []
    for name, f, c, _ in _damaged(ref):
        frames += [good, f]; caps += [len(good_data), c]; names += ["good", name]
    res = _check_decode(ours, frames, caps, names)
    assert all(r == len(good_data) for r in res[0::2])
    assert sum(r >= ERROR_LIMIT for r in res[1::2]) > 30


def test_frames_of_many_tiny_blocks(ref, ours):
    """Frames whose compressed blocks are far smaller than their maximum block size (autoFlush with small updates) reserve a
    staging slot of that maximum per block: 40 blocks of a 256 MiB frame need 10 GiB, more than the arena, so the call runs
    several decode rounds.  Every frame, and the good frames around them, still gets LizardF_decompress's result."""
    good_data = _data(3 * BS + 17, 4)
    good = frame_of(ref, good_data, lz.make_prefs(21, 1, True, True, 1))
    frames, caps, names = [], [], []
    for bsid, pieces, level in ((7, 40, 10), (7, 33, 41), (1, 3000, 10)):
        data = lz.datagen(2000 * pieces, 90, bsid + pieces)           # 2000-byte updates compress to blocks of ~700 bytes
        p = lz.make_prefs(level, bsid, True, True, len(data))
        p.autoFlush = 1
        f = _stream(ref, data, p, [2000] * pieces)
        frames += [good, f]; caps += [len(good_data), len(data)]; names += ["good", f"tiny{bsid}x{pieces}"]
    bad, pos = bytearray(frames[1]), 15
    for _ in range(19):                                               # damage in the 20th block of the first one
        pos += 4 + (int.from_bytes(bad[pos:pos + 4], "little") & 0x7FFFFFFF)
    assert not bad[pos + 3] & 0x80
    bad[pos + 4 + 40] ^= 0xFF
    frames += [bytes(bad), good]; caps += [caps[1], len(good_data)]; names += ["tiny_damaged", "good"]
    res = _check_decode(ours, frames, caps, names)
    assert res[1] == caps[1] and res[3] == caps[3] and res[5] == caps[5]


def test_five_thousand_frames(ours):
    rng = np.random.default_rng(5)
    sizes = [int(x) for x in rng.integers(0, 40000, 5000)]
    units = [lz.datagen(n, 50, i)[:n] for i, n in enumerate(sizes)]
    p = lz.make_prefs(10, 1, True, True, 1)
    caps = [ours.LizardF_compressFrameBound(n, ctypes.byref(p)) for n in sizes]
    res, out, off = run_compress(units, caps, p)
    frames = [out[o:o + r] for o, r in zip(off, res)]
    for k in range(0, 5000, 97):
        expect(frames[k] == host_compress(ours, units[k], p, caps[k])[1], k)
    res, out, off = run_decompress(frames, sizes)
    for k, (u, r, o) in enumerate(zip(units, res, off)):
        expect(r == len(u) and out[o:o + r] == u, k, r, len(u))


def test_two_streams_share_the_workspace(ours):
    torch = _torch()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    a = [_data(2 * BS + i * 1000, i) for i in range(20)]
    b = [lz.datagen(BS // 2 + i, 50, 100 + i) for i in range(30)]
    pa, pb = lz.make_prefs(41, 1, True, True, 0), lz.make_prefs(17, 1, True, False, 1)
    for _ in range(2):
        for units, p, s in ((a, pa, s1), (b, pb, s2)):
            caps = [ours.LizardF_compressFrameBound(len(u), ctypes.byref(p)) for u in units]
            res, out, off = run_compress(units, caps, p, s.cuda_stream)
            frames = [out[o:o + r] for o, r in zip(off, res)]
            expect(frames == [host_compress(ours, u, p, c)[1] for u, c in zip(units, caps)], "compress", p.compressionLevel)
            res, out, off = run_decompress(frames, [len(u) for u in units], s.cuda_stream)
            expect([out[o:o + r] for o, r in zip(off, res)] == units, "decompress", res)


def test_launches_do_not_grow_with_frames(ours):
    p = lz.make_prefs(10, 1, True, True, 1)
    counts = []
    for n in (40, 400):                                               # both above the decoder's pre-pass threshold (32 units)
        units = [lz.datagen(BS + 77, 50, i) for i in range(n)]
        caps = [ours.LizardF_compressFrameBound(len(u), ctypes.byref(p)) for u in units]
        before = ours.LizardB200_launchCount()
        res, out, off = run_compress(units, caps, p)
        mid = ours.LizardB200_launchCount()
        frames = [out[o:o + r] for o, r in zip(off, res)]
        res, _, _ = run_decompress(frames, [len(u) for u in units])
        after = ours.LizardB200_launchCount()
        assert all(r == BS + 77 for r in res)
        counts.append((mid - before, after - mid))
    assert counts[0] == counts[1], counts


def test_one_gib_frame_round_trip(ours):
    torch = _torch()
    n = 1 << 30
    host = torch.empty(n, dtype=torch.uint8).pin_memory()
    lz.datagen_into(host.data_ptr(), n, 50, 0)
    p = lz.make_prefs(10, 1, True, True, 0)
    cap = ours.LizardF_compressFrameBound(n, ctypes.byref(p))
    want = torch.empty(cap, dtype=torch.uint8)
    wr = ours.LizardF_compressFrame(want.data_ptr(), cap, host.data_ptr(), n, ctypes.byref(p))
    assert not ours.LizardF_isError(wr)
    d_src = host.to("cuda:0")
    d_frame = torch.empty(cap, dtype=torch.uint8, device="cuda:0")
    r = lz.compress_frames(d_src.data_ptr(), [0], [n], d_frame.data_ptr(), [0], [cap], p)
    assert r == [wr]
    expect(torch.equal(d_frame[:wr].cpu(), want[:wr]), "1 GiB frame differs from the host path's")
    d_back = torch.empty(n, dtype=torch.uint8, device="cuda:0")
    r = lz.decompress_frames(d_frame.data_ptr(), [0], [wr], d_back.data_ptr(), [0], [n])
    assert r == [n]
    expect(torch.equal(d_back, d_src), "1 GiB round trip")
