"""The device-memory frame calls (LizardB200_compressFrames / LizardB200_decompressFrames, DESIGN.md 3.4a) on the CPU: the
host build of their serial code (lizard_b200/libhostshim.so, TEST-ONLY) against the compiled reference.

- XXH32 (frame_device.cuh: xxh32_serial, whose helpers the hash kernel runs) equals the reference's xxhash.c.
- The header check, block walk and verdict rules (frame_walk + frame_settle, what the index kernel and the host side of
  LizardB200_decompressFrames run), with the blocks decoded by the one-lane decoder, give what the reference's
  LizardF_decompress gives when handed the whole frame and the capacity in one call: reference-written frames, streamed frames
  with short blocks, skippable frames, and damaged ones.
- The new kernels' registers, stack and local memory, read with cuobjdump -res-usage."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import lizard_b200 as lz
from tests import refs
from tests.test_encode_resources_cpu import _cuobjdump

BS = lz.BLOCK_SIZE
SZ = ctypes.c_size_t
FE = {"GENERIC": 1, "maxBlockSize_invalid": 2, "blockMode_invalid": 3, "headerVersion_wrong": 6,
      "blockChecksum_unsupported": 7, "reservedFlag_set": 8, "dstMaxSize_tooSmall": 11, "frameType_unknown": 13,
      "frameSize_wrong": 14, "decompressionFailed": 16, "headerChecksum_invalid": 17, "contentChecksum_invalid": 18}


def err(name):
    return (1 << 64) - FE[name]


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built")
    lz.bind_frame_api(L)
    L.Lizard_XXH32.argtypes = [ctypes.c_void_p, SZ, ctypes.c_uint]
    L.Lizard_XXH32.restype = ctypes.c_uint
    return L


@pytest.fixture(scope="module")
def shim():
    p = os.path.join(refs.ROOT, "lizard_b200", "libhostshim.so")
    if not os.path.exists(p):
        pytest.skip("libhostshim.so not built")
    L = ctypes.CDLL(p)
    L.lzb_host_xxh32.argtypes = [ctypes.c_char_p, ctypes.c_ulonglong, ctypes.c_uint]
    L.lzb_host_xxh32.restype = ctypes.c_uint
    L.lzb_host_frame_decode.argtypes = [ctypes.c_char_p, ctypes.c_ulonglong, ctypes.c_void_p, ctypes.c_ulonglong,
                                        ctypes.POINTER(ctypes.c_uint)]
    L.lzb_host_frame_decode.restype = ctypes.c_ulonglong
    return L


def ref_one_call(L, frame: bytes, cap: int):
    """The reference's LizardF_decompress on a fresh context, given the whole frame and cap bytes of room in one call, read
    the way LizardB200_decompressFrames reports it: (result, bytes)."""
    ctx = ctypes.c_void_p()
    L.LizardF_createDecompressionContext(ctypes.byref(ctx), 100)
    src = ctypes.create_string_buffer(frame, max(len(frame), 1))
    # room behind the capacity: the reference does not charge a raw inner block against it (DESIGN.md 3.5)
    dst = ctypes.create_string_buffer(cap + (4 << 20) + 64)
    si, so = SZ(len(frame)), SZ(cap)
    try:
        r = L.LizardF_decompress(ctx, dst, ctypes.byref(so), src, ctypes.byref(si), None)
    finally:
        L.LizardF_freeDecompressionContext(ctx)
    if L.LizardF_isError(r):
        return r, b""
    if r == 0 and si.value == len(frame):
        return so.value, dst.raw[:so.value]
    if si.value == len(frame) or r == 0:
        return err("frameSize_wrong"), b""                  # waits for more input, or stopped in front of trailing bytes
    return err("dstMaxSize_tooSmall"), b""                  # stopped with input left: the output is full


def host_frames(shim, frame: bytes, cap: int):
    dst = ctypes.create_string_buffer(b"\xA5" * (cap + 64), cap + 64)
    nb = ctypes.c_uint()
    r = shim.lzb_host_frame_decode(frame, len(frame), dst, cap, ctypes.byref(nb))
    assert dst.raw[cap:] == b"\xA5" * 64, "wrote behind the capacity"
    ok = r < (1 << 63)
    return r, dst.raw[:r] if ok else b""


def same_verdict(want, got, decode_damage=False):
    if want == got:
        return True
    # a block that fails to decode is ERROR_GENERIC or ERROR_decompressionFailed by where it was decoded (directly into the
    # output or through the one-block buffer); with short blocks in front the reference measures that room at the compacted
    # position and this library at the max-block-spaced one (frame.inl's batches)
    both = {err("GENERIC"), err("decompressionFailed")}
    return decode_damage and want in both and got in both


def _data(n, seed, raw=True):
    a = bytearray(lz.datagen(n, 50, seed))
    if raw and n > 3 * BS:
        rng = np.random.default_rng(seed)
        a[2 * BS + 17:3 * BS + 400] = rng.integers(0, 256, BS + 383, dtype=np.uint8).tobytes()
    return bytes(a)


def _stream(L, data, prefs, pieces, flush_after=()):
    """compressBegin / compressUpdate per piece (LizardF_flush after the listed ones) / compressEnd on a library handle."""
    ctx = ctypes.c_void_p()
    L.LizardF_createCompressionContext(ctypes.byref(ctx), 100)
    out = bytearray()
    cap = L.LizardF_compressFrameBound(len(data), ctypes.byref(prefs)) * 2 + 1024
    buf = ctypes.create_string_buffer(cap)
    try:
        r = L.LizardF_compressBegin(ctx, buf, cap, ctypes.byref(prefs))
        assert not L.LizardF_isError(r)
        out += buf.raw[:r]
        at = 0
        for k, n in enumerate(pieces):
            piece = data[at:at + n]
            at += n
            r = L.LizardF_compressUpdate(ctx, buf, cap, piece, len(piece), None)
            assert not L.LizardF_isError(r)
            out += buf.raw[:r]
            if k in flush_after:
                r = L.LizardF_flush(ctx, buf, cap, None)
                assert not L.LizardF_isError(r)
                out += buf.raw[:r]
        r = L.LizardF_compressEnd(ctx, buf, cap, None)
        assert not L.LizardF_isError(r)
        out += buf.raw[:r]
    finally:
        L.LizardF_freeCompressionContext(ctx)
    return bytes(out)


def frame_of(L, data: bytes, prefs) -> bytes:
    """LizardF_compressFrame with slack behind the bound: a 1-byte input whose header carries the content size takes more than
    LizardF_compressFrameBound counts (include/lizard_b200.h), in the reference as in this library."""
    cap = L.LizardF_compressFrameBound(len(data), ctypes.byref(prefs)) + 64
    dst = ctypes.create_string_buffer(cap)
    n = L.LizardF_compressFrame(dst, cap, data, len(data), ctypes.byref(prefs))
    assert not L.LizardF_isError(n), L.LizardF_getErrorName(n)
    return dst.raw[:n]


def _fix_hc(frame: bytearray, L):
    """Rewrite the header checksum byte after a change to the descriptor."""
    fh = 15 if (frame[4] >> 3) & 1 else 7
    desc = bytes(frame[4:fh - 1])
    frame[fh - 1] = (L.Lizard_XXH32(desc, len(desc), 0) >> 8) & 0xFF
    return frame


# ---- XXH32 -------------------------------------------------------------------------------------------------------------
def test_xxh32_equals_reference(ref, shim):
    rng = np.random.default_rng(7)
    big = rng.integers(0, 256, 5 << 20, dtype=np.uint8).tobytes()
    lengths = set(range(0, 65))
    for k in range(1, 80):
        lengths.update((16 * k - 1, 16 * k, 16 * k + 1))
    lengths.update((4095, 4096, 4097, 4096 + 15, 5 << 20))
    for seed in (0, 1):
        for n in sorted(lengths):
            for start in (0, 3):                                     # the routine reads any alignment
                p = big[start:start + n]
                assert shim.lzb_host_xxh32(p, len(p), seed) == ref.Lizard_XXH32(p, len(p), seed), (seed, n, start)


# ---- header check, block walk, verdicts ----------------------------------------------------------------------------------
def _ref_frames(ref):
    """(name, frame, decoded size) written by the reference."""
    out = []
    for level in (10, 17, 21, 26, 41, 49):
        for checksum, csize in ((False, 0), (True, 1)):
            data = _data(5 * BS + 777, level)
            out.append((f"L{level}c{int(checksum)}s{csize}", frame_of(ref, data, lz.make_prefs(level, 1, True, checksum, csize)),
                        len(data)))
    for bsid in (2, 3, 4):
        data = _data(3 * BS + 5, bsid)
        out.append((f"bsid{bsid}", frame_of(ref, data, lz.make_prefs(10, bsid, True, True, 0)), len(data)))
    for n in (0, 1, 15, BS - 1, BS, BS + 1):
        data = _data(n, n, raw=False)
        out.append((f"n{n}", frame_of(ref, data, lz.make_prefs(41, 1, True, True, 1)), n))
    data = _data(6 * BS + 999, 5)
    for af in (0, 1):                                                # short blocks in the middle of the frame
        p = lz.make_prefs(21, 1, True, True, 0)
        p.autoFlush = af
        out.append((f"stream_af{af}", _stream(ref, data, p, [1000, BS, 3 * BS + 5, 7, BS + 1 + 2 * BS - 8000], {0, 2}), len(data)))
    p = lz.make_prefs(10, 3, True, False, 0)
    p.autoFlush = 1
    out.append(("stream_1mb", _stream(ref, data, p, [BS, 2 * BS + 1, 3 * BS + 998]), len(data)))
    return out


def test_reference_frames_and_capacities(ref, shim):
    for name, frame, n in _ref_frames(ref):
        for cap in sorted({n, n + 1, n + 1000, max(n - 1, 0), n // 2, 0, 3 * BS + 11}):
            want = ref_one_call(ref, frame, cap)
            got = host_frames(shim, frame, cap)
            assert got[0] == want[0], (name, cap, want[0], got[0])
            assert got[1] == want[1], (name, cap)


def test_skippable_frames(ref, shim):
    body = b"skip me" * 10
    sk = (0x184D2A53).to_bytes(4, "little") + len(body).to_bytes(4, "little") + body
    for frame in (sk, sk[:-1], sk + b"x", sk[:7], sk[:8], sk[:3]):
        for cap in (0, 100):
            want = ref_one_call(ref, frame, cap)
            assert host_frames(shim, frame, cap) == want, (len(frame), cap)


def _damaged(ref):
    """(name, frame, capacity, decode_damage) for every class of damage the walk and the verdict rules handle."""
    data = _data(4 * BS + 4321, 11)
    good = frame_of(ref, data, lz.make_prefs(41, 1, True, True, 1))
    plain = frame_of(ref, data, lz.make_prefs(10, 1, True, False, 0))
    n = len(data)
    out = []
    fh = 15
    for cut in (1, 4, 6, 7, 8, 14, 15, 16, 18, 19, 20, 100, len(good) // 2, len(good) - 9, len(good) - 8, len(good) - 5,
                len(good) - 4, len(good) - 1):
        out.append((f"truncated{cut}", good[:cut], n, False))
    out.append(("trailing", good + b"\0", n, False))
    out.append(("trailing_frame", good + good, n, False))
    out.append(("plain_trailing", plain + b"abc", n, False))
    f = bytearray(good); f[0] ^= 1; out.append(("magic", bytes(f), n, False))
    f = bytearray(good); f[4] ^= 0x80; out.append(("version", bytes(_fix_hc(f, ref)), n, False))
    f = bytearray(good); f[4] |= 0x10; out.append(("block_checksum", bytes(_fix_hc(f, ref)), n, False))
    f = bytearray(good); f[4] |= 0x01; out.append(("reserved_flg", bytes(_fix_hc(f, ref)), n, False))
    f = bytearray(good); f[5] |= 0x80; out.append(("reserved_bd7", bytes(_fix_hc(f, ref)), n, False))
    f = bytearray(good); f[5] |= 0x01; out.append(("reserved_bd", bytes(_fix_hc(f, ref)), n, False))
    f = bytearray(good); f[5] &= 0x0F; out.append(("bsid0", bytes(_fix_hc(f, ref)), n, False))
    f = bytearray(good); f[fh - 1] ^= 0x55; out.append(("header_checksum", bytes(f), n, False))
    f = bytearray(good); f[4] &= ~0x20; out.append(("linked", bytes(_fix_hc(f, ref)), n, False))
    f = bytearray(good); f[6] ^= 1; out.append(("content_size", bytes(_fix_hc(f, ref)), n, False))
    f = bytearray(good); f[-1] ^= 1; out.append(("content_checksum", bytes(f), n, False))
    f = bytearray(good); f[fh:fh + 4] = (BS + 1).to_bytes(4, "little"); out.append(("block_too_big", bytes(f), n, False))
    first = int.from_bytes(good[fh:fh + 4], "little") & 0x7FFFFFFF
    f = bytearray(good); f[fh + 4 + first // 2] ^= 0xFF; out.append(("payload", bytes(f), n, True))
    f = bytearray(good); f[fh + 4] ^= 0xFF; out.append(("payload_level", bytes(f), n, True))
    f = bytearray(good); f[fh:fh + 4] = (first - 1).to_bytes(4, "little"); out.append(("block_size_word", bytes(f), n, True))
    for cap in (0, 1, BS - 1, BS, BS + 1, n - 1):
        out.append((f"cap{cap}", good, cap, False))
        out.append((f"cap{cap}_payload", bytes(_payload_damage(good, fh)), cap, True))
    out += _block_size_damage(ref)
    return out


MAX_BLOCK = {1: 128 << 10, 2: 256 << 10, 3: 1 << 20, 4: 4 << 20, 5: 16 << 20, 6: 64 << 20, 7: 256 << 20}   # lib/lizard_frame.c:194


def _header(ref, bsid):
    """A 7-byte frame header: independent blocks, no checksum, no content size."""
    f = bytearray((0x184D2206).to_bytes(4, "little") + bytes([0x60, bsid << 4, 0]))
    return bytes(_fix_hc(f, ref))


def _block_size_damage(ref):
    """Block size IDs 2-7: block words just above the frame's maximum block size (raw and compressed; the check comes before
    the payload is read), a raw block of exactly the maximum, and compressed blocks that decode past the maximum."""
    out = []
    for bsid in range(2, 8):
        mb = MAX_BLOCK[bsid]
        h = _header(ref, bsid)
        for raw in (0, 1):
            word = (mb + 1) | (raw << 31)
            out.append((f"bsid{bsid}_above_max_raw{raw}", h + word.to_bytes(4, "little") + bytes(100), 2 * mb, False))
        if bsid <= 3:
            body = _data(mb, bsid, raw=False)
            out.append((f"bsid{bsid}_raw_max", h + (mb | 1 << 31).to_bytes(4, "little") + body + bytes(4), mb, False))
        if bsid <= 4:
            data = _data(mb + 1000, bsid, raw=False)
            comp = refs.ref_compress(ref, data, 10)
            frame = h + len(comp).to_bytes(4, "little") + comp + bytes(4)
            for cap in (mb + 1000, mb - 1):                          # decoded in place / through the one-block buffer
                out.append((f"bsid{bsid}_decodes_past_max_cap{cap}", frame, cap, True))
    return out


def _payload_damage(good, fh):
    f = bytearray(good)
    first = int.from_bytes(good[fh:fh + 4], "little") & 0x7FFFFFFF
    at = fh + 4 + first + 4                                          # inside the second block
    f[at + 30] ^= 0xFF
    return f


def test_damaged_frames(ref, shim):
    for name, frame, cap, dd in _damaged(ref):
        # linked blocks are out of scope here: this library's LizardF_decompress refuses them, the reference decodes them
        want = (err("blockMode_invalid"), b"") if name == "linked" else ref_one_call(ref, frame, cap)
        got = host_frames(shim, frame, cap)
        assert same_verdict(want[0], got[0], dd), (name, cap, want[0], got[0])
        if want[0] < (1 << 63):
            assert got[1] == want[1], name


# ---- resource figures of the new kernels --------------------------------------------------------------------------------
FRAME_KERNELS = {"lizard_frame_index_kernel", "lizard_frame_hash_kernel", "lizard_frame_scan_kernel",
                 "lizard_frame_assemble_kernel"}


def _frame_kernel_resources():
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
            for k in FRAME_KERNELS:
                if re.search(r"\d" + k + r"[A-Z]", name) or name == k:
                    found[k] = {a: int(b) for a, b in re.findall(r"(REG|STACK|LOCAL|SHARED):(\d+)", line)}
            name = None
    return found


# DESIGN.md 3.4a lists these figures
FRAME_KERNEL_LIMITS = {
    "lizard_frame_index_kernel": (32, 0),
    "lizard_frame_hash_kernel": (78, 0),       # the next 4 KiB piece in flight: 9 16-byte words per lane
    "lizard_frame_scan_kernel": (32, 0),
    "lizard_frame_assemble_kernel": (40, 0),
}


def test_frame_kernel_resources():
    found = _frame_kernel_resources()
    assert set(found) == FRAME_KERNELS, found
    for k, (reg, stack) in FRAME_KERNEL_LIMITS.items():
        r = found[k]
        assert r["REG"] <= reg and r["STACK"] <= stack and r["LOCAL"] == 0, (k, r)
