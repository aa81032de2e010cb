"""GPU parity of the frame pipeline across several pipeline chunks: LizardF_compressFrame at every GPU level and block size,
streaming compression call by call, LizardF_decompress at every level 10-49 on both decoder generations (variants 7 and
23) under fixed feeding schedules, reference frames with short blocks, skippable frames and concatenations, damaged
frames, and LizardB200_gather_device.  The reference built with -DLIZARD_RESET_MEM (bound with lz.bind_frame_api) is the
yardstick: frame bytes, LizardF return values, bytes consumed and produced per call, error names.

The pipeline chunk (LIZARDB200_FRAME_CHUNK_MIB) is read once per process, so the multi-chunk groups run in a child process
(`python -m tests.test_gpu_frame_pipeline <group> <payload>`); the parent builds the inputs and the reference frames
(cached per level) and hands them over in a pickle.  At 1 MiB chunks a call of 128 KiB blocks has 8 units per chunk and no
decoder ramp (8 % 16 != 0); at 2 MiB chunks it has 16 and, from 32 units on, the ramp of 1 / 2 / 4 / 8 units.  Every group
asserts how many chunks its calls span (LizardB200_chunkPlan), so an input that shrinks below that fails loudly."""
import contextlib
import ctypes
import functools
import itertools
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

import lizard_b200 as lz
from tests import corpus, refs
from tests.test_gpu_corpus import HAS_SMEM_TABLE, SHAPES

pytestmark = pytest.mark.gpu
BS = lz.BLOCK_SIZE
MIB = 1 << 20
RAW = 0x80000000
DEFAULT_VARIANT = 7                      # api.cu Context::dec_variant: first generation behind the Huffman pre-pass
VARIANTS = (7, 23)                       # 23 = bit 16: the second-generation kernel (lizard_decode2_units_kernel)
GPU_LEVELS = corpus.ENCODE_LEVELS + corpus.LP_ENCODE_LEVELS + [18, 19, 39]
UNITS_KERNEL_LEVELS = (10, 20, 17, 41)   # <Fast>, <FastBig>, <Generic> (hashChain), the LIZv1 fast parser behind Huffman
KERNEL_LEVELS = UNITS_KERNEL_LEVELS + (24, 19)                         # + lowestPrice, optimal
UNSUPPORTED_LEVELS = (12, 26, 27, 28, 29, 32, 33, 46, 47, 48, 49)
CODEWORD_LEVELS = (10, 21, 41, 45)       # fastLZ4, LIZv1, LIZv1 + Huffman, lowestPrice LIZv1 + Huffman


# ---------------------------------------------------------------------------------------------------------------------
# inputs and reference frames (parent side)
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _ref():
    L = refs.ref_parity()
    return None if L is None else lz.bind_frame_api(L)


@functools.lru_cache(maxsize=None)
def _input(name):
    """big: 25 units of 128 KiB at 1 MiB chunks = 4 chunks [0-7] [8-15] [16-23] [24]: datagen and corpus units, then
    incompressible blocks 7-15 (raw records on both sides of the first chunk boundary, chunk 1 raw only), datagen again,
    and a last block of exactly 1 byte alone in the last chunk (a 6-byte record).  small: 6 units, below the 1 MiB of kHashThreadMin.
    ramp: 41 units (40 blocks + 777 bytes) for the decoder's ramp at 2 MiB chunks.  bs<id>: three blocks of that
    blockSizeID (nine of 256 KiB) and a short last one."""
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "big":
        fams = corpus.corpus()
        pool = b"".join(u for units in fams.values() for u in units)
        out = (lz.datagen(3 * BS, 50, 31) + pool[12345:12345 + 4 * BS] + rng.integers(0, 256, 9 * BS, dtype=np.uint8).tobytes()
               + lz.datagen(8 * BS, 40, 32) + b"\xa7")
        assert len(out) == 24 * BS + 1
        return out
    if name == "small":
        return lz.datagen(5 * BS + 4321, 50, 77)
    if name == "ramp":
        a = bytearray(lz.datagen(40 * BS + 777, 50, 78))
        a[20 * BS + 99:21 * BS + 5000] = rng.integers(0, 256, BS + 4901, dtype=np.uint8).tobytes()
        return bytes(a)
    if name == "stream":
        a = bytearray(lz.datagen(7 * BS + 2 * MIB + 3 * BS + 64, 50, 79))
        a[5 * BS:6 * BS + 3000] = rng.integers(0, 256, BS + 3000, dtype=np.uint8).tobytes()
        return bytes(a)
    if name.startswith("bs"):
        size = _block_bytes(int(name[2:]))
        k = 9 if size == 256 << 10 else 3
        return lz.datagen(k * size + size // 3 + 5, 50, 80 + int(name[2:]))
    raise KeyError(name)


def _block_bytes(bsid):
    return {1: BS, 2: 256 << 10, 3: MIB, 4: 4 * MIB, 5: 16 * MIB}[bsid]


@functools.lru_cache(maxsize=None)
def _ref_frame(name, level, bsid, checksum, csize):
    return lz.frame_compress(_ref(), _input(name), lz.make_prefs(level, bsid, True, checksum, csize))


def _records(frame):
    """(header size, [(record position, payload size, raw)], end mark position) of a frame (stops at a damaged record)."""
    fh = 15 if frame[4] & 8 else 7
    pos, recs = fh, []
    while pos + 4 <= len(frame):
        w = int.from_bytes(frame[pos:pos + 4], "little")
        if w == 0:
            break
        recs.append((pos, w & 0x7FFFFFFF, bool(w & RAW)))
        pos += 4 + (w & 0x7FFFFFFF)
    return fh, recs, pos


def _ref_begin(prefs):
    """The frame header the reference writes for these preferences."""
    L = _ref()
    ctx = ctypes.c_void_p()
    assert L.LizardF_createCompressionContext(ctypes.byref(ctx), 100) == 0
    buf = ctypes.create_string_buffer(64)
    n = L.LizardF_compressBegin(ctx, buf, 64, ctypes.byref(prefs))
    L.LizardF_freeCompressionContext(ctx)
    assert not L.LizardF_isError(n)
    return buf.raw[:n]


def _skippable(magic_low, payload):
    return (0x184D2A50 + magic_low).to_bytes(4, "little") + len(payload).to_bytes(4, "little") + payload


def _ref_stream_frame(data, level, bsid, cuts):
    """A reference frame written with LizardF_compressUpdate pieces and a LizardF_flush after each: short blocks inside."""
    L = _ref()
    p = lz.make_prefs(level, bsid, True, True, 0)
    ctx = ctypes.c_void_p()
    assert L.LizardF_createCompressionContext(ctypes.byref(ctx), 100) == 0
    buf = ctypes.create_string_buffer(L.LizardF_compressBound(len(data), ctypes.byref(p)) + 64)
    n = L.LizardF_compressBegin(ctx, buf, len(buf), ctypes.byref(p))
    out = bytearray(buf.raw[:n])
    pos = 0
    for n in cuts + [len(data) - sum(cuts)]:
        for fn, args in ((L.LizardF_compressUpdate, (data[pos:pos + n], n, None)), (L.LizardF_flush, (None,))):
            r = fn(ctx, buf, len(buf), *args)
            assert not L.LizardF_isError(r), L.LizardF_getErrorName(r)
            out += buf.raw[:r]
        pos += n
    r = L.LizardF_compressEnd(ctx, buf, len(buf), None)
    assert not L.LizardF_isError(r)
    out += buf.raw[:r]
    L.LizardF_freeCompressionContext(ctx)
    return bytes(out)


def _damaged(level):
    """The big frame at `level` damaged one way each: name -> bytes."""
    f = _ref_frame("big", level, 1, True, 1)
    fh, recs, end = _records(f)
    assert len(recs) == 25 and end == len(f) - 8
    rnd = np.random.default_rng(level)

    def word(i, w):
        b = bytearray(f)
        b[recs[i][0]:recs[i][0] + 4] = (w & 0xFFFFFFFF).to_bytes(4, "little")
        return bytes(b)

    def payload(i, at, data):
        b = bytearray(f)
        p = recs[i][0] + 4 + at
        b[p:p + len(data)] = data
        return bytes(b)

    def flip(i, frac, bit):
        p, n, _ = recs[i]
        at = int(n * frac)
        return payload(i, at, bytes([f[p + 4 + at] ^ (1 << bit)]))

    n = len(_input("big"))
    out = {
        "flip-early": flip(1, 0.5, 4), "flip-head": flip(2, 0.0, 0), "flip-late": flip(17, 0.7, 7),
        "random-bytes": payload(3, recs[3][1] // 3, rnd.integers(0, 256, 16, dtype=np.uint8).tobytes()),
        "random-tail": payload(20, recs[20][1] - 9, rnd.integers(0, 256, 9, dtype=np.uint8).tobytes()),
        "size-above-max": word(2, BS + 1), "raw-size-above-max": word(9, RAW | (BS + 1)),
        "raw-flag-on": word(4, RAW | recs[4][1]), "raw-flag-off": word(8, recs[8][1]),
        "zero-size-early": word(1, 0),
        "cut-in-block": f[:recs[5][0] + 4 + recs[5][1] // 2], "cut-in-size-word": f[:recs[6][0] + 2],
        "cut-in-raw-block": f[:recs[10][0] + 4 + 1000], "cut-in-suffix": f[:-2], "cut-before-end-mark": f[:end],
        "content-checksum": f[:-1] + bytes([f[-1] ^ 1]),
    }
    for name, cs in (("content-size+1", n + 1), ("content-size-1", n - 1)):
        hdr = _ref_begin(lz.make_prefs(level, 1, True, True, cs))
        assert len(hdr) == fh
        out[name] = hdr + f[fh:]
    return out


# ---------------------------------------------------------------------------------------------------------------------
# drivers (used on both libraries)
# ---------------------------------------------------------------------------------------------------------------------
def _ret(L, r):
    """A LizardF return value as the number, or the error's name."""
    if L.LizardF_isError(r):
        return L.LizardF_getErrorName(r).decode()
    return r


def _schedule(spec):
    """Piece sizes: spec None = everything left each call; else (prefix, cycle) of piece sizes."""
    if spec is None:
        return None
    prefix, cycle = spec
    return itertools.chain(prefix, itertools.cycle(cycle))


def decode_calls(L, stream, out_cap, src_spec=None, dst_spec=None, info_at=(), max_calls=400000):
    """Feed `stream` to one LizardF_decompress context piece by piece.  Returns ([(return or error name, consumed,
    produced), ...], bytes produced).  Stops after an error, at the end of the input once a frame is complete, or after two
    calls without progress.  `info_at`: input positions at which LizardF_getFrameInfo is called first (logged as
    ("info", return, consumed, frame info fields))."""
    ctx = ctypes.c_void_p()
    assert L.LizardF_createDecompressionContext(ctypes.byref(ctx), 100) == 0
    out = ctypes.create_string_buffer(out_cap + 2 * BS + 64)     # slack: the caller never offers it
    src = ctypes.create_string_buffer(bytes(stream), max(len(stream), 1))
    si_it, so_it = _schedule(src_spec), _schedule(dst_spec)
    log, ip, op, idle = [], 0, 0, 0
    info_at = list(info_at)
    try:
        while len(log) < max_calls:
            if info_at and ip == info_at[0]:
                info_at.pop(0)
                fi = lz.FrameInfo()
                sz = ctypes.c_size_t(len(stream) - ip)
                r = L.LizardF_getFrameInfo(ctx, ctypes.byref(fi), ctypes.byref(src, ip), ctypes.byref(sz))
                log.append(("info", _ret(L, r), sz.value, fi.blockSizeID, fi.blockMode, fi.contentChecksumFlag,
                            fi.frameType, fi.contentSize))
                if L.LizardF_isError(r):
                    break
                ip += sz.value
                continue
            n_in = len(stream) - ip if si_it is None else min(next(si_it), len(stream) - ip)
            n_out = out_cap - op if so_it is None else min(next(so_it), out_cap - op)
            si, so = ctypes.c_size_t(n_in), ctypes.c_size_t(n_out)
            r = L.LizardF_decompress(ctx, ctypes.byref(out, op), ctypes.byref(so), ctypes.byref(src, ip), ctypes.byref(si), None)
            log.append((_ret(L, r), si.value, so.value))
            if L.LizardF_isError(r):
                break
            ip += si.value
            op += so.value
            if r == 0 and ip >= len(stream):
                break
            idle = idle + 1 if si.value == 0 and so.value == 0 else 0
            if idle >= 2:
                break
    finally:
        L.LizardF_freeDecompressionContext(ctx)
    return log, out.raw[:op]


def _first_diff(a, b):
    for i, (x, y) in enumerate(zip(a, b)):
        if x != y:
            return i, x, y
    return min(len(a), len(b)), a[len(b):][:2], b[len(a):][:2]


def assert_same_calls(ours, want, what, bytes_defined=True):
    (olog, oout), (rlog, rout) = ours, want
    assert olog == rlog, (what, "calls", len(olog), len(rlog), _first_diff(olog, rlog))
    assert oout == rout or not bytes_defined, (what, "bytes", len(oout), len(rout), _first_diff(oout, rout)[0])


@contextlib.contextmanager
def decode_variant(variant):
    L = lz.lib()
    L.LizardB200_setDecodeVariant.argtypes = [ctypes.c_int]
    assert L.LizardB200_setDecodeVariant(variant) == 0
    try:
        yield
    finally:
        L.LizardB200_setDecodeVariant(DEFAULT_VARIANT)


@contextlib.contextmanager
def enc_shape(value):
    old = os.environ.pop("LIZARDB200_ENC_SHAPE", None)
    if value is not None:
        os.environ["LIZARDB200_ENC_SHAPE"] = value
    try:
        yield
    finally:
        os.environ.pop("LIZARDB200_ENC_SHAPE", None)
        if old is not None:
            os.environ["LIZARDB200_ENC_SHAPE"] = old


def _shape(level):
    v = [ctypes.c_int() for _ in range(4)]
    assert lz.lib().LizardB200_encodeShape(level, *[ctypes.byref(x) for x in v]) == 0
    return tuple(x.value for x in v[:3])


def chunks(n_units, per_chunk, ramp):
    """Pipeline chunks of a call of n_units (LizardB200_chunkPlan: the host's and the kernels' arithmetic agree)."""
    L = lz.lib()
    L.LizardB200_chunkPlan.argtypes = [ctypes.c_uint, ctypes.c_uint, ctypes.c_int, ctypes.c_uint] + [ctypes.POINTER(ctypes.c_uint)] * 3
    for u in range(n_units):
        assert L.LizardB200_chunkPlan(n_units, per_chunk, int(ramp), u, None, None, None) > 0, (n_units, per_chunk, u)
    return L.LizardB200_chunkPlan(n_units, per_chunk, int(ramp), n_units, None, None, None)


def _units_per_chunk(block):
    return max(int(os.environ["LIZARDB200_FRAME_CHUNK_MIB"]) * MIB // block, 1)


def _libs():
    return lz.bind_frame_api(lz.lib()), lz.bind_frame_api(refs.ref_parity())


# ---------------------------------------------------------------------------------------------------------------------
# child-side case groups
# ---------------------------------------------------------------------------------------------------------------------
def group_encode(pl):
    """A. One-shot LizardF_compressFrame at every GPU level across 4 chunks, byte for byte, then decoded by both libraries;
    checksum off / on above and below kHashThreadMin, content size off / on; four launch shapes at one level per
    units-kernel instance."""
    ours, ref = _libs()
    big, small = pl["inputs"]["big"], pl["inputs"]["small"]
    assert chunks(25, _units_per_chunk(BS), False) == 4 and len(big) == 24 * BS + 1
    for level in GPU_LEVELS:
        for name, data, ck, cs in (("big", big, True, 1), ("big", big, False, 0), ("small", small, True, 0), ("small", small, False, 1)):
            want = pl["frames"][(name, level, ck, cs)]
            if name == "big":
                fh, recs, _ = _records(want)
                # the 1-byte last block is the reference's 6-byte record (DESIGN.md 3.5), which pack_unit special-cases
                assert len(recs) == 25 and all(r[2] for r in recs[7:16]) and recs[24][1:] == (6, False), level
                assert not any(r[2] for r in recs[16:24]), level
            got = lz.frame_compress(ours, data, lz.make_prefs(level, 1, True, ck, cs))
            assert got == want, (level, name, ck, cs, len(got), len(want), _first_diff(got, want)[0])
            for L in (ours, ref):
                r, back = lz.frame_decompress(L, got, len(data))
                assert r == 0 and back == data, (level, name, ck, cs, L is ours)
    for level in UNITS_KERNEL_LEVELS:
        want = pl["frames"][("big", level, True, 1)]
        for name, value in SHAPES + (("one-warp", "1,1,1"),):
            with enc_shape(value):
                if value is not None:
                    w, t, k = (int(x) for x in value.split(","))
                    assert _shape(level) == (w, t if level in HAS_SMEM_TABLE else 0, k), (level, value)
                got = lz.frame_compress(ours, big, lz.make_prefs(level, 1, True, True, 1))
            assert got == want, (level, name, _first_diff(got, want)[0])


def group_blocksizes(pl):
    """B. blockSizeID 2-5 (256 KiB to 16 MiB): units of several inner blocks, 4 / 1 / 1 / 1 units per 1 MiB chunk; each
    frame has at least 3 blocks and a short last one; decoded by both libraries and both generations."""
    ours, ref = _libs()
    for (bsid, level), want in sorted(pl["frames"].items()):
        data, size = pl["inputs"][bsid], _block_bytes(bsid)
        nblk = -(-len(data) // size)
        assert nblk >= 4 and len(data) % size and chunks(nblk, _units_per_chunk(size), False) >= 3, (bsid, nblk)
        got = lz.frame_compress(ours, data, lz.make_prefs(level, bsid, True, True, 1))
        assert got == want, (bsid, level, len(got), len(want), _first_diff(got, want)[0])
        assert len(_records(got)[1]) == nblk
        for variant in VARIANTS:
            with decode_variant(variant):
                r, back = lz.frame_decompress(ours, got, len(data))
            assert r == 0 and back == data, (bsid, level, variant, r, len(back))
        r, back = lz.frame_decompress(ref, got, len(data))
        assert r == 0 and back == data, (bsid, level)


def _stream_calls(L, data, prefs, ops):
    """compressBegin, the ops ("u", n) = compressUpdate of the next n bytes, ("f",) = LizardF_flush, then compressEnd:
    [(call, return or error name, bytes written)]."""
    ctx = ctypes.c_void_p()
    assert L.LizardF_createCompressionContext(ctypes.byref(ctx), 100) == 0
    cap = L.LizardF_compressBound(len(data), ctypes.byref(prefs)) + 64
    buf = ctypes.create_string_buffer(cap)
    log, pos = [], 0

    def rec(what, r):
        log.append((what, _ret(L, r), buf.raw[:r] if not L.LizardF_isError(r) else b""))

    try:
        rec("begin", L.LizardF_compressBegin(ctx, buf, cap, ctypes.byref(prefs)))
        for op in ops:
            if op[0] == "u":
                n = op[1]
                rec(("update", n), L.LizardF_compressUpdate(ctx, buf, cap, data[pos:pos + n], n, None))
                pos += n
            else:
                rec("flush", L.LizardF_flush(ctx, buf, cap, None))
        rec("end", L.LizardF_compressEnd(ctx, buf, cap, None))
    finally:
        L.LizardF_freeCompressionContext(ctx)
    assert pos == len(data)
    return log


def group_stream(pl):
    """C. compressBegin / compressUpdate / LizardF_flush / compressEnd call by call against the reference at autoFlush 0
    and 1, one level per kernel instance; the errors; the levels the GPU refuses."""
    ours, ref = _libs()
    data = pl["inputs"]["stream"]
    multi = 2 * MIB + 3 * BS + 11
    assert chunks(-(-multi // BS), _units_per_chunk(BS), False) >= 3
    ops = [("u", 1), ("f",), ("u", BS - 1), ("u", BS), ("f",), ("u", BS + 1), ("u", 3 * BS + 5), ("u", multi), ("f",),
           ("u", 1), ("u", 7), ("f",), ("f",), ("u", BS + 1)]
    ops.append(("u", len(data) - sum(o[1] for o in ops if o[0] == "u")))
    assert ops[-1][1] > 0
    for level in KERNEL_LEVELS:
        for auto, ck, cs in ((0, True, 0), (1, True, len(data)), (1, False, 0)):
            p = lz.make_prefs(level, 1, True, ck, cs)
            p.autoFlush = auto
            want = _stream_calls(ref, data, p, ops)
            got = _stream_calls(ours, data, p, ops)
            assert got == want, (level, auto, ck, _first_diff([g[:2] for g in got], [w[:2] for w in want]),
                                 _first_diff(got, want)[0])
    # errors, each against the reference
    p = lz.make_prefs(10, 1, True, True, 0)
    for auto in (0, 1):
        p.autoFlush = auto
        for L in (ours, ref):
            ctx = ctypes.c_void_p()
            L.LizardF_createCompressionContext(ctypes.byref(ctx), 100)
            buf = ctypes.create_string_buffer(len(data) + 4096)
            assert not L.LizardF_isError(L.LizardF_compressBegin(ctx, buf, len(buf), ctypes.byref(p)))
            for n in (1, BS - 1, BS, 3 * BS + 5):
                bound = L.LizardF_compressBound(n, ctypes.byref(p))
                assert _ret(L, L.LizardF_compressUpdate(ctx, buf, bound - 1, data[:n], n, None)) == "ERROR_dstMaxSize_tooSmall"
            L.LizardF_freeCompressionContext(ctx)
    for cs in (len(data) - 1, len(data) + 1):
        p = lz.make_prefs(41, 1, True, True, cs)
        pieces = [("u", BS + 3), ("u", len(data) - BS - 3)]
        got, want = _stream_calls(ours, data, p, pieces), _stream_calls(ref, data, p, pieces)
        assert got == want and want[-1][1] == "ERROR_frameSize_wrong", (cs, got[-1][:2], want[-1][:2])
    for L in (ours, ref):
        ctx = ctypes.c_void_p()
        L.LizardF_createCompressionContext(ctypes.byref(ctx), 100)
        buf = ctypes.create_string_buffer(4 * BS)
        assert _ret(L, L.LizardF_compressUpdate(ctx, buf, len(buf), data[:1000], 1000, None)) == "ERROR_GENERIC"
        L.LizardF_freeCompressionContext(ctx)
    # the levels with no GPU parser: refused, nothing written
    for level in UNSUPPORTED_LEVELS:
        p = lz.make_prefs(level, 1, True, True, 0)
        ctx = ctypes.c_void_p()
        ours.LizardF_createCompressionContext(ctypes.byref(ctx), 100)
        buf = ctypes.create_string_buffer(b"\xee" * 64, 64)
        assert _ret(ours, ours.LizardF_compressBegin(ctx, buf, 64, ctypes.byref(p))) == "ERROR_compressionLevel_invalid", level
        ours.LizardF_freeCompressionContext(ctx)
        assert buf.raw == b"\xee" * 64, level
        cap = ours.LizardF_compressFrameBound(BS, ctypes.byref(p))
        dst = ctypes.create_string_buffer(b"\xee" * cap, cap)
        r = ours.LizardF_compressFrame(dst, cap, data[:BS], BS, ctypes.byref(p))
        assert _ret(ours, r) == "ERROR_compressionLevel_invalid" and dst.raw == b"\xee" * cap, level


# feeding schedules: (name, source pieces, destination pieces); None = all that is left, else (prefix, cycle)
SCHEDULES = (
    ("whole", None, None),
    ("src-mixed", ((), (1, 3, 4093, BS + 7)), None),
    ("src-4093", ((), (4093,)), None),
    ("src-BS+7", ((), (BS + 7,)), None),
    ("dst-small", None, ((), (BS // 2 + 3,))),
    ("both-small", ((), (4093,)), ((), (BS // 3,))),
)
BYTE_SCHEDULES = (                       # pure 1- and 3-byte feeding over the header and the first blocks, then larger pieces
    ("src-1", ((1,) * 90000, (BS + 7,)), None),
    ("src-3", ((3,) * 40000, (4093,)), None),
)


def _decode_both(ours, ref, stream, out_cap, what, schedules=SCHEDULES, info_at=()):
    for name, s_in, s_out in schedules:
        want = decode_calls(ref, stream, out_cap, s_in, s_out, info_at)
        assert want[0] and not isinstance(want[0][-1][0], str), (what, name, want[0][-1])
        for variant in VARIANTS:
            with decode_variant(variant):
                got = decode_calls(ours, stream, out_cap, s_in, s_out, info_at)
            assert_same_calls(got, want, (what, name, variant))


def group_decode(pl):
    """D. Reference frames at every level 10-49 (4 chunks, raw blocks inside, checksum and content size on) under both
    generations and the fixed feeding schedules, call by call; streaming frames with short blocks inside; skippable and
    concatenated frames with LizardF_getFrameInfo before and between."""
    ours, ref = _libs()
    data = pl["inputs"]["big"]
    assert chunks(25, _units_per_chunk(BS), True) == 4
    for level in range(10, 50):
        frame = pl["frames"][("big", level, True, 1)]
        fh, recs, _ = _records(frame)
        assert len(recs) == 25 and all(r[2] for r in recs[7:16]), level
        scheds = SCHEDULES + (BYTE_SCHEDULES if level in CODEWORD_LEVELS else ())
        _decode_both(ours, ref, frame, len(data), level, scheds)
        for variant in VARIANTS:
            with decode_variant(variant):
                r, back = lz.frame_decompress(ours, frame, len(data))
            assert r == 0 and back == data, (level, variant)
    for key, (stream, content) in pl["streams"].items():
        _decode_both(ours, ref, stream, len(content), key, SCHEDULES[:5])
        got = decode_calls(ours, stream, len(content))
        assert got[1] == content, key
    for key, (stream, content, starts) in pl["multi"].items():
        _decode_both(ours, ref, stream, len(content), key, SCHEDULES[:5:2], info_at=starts)
        assert decode_calls(ours, stream, len(content), info_at=starts)[1] == content, key
    # LizardF_getFrameInfo on an empty skippable frame: the frame is over within the call, the context is back at a header,
    # and the reference reports ERROR_frameHeader_incomplete after consuming the 8 bytes
    stream, content, _ = pl["multi"]["skippable-empty-and-end"]
    at = [stream.index(_skippable(3, b""))]
    want = decode_calls(ref, stream, len(content), info_at=at)
    assert want[0][-1][:2] == ("info", "ERROR_frameHeader_incomplete"), want[0][-1]
    assert_same_calls(decode_calls(ours, stream, len(content), info_at=at), want, "empty skippable")


def group_ramp(pl):
    """D (ramp). 41 units at 2 MiB chunks: the decoder's ramp of 1 / 2 / 4 / 8 units, then full chunks, with the content
    checksum hashed chunk by chunk (ChunkHasher), one level per codeword path, both generations."""
    ours, ref = _libs()
    data = pl["inputs"]["ramp"]
    assert _units_per_chunk(BS) == 16 and chunks(41, 16, True) == 6 and chunks(33, 16, True) == 6
    for level in CODEWORD_LEVELS:
        frame = pl["frames"][("ramp", level, True, 0)]
        scheds = (SCHEDULES[0], ("dst-33-blocks", None, ((), (33 * BS,))), ("src-3MiB", ((), (3 * MIB,)), None))
        _decode_both(ours, ref, frame, len(data), ("ramp", level), scheds)
        for variant in VARIANTS:
            with decode_variant(variant):
                r, back = lz.frame_decompress(ours, frame, len(data))
            assert r == 0 and back == data, (level, variant)


def _reference_caveats(frame):
    """(overrun, bytes defined) of a damaged frame (DESIGN.md 3.5): overrun when the reference would decode a compressed
    record past max_block behind a raw inner block; bytes undefined when a record that decodes has a match offset below 8,
    where the reference's output depends on stale bytes."""
    L, O = refs.ref_parity(), refs.oracle()
    _, recs, _ = _records(frame)
    overrun, defined = False, True
    for pos, n, raw in recs:
        if not raw and n <= BS and pos + 4 + n <= len(frame):
            payload = frame[pos + 4:pos + 4 + n]
            overrun |= refs.ref_decompress(L, payload, BS)[0] > BS
            dst = ctypes.create_string_buffer(BS + 64)
            if O.oracle_Lizard_decompress_safe(payload, dst, n, BS) > 0 and O.oracle_last_min_offset() < 8:
                defined = False
    return overrun, defined


def group_damage(pl):
    """E. Damaged reference frames fed whole (the batch path) and in small destination pieces (tmp_out), both generations:
    the reference's calls up to and including its error, and the bytes produced before it."""
    ours, ref = _libs()
    n = len(pl["inputs"]["big"])
    errors = set()
    for (level, name), frame in sorted(pl["damaged"].items()):
        overrun, defined = _reference_caveats(frame)
        for sname, s_in, s_out in (SCHEDULES[0], SCHEDULES[4], SCHEDULES[2]):
            want = None if overrun else decode_calls(ref, frame, n, s_in, s_out)
            for variant in VARIANTS:
                with decode_variant(variant):
                    got = decode_calls(ours, frame, n, s_in, s_out)
                if overrun:                      # the reference reports success behind a raw inner block; we refuse
                    assert isinstance(got[0][-1][0], str), (level, name, sname, variant, got[0][-1])
                    continue
                assert_same_calls(got, want, (level, name, sname, variant), defined)
            if want and isinstance(want[0][-1][0], str):
                errors.add(want[0][-1][0])
    assert {"ERROR_GENERIC", "ERROR_decompressionFailed", "ERROR_contentChecksum_invalid", "ERROR_frameSize_wrong"} <= errors, errors


GROUPS = {"encode": group_encode, "blocksizes": group_blocksizes, "stream": group_stream, "decode": group_decode,
          "ramp": group_ramp, "damage": group_damage}


# ---------------------------------------------------------------------------------------------------------------------
# parent-side tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref():
    if _ref() is None:
        pytest.skip("oracle/_ref not built")
    return _ref()


def _run_group(tmp_path, group, chunk_mib, payload):
    path = tmp_path / (group + ".pkl")
    with open(path, "wb") as f:
        pickle.dump(payload, f)
    env = dict(os.environ, LIZARDB200_FRAME_CHUNK_MIB=str(chunk_mib))
    env.pop("LIZARDB200_ENC_SHAPE", None)
    env.pop("LIZARDB200_DEC_VARIANT", None)
    out = subprocess.run([sys.executable, "-m", "tests.test_gpu_frame_pipeline", group, str(path)], cwd=refs.ROOT, env=env,
                         capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0 and ("group ok: " + group) in out.stdout, out.stdout[-3000:] + out.stderr[-6000:]


def test_compress_frame_every_gpu_level_across_chunks(ref, tmp_path):
    frames = {}
    for level in GPU_LEVELS:
        for name, ck, cs in (("big", True, 1), ("big", False, 0), ("small", True, 0), ("small", False, 1)):
            frames[(name, level, ck, cs)] = _ref_frame(name, level, 1, ck, cs)
    _run_group(tmp_path, "encode", 1, {"inputs": {"big": _input("big"), "small": _input("small")}, "frames": frames})


def test_compress_frame_large_block_sizes(ref, tmp_path):
    frames, inputs = {}, {}
    for bsid in (2, 3, 4, 5):
        inputs[bsid] = _input("bs%d" % bsid)
        for level in (KERNEL_LEVELS if bsid < 5 else (10, 20, 41)):      # 16 MiB blocks: the fast levels only
            frames[(bsid, level)] = _ref_frame("bs%d" % bsid, level, bsid, True, 1)
    _run_group(tmp_path, "blocksizes", 1, {"inputs": inputs, "frames": frames})


def test_streaming_compress_call_by_call(ref, tmp_path):
    _run_group(tmp_path, "stream", 1, {"inputs": {"stream": _input("stream")}})


def test_decompress_every_level_both_generations_across_chunks(ref, tmp_path):
    big = _input("big")
    frames = {("big", level, True, 1): _ref_frame("big", level, 1, True, 1) for level in range(10, 50)}
    streams = {}
    for level, bsid, cuts in ((10, 1, [70000, 1, BS + 5, 2 * BS]), (41, 1, [3 * BS + 1, 5, 40000]),
                              (21, 3, [MIB + 7, 300000, 1]), (45, 3, [5, 2 * MIB + 9])):
        streams[("short-blocks", level, bsid)] = (_ref_stream_frame(big, level, bsid, cuts), big)
    small = _input("small")
    f1, f2 = _ref_frame("big", 17, 1, True, 1), _ref_frame("small", 41, 1, True, 0)
    multi = {}
    for key, parts in (("two-frames", [f1, f2]),
                       ("skippable-front-and-between", [_skippable(0, b"\x01" * 100), f1, _skippable(15, b"xyz" * 3), f2]),
                       ("skippable-empty-and-end", [f2, _skippable(3, b""), f1, _skippable(7, bytes(range(256)))])):
        starts, at = [], 0
        for p in parts:
            starts.append(at)
            at += len(p)
        content = b"".join(big if p is f1 else small if p is f2 else b"" for p in parts)
        # not at an empty skippable frame: there LizardF_getFrameInfo ends with an error (checked on its own)
        multi[key] = (b"".join(parts), content, [at for at, p in zip(starts, parts) if len(p) > 8 or p[:4] != _skippable(3, b"")[:4]])
    _run_group(tmp_path, "decode", 1, {"inputs": {"big": big}, "frames": frames, "streams": streams, "multi": multi})


def test_decompress_ramp_frames_both_generations(ref, tmp_path):
    frames = {("ramp", level, True, 0): _ref_frame("ramp", level, 1, True, 0) for level in CODEWORD_LEVELS}
    _run_group(tmp_path, "ramp", 2, {"inputs": {"ramp": _input("ramp")}, "frames": frames})


def test_damaged_frames_match_reference(ref, tmp_path):
    damaged = {(level, name): b for level in CODEWORD_LEVELS for name, b in _damaged(level).items()}
    _run_group(tmp_path, "damage", 1, {"inputs": {"big": _input("big")}, "damaged": damaged})


# ---------------------------------------------------------------------------------------------------------------------
# F. LizardB200_gather_device
# ---------------------------------------------------------------------------------------------------------------------
def _place(rng, sizes, residue, gap):
    """Offsets with the given residue mod 16 per segment and `gap` + 0..47 bytes between segments."""
    offs, p = [], 64
    for i, n in enumerate(sizes):
        p += (residue(i) - p) % 16 + 16 * int(rng.integers(0, 3))
        offs.append(p)
        p += max(n, 0) + gap
    return offs, p + 64


def _gather(src_bytes, src_off, lens, dst_bytes, dst_off, stream):
    import torch
    dev = torch.device("cuda", 0)
    d_src = torch.frombuffer(bytearray(src_bytes), dtype=torch.uint8).to(dev)
    d_dst = torch.frombuffer(bytearray(dst_bytes), dtype=torch.uint8).to(dev)
    t_so = torch.tensor(src_off, dtype=torch.int64, device=dev)
    t_do = torch.tensor(dst_off, dtype=torch.int64, device=dev)
    t_len = torch.tensor(lens, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    L = lz.lib()
    assert L.LizardB200_gather_device(d_src.data_ptr(), t_so.data_ptr(), t_len.data_ptr(), d_dst.data_ptr(), t_do.data_ptr(),
                                      len(lens), stream.cuda_stream) == 0, L.LizardB200_lastError()
    stream.synchronize()
    return bytes(d_dst.cpu().numpy())


def test_gather_segments_match_numpy_concatenation():
    """Segment lengths 0, -1, 1-17, around 4 KiB and the 8-warp x 4 KiB tile stride, 1 MiB + 3; every source and destination
    residue mod 16; more segments than the grid (8 CTAs per SM) so that the CTAs loop; guard bytes around every
    destination untouched; a non-default stream."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(17)
    fixed = [0, -1] + list(range(1, 18)) + [4095, 4096, 4097, 32767, 32768, 32769, MIB + 3]
    n = 8 * sms + 333
    lens = fixed + [int(x) for x in rng.integers(-3, 40000, n - len(fixed))]
    lens = [lens[i] for i in rng.permutation(n)]
    src_off, n_src = _place(rng, lens, lambda i: i % 16, 0)
    dst_off, n_dst = _place(rng, lens, lambda i: (7 * i + 3) % 16, 16)
    src = rng.integers(0, 256, n_src, dtype=np.uint8)
    want = np.full(n_dst, 0xEE, dtype=np.uint8)
    for so, do, k in zip(src_off, dst_off, lens):
        if k > 0:
            want[do:do + k] = src[so:so + k]
    assert sum(1 for k in lens if k > 0) > 8 * sms
    got = _gather(src.tobytes(), src_off, lens, b"\xEE" * n_dst, dst_off, torch.cuda.Stream())
    assert got == want.tobytes(), next(i for i in range(n_dst) if got[i] != want[i])


@pytest.mark.parametrize("level", [10, 41])
def test_gather_packs_compress_device_results(ref, level):
    """The documented use: LizardB200_compress_device at a fixed stride, the exclusive prefix sum of its results, then
    LizardB200_gather_device: the reference's blocks back to back, on a non-default stream."""
    import torch
    L = lz.lib()
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(level)
    pool = lz.datagen(4 * MIB, 50, 5) + b"".join(u for units in corpus.corpus().values() for u in units)[:4 * MIB]
    sizes = [int(x) for x in rng.choice([1, 17, 4096, 70000, BS - 1, BS], 300)]
    units = [pool[a:a + k] for a, k in zip((int(x) for x in rng.integers(0, len(pool) - BS, 300)), sizes)]
    want = [refs.ref_compress(refs.ref_parity(), u, level) for u in units]
    stride = (L.Lizard_compressBound(BS) + 15) // 16 * 16
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        h_src = b"".join(u + bytes(BS - len(u)) for u in units)
        d_src = torch.frombuffer(bytearray(h_src), dtype=torch.uint8).to(dev)
        t_so = torch.arange(300, dtype=torch.int64, device=dev) * BS
        t_sl = torch.tensor(sizes, dtype=torch.int32, device=dev)
        d_out = torch.zeros(300 * stride, dtype=torch.uint8, device=dev)
        t_oo = torch.arange(300, dtype=torch.int64, device=dev) * stride
        t_cap = torch.tensor([L.Lizard_compressBound(k) for k in sizes], dtype=torch.int32, device=dev)
        t_res = torch.zeros(300, dtype=torch.int32, device=dev)
        s.synchronize()
        assert L.LizardB200_compress_device(d_src.data_ptr(), t_so.data_ptr(), t_sl.data_ptr(), d_out.data_ptr(),
                                            t_oo.data_ptr(), t_cap.data_ptr(), t_res.data_ptr(), 300, level, s.cuda_stream) == 0
        t_at = torch.cumsum(t_res.to(torch.int64), 0) - t_res.to(torch.int64)
        total = int(t_res.to(torch.int64).sum().item())
        d_packed = torch.full((total + 64,), 0xEE, dtype=torch.uint8, device=dev)
        assert L.LizardB200_gather_device(d_out.data_ptr(), t_oo.data_ptr(), t_res.data_ptr(), d_packed.data_ptr(),
                                          t_at.data_ptr(), 300, s.cuda_stream) == 0, L.LizardB200_lastError()
        s.synchronize()
    assert t_res.cpu().tolist() == [len(w) for w in want]
    got = bytes(d_packed.cpu().numpy())
    assert got == b"".join(want) + b"\xEE" * 64


if __name__ == "__main__":
    with open(sys.argv[2], "rb") as f:
        payload = pickle.load(f)
    GROUPS[sys.argv[1]](payload)
    print("group ok: " + sys.argv[1])
